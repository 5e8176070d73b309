// TrackPlane::perform_plane_detection_monocular (track_plane/TrackPlane.cpp:580-1121) on the device: one CTA per frame.
// The tracker's histories live in device memory across frames, indexed by a slot per feature id that the host assigns (the mapping depends
// only on the ids the caller passes).  A frame is one upload (pose, calibration, slots, pixels, normalised coordinates, ascending-id order,
// the previous frame's features that left) and one launch; nothing is read back unless the caller asks.
//
// Phases of plane_track_kernel, in the reference's order:
//   1  a thread per feature: accumulate the bearing system, solve it once enough observations are in (remove_feats is the host's slot reset)
//   2  keep the features with a 3D estimate, in order
//   3  Delaunay mesh of their pixels: CDT's incremental insertion restated (super-triangle, insertion in the order given, the same triangle
//      layout, vertex rotations and edge-flip stack), with sign-exact orient2d / incircle on the float inputs.  The triangle containing a
//      point is located by the whole CTA, each insertion and its flips run on thread 0.
//   4  a thread per triangle for the normals, a thread per vertex for its normal window (pushes in triangle order) and its average
//   5  the matching and merging loop, serial over features in ascending id on warp 0; relabel sweeps spread over its lanes
//   6  the spatial filter (k-NN z-test) and the pruning to the frame's planes with more than 3 features, a thread per feature
#include "ovp_internal.h"
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <unordered_map>
#include <unordered_set>

namespace ovp {
namespace ptrack {

constexpr int NMAX = OVP_PLANE_TRACK_MAX_POINTS;
constexpr int NSLOT = 2 * NMAX; // the frame's features + the previous frame's that left (their plane labels live until the frame ends)
constexpr int TMAX = 2 * NMAX + 1; // triangles of NMAX points and the super-triangle's 3
constexpr int WCAP = OVP_PLANE_TRACK_MAX_NORM_COUNT;
constexpr int KCAP = OVP_PLANE_TRACK_MAX_FILTER_FEAT;
constexpr int PCAP = OVP_PLANE_TRACK_MAX_MERGES;
constexpr int THREADS = 1024;
constexpr int HIST = 18 + 3 * WCAP; // ovp_debug_plane_track_history's record

// device-resident tracker state
struct Dev {
  double *A, *b, *inG, *win; // per slot: 9, 3, 3, 3 * WCAP
  int *cnt, *has, *wlen;
  long long *label;          // hist_feat_to_plane, -1: no entry
  long long *pair_old, *pair_owner; // hist_plane_to_oldplanes: old plane -> the plane it was merged into
  int *npair;                // [0] pairs, [1] overflow flag (sticky)
  long long *planeid_ctr;    // currplaneid
  // last frame's outputs
  int *ntri, *tri;           // [0] triangles; 3 per triangle
  double *tnorm;             // 3 per triangle
  long long *frame_label;    // label of each of the frame's features after the frame
  // per-frame scratch
  int *inc_off, *inc_list;   // incident triangles of each surviving vertex, in triangle order
  int *match;                // the matches of the feature the merging loop is at (slots)
  int *surv;                 // [0] surviving features m, then their frame indices (the mesh's vertices, in order)
  int *tacc;                 // triangle gave a normal
  double *avg;               // average normal of each surviving vertex (3)
  double *knn;               // k-NN mean distance of each surviving vertex
  double *zstat;             // plane mean / std at the plane's first member (2)
};

// the frame as uploaded: header then the arrays (Frame::layout)
struct FrameArgs {
  const double *pose;  // 14: pose_GtoI7, calib7
  const int *slot;     // n: slot of each feature, bit 30 set: a fresh slot (history reset first)
  const float2 *uv, *uvn;
  const int *asc;      // n: frame indices in ascending featid
  const int *stale;    // nstale slots of the previous frame's features not in this frame
  int n, nstale, nslot;
};

// ---- sign-exact predicates on float inputs -------------------------------------------------------------------------------------------
__device__ __forceinline__ void two_sum(double a, double b, double &s, double &e) {
  s = __dadd_rn(a, b);
  const double bb = __dsub_rn(s, a);
  e = __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb));
}
// sign of the exact sum of t[0..n): grow an expansion term by term (zero components dropped); it is nonoverlapping and ordered by
// magnitude, so its sign is its last component's.  t is overwritten.
__device__ int exact_sum_sign(double *t, int n) {
  int m = 0;
  for (int i = 0; i < n; i++) {
    double q = t[i];
    int k = 0;
    for (int j = 0; j < m; j++) {
      double s, h;
      two_sum(q, t[j], s, h);
      q = s;
      if (h != 0.0)
        t[k++] = h;
    }
    if (q != 0.0)
      t[k++] = q;
    m = k;
  }
  return m == 0 ? 0 : (t[m - 1] > 0 ? 1 : -1);
}
__device__ __forceinline__ double fprod(float a, float b) { return __dmul_rn((double)a, (double)b); } // exact: 24 + 24 bits
// sign of CDT's orient2D(p, v1, v2) = orient2d(v1, v2, p) = (v1 - p) x (v2 - p): > 0 p left of v1 -> v2
__device__ int orient_sign(float px, float py, float ax, float ay, float bx, float by) {
  // (ax - px)(by - py) - (ay - py)(bx - px) expanded into six products of floats, each exact in double
  double t[6] = {fprod(ax, by), -fprod(ax, py), -fprod(px, by), -fprod(ay, bx), fprod(ay, px), fprod(py, bx)};
  double s = 0.0, mag = 0.0;
  for (int i = 0; i < 6; i++) {
    s = __dadd_rn(s, t[i]);
    mag = __dadd_rn(mag, fabs(t[i]));
  }
  if (fabs(s) > __dmul_rn(mag, 8.0 * 1.1102230246251565e-16)) // 5 roundings of exact terms, with margin
    return s > 0 ? 1 : -1;
  return exact_sum_sign(t, 6);
}
__device__ void push_lift_cross(double *t, int &n, bool neg, float px, float py, float qx, float qy, float rx, float ry) {
  // +-(px^2 + py^2)(qx ry - qy rx) as eight exact doubles
  const double l[2] = {fprod(px, px), fprod(py, py)};
  const double c[2] = {fprod(qx, ry), -fprod(qy, rx)};
  for (int i = 0; i < 2; i++)
    for (int j = 0; j < 2; j++) {
      const double p = __dmul_rn(l[i], c[j]);
      const double e = __fma_rn(l[i], c[j], -p);
      t[n++] = neg ? -p : p;
      t[n++] = neg ? -e : e;
    }
}
__device__ void push_det3(double *t, int &n, bool neg, float2 p, float2 q, float2 r) {
  // det [p, |p|^2; q, |q|^2; r, |r|^2] = |p|^2 (q x r) - |q|^2 (p x r) + |r|^2 (p x q)
  push_lift_cross(t, n, neg, p.x, p.y, q.x, q.y, r.x, r.y);
  push_lift_cross(t, n, !neg, q.x, q.y, p.x, p.y, r.x, r.y);
  push_lift_cross(t, n, neg, r.x, r.y, p.x, p.y, q.x, q.y);
}
// sign of incircle(a, b, c, d): > 0 d inside the circle through a, b, c (counter-clockwise)
__device__ int incircle_sign(float2 a, float2 b, float2 c, float2 d) {
  const double adx = __dsub_rn(a.x, d.x), ady = __dsub_rn(a.y, d.y), bdx = __dsub_rn(b.x, d.x), bdy = __dsub_rn(b.y, d.y);
  const double cdx = __dsub_rn(c.x, d.x), cdy = __dsub_rn(c.y, d.y);
  const double bdxcdy = __dmul_rn(bdx, cdy), cdxbdy = __dmul_rn(cdx, bdy), cdxady = __dmul_rn(cdx, ady), adxcdy = __dmul_rn(adx, cdy);
  const double adxbdy = __dmul_rn(adx, bdy), bdxady = __dmul_rn(bdx, ady);
  const double al = __dadd_rn(__dmul_rn(adx, adx), __dmul_rn(ady, ady)), bl = __dadd_rn(__dmul_rn(bdx, bdx), __dmul_rn(bdy, bdy));
  const double cl = __dadd_rn(__dmul_rn(cdx, cdx), __dmul_rn(cdy, cdy));
  const double det = __dadd_rn(__dadd_rn(__dmul_rn(al, __dsub_rn(bdxcdy, cdxbdy)), __dmul_rn(bl, __dsub_rn(cdxady, adxcdy))),
                               __dmul_rn(cl, __dsub_rn(adxbdy, bdxady)));
  const double perm = __dadd_rn(__dadd_rn(__dmul_rn(__dadd_rn(fabs(bdxcdy), fabs(cdxbdy)), al), __dmul_rn(__dadd_rn(fabs(cdxady), fabs(adxcdy)), bl)),
                                __dmul_rn(__dadd_rn(fabs(adxbdy), fabs(bdxady)), cl));
  if (fabs(det) > __dmul_rn(perm, 12.0 * 1.1102230246251565e-16)) // Shewchuk's first bound (10 + 96 eps) eps, with margin
    return det > 0 ? 1 : -1;
  // exact: the 4 x 4 determinant [x, y, x^2 + y^2, 1] expanded along its column of ones, 96 exact doubles
  double t[96];
  int n = 0;
  push_det3(t, n, true, b, c, d);
  push_det3(t, n, false, a, c, d);
  push_det3(t, n, true, a, b, d);
  push_det3(t, n, false, a, b, c);
  return exact_sum_sign(t, n);
}

// ---- CDT's triangle layout ----------------------------------------------------------------------------------------------------------
// triangle i: T[6i + 0..2] vertices (counter-clockwise), T[6i + 3..5] neighbours, neighbour k across the edge (v_k, v_{k+1}); -1: none
__device__ __forceinline__ int ccw3(int i) { return (i + 1) % 3; }
__device__ __forceinline__ int cw3(int i) { return (i + 2) % 3; }
__device__ __forceinline__ int opo_nbr(int vi) { return vi == 0 ? 1 : (vi == 1 ? 2 : 0); }
__device__ __forceinline__ int opo_vrt(int ni) { return ni == 0 ? 2 : (ni == 1 ? 0 : 1); }
__device__ __forceinline__ int nbr_ind(const int *t, int iTn) { return t[3] == iTn ? 0 : (t[4] == iTn ? 1 : 2); }
__device__ __forceinline__ void set_tri(int *T, int i, int v0, int v1, int v2, int n0, int n1, int n2) {
  int *t = T + 6 * i;
  t[0] = v0, t[1] = v1, t[2] = v2, t[3] = n0, t[4] = n1, t[5] = n2;
}
__device__ __forceinline__ void change_nbr(int *T, int iT, int oldN, int newN) {
  if (iT < 0)
    return;
  int *t = T + 6 * iT;
  t[3 + nbr_ind(t, oldN)] = newN;
}
// CDT's locatePointTriangle: 0 outside, 1 inside, 2..4 on edge 1..3 (the last edge the point lies on)
__device__ int locate_in_tri(const float2 *V, const int *t, float2 p) {
  int res = 1;
  for (int e = 0; e < 3; e++) {
    const float2 a = V[t[e]], b = V[t[(e + 1) % 3]];
    const int o = orient_sign(p.x, p.y, a.x, a.y, b.x, b.y);
    if (o < 0)
      return 0;
    if (o == 0)
      res = 2 + e;
  }
  return res;
}
// side of p against the line v1 -> v2: CDT's locatePointLine as a sign
__device__ __forceinline__ int side(const float2 *V, int ip, int i1, int i2) {
  return orient_sign(V[ip].x, V[ip].y, V[i1].x, V[i1].y, V[i2].x, V[i2].y);
}
// CDT's isFlipNeeded for the new vertex iV (never a super-triangle vertex) against the edge (iV1, iV3) of the triangle with apex iV2
__device__ bool flip_needed(const float2 *V, int iV, int iV1, int iV2, int iV3) {
  if (iV2 < 3) {
    if (iV1 < 3)
      return side(V, iV1, iV, iV3) == side(V, iV2, iV, iV3);
    if (iV3 < 3)
      return side(V, iV3, iV1, iV) == side(V, iV2, iV1, iV);
    return false;
  }
  if (iV1 < 3)
    return side(V, iV1, iV2, iV3) == side(V, iV, iV2, iV3);
  if (iV3 < 3)
    return side(V, iV3, iV1, iV2) == side(V, iV, iV1, iV2);
  return incircle_sign(V[iV1], V[iV2], V[iV3], V[iV]) > 0;
}
__device__ void flip_edge(int *T, int iT, int iTopo) {
  int *t = T + 6 * iT, *to = T + 6 * iTopo;
  int i = opo_vrt(nbr_ind(t, iTopo));
  const int v1 = t[i], v2 = t[ccw3(i)], n1 = t[3 + i], n3 = t[3 + cw3(i)];
  i = opo_vrt(nbr_ind(to, iT));
  const int v3 = to[i], v4 = to[ccw3(i)], n4 = to[3 + i], n2 = to[3 + cw3(i)];
  set_tri(T, iT, v4, v1, v3, n3, iTopo, n4);
  set_tri(T, iTopo, v2, v3, v1, n2, iT, n1);
  change_nbr(T, n1, iT, iTopo);
  change_nbr(T, n4, iTopo, iT);
}
// insert vertex v located in triangle iT (loc 1) or on its edge loc - 2 (loc 2..4), then restore the Delaunay property with CDT's flip
// stack.  Thread 0 only.
__device__ void insert_vertex(const float2 *V, int *T, int *stack, int &ntri, int v, int iT, int loc) {
  int top = 0;
  if (loc > 1 && T[6 * iT + 3 + (loc - 2)] < 0) // on an edge without a neighbour (one point: a flat super-triangle): CDT splits the triangle
    loc = 1;
  if (loc == 1) {
    const int iN1 = ntri, iN2 = ntri + 1;
    ntri += 2;
    const int *t = T + 6 * iT;
    const int v1 = t[0], v2 = t[1], v3 = t[2], n1 = t[3], n2 = t[4], n3 = t[5];
    set_tri(T, iN1, v2, v3, v, n2, iN2, iT);
    set_tri(T, iN2, v3, v1, v, n3, iT, iN1);
    set_tri(T, iT, v1, v2, v, n1, iN1, iN2);
    change_nbr(T, n2, iT, iN1);
    change_nbr(T, n3, iT, iN2);
    stack[top++] = iT;
    stack[top++] = iN1;
    stack[top++] = iN2;
  } else {
    const int iT1 = iT, iT2 = T[6 * iT + 3 + (loc - 2)];
    const int iN1 = ntri, iN2 = ntri + 1;
    ntri += 2;
    const int *t1 = T + 6 * iT1, *t2 = T + 6 * iT2;
    int i = opo_vrt(nbr_ind(t1, iT2));
    const int v1 = t1[i], v2 = t1[ccw3(i)], n1 = t1[3 + i], n4 = t1[3 + cw3(i)];
    i = opo_vrt(nbr_ind(t2, iT1));
    const int v3 = t2[i], v4 = t2[ccw3(i)], n3 = t2[3 + i], n2 = t2[3 + cw3(i)];
    set_tri(T, iT1, v1, v2, v, n1, iN2, iN1);
    set_tri(T, iT2, v3, v4, v, n3, iN1, iN2);
    set_tri(T, iN1, v1, v, v4, iT1, iT2, n4);
    set_tri(T, iN2, v3, v, v2, iT2, iT1, n2);
    change_nbr(T, n4, iT1, iN1);
    change_nbr(T, n2, iT2, iN2);
    stack[top++] = iT1;
    stack[top++] = iN2;
    stack[top++] = iT2;
    stack[top++] = iN1;
  }
  while (top > 0) {
    const int a = stack[--top];
    const int *t = T + 6 * a;
    const int vi = t[0] == v ? 0 : (t[1] == v ? 1 : 2);
    const int o = t[3 + opo_nbr(vi)];
    if (o < 0)
      continue;
    const int *to = T + 6 * o;
    const int i = opo_vrt(nbr_ind(to, a));
    if (flip_needed(V, v, to[cw3(i)], to[i], to[ccw3(i)])) {
      flip_edge(T, a, o);
      stack[top++] = a;
      stack[top++] = o;
    }
  }
}

// ---- small dense helpers (double) --------------------------------------------------------------------------------------------------
__device__ void solve3(const double *A, const double *b, double *x) { // Gaussian elimination with complete pivoting
  double M[3][4];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++)
      M[i][j] = A[3 * i + j];
    M[i][3] = b[i];
  }
  int col[3] = {0, 1, 2};
  for (int k = 0; k < 3; k++) {
    int pi = k, pj = k;
    for (int i = k; i < 3; i++)
      for (int j = k; j < 3; j++)
        if (fabs(M[i][j]) > fabs(M[pi][pj]))
          pi = i, pj = j;
    for (int j = 0; j < 4; j++) {
      const double s = M[k][j];
      M[k][j] = M[pi][j];
      M[pi][j] = s;
    }
    for (int i = 0; i < 3; i++) {
      const double s = M[i][k];
      M[i][k] = M[i][pj];
      M[i][pj] = s;
    }
    const int s = col[k];
    col[k] = col[pj];
    col[pj] = s;
    for (int i = k + 1; i < 3; i++) {
      const double f = M[i][k] / M[k][k];
      for (int j = k; j < 4; j++)
        M[i][j] -= f * M[k][j];
    }
  }
  double y[3];
  for (int k = 2; k >= 0; k--) {
    double s = M[k][3];
    for (int j = k + 1; j < 3; j++)
      s -= M[k][j] * y[j];
    y[k] = s / M[k][k];
  }
  for (int k = 0; k < 3; k++)
    x[col[k]] = y[k];
}
// singular values of a symmetric 3 x 3 matrix: |eigenvalues|, cyclic Jacobi; returns max / min
__device__ double cond_sym3(const double *A) {
  double a[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      a[i][j] = A[3 * i + j];
  for (int sweep = 0; sweep < 30; sweep++) {
    const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
    if (off == 0.0)
      break;
    for (int p = 0; p < 2; p++)
      for (int q = p + 1; q < 3; q++) {
        if (a[p][q] == 0.0)
          continue;
        const double th = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
        for (int k = 0; k < 3; k++) { // A <- J^T A J
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = cs * akp - sn * akq;
          a[k][q] = sn * akp + cs * akq;
        }
        for (int k = 0; k < 3; k++) {
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = cs * apk - sn * aqk;
          a[q][k] = sn * apk + cs * aqk;
        }
      }
  }
  const double s0 = fabs(a[0][0]), s1 = fabs(a[1][1]), s2 = fabs(a[2][2]);
  return fmax(s0, fmax(s1, s2)) / fmin(s0, fmin(s1, s2));
}
__device__ __forceinline__ double norm3(const double *v) {
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])), __dmul_rn(v[2], v[2])));
}
__device__ __forceinline__ double dot3(const double *a, const double *b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}
// cv::norm of a float Point2f difference, in double
__device__ __forceinline__ double px_dist(float2 a, float2 b) {
  const float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y);
  return __dsqrt_rn(__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)));
}

// TrackPlane::avg_norm (:1123-1171) over a window of w normals; zero when rejected
__device__ void avg_norm(const double *win, int w, const ovp_plane_track_options &o, double *out) {
  out[0] = out[1] = out[2] = 0.0;
  if (w == 0)
    return;
  int count = 0;
  double s[3] = {0, 0, 0};
  for (int k = 0; k < w; k++) {
    const double *nk = win + 3 * k;
    if (norm3(nk) <= 0)
      continue;
    for (int j = 0; j < 3; j++)
      s[j] = __dadd_rn(s[j], nk[j]);
    count++;
  }
  const double sn = norm3(s);
  for (int j = 0; j < 3; j++)
    s[j] = __ddiv_rn(s[j], sn);
  if (count < 2)
    return;
  double max_deg = 0.0, var_deg = 0.0;
  for (int k = 0; k < w; k++) {
    const double *nk = win + 3 * k;
    if (norm3(nk) <= 0)
      continue;
    const double d = __dmul_rn(180.0 / M_PI, acos(dot3(nk, s)));
    var_deg = __dadd_rn(var_deg, __dmul_rn(d, d));
    max_deg = (max_deg < d) ? d : max_deg; // std::max: a NaN deviation never becomes the maximum
  }
  var_deg = __ddiv_rn(var_deg, (double)(count - 1));
  if (sqrt(var_deg) > o.max_norm_avg_var || max_deg > o.max_norm_avg_max)
    return;
  out[0] = s[0], out[1] = s[1], out[2] = s[2];
}

__device__ void relabel(Dev &D, const FrameArgs &F, long long minp, long long oldp, int lane) {
  if (minp == oldp)
    return;
  for (int s = lane; s < F.nslot; s += 32)
    if (D.label[s] == oldp)
      D.label[s] = minp;
  const int np = D.npair[0];
  for (int k = lane; k < np; k += 32)
    if (D.pair_owner[k] == oldp)
      D.pair_owner[k] = minp;
  __syncwarp();
  if (lane == 0) {
    if (np < PCAP) {
      D.pair_old[np] = oldp;
      D.pair_owner[np] = minp;
      D.npair[0] = np + 1;
    } else {
      D.npair[1] = 1;
    }
  }
  __syncwarp();
}

__global__ void __launch_bounds__(THREADS, 1) plane_track_kernel(Dev D, FrameArgs F, ovp_plane_track_options o) {
  extern __shared__ __align__(16) unsigned char smem[];
  float2 *V = (float2 *)smem;                  // NMAX + 3 mesh vertices (the super-triangle's first)
  int *T = (int *)(V + NMAX + 3);              // TMAX triangles
  int *stack = T + 6 * TMAX;                   // TMAX + 8 flip stack
  int *surv = stack + TMAX + 8;                // NMAX: frame index of each surviving vertex
  int *sidx = surv + NMAX;                     // NMAX: surviving index of each frame feature, -1 dropped
  unsigned char *done = (unsigned char *)(sidx + NMAX); // NMAX: done_verts_ids, by surviving index
  __shared__ double R[9], pc[3];               // R_GtoCi, p_CiinG
  __shared__ int s_m, s_ntri, s_loc;
  __shared__ float s_box[4];
  const int tid = threadIdx.x, n = F.n;

  if (tid == 0) {
    const double *q = F.pose, *qc = F.pose + 7;
    double Ri[9], Rc[9];
    for (int k = 0; k < 2; k++) { // JPL quat_2_Rot: (2 q4^2 - 1) I - 2 q4 [q]x + 2 q q^T
      const double *qq = k == 0 ? q : qc;
      double *Rk = k == 0 ? Ri : Rc;
      const double w = qq[3];
      const double sk[9] = {0, -qq[2], qq[1], qq[2], 0, -qq[0], -qq[1], qq[0], 0};
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
          Rk[3 * i + j] = (i == j ? 2 * w * w - 1 : 0.0) - 2 * w * sk[3 * i + j] + 2 * qq[i] * qq[j];
    }
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        R[3 * i + j] = Rc[3 * i] * Ri[j] + Rc[3 * i + 1] * Ri[3 + j] + Rc[3 * i + 2] * Ri[6 + j];
    for (int i = 0; i < 3; i++)
      pc[i] = q[4 + i] - (R[i] * qc[4] + R[3 + i] * qc[5] + R[6 + i] * qc[6]);
  }
  __syncthreads();

  // ---- 1: bearing systems and their solves (:632-694) ----
  for (int i = tid; i < n; i += THREADS) {
    const int s = F.slot[i] & 0x3fffffff;
    if (F.slot[i] & 0x40000000) { // remove_feats dropped this id's history (or it is new)
      for (int k = 0; k < 9; k++)
        D.A[9 * s + k] = 0.0;
      for (int k = 0; k < 3; k++)
        D.b[3 * s + k] = 0.0;
      D.cnt[s] = 0, D.has[s] = 0, D.wlen[s] = 0, D.label[s] = -1;
    }
    const float2 z = F.uvn[i];
    double bv[3];
    for (int r = 0; r < 3; r++)
      bv[r] = R[r] * (double)z.x + R[3 + r] * (double)z.y + R[6 + r];
    const double nb = norm3(bv);
    for (int r = 0; r < 3; r++)
      bv[r] /= nb;
    const double B[9] = {0, -bv[2], bv[1], bv[2], 0, -bv[0], -bv[1], bv[0], 0};
    double Ai[9], bi[3];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++)
        Ai[3 * r + c] = B[r] * B[c] + B[3 + r] * B[3 + c] + B[6 + r] * B[6 + c];
    for (int r = 0; r < 3; r++)
      bi[r] = Ai[3 * r] * pc[0] + Ai[3 * r + 1] * pc[1] + Ai[3 * r + 2] * pc[2];
    double A[9], b[3];
    for (int k = 0; k < 9; k++)
      A[k] = D.A[9 * s + k] = Ai[k] + D.A[9 * s + k];
    for (int k = 0; k < 3; k++)
      b[k] = D.b[3 * s + k] = bi[k] + D.b[3 * s + k];
    const int cnt = D.cnt[s] = D.cnt[s] + 1;
    if (cnt >= o.feat_init_min_obs) {
      double p[3];
      solve3(A, b, p);
      const double cond = cond_sym3(A);
      double pz = 0.0, nn = 0.0;
      for (int r = 0; r < 3; r++) {
        const double v = R[3 * r] * (p[0] - pc[0]) + R[3 * r + 1] * (p[1] - pc[1]) + R[3 * r + 2] * (p[2] - pc[2]);
        nn += v * v;
        if (r == 2)
          pz = v;
      }
      if (fabs(cond) <= o.max_cond_number && pz >= o.min_dist && pz <= o.max_dist && !isnan(sqrt(nn))) {
        for (int r = 0; r < 3; r++)
          D.inG[3 * s + r] = p[r];
        D.has[s] = 1;
      }
    }
  }
  __syncthreads();

  // ---- 2: the features with a 3D estimate, in order (:696-708) ----
  if (tid == 0) {
    int m = 0;
    float mnx = 0, mny = 0, mxx = 0, mxy = 0;
    for (int i = 0; i < n; i++) {
      if (!D.has[F.slot[i] & 0x3fffffff]) {
        sidx[i] = -1;
        continue;
      }
      const float2 u = F.uv[i];
      if (m == 0)
        mnx = mxx = u.x, mny = mxy = u.y;
      mnx = fminf(mnx, u.x), mny = fminf(mny, u.y), mxx = fmaxf(mxx, u.x), mxy = fmaxf(mxy, u.y);
      sidx[i] = m;
      surv[m++] = i;
    }
    s_m = m;
    s_box[0] = mnx, s_box[1] = mny, s_box[2] = mxx, s_box[3] = mxy;
  }
  __syncthreads();
  const int m = s_m;

  // ---- 3: Delaunay triangulation (:715-723) ----
  for (int k = tid; k < m; k += THREADS)
    V[3 + k] = F.uv[surv[k]];
  if (tid == 0) {
    // CDT's super-triangle around the envelope box, in float and unfused
    const float cx = __fdiv_rn(__fadd_rn(s_box[0], s_box[2]), 2.0f), cy = __fdiv_rn(__fadd_rn(s_box[1], s_box[3]), 2.0f);
    const float w = __fsub_rn(s_box[2], s_box[0]), h = __fsub_rn(s_box[3], s_box[1]);
    float r = __fdiv_rn(__fsqrt_rn(__fadd_rn(__fmul_rn(w, w), __fmul_rn(h, h))), 2.0f);
    r = __fmul_rn(r, 1.1f);
    const float Rr = __fmul_rn(2.0f, r);
    const float sx = __fdiv_rn(__fmul_rn(Rr, __fsqrt_rn(3.0f)), 2.0f);
    V[0] = make_float2(__fsub_rn(cx, sx), __fsub_rn(cy, r));
    V[1] = make_float2(__fadd_rn(cx, sx), __fsub_rn(cy, r));
    V[2] = make_float2(cx, __fadd_rn(cy, Rr));
    set_tri(T, 0, 0, 1, 2, -1, -1, -1);
    s_ntri = 1;
  }
  __syncthreads();
  for (int k = 0; k < m; k++) {
    const float2 p = V[3 + k];
    if (tid == 0)
      s_loc = INT_MAX;
    __syncthreads();
    const int ntri = s_ntri;
    for (int t = tid; t < ntri; t += THREADS) {
      const int loc = locate_in_tri(V, T + 6 * t, p);
      if (loc)
        atomicMin(&s_loc, t * 4 + (loc - 1));
    }
    __syncthreads();
    if (tid == 0 && s_loc != INT_MAX) { // every point lies in the super-triangle; CDT throws where none is found
      int nt = s_ntri;
      insert_vertex(V, T, stack, nt, 3 + k, s_loc >> 2, (s_loc & 3) + 1);
      s_ntri = nt;
    }
    __syncthreads();
  }
  // eraseSuperTriangle: the triangles without a super-triangle vertex, in order, vertices renumbered
  if (tid == 0) {
    int nt = 0;
    for (int t = 0; t < s_ntri; t++) {
      const int *tt = T + 6 * t;
      if (tt[0] < 3 || tt[1] < 3 || tt[2] < 3)
        continue;
      for (int j = 0; j < 3; j++)
        D.tri[3 * nt + j] = tt[j] - 3;
      nt++;
    }
    D.ntri[0] = nt;
    s_ntri = nt;
    // incident triangles of every surviving vertex, in triangle order
    for (int v = 0; v <= m; v++)
      D.inc_off[v] = 0;
    for (int t = 0; t < nt; t++)
      for (int j = 0; j < 3; j++)
        D.inc_off[D.tri[3 * t + j] + 1]++;
    for (int v = 0; v < m; v++)
      D.inc_off[v + 1] += D.inc_off[v];
    for (int v = 0; v < m; v++)
      stack[v] = D.inc_off[v];
    for (int t = 0; t < nt; t++)
      for (int j = 0; j < 3; j++)
        D.inc_list[stack[D.tri[3 * t + j]]++] = t;
  }
  __syncthreads();
  const int ntri = s_ntri;

  // ---- 4: triangle normals (:733-776), windows (:778-795), average normals (:801-806) ----
  for (int t = tid; t < ntri; t += THREADS) {
    const int v0 = D.tri[3 * t], v1 = D.tri[3 * t + 1], v2 = D.tri[3 * t + 2];
    const float2 u0 = V[3 + v0], u1 = V[3 + v1], u2 = V[3 + v2];
    double nrm[3] = {0, 0, 0};
    const double side_max = (double)o.max_tri_side_px;
    const bool ok = !(px_dist(u0, u1) > side_max || px_dist(u1, u2) > side_max || px_dist(u2, u0) > side_max);
    if (ok) {
      const double *p1 = D.inG + 3 * (F.slot[surv[v0]] & 0x3fffffff), *p2 = D.inG + 3 * (F.slot[surv[v1]] & 0x3fffffff);
      const double *p3 = D.inG + 3 * (F.slot[surv[v2]] & 0x3fffffff);
      double d1[3], d2[3];
      for (int j = 0; j < 3; j++)
        d1[j] = __dsub_rn(p2[j], p1[j]), d2[j] = __dsub_rn(p3[j], p1[j]);
      const double n1 = norm3(d1), n2 = norm3(d2);
      for (int j = 0; j < 3; j++)
        d1[j] = __ddiv_rn(d1[j], n1), d2[j] = __ddiv_rn(d2[j], n2);
      nrm[0] = __dsub_rn(__dmul_rn(d1[1], d2[2]), __dmul_rn(d1[2], d2[1]));
      nrm[1] = __dsub_rn(__dmul_rn(d1[2], d2[0]), __dmul_rn(d1[0], d2[2]));
      nrm[2] = __dsub_rn(__dmul_rn(d1[0], d2[1]), __dmul_rn(d1[1], d2[0]));
      const double nn = norm3(nrm);
      for (int j = 0; j < 3; j++)
        nrm[j] = __ddiv_rn(nrm[j], nn);
      double pf[3], nc[3];
      for (int r = 0; r < 3; r++) {
        pf[r] = R[3 * r] * (p1[0] - pc[0]) + R[3 * r + 1] * (p1[1] - pc[1]) + R[3 * r + 2] * (p1[2] - pc[2]);
        nc[r] = R[3 * r] * nrm[0] + R[3 * r + 1] * nrm[1] + R[3 * r + 2] * nrm[2];
      }
      if (dot3(nc, pf) < 0)
        for (int j = 0; j < 3; j++)
          nrm[j] = -nrm[j];
    }
    D.tacc[t] = ok;
    for (int j = 0; j < 3; j++)
      D.tnorm[3 * t + j] = nrm[j];
  }
  __syncthreads();
  for (int v = tid; v < m; v += THREADS) {
    const int s = F.slot[surv[v]] & 0x3fffffff;
    double *w = D.win + 3 * WCAP * s;
    int len = D.wlen[s];
    for (int k = D.inc_off[v]; k < D.inc_off[v + 1]; k++) {
      const int t = D.inc_list[k];
      if (!D.tacc[t])
        continue;
      if (len == o.max_norm_count) { // keep the newest max_norm_count
        for (int q = 0; q < 3 * (len - 1); q++)
          w[q] = w[q + 3];
        len--;
      }
      for (int j = 0; j < 3; j++)
        w[3 * len + j] = D.tnorm[3 * t + j];
      len++;
    }
    D.wlen[s] = len;
    avg_norm(w, len, o, D.avg + 3 * v);
    done[v] = 0;
  }
  __syncthreads();

  // ---- 5: matching and merging, serial in ascending id (:816-979) ----
  if (tid < 32 && ntri > 0) {
    const int lane = tid;
    for (int a = 0; a < n; a++) {
      const int fi = F.asc[a], v = sidx[fi];
      if (v < 0)
        continue;
      const int s = F.slot[fi] & 0x3fffffff;
      const int wl = D.wlen[s];
      if (wl == 0 || wl < o.min_norms) // a feature without a window has no entry in hist_feat_norms_inG
        continue;
      const double *nv = D.avg + 3 * v;
      if (norm3(nv) <= 0)
        continue;
      const double *pf = D.inG + 3 * s;
      const double d = dot3(pf, nv);
      if (!o.check_old_feats && D.label[s] >= 0)
        continue;
      if (D.inc_off[v + 1] == D.inc_off[v])
        continue;
      // the neighbours through every triangle (lane 0; duplicates are harmless: a second match changes nothing)
      int *s_match = D.match;
      __shared__ int s_nmatch;
      if (lane == 0) {
        int nm = 0;
        for (int k = D.inc_off[v]; k < D.inc_off[v + 1]; k++) {
          const int t = D.inc_list[k];
          for (int j = 0; j < 3; j++) {
            const int g = D.tri[3 * t + j];
            if (g == v)
              continue;
            const int sg = F.slot[surv[g]] & 0x3fffffff;
            const int wg = D.wlen[sg];
            if (wg == 0 || wg < o.min_norms)
              continue;
            const double *ng = D.avg + 3 * g;
            if (norm3(ng) <= 0 || done[g])
              continue;
            if (px_dist(F.uv[fi], F.uv[surv[g]]) > (double)o.max_pairwise_px)
              continue;
            const double plane_dist = __dsub_rn(dot3(D.inG + 3 * sg, nv), d);
            const double angle = __dmul_rn(180.0 / M_PI, acos(dot3(nv, ng)));
            if (!isnan(angle) && angle < o.max_norm_deg && fabs(plane_dist) < o.max_dist_between_z) {
              bool dup = false;
              for (int q = 0; q < nm; q++)
                dup |= s_match[q] == sg;
              if (!dup)
                s_match[nm++] = sg;
            }
          }
        }
        s_nmatch = nm;
      }
      __syncwarp();
      const int nm = s_nmatch;
      if (nm == 0)
        continue;
      long long minp = D.label[s];
      for (int q = 0; q < nm; q++) {
        const long long lg = D.label[s_match[q]];
        if (lg >= 0 && (minp < 0 || lg < minp))
          minp = lg;
      }
      if (minp >= 0) {
        // each old label is read by lane 0 and broadcast: the sweep of relabel() writes the slots the lanes would otherwise read
        for (int q = 0; q <= nm; q++) {
          const int sq = q < nm ? s_match[q] : s;
          const long long lg = __shfl_sync(0xffffffffu, lane == 0 ? D.label[sq] : 0ll, 0);
          if (lg >= 0)
            relabel(D, F, minp, lg, lane);
        }
        if (lane == 0) {
          for (int q = 0; q < nm; q++)
            D.label[s_match[q]] = minp;
          D.label[s] = minp;
          done[v] = 1;
        }
      } else if (lane == 0) {
        const long long id = ++D.planeid_ctr[0];
        for (int q = 0; q < nm; q++)
          D.label[s_match[q]] = id;
        D.label[s] = id;
      }
      __syncwarp();
    }
  }
  __syncthreads();

  // ---- 6: spatial filter (:989-1058) ----
  // every active feature (a survivor with a plane): its plane's member count and first member in ascending id, its k-NN mean distance
  for (int v = tid; v < m; v += THREADS) {
    const int s = F.slot[surv[v]] & 0x3fffffff;
    const long long lp = D.label[s];
    D.knn[v] = 0.0;
    if (lp < 0)
      continue;
    int members = 0;
    for (int u = 0; u < m; u++)
      members += D.label[F.slot[surv[u]] & 0x3fffffff] == lp;
    if (members <= o.filter_num_feat)
      continue;
    const float x = (float)D.inG[3 * s], y = (float)D.inG[3 * s + 1], z = (float)D.inG[3 * s + 2];
    float best[KCAP];
    int nb = 0;
    for (int u = 0; u < m; u++) {
      if (u == v)
        continue;
      const int su = F.slot[surv[u]] & 0x3fffffff;
      if (D.label[su] != lp)
        continue;
      const float dx = __fsub_rn(x, (float)D.inG[3 * su]), dy = __fsub_rn(y, (float)D.inG[3 * su + 1]), dz = __fsub_rn(z, (float)D.inG[3 * su + 2]);
      const float dd = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)); // ikd-tree's calc_dist, unfused
      if (nb == o.filter_num_feat && !(dd < best[nb - 1]))
        continue;
      int q = nb < o.filter_num_feat ? nb++ : nb - 1;
      while (q > 0 && best[q - 1] > dd) {
        best[q] = best[q - 1];
        q--;
      }
      best[q] = dd;
    }
    double acc = 0.0;
    for (int q = 0; q < nb; q++)
      acc += (double)best[q];
    D.knn[v] = acc / (double)nb;
  }
  __syncthreads();
  // the plane's mean and n - 1 standard deviation at its first member in ascending id, summed in ascending id
  for (int v = tid; v < m; v += THREADS) {
    const long long lp = D.label[F.slot[surv[v]] & 0x3fffffff];
    if (lp < 0)
      continue;
    int cntp = 0, rep = -1;
    double sum = 0.0;
    for (int a = 0; a < n; a++) {
      const int fj = F.asc[a];
      if (sidx[fj] < 0 || D.label[F.slot[fj] & 0x3fffffff] != lp)
        continue;
      if (rep < 0)
        rep = sidx[fj];
      sum += D.knn[sidx[fj]];
      cntp++;
    }
    if (rep != v || cntp <= o.filter_num_feat)
      continue;
    const double mean = sum / (double)cntp;
    double ss = 0.0;
    for (int a = 0; a < n; a++) {
      const int fj = F.asc[a];
      if (sidx[fj] < 0 || D.label[F.slot[fj] & 0x3fffffff] != lp)
        continue;
      const double e = D.knn[sidx[fj]] - mean;
      ss += e * e;
    }
    D.zstat[2 * v] = mean;
    D.zstat[2 * v + 1] = sqrt(ss / ((double)cntp - 1));
  }
  __syncthreads();
  // z-test: find the plane's first member again, drop the features above the threshold
  for (int v = tid; v < m; v += THREADS) {
    const int s = F.slot[surv[v]] & 0x3fffffff;
    const long long lp = D.label[s];
    stack[v] = 0;
    if (lp < 0)
      continue;
    int rep = -1, members = 0;
    for (int a = 0; a < n; a++) {
      const int fj = F.asc[a];
      if (sidx[fj] < 0 || D.label[F.slot[fj] & 0x3fffffff] != lp)
        continue;
      if (rep < 0)
        rep = sidx[fj];
      members++;
    }
    if (members <= o.filter_num_feat)
      continue;
    const double sigma = fabs(D.knn[v] - D.zstat[2 * rep]) / D.zstat[2 * rep + 1];
    stack[v] = sigma > o.filter_z_thresh; // erase after every plane has been read
  }
  __syncthreads();
  for (int v = tid; v < m; v += THREADS)
    if (stack[v])
      D.label[F.slot[surv[v]] & 0x3fffffff] = -1;
  __syncthreads();

  // ---- 7: keep the frame's planes with more than 3 active features, and their merge history (:1064-1095) ----
  for (int v = tid; v < m; v += THREADS) {
    const long long lp = D.label[F.slot[surv[v]] & 0x3fffffff];
    int members = 0;
    if (lp >= 0)
      for (int u = 0; u < m; u++)
        members += D.label[F.slot[surv[u]] & 0x3fffffff] == lp;
    stack[v] = lp >= 0 && members > 3;
  }
  __syncthreads();
  for (int i = tid; i < n; i += THREADS) // features with no 3D estimate lose their entry
    if (sidx[i] < 0)
      D.label[F.slot[i] & 0x3fffffff] = -1;
  for (int k = tid; k < F.nstale; k += THREADS)
    D.label[F.stale[k]] = -1;
  const int np = D.npair[0];
  for (int k = tid; k < np; k += THREADS) { // owner of each pair still a kept plane?
    bool keep = false;
    for (int v = 0; v < m && !keep; v++)
      keep = stack[v] && D.label[F.slot[surv[v]] & 0x3fffffff] == D.pair_owner[k];
    if (!keep)
      D.pair_owner[k] = -1;
  }
  __syncthreads();
  for (int v = tid; v < m; v += THREADS)
    if (!stack[v])
      D.label[F.slot[surv[v]] & 0x3fffffff] = -1;
  __syncthreads();
  if (tid == 0) {
    int w = 0;
    for (int k = 0; k < np; k++)
      if (D.pair_owner[k] >= 0) {
        D.pair_old[w] = D.pair_old[k];
        D.pair_owner[w] = D.pair_owner[k];
        w++;
      }
    D.npair[0] = w;
  }
  for (int i = tid; i < n; i += THREADS)
    D.frame_label[i] = D.label[F.slot[i] & 0x3fffffff];
  for (int v = tid; v < m; v += THREADS)
    D.surv[1 + v] = surv[v];
  if (tid == 0)
    D.surv[0] = m;
}

constexpr size_t smem_bytes() {
  return sizeof(float2) * (NMAX + 3) + sizeof(int) * (6 * TMAX + TMAX + 8 + 2 * NMAX) + NMAX;
}

} // namespace ptrack

// host side of one context's tracker
struct PlaneTrack {
  bool has_opt = false, started = false, attr_set = false;
  ovp_plane_track_options opt;
  std::unordered_map<int64_t, int> slot_of; // the features of the last frame
  std::vector<int> free_slots;
  std::vector<int64_t> last_ids;            // the last frame's featids, in its order
  std::vector<float> last_uv;               // and its pixels
  int nslot = 0;                            // slots ever used (hi-water mark)
  ptrack::Dev d = {};
  void *dmem = nullptr;
};

static void plane_track_defaults(ovp_plane_track_options &o) {
  o.max_tri_side_px = 200;
  o.max_norm_count = 5;
  o.max_norm_avg_max = 25.0;
  o.max_norm_avg_var = 25.0;
  o.max_norm_deg = 25.0;
  o.max_dist_between_z = 0.10;
  o.max_pairwise_px = 100;
  o.min_norms = 3;
  o.check_old_feats = 1;
  o.filter_num_feat = 4;
  o.filter_z_thresh = 1.2;
  o.feat_init_min_obs = 4;
  o.min_dist = 0.10;
  o.max_dist = 60;
  o.max_cond_number = 8000;
}

static int plane_track_alloc(Ctx *c, PlaneTrack *pt) {
  using namespace ptrack;
  const size_t nd = (size_t)NSLOT * (9 + 3 + 3 + 3 * WCAP) + 3 * TMAX + 3 * NMAX + NMAX + 2 * NMAX;
  const size_t nl = (size_t)NSLOT + 2 * PCAP + 1 + NMAX;
  const size_t ni = (size_t)3 * NSLOT + 2 + 1 + 3 * TMAX + (NMAX + 1) + 3 * TMAX + TMAX + NMAX + NMAX + 1;
  const size_t bytes = nd * 8 + nl * 8 + ni * 4;
  OVP_CUDA(cudaMalloc(&pt->dmem, bytes));
  OVP_CUDA(cudaMemsetAsync(pt->dmem, 0, bytes, c->stream));
  double *pd = (double *)pt->dmem;
  Dev &D = pt->d;
  D.A = pd, pd += (size_t)9 * NSLOT;
  D.b = pd, pd += (size_t)3 * NSLOT;
  D.inG = pd, pd += (size_t)3 * NSLOT;
  D.win = pd, pd += (size_t)3 * WCAP * NSLOT;
  D.tnorm = pd, pd += 3 * TMAX;
  D.avg = pd, pd += 3 * NMAX;
  D.knn = pd, pd += NMAX;
  D.zstat = pd, pd += 2 * NMAX;
  long long *pl = (long long *)pd;
  D.label = pl, pl += NSLOT;
  D.pair_old = pl, pl += PCAP;
  D.pair_owner = pl, pl += PCAP;
  D.planeid_ctr = pl, pl += 1;
  D.frame_label = pl, pl += NMAX;
  int *pi = (int *)pl;
  D.cnt = pi, pi += NSLOT;
  D.has = pi, pi += NSLOT;
  D.wlen = pi, pi += NSLOT;
  D.npair = pi, pi += 2;
  D.ntri = pi, pi += 1;
  D.tri = pi, pi += 3 * TMAX;
  D.inc_off = pi, pi += NMAX + 1;
  D.inc_list = pi, pi += 3 * TMAX;
  D.tacc = pi, pi += TMAX;
  D.match = pi, pi += NMAX;
  D.surv = pi, pi += NMAX + 1;
  OVP_CUDA(cudaMemsetAsync(D.label, 0xff, sizeof(long long) * NSLOT, c->stream)); // no plane
  return OVP_OK;
}

void plane_track_free(Ctx *c) {
  if (!c->ptrack)
    return;
  cudaFree(c->ptrack->dmem);
  delete c->ptrack;
  c->ptrack = nullptr;
}

static PlaneTrack *tracker(Ctx *c) {
  if (!c->ptrack)
    c->ptrack = new PlaneTrack();
  return c->ptrack;
}

// the readbacks below see every frame enqueued before them; a merge history that outgrew its capacity fails them
static int plane_track_check(Ctx *c, PlaneTrack *pt) {
  int np[2] = {0, 0};
  int st;
  if ((st = stage_copy_out(c, np, pt->d.npair, sizeof(np))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  if (np[1])
    return fail(c, OVP_ERR_CAPACITY, "plane tracker: merge history above %d pairs", OVP_PLANE_TRACK_MAX_MERGES);
  return OVP_OK;
}

} // namespace ovp

using namespace ovp;

extern "C" {

int ovp_plane_track_set_options(ovp_ctx *h, const ovp_plane_track_options *opt) {
  Ctx *c = ovp::enter(h);
  PlaneTrack *pt = tracker(c);
  if (pt->started)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_set_options: the tracker has already run a frame");
  ovp_plane_track_options o;
  if (opt)
    o = *opt;
  else
    plane_track_defaults(o);
  const double d[] = {o.max_norm_avg_max, o.max_norm_avg_var, o.max_norm_deg, o.max_dist_between_z, o.filter_z_thresh, o.min_dist,
                      o.max_dist, o.max_cond_number};
  for (double v : d)
    if (std::isnan(v))
      return fail(c, OVP_ERR_BAD_ARGS, "plane_track_set_options: NaN threshold");
  if (o.max_norm_count < 1 || o.max_norm_count > OVP_PLANE_TRACK_MAX_NORM_COUNT)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_set_options: max_norm_count %d outside 1..%d", o.max_norm_count,
                OVP_PLANE_TRACK_MAX_NORM_COUNT);
  if (o.filter_num_feat <= 1 || o.filter_num_feat > OVP_PLANE_TRACK_MAX_FILTER_FEAT)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_set_options: filter_num_feat %d outside 2..%d", o.filter_num_feat,
                OVP_PLANE_TRACK_MAX_FILTER_FEAT);
  if ((o.check_old_feats != 0 && o.check_old_feats != 1) || o.feat_init_min_obs < 1)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_set_options: check_old_feats must be 0 / 1 and feat_init_min_obs >= 1");
  pt->opt = o;
  pt->has_opt = true;
  return OVP_OK;
}

int ovp_plane_track_frame(ovp_ctx *h, const double pose_GtoI7[7], const double calib7[7], int n, const int64_t *featid, const float *uv,
                          const float *uv_norm) {
  using namespace ptrack;
  Ctx *c = ovp::enter(h);
  PlaneTrack *pt = tracker(c);
  if (!pt->has_opt)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_frame: call ovp_plane_track_set_options first");
  if (n == 0)
    return OVP_OK;
  if (n < 0 || n > NMAX)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_frame: n = %d outside 0..%d", n, NMAX);
  if (!pose_GtoI7 || !calib7 || !featid || !uv || !uv_norm)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_frame: null pointer");
  {
    std::unordered_set<int64_t> ids;
    std::unordered_set<uint64_t> px;
    for (int i = 0; i < n; i++) {
      if (featid[i] < 0 || !ids.insert(featid[i]).second)
        return fail(c, OVP_ERR_BAD_ARGS, "plane_track_frame: featid %lld negative or given twice", (long long)featid[i]);
      float u = uv[2 * i], v = uv[2 * i + 1];
      if (!std::isfinite(u) || !std::isfinite(v)) // CDT throws: no triangle holds such a point
        return fail(c, OVP_ERR_BAD_ARGS, "plane_track_frame: featid %lld has a non-finite pixel", (long long)featid[i]);
      u = u == 0.0f ? 0.0f : u; // -0 and +0 are the same pixel
      v = v == 0.0f ? 0.0f : v;
      uint32_t bu, bv;
      memcpy(&bu, &u, 4);
      memcpy(&bv, &v, 4);
      if (!px.insert(((uint64_t)bu << 32) | bv).second)
        return fail(c, OVP_ERR_BAD_ARGS, "plane_track_frame: two features on pixel (%g, %g)", u, v);
    }
  }
  int st;
  if (!pt->dmem && (st = plane_track_alloc(c, pt)))
    return st;
  if (!pt->attr_set) {
    OVP_CUDA(cudaFuncSetAttribute(plane_track_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
    pt->attr_set = true;
  }
  // slots: the frame's features keep theirs, new ones take free ones (fresh: reset on the device); the last frame's features that left
  // keep theirs through this frame (their plane labels still take part in the relabelling) and are freed after it
  // built in locals, committed once the frame has run
  std::vector<int> slot(n), stale, free_slots = pt->free_slots;
  int nslot = pt->nslot;
  std::unordered_map<int64_t, int> next;
  next.reserve(2 * n);
  std::vector<int> order(n);
  for (int i = 0; i < n; i++)
    order[i] = i;
  std::sort(order.begin(), order.end(), [&](int a, int b) { return featid[a] < featid[b]; });
  std::unordered_set<int64_t> cur(featid, featid + n);
  for (int64_t id : pt->last_ids)
    if (!cur.count(id))
      stale.push_back(pt->slot_of.at(id));
  for (int i = 0; i < n; i++) {
    auto it = pt->slot_of.find(featid[i]);
    if (it != pt->slot_of.end()) {
      slot[i] = it->second;
    } else {
      int s;
      if (!free_slots.empty()) {
        s = free_slots.back();
        free_slots.pop_back();
      } else {
        s = nslot++;
      }
      slot[i] = s | 0x40000000;
    }
    next[featid[i]] = slot[i] & 0x3fffffff;
  }
  StageLayout L;
  const size_t o_pose = L.take(14 * sizeof(double)), o_slot = L.take(n * sizeof(int)), o_uv = L.take(n * sizeof(float2)),
               o_uvn = L.take(n * sizeof(float2)), o_asc = L.take(n * sizeof(int)), o_stale = L.take(stale.size() * sizeof(int));
  std::vector<unsigned char> hbuf(L.top);
  memcpy(hbuf.data() + o_pose, pose_GtoI7, 7 * sizeof(double));
  memcpy(hbuf.data() + o_pose + 7 * sizeof(double), calib7, 7 * sizeof(double));
  memcpy(hbuf.data() + o_slot, slot.data(), n * sizeof(int));
  memcpy(hbuf.data() + o_uv, uv, n * sizeof(float2));
  memcpy(hbuf.data() + o_uvn, uv_norm, n * sizeof(float2));
  memcpy(hbuf.data() + o_asc, order.data(), n * sizeof(int));
  if (!stale.empty())
    memcpy(hbuf.data() + o_stale, stale.data(), stale.size() * sizeof(int));
  if ((st = ensure_stage(c, L)))
    return st;
  if ((st = stage_copy_in(c, c->d_stage, hbuf.data(), L.top)))
    return st;
  FrameArgs F;
  F.pose = (const double *)(c->d_stage + o_pose);
  F.slot = (const int *)(c->d_stage + o_slot);
  F.uv = (const float2 *)(c->d_stage + o_uv);
  F.uvn = (const float2 *)(c->d_stage + o_uvn);
  F.asc = (const int *)(c->d_stage + o_asc);
  F.stale = (const int *)(c->d_stage + o_stale);
  F.n = n;
  F.nstale = (int)stale.size();
  F.nslot = nslot;
  plane_track_kernel<<<1, THREADS, smem_bytes(), c->stream>>>(pt->d, F, pt->opt);
  c->launches++;
  OVP_CUDA(cudaGetLastError());
  OVP_CUDA(cudaStreamSynchronize(c->stream)); // the host buffer is staged from pageable memory; the next frame reuses the staging area
  for (int s : stale)
    free_slots.push_back(s);
  pt->free_slots.swap(free_slots);
  pt->nslot = nslot;
  pt->slot_of.swap(next);
  pt->last_ids.assign(featid, featid + n);
  pt->last_uv.assign(uv, uv + 2 * (size_t)n);
  pt->started = true;
  return OVP_OK;
}

int ovp_plane_track_feature2plane(ovp_ctx *h, int cap, int64_t *featid, int64_t *planeid, int *n) {
  Ctx *c = ovp::enter(h);
  PlaneTrack *pt = tracker(c);
  if (!n || (cap > 0 && (!featid || !planeid)))
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_feature2plane: null pointer");
  *n = 0;
  if (!pt->started)
    return OVP_OK;
  int st;
  if ((st = plane_track_check(c, pt)))
    return st;
  const int nf = (int)pt->last_ids.size();
  std::vector<long long> lab(nf);
  if ((st = stage_copy_out(c, lab.data(), pt->d.frame_label, nf * sizeof(long long))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  std::vector<std::pair<int64_t, int64_t>> out;
  for (int i = 0; i < nf; i++)
    if (lab[i] >= 0)
      out.push_back({pt->last_ids[i], (int64_t)lab[i]});
  std::sort(out.begin(), out.end());
  *n = (int)out.size();
  if ((int)out.size() > cap)
    return fail(c, OVP_ERR_CAPACITY, "plane_track_feature2plane: %d entries, cap %d", (int)out.size(), cap);
  for (size_t k = 0; k < out.size(); k++)
    featid[k] = out[k].first, planeid[k] = out[k].second;
  return OVP_OK;
}

int ovp_plane_track_plane2oldplane(ovp_ctx *h, int cap, int64_t *planeid, int64_t *oldplaneid, int *n) {
  Ctx *c = ovp::enter(h);
  PlaneTrack *pt = tracker(c);
  if (!n || (cap > 0 && (!planeid || !oldplaneid)))
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_plane2oldplane: null pointer");
  *n = 0;
  if (!pt->started)
    return OVP_OK;
  int np[2] = {0, 0};
  int st;
  if ((st = stage_copy_out(c, np, pt->d.npair, sizeof(np))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  if (np[1])
    return fail(c, OVP_ERR_CAPACITY, "plane tracker: merge history above %d pairs", OVP_PLANE_TRACK_MAX_MERGES);
  std::vector<long long> po(np[0]), pw(np[0]);
  if ((st = stage_copy_out(c, po.data(), pt->d.pair_old, np[0] * sizeof(long long))) ||
      (st = stage_copy_out(c, pw.data(), pt->d.pair_owner, np[0] * sizeof(long long))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  std::vector<std::pair<int64_t, int64_t>> out(np[0]);
  for (int k = 0; k < np[0]; k++)
    out[k] = {(int64_t)pw[k], (int64_t)po[k]};
  std::sort(out.begin(), out.end());
  *n = np[0];
  if (np[0] > cap)
    return fail(c, OVP_ERR_CAPACITY, "plane_track_plane2oldplane: %d pairs, cap %d", np[0], cap);
  for (int k = 0; k < np[0]; k++)
    planeid[k] = out[k].first, oldplaneid[k] = out[k].second;
  return OVP_OK;
}

int ovp_plane_track_mesh(ovp_ctx *h, int cap, int *tri3, double *normal3, int *n_tri) {
  Ctx *c = ovp::enter(h);
  PlaneTrack *pt = tracker(c);
  if (!n_tri)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_mesh: null pointer");
  *n_tri = 0;
  if (!pt->started)
    return OVP_OK;
  int nt = 0, st;
  if ((st = stage_copy_out(c, &nt, pt->d.ntri, sizeof(int))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  *n_tri = nt;
  if (nt > cap && (tri3 || normal3))
    return fail(c, OVP_ERR_CAPACITY, "plane_track_mesh: %d triangles, cap %d", nt, cap);
  if (tri3 && (st = stage_copy_out(c, tri3, pt->d.tri, (size_t)3 * nt * sizeof(int))))
    return st;
  if (normal3 && (st = stage_copy_out(c, normal3, pt->d.tnorm, (size_t)3 * nt * sizeof(double))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  return OVP_OK;
}

int ovp_plane_track_vertices(ovp_ctx *h, int cap, int64_t *featid, float *uv, int *n) {
  Ctx *c = ovp::enter(h);
  PlaneTrack *pt = tracker(c);
  if (!n || (cap > 0 && (!featid || !uv)))
    return fail(c, OVP_ERR_BAD_ARGS, "plane_track_vertices: null pointer");
  *n = 0;
  if (!pt->started)
    return OVP_OK;
  std::vector<int> sv(pt->last_ids.size() + 1);
  int st;
  if ((st = stage_copy_out(c, sv.data(), pt->d.surv, sizeof(int))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  const int m = sv[0];
  *n = m;
  if (m > cap)
    return fail(c, OVP_ERR_CAPACITY, "plane_track_vertices: %d vertices, cap %d", m, cap);
  if ((st = stage_copy_out(c, sv.data() + 1, pt->d.surv + 1, (size_t)m * sizeof(int))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  for (int k = 0; k < m; k++) {
    const int i = sv[1 + k];
    featid[k] = pt->last_ids[i];
    uv[2 * k] = pt->last_uv[2 * i];
    uv[2 * k + 1] = pt->last_uv[2 * i + 1];
  }
  return OVP_OK;
}

#ifdef OVP_DEBUG
int ovp_debug_plane_track_history(ovp_ctx *h, int n, const int64_t *featid, double *out) {
  using namespace ptrack;
  Ctx *c = ovp::enter(h);
  PlaneTrack *pt = tracker(c);
  if (n < 0 || (n > 0 && (!featid || !out)))
    return fail(c, OVP_ERR_BAD_ARGS, "debug_plane_track_history: bad arguments");
  std::fill(out, out + (size_t)n * HIST, 0.0);
  if (!pt->dmem)
    return OVP_OK;
  const int ns = std::max(pt->nslot, 1);
  std::vector<double> A(9 * ns), b(3 * ns), p(3 * ns), w((size_t)3 * WCAP * ns);
  std::vector<int> cnt(ns), has(ns), wl(ns);
  int st;
  const Dev &D = pt->d;
  if ((st = stage_copy_out(c, A.data(), D.A, A.size() * 8)) || (st = stage_copy_out(c, b.data(), D.b, b.size() * 8)) ||
      (st = stage_copy_out(c, p.data(), D.inG, p.size() * 8)) || (st = stage_copy_out(c, w.data(), D.win, w.size() * 8)) ||
      (st = stage_copy_out(c, cnt.data(), D.cnt, ns * 4)) || (st = stage_copy_out(c, has.data(), D.has, ns * 4)) ||
      (st = stage_copy_out(c, wl.data(), D.wlen, ns * 4)))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < n; i++) {
    auto it = pt->slot_of.find(featid[i]);
    if (it == pt->slot_of.end())
      continue;
    const int s = it->second;
    double *o = out + (size_t)i * HIST;
    std::copy(&A[9 * s], &A[9 * s] + 9, o);
    std::copy(&b[3 * s], &b[3 * s] + 3, o + 9);
    o[12] = cnt[s];
    o[13] = has[s];
    std::copy(&p[3 * s], &p[3 * s] + 3, o + 14);
    o[17] = wl[s];
    std::copy(&w[(size_t)3 * WCAP * s], &w[(size_t)3 * WCAP * s] + 3 * wl[s], o + 18);
  }
  return OVP_OK;
}
#endif

} // extern "C"

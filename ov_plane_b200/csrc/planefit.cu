// PlaneFitting on the device: the plane hypotheses / refinement the updaters call right before they build Jacobians
// (reference: ov_plane/src/track_plane/PlaneFitting.cpp; call sites UpdaterMSCKF.cpp:267-360, UpdaterPlane.cpp:230-267, UpdaterSLAM.cpp:171).
//
//   ovp_plane_fitting   = PlaneFitting::plane_fitting (:83-195) for a BATCH of candidate planes.  The reference draws 200 five-point sets one
//     after the other with std::shuffle(std::mt19937(8888)); the draws do not depend on the fits, so the 200 permutations are produced on the
//     host (they depend only on the number of points: cached per size) and the 200 hypotheses of every plane are evaluated concurrently, one warp
//     per hypothesis: greedy minimum-distance selection, 5 x 3 condition check + least squares, inlier count over all points.  A second launch
//     picks the winner exactly like the sequential loop (more inliers, then smaller mean error, then the earlier draw) and refits it.
//   ovp_optimize_plane  = PlaneFitting::optimize_plane (:197-514).  The reference hands the problem to Ceres (DENSE_SCHUR + DOGLEG, Cauchy loss,
//     12 iterations).  Ceres is not part of the reference tree (libceres-dev 1.14, package.xml:47); the algorithm of its TrustRegionMinimizer +
//     DoglegStrategy is restated here as ONE kernel launch per batch of planes: a CTA per plane; the residual / Jacobian pass runs a warp per feature (lane = measurement), the 3 x 3 algebra a thread per feature.  Every free feature is a
//     3 x 3 block that only couples to the 3 plane parameters, so the whole iteration (Jacobi scaling, gradient, Cauchy point, regularised
//     Gauss-Newton step through the Schur complement on the plane, dogleg interpolation, model / true cost change, radius and mu updates,
//     the three convergence tests) runs on per-feature normal-equation blocks plus a handful of block reductions - no Jacobian rows are stored,
//     nothing returns to the host between iterations.
// std::shuffle / std::uniform_int_distribution are implementation-defined; libstdc++'s two variants are restated (shuffle_kind) so that the
// draws do not depend on the compiler that builds this library (the reference's Docker images use GCC 7 / 9 = the classic variant).
#include <cfloat>
#include <cstring>
#include <map>
#include <mutex>

namespace ovp {

// ---- host: std::mt19937 + libstdc++ std::shuffle, restated ----------------------------------------------------------------------------
struct Mt19937 {
  uint32_t s[624];
  int idx;
  explicit Mt19937(uint32_t seed) {
    s[0] = seed;
    for (int i = 1; i < 624; i++)
      s[i] = 1812433253u * (s[i - 1] ^ (s[i - 1] >> 30)) + (uint32_t)i;
    idx = 624;
  }
  uint32_t next() {
    if (idx >= 624) {
      for (int i = 0; i < 624; i++) {
        const uint32_t y = (s[i] & 0x80000000u) | (s[(i + 1) % 624] & 0x7fffffffu);
        s[i] = s[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
      }
      idx = 0;
    }
    uint32_t y = s[idx++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
  }
};
static uint64_t pf_uniform_below(Mt19937 &g, uint64_t n, int kind) { // uniform_int_distribution<unsigned long>{0, n - 1}(g), n <= 2^32
  if (kind == 1) {                                                    // GCC >= 11: Lemire's nearly divisionless method on 32-bit draws
    const uint32_t range = (uint32_t)n;
    uint64_t product = (uint64_t)g.next() * (uint64_t)range;
    uint32_t low = (uint32_t)product;
    if (low < range) {
      const uint32_t threshold = (uint32_t)(0u - range) % range;
      while (low < threshold) {
        product = (uint64_t)g.next() * (uint64_t)range;
        low = (uint32_t)product;
      }
    }
    return product >> 32;
  }
  const uint64_t scaling = 0xFFFFFFFFull / n, past = n * scaling; // GCC <= 10: down-scaling with rejection
  uint64_t ret;
  do
    ret = (uint64_t)g.next();
  while (ret >= past);
  return ret / scaling;
}
static void pf_shuffle(int *v, int n, Mt19937 &g, int kind) { // libstdc++ std::shuffle: two swap positions per draw while n^2 fits the generator
  if (n == 0)
    return;
  if (0xFFFFFFFFull / (uint64_t)n >= (uint64_t)n) {
    int i = 1;
    if ((n % 2) == 0) {
      std::swap(v[i], v[pf_uniform_below(g, 2, kind)]);
      i++;
    }
    while (i != n) {
      const uint64_t r = (uint64_t)i + 1;
      const uint64_t x = pf_uniform_below(g, r * (r + 1), kind);
      std::swap(v[i], v[x / (r + 1)]);
      i++;
      std::swap(v[i], v[x % (r + 1)]);
      i++;
    }
    return;
  }
  for (int i = 1; i < n; i++)
    std::swap(v[i], v[pf_uniform_below(g, (uint64_t)i + 1, kind)]);
}

#define PF_HYP 200            // max_iter_num (PlaneFitting.cpp:88)
#define PF_SET 5              // ransac_solver_feat_num (:87)
#define PF_MAX_POINTS 1900    // points of one candidate plane (shared-memory staging: 24 bytes each + the warps' work rows <= 48 KB)
#define PF_WARPS 8

struct PfHyp { // result of one draw
  int state;   // 0 fit rejected, 1 candidate (counts below valid), 2 fewer than 5 separated points (the reference returns false outright)
  int count;
  double avg;
  double abcd[4];
};

__device__ __forceinline__ double pf_warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1)
    v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// Least squares [A | b] (K rows x 4, row-major in shared or local memory, overwritten) -> x (3) by Householder QR with column pivoting,
// executed by ONE warp (rows strided over the lanes).  Eigen::ColPivHouseholderQR::solve (PlaneFitting.cpp:70).
__device__ void pf_warp_lstsq3(double *Ab, int K, double *x) {
  const int lane = threadIdx.x & 31;
  int perm[3] = {0, 1, 2};
  for (int j = 0; j < 3; j++) {
    double nrm[3] = {0.0, 0.0, 0.0};
    for (int i = j + lane; i < K; i += 32)
      for (int c = j; c < 3; c++)
        nrm[c] += Ab[4 * i + c] * Ab[4 * i + c];
    int best = j;
    double bn = -1.0;
    for (int c = j; c < 3; c++) {
      nrm[c] = pf_warp_sum(nrm[c]);
      if (nrm[c] > bn) {
        bn = nrm[c];
        best = c;
      }
    }
    if (best != j) {
      for (int i = lane; i < K; i += 32) {
        const double t = Ab[4 * i + j];
        Ab[4 * i + j] = Ab[4 * i + best];
        Ab[4 * i + best] = t;
      }
      const int t = perm[j];
      perm[j] = perm[best];
      perm[best] = t;
      __syncwarp();
    }
    const double sigma = sqrt(bn);
    if (sigma == 0.0)
      continue;
    const double ajj = Ab[4 * j + j];
    const double alpha = (ajj > 0.0) ? -sigma : sigma;
    // v = column j below the diagonal with v_j = a_jj - alpha; |v|^2 = 2 sigma (sigma + |a_jj|)
    const double vj = ajj - alpha, vn = sigma * sigma - ajj * ajj + vj * vj;
    if (vn == 0.0)
      continue;
    double dots[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = j + lane; i < K; i += 32) {
      const double vi = (i == j) ? vj : Ab[4 * i + j];
      for (int c = j + 1; c < 4; c++)
        dots[c] += vi * Ab[4 * i + c];
    }
    for (int c = j + 1; c < 4; c++)
      dots[c] = 2.0 * pf_warp_sum(dots[c]) / vn;
    __syncwarp();
    for (int i = j + lane; i < K; i += 32) {
      const double vi = (i == j) ? vj : Ab[4 * i + j];
      for (int c = j + 1; c < 4; c++)
        Ab[4 * i + c] -= dots[c] * vi;
    }
    __syncwarp();
    if (lane == 0)
      Ab[4 * j + j] = alpha;
    __syncwarp();
  }
  double y[3];
  for (int j = 2; j >= 0; j--) {
    double s = Ab[4 * j + 3];
    for (int c = j + 1; c < 3; c++)
      s -= Ab[4 * j + c] * y[c];
    y[j] = s / Ab[4 * j + j];
  }
  for (int j = 0; j < 3; j++)
    x[perm[j]] = y[j];
  __syncwarp();
}
// abcd from the least-squares normal (PlaneFitting.cpp:70-80); returns cp.norm() > 0.02
__device__ __forceinline__ bool pf_finish_plane(const double *n, double *abcd) {
  const double nn = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  abcd[0] = n[0] / nn;
  abcd[1] = n[1] / nn;
  abcd[2] = n[2] / nn;
  abcd[3] = 1.0 / nn;
  const double cpn = fabs(abcd[3]) * sqrt(abcd[0] * abcd[0] + abcd[1] * abcd[1] + abcd[2] * abcd[2]);
  return cpn > 0.02;
}

// grid (ceil(200 / 8), planes), 8 warps: one warp per draw
__global__ void __launch_bounds__(32 * PF_WARPS) plane_ransac_kernel(const int *feat_offset, const double *pts, const int *perm_base, const int *perm_offset,
                                                                      double max_cond, PfHyp *hyp) {
  extern __shared__ double sm_pts[]; // F x 3, then 8 x (5 x 4) work rows
  const int plane = blockIdx.y, f0 = feat_offset[plane], F = feat_offset[plane + 1] - f0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, h = blockIdx.x * PF_WARPS + warp;
  for (int i = threadIdx.x; i < 3 * F; i += blockDim.x)
    sm_pts[i] = pts[3 * (size_t)f0 + i];
  __syncthreads();
  if (h >= PF_HYP || F == 0)
    return;
  double *Ab = sm_pts + 3 * (size_t)F + 20 * warp;
  const int *perm = perm_base + perm_offset[plane] + (size_t)h * F;
  // greedy selection of 5 points that are >= 0.05 m apart, walking the shuffled order (:106-130)
  int sel[PF_SET], nsel = 0;
  if (lane == 0) {
    for (int it = 0; it < F && nsel < PF_SET; it++) {
      const int c = perm[it];
      bool good = true;
      for (int q = 0; q < nsel; q++) {
        const double dx = sm_pts[3 * sel[q]] - sm_pts[3 * c], dy = sm_pts[3 * sel[q] + 1] - sm_pts[3 * c + 1], dz = sm_pts[3 * sel[q] + 2] - sm_pts[3 * c + 2];
        if (sqrt(dx * dx + dy * dy + dz * dz) < 0.05) {
          good = false;
          break;
        }
      }
      if (good)
        sel[nsel++] = c;
    }
  }
  nsel = __shfl_sync(0xffffffffu, nsel, 0);
  for (int q = 0; q < PF_SET; q++)
    sel[q] = __shfl_sync(0xffffffffu, sel[q], 0);
  PfHyp out;
  out.state = 0;
  out.count = 0;
  out.avg = 0.0;
  out.abcd[0] = out.abcd[1] = out.abcd[2] = out.abcd[3] = 0.0;
  if (nsel != PF_SET) {
    out.state = 2;
  } else {
    // condition number of the 5 x 3 system from the extreme eigenvalues of A^T A (:60-67)
    double AtA[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int q = 0; q < PF_SET; q++) {
      const double *p = sm_pts + 3 * sel[q];
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++)
          AtA[3 * a + b] += p[a] * p[b];
    }
    double emin, emax;
    tri_eig_minmax(AtA, emin, emax);
    const bool cond_ok = (emin > 0.0) && (sqrt(emax / emin) <= max_cond);
    if (cond_ok) {
      if (lane < PF_SET) {
        const double *p = sm_pts + 3 * sel[lane];
        Ab[4 * lane] = p[0];
        Ab[4 * lane + 1] = p[1];
        Ab[4 * lane + 2] = p[2];
        Ab[4 * lane + 3] = -1.0;
      }
      __syncwarp();
      double n[3];
      pf_warp_lstsq3(Ab, PF_SET, n);
      if (pf_finish_plane(n, out.abcd)) {
        int cnt = 0;
        double sum = 0.0;
        for (int f = lane; f < F; f += 32) {
          const double e = fabs(sm_pts[3 * f] * out.abcd[0] + sm_pts[3 * f + 1] * out.abcd[1] + sm_pts[3 * f + 2] * out.abcd[2] + out.abcd[3]);
          if (e < 0.05) {
            cnt++;
            sum += e;
          }
        }
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        sum = pf_warp_sum(sum);
        out.state = 1;
        out.count = cnt;
        out.avg = sum / (double)cnt;
      }
    }
  }
  if (lane == 0)
    hyp[(size_t)plane * PF_HYP + h] = out;
}

// grid (planes), one warp: the sequential "better set" rule of :147-155 as a reduction, then the refit on the inliers (:161-181)
__global__ void __launch_bounds__(32) plane_ransac_select_kernel(const int *feat_offset, const double *pts, const PfHyp *hyp, int min_inlier_num,
                                                                  double *work, int *status, double *abcd_out, int *inlier) {
  const int plane = blockIdx.x, f0 = feat_offset[plane], F = feat_offset[plane + 1] - f0, lane = threadIdx.x;
  const double *P = pts + 3 * (size_t)f0;
  int *inl = inlier + f0;
  for (int f = lane; f < F; f += 32)
    inl[f] = 0;
  if (lane < 4)
    abcd_out[4 * plane + lane] = 0.0;
  if (lane == 0)
    status[plane] = 0;
  if (F < min_inlier_num || F == 0)
    return;
  const int thr = max(min_inlier_num, (int)((double)F * 0.80));
  int best = -1, bcount = 0, anyshort = 0;
  double bavg = 0.0;
  for (int h = lane; h < PF_HYP; h += 32) {
    const PfHyp &H = hyp[(size_t)plane * PF_HYP + h];
    if (H.state == 2)
      anyshort = 1;
    if (H.state != 1 || !(H.count > thr && H.avg < 0.05))
      continue;
    if (best < 0 || H.count > bcount || (H.count == bcount && H.avg < bavg)) { // ascending h within a lane: ties keep the earlier draw
      best = h;
      bcount = H.count;
      bavg = H.avg;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const int ob = __shfl_xor_sync(0xffffffffu, best, o), oc = __shfl_xor_sync(0xffffffffu, bcount, o);
    const double oa = __shfl_xor_sync(0xffffffffu, bavg, o);
    const bool take = ob >= 0 && (best < 0 || oc > bcount || (oc == bcount && (oa < bavg || (oa == bavg && ob < best))));
    if (take) {
      best = ob;
      bcount = oc;
      bavg = oa;
    }
  }
  anyshort = __any_sync(0xffffffffu, anyshort);
  if (anyshort || best < 0)
    return;
  const PfHyp &B = hyp[(size_t)plane * PF_HYP + best];
  double *Ab = work + 4 * (size_t)f0;
  // inlier flags of the winning draw, compacted rows for the refit (order preserved)
  int K = 0;
  for (int base = 0; base < F; base += 32) {
    const int f = base + lane;
    bool in = false;
    if (f < F)
      in = fabs(P[3 * f] * B.abcd[0] + P[3 * f + 1] * B.abcd[1] + P[3 * f + 2] * B.abcd[2] + B.abcd[3]) < 0.05;
    const unsigned m = __ballot_sync(0xffffffffu, in);
    if (in) {
      const int r = K + __popc(m & ((1u << lane) - 1u));
      Ab[4 * r] = P[3 * f];
      Ab[4 * r + 1] = P[3 * f + 1];
      Ab[4 * r + 2] = P[3 * f + 2];
      Ab[4 * r + 3] = -1.0;
      inl[f] = 1;
    }
    K += __popc(m);
  }
  __syncwarp();
  double n[3], abcd[4];
  pf_warp_lstsq3(Ab, K, n);
  const bool ok = (K >= 3) && pf_finish_plane(n, abcd);
  if (!ok) {
    for (int f = lane; f < F; f += 32)
      inl[f] = 0;
    return;
  }
  if (lane < 4)
    abcd_out[4 * plane + lane] = abcd[lane];
  if (lane == 0)
    status[plane] = 1;
}

// ---- optimize_plane: restated Ceres dogleg on per-feature normal blocks -----------------------------------------------------------------
#define PO_THREADS 256
#define PO_FIELDS 42 // per-feature scratch doubles: x 3, cand 3, Uu 6, Wu 9, bu 3, sc 3, D 3, g 3, gn 3, st 3 + 3 spare
enum { PO_X = 0, PO_CAND = 3, PO_U = 6, PO_W = 12, PO_B = 21, PO_SC = 24, PO_D = 27, PO_G = 30, PO_GN = 33, PO_ST = 36 };

template <int N> __device__ void po_block_sum(double *v, double *red) { // deterministic: lanes by shuffle tree, warps in order; result to all threads
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int k = 0; k < N; k++)
    v[k] = pf_warp_sum(v[k]);
  __syncthreads();
  if (lane == 0)
    for (int k = 0; k < N; k++)
      red[warp * N + k] = v[k];
  __syncthreads();
  for (int k = 0; k < N; k++) {
    double s = 0.0;
    for (int w = 0; w < nw; w++)
      s += red[w * N + k];
    v[k] = s;
  }
}
__device__ double po_block_max(double v, double *red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int o = 16; o > 0; o >>= 1)
    v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0)
    red[warp] = v;
  __syncthreads();
  double s = red[0];
  for (int w = 1; w < nw; w++)
    s = fmax(s, red[w]);
  return s;
}
// lower Cholesky of a symmetric 3x3 given as {a00,a10,a11,a20,a21,a22}; false when not positive definite
__device__ __forceinline__ bool po_chol3(const double *A, double *L) {
  if (!(A[0] > 0.0))
    return false;
  L[0] = sqrt(A[0]);
  L[1] = A[1] / L[0];
  L[3] = A[3] / L[0];
  const double d1 = A[2] - L[1] * L[1];
  if (!(d1 > 0.0))
    return false;
  L[2] = sqrt(d1);
  L[4] = (A[4] - L[3] * L[1]) / L[2];
  const double d2 = A[5] - L[3] * L[3] - L[4] * L[4];
  if (!(d2 > 0.0))
    return false;
  L[5] = sqrt(d2);
  return true;
}
__device__ __forceinline__ void po_chol3_solve(const double *L, const double *b, double *x) {
  const double y0 = b[0] / L[0], y1 = (b[1] - L[1] * y0) / L[2], y2 = (b[2] - L[3] * y0 - L[4] * y1) / L[5];
  x[2] = y2 / L[5];
  x[1] = (y1 - L[4] * x[2]) / L[2];
  x[0] = (y0 - L[1] * x[1] - L[3] * x[2]) / L[0];
}
__device__ __forceinline__ double po_sym(const double *S, int i, int j) { // packed lower {00,10,11,20,21,22}
  const int a = i > j ? i : j, b = i > j ? j : i;
  return S[a * (a + 1) / 2 + b];
}

struct PoArgs {
  const int *feat_offset, *meas_offset, *meas_clone, *fix_plane;
  const float *uvn;
  const double *p0, *cp0, *Rc, *pc; // camera pose table by clone handle (cam_pose_kernel)
  double sigma_px_norm, sigma_c;
  int max_iter;
  double R_cur[9], p_cur[3]; // current camera pose R_GtoC, p_CinG (for the in-front-of-camera test, :471-474)
  double *scratch;           // PO_FIELDS per feature
  double *p_out, *cp_out, *info;
  int *inlier, *status;
};

// Cost contribution and (optionally) the UNSCALED normal-equation blocks of one feature at position p with plane cp (n, d precomputed), computed
// by ONE WARP: lane = measurement (strided when a track is longer than 32), per-lane partial sums combined by an xor butterfly (every lane ends
// with the same bits), the point-on-plane block evaluated redundantly by every lane.  Outputs are SET, not accumulated, and identical in all
// lanes: U (6, packed lower), W (9), bf (3): feature blocks; Vf (6), bcf (3): this feature's share of the plane block.
// Loss: Cauchy a = 1 on every residual block (PlaneFitting.cpp:252,363): rho = log(1 + s); corrector.cc with rho'' <= 0: residual and
// Jacobian are scaled by sqrt(rho') = 1 / sqrt(1 + s).
__device__ double po_feature_warp(const PoArgs &A, int fg, const double *p, const double *nrm, double d, bool cp_free, bool feat_free, bool want,
                                  double *U, double *W, double *bf, double *Vf, double *bcf) {
  const int lane = threadIdx.x & 31;
  const int m0 = A.meas_offset[fg], m = A.meas_offset[fg + 1] - m0;
  double part[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; // cost, U (6), bf (3) of this lane's measurements
  const double w = 1.0 / A.sigma_px_norm;
  for (int k = lane; k < m; k += 32) {
    const int hc = A.meas_clone[m0 + k];
    const double *R = A.Rc + 9 * (size_t)hc, *pc = A.pc + 3 * (size_t)hc;
    const double dx = p[0] - pc[0], dy = p[1] - pc[1], dz = p[2] - pc[2];
    const double X = R[0] * dx + R[1] * dy + R[2] * dz, Y = R[3] * dx + R[4] * dy + R[5] * dz, Z = R[6] * dx + R[7] * dy + R[8] * dz;
    const double r0 = w * (X / Z - (double)A.uvn[2 * (size_t)(m0 + k)]), r1 = w * (Y / Z - (double)A.uvn[2 * (size_t)(m0 + k) + 1]);
    const double s = r0 * r0 + r1 * r1;
    part[0] += 0.5 * log(1.0 + s);
    if (want) {
      const double rho1 = fmax(DBL_MIN, 1.0 / (1.0 + s)), sq = sqrt(rho1), sc = sq * w;
      const double iz = 1.0 / Z, xz = -X / (Z * Z), yz = -Y / (Z * Z);
      double J0[3], J1[3];
      for (int i = 0; i < 3; i++) {
        J0[i] = sc * (iz * R[i] + xz * R[6 + i]);
        J1[i] = sc * (iz * R[3 + i] + yz * R[6 + i]);
      }
      const double q0 = sq * r0, q1 = sq * r1;
      for (int i = 0; i < 3; i++) {
        for (int j = 0; j <= i; j++)
          part[1 + i * (i + 1) / 2 + j] += J0[i] * J0[j] + J1[i] * J1[j];
        part[7 + i] += J0[i] * q0 + J1[i] * q1;
      }
    }
  }
  const int nred = want ? 10 : 1;
  for (int k = 0; k < nred; k++)
    part[k] = pf_warp_sum(part[k]);
  double cost = part[0];
  if (want) {
    for (int i = 0; i < 6; i++)
      U[i] = part[1 + i];
    for (int i = 0; i < 3; i++)
      bf[i] = part[7 + i];
    for (int i = 0; i < 9; i++)
      W[i] = 0.0;
    for (int i = 0; i < 6; i++)
      Vf[i] = 0.0;
    for (int i = 0; i < 3; i++)
      bcf[i] = 0.0;
  }
  // point-on-plane block (Factor_PointOnPlane.cpp:39-70): m identical copies for a measured feature (:367-369), one inflated copy for a
  // constant (SLAM) feature (:274-277) - and none at all when neither the feature nor the plane is free (Ceres drops constant blocks)
  if (!feat_free && !cp_free)
    return cost;
  const double mult = (m > 0) ? (double)m : 1.0, wc = 1.0 / ((m > 0) ? A.sigma_c : 2.0 * A.sigma_c);
  const double ndp = nrm[0] * p[0] + nrm[1] * p[1] + nrm[2] * p[2];
  const double r = wc * (ndp - d), s = r * r;
  cost += mult * 0.5 * log(1.0 + s);
  if (want) {
    const double rho1 = fmax(DBL_MIN, 1.0 / (1.0 + s)), sq = sqrt(rho1), q = sq * r;
    double Jp[3], Jc[3];
    for (int i = 0; i < 3; i++) {
      Jp[i] = sq * wc * nrm[i];
      Jc[i] = sq * wc * (1.0 / d) * (p[i] - ndp * nrm[i] - d * nrm[i]);
    }
    for (int i = 0; i < 3; i++) {
      if (feat_free) {
        for (int j = 0; j <= i; j++)
          U[i * (i + 1) / 2 + j] += mult * Jp[i] * Jp[j];
        bf[i] += mult * Jp[i] * q;
      }
      if (cp_free) {
        for (int j = 0; j <= i; j++)
          Vf[i * (i + 1) / 2 + j] += mult * Jc[i] * Jc[j];
        bcf[i] += mult * Jc[i] * q;
        if (feat_free)
          for (int j = 0; j < 3; j++)
            W[3 * i + j] += mult * Jp[i] * Jc[j];
      }
    }
  }
  return cost;
}

__global__ void __launch_bounds__(PO_THREADS) optimize_plane_kernel(PoArgs A) {
  __shared__ double red[(PO_THREADS / 32) * 12];
  const int plane = blockIdx.x, f0 = A.feat_offset[plane], F = A.feat_offset[plane + 1] - f0, tid = threadIdx.x;
  const bool fix_plane = A.fix_plane[plane] != 0, cp_free = !fix_plane;
  double *S = A.scratch + (size_t)PO_FIELDS * f0;
#define FLD(field, f, i) S[(size_t)((field) + (i)) * F + (f)]
  // outputs default to the inputs (the reference leaves everything untouched unless the solver converged)
  for (int i = tid; i < 3 * F; i += PO_THREADS)
    A.p_out[3 * (size_t)f0 + i] = A.p0[3 * (size_t)f0 + i];
  for (int f = tid; f < F; f += PO_THREADS)
    A.inlier[f0 + f] = 0;
  double cp[3] = {A.cp0[3 * plane], A.cp0[3 * plane + 1], A.cp0[3 * plane + 2]};
  if (tid < 3)
    A.cp_out[3 * plane + tid] = cp[tid];
  if (tid == 0) {
    A.status[plane] = 0;
    for (int i = 0; i < 5; i++)
      A.info[5 * plane + i] = 0.0;
  }
  if ((!fix_plane && F < 4) || (fix_plane && F == 0)) // :211-214
    return;
  // free parameters
  double cnt[1] = {0.0};
  for (int f = tid; f < F; f += PO_THREADS) {
    const bool ff = A.meas_offset[f0 + f + 1] > A.meas_offset[f0 + f];
    cnt[0] += ff ? 3.0 : 0.0;
    for (int i = 0; i < 3; i++)
      FLD(PO_X, f, i) = A.p0[3 * (size_t)(f0 + f) + i];
  }
  po_block_sum<1>(cnt, red);
  const int n_free = (int)cnt[0] + (cp_free ? 3 : 0);

  const double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8, min_relative_decrease = 1e-3;
  const double min_diagonal = 1e-6, max_diagonal = 1e32, min_mu = 1e-8, max_mu = 1.0, mu_increase_factor = 10.0;
  double radius = 1e4, mu = min_mu, alpha = 0.0, dogleg_step_norm = 0.0;
  bool reuse = false, converged = false, last_successful = false;
  int reason = 0, iteration = 0, num_invalid = 0;
  double x_cost = 0.0, initial_cost = 0.0, gmax = 0.0, x_norm = 0.0;
  double Vu[6], bcu[3], scc[3] = {0, 0, 0}, Dc[3] = {1, 1, 1}, gc[3] = {0, 0, 0}, gnc[3] = {0, 0, 0}, stc[3] = {0, 0, 0};

  // evaluation with Jacobian at (x, cp): a warp per feature (lane = measurement); per-feature blocks to scratch, plane blocks + cost + gradient
  // max norm + |x| reduced over the block.  The other phases of an iteration are 3 x 3 algebra per feature and stay one thread per feature:
  // the two mappings meet in the scratch arrays, with a block barrier in between.
  const int lane = tid & 31, warp = tid >> 5, nwarps = PO_THREADS / 32;
  auto evaluate_full = [&]() {
    const double d = sqrt(cp[0] * cp[0] + cp[1] * cp[1] + cp[2] * cp[2]);
    const double nrm[3] = {cp[0] / d, cp[1] / d, cp[2] / d};
    double acc[11] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; // cost, V(6), bc(3), |x|^2   (lane 0 of every warp accumulates)
    double gm = 0.0;
    __syncthreads();
    for (int f = warp; f < F; f += nwarps) {
      const bool ff = A.meas_offset[f0 + f + 1] > A.meas_offset[f0 + f];
      const double p[3] = {FLD(PO_X, f, 0), FLD(PO_X, f, 1), FLD(PO_X, f, 2)};
      double U[6], W[9], bf[3], Vf[6], bcf[3];
      const double cf = po_feature_warp(A, f0 + f, p, nrm, d, cp_free, ff, true, U, W, bf, Vf, bcf);
      if (lane == 0) {
        acc[0] += cf;
        for (int i = 0; i < 6; i++) {
          FLD(PO_U, f, i) = U[i];
          acc[1 + i] += Vf[i];
        }
        for (int i = 0; i < 9; i++)
          FLD(PO_W, f, i) = W[i];
        for (int i = 0; i < 3; i++) {
          FLD(PO_B, f, i) = bf[i];
          acc[7 + i] += bcf[i];
          if (ff) {
            gm = fmax(gm, fabs(bf[i]));
            acc[10] += p[i] * p[i];
          }
        }
      }
    }
    po_block_sum<11>(acc, red);
    x_cost = acc[0];
    for (int i = 0; i < 6; i++)
      Vu[i] = acc[1 + i];
    for (int i = 0; i < 3; i++)
      bcu[i] = acc[7 + i];
    gm = po_block_max(gm, red);
    double xn = acc[10];
    if (cp_free)
      for (int i = 0; i < 3; i++) {
        gm = fmax(gm, fabs(bcu[i]));
        xn += cp[i] * cp[i];
      }
    gmax = gm;
    x_norm = sqrt(xn);
  };
  auto traditional_dogleg = [&]() { // DoglegStrategy::ComputeTraditionalDoglegStep on (gradient, gauss_newton_step, alpha, radius)
    double acc[3] = {0, 0, 0};      // |g|^2, |gn|^2, g.gn
    for (int f = tid; f < F; f += PO_THREADS) {
      if (!(A.meas_offset[f0 + f + 1] > A.meas_offset[f0 + f]))
        continue;
      for (int i = 0; i < 3; i++) {
        const double g = FLD(PO_G, f, i), q = FLD(PO_GN, f, i);
        acc[0] += g * g;
        acc[1] += q * q;
        acc[2] += g * q;
      }
    }
    po_block_sum<3>(acc, red);
    if (cp_free)
      for (int i = 0; i < 3; i++) {
        acc[0] += gc[i] * gc[i];
        acc[1] += gnc[i] * gnc[i];
        acc[2] += gc[i] * gnc[i];
      }
    const double gnorm = sqrt(acc[0]), gnn = sqrt(acc[1]);
    double ca, cb; // step = ca * gradient + cb * gn
    bool need_norm = false;
    if (gnn <= radius) {
      ca = 0.0;
      cb = 1.0;
      dogleg_step_norm = gnn;
    } else if (gnorm * alpha >= radius) {
      ca = -(radius / gnorm);
      cb = 0.0;
      dogleg_step_norm = radius;
    } else {
      const double b_dot_a = -alpha * acc[2];
      const double a_sq = (alpha * gnorm) * (alpha * gnorm);
      const double bma_sq = a_sq - 2.0 * b_dot_a + gnn * gnn;
      const double c = b_dot_a - a_sq;
      const double dd = sqrt(c * c + bma_sq * (radius * radius - a_sq));
      const double beta = (c <= 0.0) ? (dd - c) / bma_sq : (radius * radius - a_sq) / (dd + c);
      ca = -alpha * (1.0 - beta);
      cb = beta;
      need_norm = true;
    }
    double sn[1] = {0.0};
    for (int f = tid; f < F; f += PO_THREADS) {
      if (!(A.meas_offset[f0 + f + 1] > A.meas_offset[f0 + f]))
        continue;
      for (int i = 0; i < 3; i++) {
        const double s = (cb == 0.0 ? 0.0 : cb * FLD(PO_GN, f, i)) + (ca == 0.0 ? 0.0 : ca * FLD(PO_G, f, i));
        sn[0] += s * s;
        FLD(PO_ST, f, i) = s / FLD(PO_D, f, i);
      }
    }
    if (need_norm)
      po_block_sum<1>(sn, red);
    for (int i = 0; i < 3; i++) {
      const double s = cp_free ? ((cb == 0.0 ? 0.0 : cb * gnc[i]) + (ca == 0.0 ? 0.0 : ca * gc[i])) : 0.0;
      if (need_norm)
        sn[0] += s * s;
      stc[i] = cp_free ? s / Dc[i] : 0.0;
    }
    if (need_norm)
      dogleg_step_norm = sqrt(sn[0]);
  };

  if (n_free == 0) { // "No non-constant parameter blocks found": Ceres reports CONVERGENCE without iterating
    converged = true;
    reason = 4;
  } else {
    evaluate_full();
    initial_cost = x_cost;
    // Jacobi scaling from the first Jacobian (trust_region_minimizer.cc: 1 / (1 + column norm))
    for (int f = tid; f < F; f += PO_THREADS)
      for (int i = 0; i < 3; i++)
        FLD(PO_SC, f, i) = 1.0 / (1.0 + sqrt(FLD(PO_U, f, i * (i + 1) / 2 + i)));
    if (cp_free)
      for (int i = 0; i < 3; i++)
        scc[i] = 1.0 / (1.0 + sqrt(Vu[i * (i + 1) / 2 + i]));
    while (true) {
      if (iteration >= A.max_iter) {
        reason = -1;
        break;
      }
      if (last_successful && gmax <= gradient_tolerance) {
        converged = true;
        reason = 1;
        break;
      }
      iteration++;
      last_successful = false;
      bool solve_ok = true;
      if (reuse) {
        traditional_dogleg();
      } else {
        reuse = true;
        // diagonal, gradient, Cauchy point
        double acc[2] = {0, 0}; // |g|^2, u^T H u with u = g * sc / D
        double uc[3] = {0, 0, 0};
        if (cp_free)
          for (int i = 0; i < 3; i++) {
            const double cn = Vu[i * (i + 1) / 2 + i] * scc[i] * scc[i];
            Dc[i] = sqrt(fmin(fmax(cn, min_diagonal), max_diagonal));
            gc[i] = scc[i] * bcu[i] / Dc[i];
            uc[i] = gc[i] / Dc[i] * scc[i];
            acc[0] += (tid == 0) ? gc[i] * gc[i] : 0.0;
          }
        if (cp_free && tid == 0)
          for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++)
              acc[1] += uc[i] * po_sym(Vu, i, j) * uc[j];
        for (int f = tid; f < F; f += PO_THREADS) {
          if (!(A.meas_offset[f0 + f + 1] > A.meas_offset[f0 + f]))
            continue;
          double u[3], U[6];
          for (int i = 0; i < 6; i++)
            U[i] = FLD(PO_U, f, i);
          for (int i = 0; i < 3; i++) {
            const double sc = FLD(PO_SC, f, i);
            const double D = sqrt(fmin(fmax(U[i * (i + 1) / 2 + i] * sc * sc, min_diagonal), max_diagonal));
            const double g = sc * FLD(PO_B, f, i) / D;
            FLD(PO_D, f, i) = D;
            FLD(PO_G, f, i) = g;
            u[i] = g / D * sc;
            acc[0] += g * g;
          }
          for (int i = 0; i < 3; i++) {
            for (int j = 0; j < 3; j++)
              acc[1] += u[i] * po_sym(U, i, j) * u[j];
            if (cp_free)
              for (int j = 0; j < 3; j++)
                acc[1] += 2.0 * u[i] * FLD(PO_W, f, 3 * i + j) * uc[j];
          }
        }
        po_block_sum<2>(acc, red);
        alpha = acc[0] / acc[1];
        // Gauss-Newton step (J^T J + mu D^2) y = J^T r through the Schur complement on the plane block; gn = -D y
        solve_ok = false;
        while (mu < max_mu) {
          double sacc[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; // S (6 packed), rhs (3), failure flag
          for (int f = tid; f < F; f += PO_THREADS) {
            if (!(A.meas_offset[f0 + f + 1] > A.meas_offset[f0 + f]))
              continue;
            double Af[6], L[6], sc[3], bs[3];
            for (int i = 0; i < 3; i++)
              sc[i] = FLD(PO_SC, f, i);
            for (int i = 0; i < 3; i++) {
              for (int j = 0; j <= i; j++)
                Af[i * (i + 1) / 2 + j] = sc[i] * sc[j] * FLD(PO_U, f, i * (i + 1) / 2 + j);
              const double D = FLD(PO_D, f, i);
              Af[i * (i + 1) / 2 + i] += mu * D * D;
              bs[i] = sc[i] * FLD(PO_B, f, i);
            }
            if (!po_chol3(Af, L)) {
              sacc[9] += 1.0;
              continue;
            }
            if (cp_free) {
              double Ws[9], AiW[9], Aib[3];
              for (int i = 0; i < 3; i++)
                for (int j = 0; j < 3; j++)
                  Ws[3 * i + j] = sc[i] * FLD(PO_W, f, 3 * i + j) * scc[j];
              for (int j = 0; j < 3; j++) {
                const double col[3] = {Ws[j], Ws[3 + j], Ws[6 + j]};
                double x3[3];
                po_chol3_solve(L, col, x3);
                AiW[j] = x3[0];
                AiW[3 + j] = x3[1];
                AiW[6 + j] = x3[2];
              }
              po_chol3_solve(L, bs, Aib);
              for (int i = 0; i < 3; i++) {
                for (int j = 0; j <= i; j++)
                  sacc[i * (i + 1) / 2 + j] += Ws[i] * AiW[j] + Ws[3 + i] * AiW[3 + j] + Ws[6 + i] * AiW[6 + j];
                sacc[6 + i] += Ws[i] * Aib[0] + Ws[3 + i] * Aib[1] + Ws[6 + i] * Aib[2];
              }
            }
          }
          po_block_sum<10>(sacc, red);
          bool ok = sacc[9] == 0.0;
          double yc[3] = {0, 0, 0};
          if (ok && cp_free) {
            double Sm[6], L[6], rhs[3];
            for (int i = 0; i < 3; i++) {
              for (int j = 0; j <= i; j++)
                Sm[i * (i + 1) / 2 + j] = scc[i] * scc[j] * Vu[i * (i + 1) / 2 + j] - sacc[i * (i + 1) / 2 + j];
              Sm[i * (i + 1) / 2 + i] += mu * Dc[i] * Dc[i];
              rhs[i] = scc[i] * bcu[i] - sacc[6 + i];
            }
            ok = po_chol3(Sm, L);
            if (ok) {
              po_chol3_solve(L, rhs, yc);
              ok = isfinite(yc[0]) && isfinite(yc[1]) && isfinite(yc[2]);
            }
          }
          double bad[1] = {0.0};
          if (ok) {
            for (int f = tid; f < F; f += PO_THREADS) {
              if (!(A.meas_offset[f0 + f + 1] > A.meas_offset[f0 + f]))
                continue;
              double Af[6], L[6], sc[3], rhs[3], y[3];
              for (int i = 0; i < 3; i++)
                sc[i] = FLD(PO_SC, f, i);
              for (int i = 0; i < 3; i++) {
                for (int j = 0; j <= i; j++)
                  Af[i * (i + 1) / 2 + j] = sc[i] * sc[j] * FLD(PO_U, f, i * (i + 1) / 2 + j);
                const double D = FLD(PO_D, f, i);
                Af[i * (i + 1) / 2 + i] += mu * D * D;
                rhs[i] = sc[i] * FLD(PO_B, f, i);
                if (cp_free)
                  for (int j = 0; j < 3; j++)
                    rhs[i] -= sc[i] * FLD(PO_W, f, 3 * i + j) * scc[j] * yc[j];
              }
              po_chol3(Af, L);
              po_chol3_solve(L, rhs, y);
              for (int i = 0; i < 3; i++) {
                if (!isfinite(y[i]))
                  bad[0] += 1.0;
                FLD(PO_GN, f, i) = -FLD(PO_D, f, i) * y[i];
              }
            }
            po_block_sum<1>(bad, red);
            ok = bad[0] == 0.0;
          }
          if (!ok) {
            mu *= mu_increase_factor;
            continue;
          }
          for (int i = 0; i < 3; i++)
            gnc[i] = cp_free ? -Dc[i] * yc[i] : 0.0;
          solve_ok = true;
          break;
        }
        if (solve_ok)
          traditional_dogleg();
      }
      // model cost change -(J s)^T (r + J s / 2) = -t^T b_u - t^T H_u t / 2 with t = step * scale (= delta), candidate point
      bool step_is_valid = false;
      double model_cost_change = 0.0, step_norm = 0.0;
      double dcp[3] = {0, 0, 0};
      if (solve_ok) {
        double acc[2] = {0, 0}; // model cost change, |delta|^2
        if (cp_free)
          for (int i = 0; i < 3; i++)
            dcp[i] = stc[i] * scc[i];
        if (cp_free && tid == 0) {
          for (int i = 0; i < 3; i++) {
            acc[0] -= dcp[i] * bcu[i];
            for (int j = 0; j < 3; j++)
              acc[0] -= 0.5 * dcp[i] * po_sym(Vu, i, j) * dcp[j];
            acc[1] += dcp[i] * dcp[i];
          }
        }
        for (int f = tid; f < F; f += PO_THREADS) {
          if (!(A.meas_offset[f0 + f + 1] > A.meas_offset[f0 + f])) {
            for (int i = 0; i < 3; i++)
              FLD(PO_CAND, f, i) = FLD(PO_X, f, i);
            continue;
          }
          double t[3], U[6];
          for (int i = 0; i < 6; i++)
            U[i] = FLD(PO_U, f, i);
          for (int i = 0; i < 3; i++) {
            t[i] = FLD(PO_ST, f, i) * FLD(PO_SC, f, i);
            FLD(PO_CAND, f, i) = FLD(PO_X, f, i) + t[i];
            acc[1] += t[i] * t[i];
          }
          for (int i = 0; i < 3; i++) {
            acc[0] -= t[i] * FLD(PO_B, f, i);
            for (int j = 0; j < 3; j++)
              acc[0] -= 0.5 * t[i] * po_sym(U, i, j) * t[j];
            if (cp_free)
              for (int j = 0; j < 3; j++)
                acc[0] -= t[i] * FLD(PO_W, f, 3 * i + j) * dcp[j];
          }
        }
        po_block_sum<2>(acc, red);
        model_cost_change = acc[0];
        step_norm = sqrt(acc[1]);
        step_is_valid = model_cost_change > 0.0;
      }
      if (!step_is_valid) { // HandleInvalidStep
        if (++num_invalid >= 5) {
          reason = -2;
          break;
        }
        mu *= mu_increase_factor;
        reuse = false;
        continue;
      }
      num_invalid = 0;
      // candidate cost
      double ccp[3] = {cp[0] + dcp[0], cp[1] + dcp[1], cp[2] + dcp[2]};
      double cc[1] = {0.0};
      {
        const double d = sqrt(ccp[0] * ccp[0] + ccp[1] * ccp[1] + ccp[2] * ccp[2]);
        const double nrm[3] = {ccp[0] / d, ccp[1] / d, ccp[2] / d};
        __syncthreads(); // the candidate positions were written one thread per feature
        for (int f = warp; f < F; f += nwarps) {
          const bool ff = A.meas_offset[f0 + f + 1] > A.meas_offset[f0 + f];
          const double p[3] = {FLD(PO_CAND, f, 0), FLD(PO_CAND, f, 1), FLD(PO_CAND, f, 2)};
          const double cf = po_feature_warp(A, f0 + f, p, nrm, d, cp_free, ff, false, nullptr, nullptr, nullptr, nullptr, nullptr);
          if (lane == 0)
            cc[0] += cf;
        }
      }
      po_block_sum<1>(cc, red);
      double cand_cost = cc[0];
      if (!isfinite(cand_cost))
        cand_cost = DBL_MAX;
      if (step_norm <= parameter_tolerance * (x_norm + parameter_tolerance)) {
        converged = true;
        reason = 2;
        break;
      }
      if (fabs(x_cost - cand_cost) <= function_tolerance * x_cost) { // the candidate is not taken
        converged = true;
        reason = 3;
        break;
      }
      const double relative_decrease = (x_cost - cand_cost) / model_cost_change;
      if (relative_decrease > min_relative_decrease) { // HandleSuccessfulStep
        for (int f = tid; f < F; f += PO_THREADS)
          for (int i = 0; i < 3; i++)
            FLD(PO_X, f, i) = FLD(PO_CAND, f, i);
        for (int i = 0; i < 3; i++)
          cp[i] = ccp[i];
        evaluate_full();
        last_successful = true;
        if (relative_decrease < 0.25)
          radius *= 0.5;
        if (relative_decrease > 0.75)
          radius = fmax(radius, 3.0 * dogleg_step_norm);
        mu = fmax(min_mu, 2.0 * mu / mu_increase_factor);
        reuse = false;
      } else {
        radius *= 0.5;
        reuse = true;
      }
    }
  }
  if (tid == 0) {
    A.info[5 * plane] = converged ? 1.0 : 0.0;
    A.info[5 * plane + 1] = (double)iteration;
    A.info[5 * plane + 2] = initial_cost;
    A.info[5 * plane + 3] = x_cost;
    A.info[5 * plane + 4] = (double)reason;
  }
  if (!converged) // summary.termination_type != CONVERGENCE (:431-438)
    return;
  // inlier pass (:441-487): distance of the ORIGINAL position to the refined plane, NaN, in front of the current camera
  const double cn = sqrt(cp[0] * cp[0] + cp[1] * cp[1] + cp[2] * cp[2]);
  const double ab[4] = {cp[0] / cn, cp[1] / cn, cp[2] / cn, -cn};
  double ninl[1] = {0.0};
  __syncthreads();
  for (int f = tid; f < F; f += PO_THREADS) {
    const double *q0 = A.p0 + 3 * (size_t)(f0 + f);
    const double after[3] = {FLD(PO_X, f, 0), FLD(PO_X, f, 1), FLD(PO_X, f, 2)};
    const double err = q0[0] * ab[0] + q0[1] * ab[1] + q0[2] * ab[2] + ab[3];
    if (fabs(err) >= 0.03)
      continue;
    if (isnan(sqrt(after[0] * after[0] + after[1] * after[1] + after[2] * after[2])))
      continue;
    const double z = A.R_cur[6] * (after[0] - A.p_cur[0]) + A.R_cur[7] * (after[1] - A.p_cur[1]) + A.R_cur[8] * (after[2] - A.p_cur[2]);
    if (z < 0.1)
      continue;
    for (int i = 0; i < 3; i++)
      A.p_out[3 * (size_t)(f0 + f) + i] = after[i];
    A.inlier[f0 + f] = 1;
    ninl[0] += 1.0;
  }
  po_block_sum<1>(ninl, red);
  if (tid < 3)
    A.cp_out[3 * plane + tid] = cp[tid];
  const int thr = max(4, (int)((double)F * 0.80)), n_inl = (int)ninl[0];
  const bool fail = (F != 1 && n_inl < thr) || (fix_plane && F == 1 && n_inl == 0);
  if (tid == 0)
    A.status[plane] = fail ? 0 : 1;
#undef FLD
}

static std::map<long long, std::vector<int>> g_perm_cache; // (shuffle_kind, F) -> 200 x F draws; depends on nothing else
static std::mutex g_perm_mutex;
// copies the 200 draws for F points into dst (200 x F ints); generated once per (kind, F) and kept, under the lock
static void pf_permutations_copy(int F, int kind, int *dst) {
  if (F <= 0)
    return;
  std::lock_guard<std::mutex> lock(g_perm_mutex);
  const long long key = ((long long)kind << 32) | (unsigned)F;
  auto it = g_perm_cache.find(key);
  if (it == g_perm_cache.end()) {
    if (g_perm_cache.size() >= 64) // a tracker sees a handful of sizes per frame; bound the table anyway
      g_perm_cache.clear();
    std::vector<int> out((size_t)PF_HYP * F);
    Mt19937 g(8888u); // std::mt19937 rand_gen(8888), PlaneFitting.cpp:93
    for (int h = 0; h < PF_HYP; h++) {
      int *v = out.data() + (size_t)h * F;
      for (int i = 0; i < F; i++)
        v[i] = i;
      pf_shuffle(v, F, g, kind);
    }
    it = g_perm_cache.emplace(key, std::move(out)).first;
  }
  std::memcpy(dst, it->second.data(), it->second.size() * sizeof(int));
}

} // namespace ovp

extern "C" {

int ovp_plane_shuffle(int n, int n_shuffles, int shuffle_kind, int *out) {
  if (n < 0 || n_shuffles < 0 || !out || (shuffle_kind != 0 && shuffle_kind != 1))
    return OVP_ERR_BAD_ARGS;
  ovp::Mt19937 g(8888u);
  for (int k = 0; k < n_shuffles; k++) {
    int *v = out + (size_t)k * n;
    for (int i = 0; i < n; i++)
      v[i] = i;
    ovp::pf_shuffle(v, n, g, shuffle_kind);
  }
  return OVP_OK;
}

int ovp_plane_fitting(ovp_ctx *h, int n_planes, const int *feat_offset, const double *p_FinG, const ovp_plane_fit_options *opt, int *status,
                      double *abcd, int *inlier) {
  using namespace ovp;
  Ctx *c = ovp::enter(h);
  if (n_planes <= 0)
    return OVP_OK;
  if (!feat_offset || !p_FinG || !opt || !status || !abcd || !inlier)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_fitting: null argument");
  if (opt->shuffle_kind != 0 && opt->shuffle_kind != 1)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_fitting: shuffle_kind %d (0 = libstdc++ GCC <= 10, 1 = GCC >= 11)", opt->shuffle_kind);
  if (feat_offset[0] != 0)
    return fail(c, OVP_ERR_BAD_ARGS, "plane_fitting: feat_offset must start at 0");
  const int Ftot = feat_offset[n_planes];
  int Fmax = 0;
  std::map<int, int> perm_off; // F -> offset (ints) into the permutation block of this call
  std::vector<int> h_perm_off(n_planes);
  size_t perm_ints = 0;
  for (int p = 0; p < n_planes; p++) {
    const int F = feat_offset[p + 1] - feat_offset[p];
    if (F < 0 || F > PF_MAX_POINTS)
      return fail(c, OVP_ERR_CAPACITY, "plane_fitting: plane %d has %d points (limit %d)", p, F, PF_MAX_POINTS);
    Fmax = std::max(Fmax, F);
    auto it = perm_off.find(F);
    if (it == perm_off.end()) {
      it = perm_off.emplace(F, (int)perm_ints).first;
      perm_ints += (size_t)PF_HYP * F;
    }
    h_perm_off[p] = it->second;
  }
  if (Ftot == 0) {
    for (int p = 0; p < n_planes; p++) {
      status[p] = 0;
      for (int i = 0; i < 4; i++)
        abcd[4 * p + i] = 0.0;
    }
    return OVP_OK;
  }
  // staging (bytes): [feat_offset | perm_off | perms | pts] in, [hyp | work | status | abcd | inlier] out
  auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
  const size_t b_fo = 0, b_po = al(b_fo + (size_t)(n_planes + 1) * 4), b_pm = al(b_po + (size_t)n_planes * 4), b_pt = al(b_pm + perm_ints * 4);
  const size_t b_in_end = al(b_pt + (size_t)Ftot * 24);
  const size_t b_hy = b_in_end, b_wk = al(b_hy + (size_t)n_planes * PF_HYP * sizeof(PfHyp)), b_st = al(b_wk + (size_t)Ftot * 32);
  const size_t b_ab = al(b_st + (size_t)n_planes * 4), b_il = al(b_ab + (size_t)n_planes * 32), b_end = al(b_il + (size_t)Ftot * 4);
  int st = ensure_stage(c, b_end / 8 + 8);
  if (st)
    return st;
  std::vector<char> hbuf(b_in_end);
  std::memcpy(hbuf.data() + b_fo, feat_offset, (size_t)(n_planes + 1) * 4);
  std::memcpy(hbuf.data() + b_po, h_perm_off.data(), (size_t)n_planes * 4);
  for (auto &kv : perm_off)
    pf_permutations_copy(kv.first, opt->shuffle_kind, (int *)(hbuf.data() + b_pm + (size_t)kv.second * 4));
  std::memcpy(hbuf.data() + b_pt, p_FinG, (size_t)Ftot * 24);
  char *d = (char *)c->d_stage;
  OVP_CUDA(cudaMemcpyAsync(d, hbuf.data(), b_in_end, cudaMemcpyHostToDevice, c->stream));
  c->h2d_bytes += (int64_t)b_in_end;
  const size_t smem = (size_t)Fmax * 24 + PF_WARPS * 20 * 8;
  plane_ransac_kernel<<<dim3((PF_HYP + PF_WARPS - 1) / PF_WARPS, n_planes), 32 * PF_WARPS, smem, c->stream>>>(
      (const int *)(d + b_fo), (const double *)(d + b_pt), (const int *)(d + b_pm), (const int *)(d + b_po), opt->max_cond_number, (PfHyp *)(d + b_hy));
  plane_ransac_select_kernel<<<n_planes, 32, 0, c->stream>>>((const int *)(d + b_fo), (const double *)(d + b_pt), (const PfHyp *)(d + b_hy), opt->min_inlier_num,
                                                             (double *)(d + b_wk), (int *)(d + b_st), (double *)(d + b_ab), (int *)(d + b_il));
  c->launches += 2;
  OVP_CUDA(cudaGetLastError());
  OVP_CUDA(cudaMemcpyAsync(status, d + b_st, (size_t)n_planes * 4, cudaMemcpyDeviceToHost, c->stream));
  OVP_CUDA(cudaMemcpyAsync(abcd, d + b_ab, (size_t)n_planes * 32, cudaMemcpyDeviceToHost, c->stream));
  OVP_CUDA(cudaMemcpyAsync(inlier, d + b_il, (size_t)Ftot * 4, cudaMemcpyDeviceToHost, c->stream));
  OVP_CUDA(cudaStreamSynchronize(c->stream)); // hbuf is pageable: the H2D copy above has completed by now as well
  c->d2h_bytes += (int64_t)n_planes * 36 + (int64_t)Ftot * 4;
  return OVP_OK;
}

int ovp_optimize_plane(ovp_ctx *h, int n_planes, const int *feat_offset, const int *meas_offset, const int *meas_clone, const float *uv_norm,
                       const double *p_FinG, const double *cp_inG, const int *fix_plane, const ovp_plane_refine_options *opt, double *p_FinG_out,
                       double *cp_out, int *inlier, int *status, double *info) {
  using namespace ovp;
  Ctx *c = ovp::enter(h);
  if (n_planes <= 0)
    return OVP_OK;
  if (!feat_offset || !meas_offset || !p_FinG || !cp_inG || !fix_plane || !opt || !p_FinG_out || !cp_out || !inlier || !status)
    return fail(c, OVP_ERR_BAD_ARGS, "optimize_plane: null argument");
  if (feat_offset[0] != 0 || meas_offset[0] != 0)
    return fail(c, OVP_ERR_BAD_ARGS, "optimize_plane: offset arrays must start at 0");
  for (int p = 0; p < n_planes; p++)
    if (feat_offset[p + 1] < feat_offset[p])
      return fail(c, OVP_ERR_BAD_ARGS, "optimize_plane: feat_offset is not non-decreasing at plane %d", p);
  const int Ftot = feat_offset[n_planes];
  for (int f = 0; f < Ftot; f++)
    if (meas_offset[f + 1] < meas_offset[f])
      return fail(c, OVP_ERR_BAD_ARGS, "optimize_plane: meas_offset is not non-decreasing at feature %d", f);
  const int M = (Ftot > 0) ? meas_offset[Ftot] : 0;
  if (M > 0 && (!meas_clone || !uv_norm))
    return fail(c, OVP_ERR_BAD_ARGS, "optimize_plane: null measurement arrays");
  if (!(opt->sigma_px_norm > 0.0) || !(opt->sigma_c > 0.0))
    return fail(c, OVP_ERR_BAD_ARGS, "optimize_plane: sigma_px_norm / sigma_c must be positive");
  for (int k = 0; k < M; k++) {
    const int hh = meas_clone[k];
    if (hh < 0 || hh >= (int)c->vars.size() || !c->vars[hh].alive || c->vars[hh].kind != OVP_KIND_POSE || c->vars[hh].id < 0 || hh == c->h_calib)
      return fail(c, OVP_ERR_BAD_ARGS, "optimize_plane: measurement %d: handle %d is not a clone in the state", k, hh);
  }
  if (Ftot == 0) {
    for (int p = 0; p < n_planes; p++) {
      status[p] = 0;
      for (int i = 0; i < 3; i++)
        cp_out[3 * p + i] = cp_inG[3 * p + i];
      if (info)
        for (int i = 0; i < 5; i++)
          info[5 * p + i] = 0.0;
    }
    return OVP_OK;
  }
  if (c->var_table_dirty) {
    int st = upload_var_table(c);
    if (st)
      return st;
  }
  int st = sync_host_values(c); // current IMU pose + extrinsics for the in-front-of-camera test (stateI, calib0: PlaneFitting.cpp:441-450)
  if (st)
    return st;
  PoArgs A;
  {
    const double *vi = c->h_val.data() + (size_t)c->h_imu * OVP_VAL_STRIDE, *vc = c->h_val.data() + (size_t)c->h_calib * OVP_VAL_STRIDE;
    double Ri[9], RC[9];
    quat_to_rot(vi, Ri);
    quat_to_rot(vc, RC);
    mat3_mul(RC, Ri, A.R_cur);
    for (int i = 0; i < 3; i++)
      A.p_cur[i] = vi[4 + i] - (A.R_cur[i] * vc[4] + A.R_cur[3 + i] * vc[5] + A.R_cur[6 + i] * vc[6]);
  }
  const int nh = (int)c->vars.size();
  auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
  const size_t b_fo = 0, b_mo = al(b_fo + (size_t)(n_planes + 1) * 4), b_mc = al(b_mo + (size_t)(Ftot + 1) * 4), b_uv = al(b_mc + (size_t)M * 4);
  const size_t b_fx = al(b_uv + (size_t)M * 8), b_p0 = al(b_fx + (size_t)n_planes * 4), b_c0 = al(b_p0 + (size_t)Ftot * 24), b_in_end = al(b_c0 + (size_t)n_planes * 24);
  const size_t b_R = b_in_end, b_pc = al(b_R + (size_t)nh * 72), b_sc = al(b_pc + (size_t)nh * 24), b_po = al(b_sc + (size_t)Ftot * PO_FIELDS * 8);
  const size_t b_co = al(b_po + (size_t)Ftot * 24), b_if = al(b_co + (size_t)n_planes * 24), b_il = al(b_if + (size_t)n_planes * 40);
  const size_t b_st = al(b_il + (size_t)Ftot * 4), b_end = al(b_st + (size_t)n_planes * 4);
  st = ensure_stage(c, b_end / 8 + 8);
  if (st)
    return st;
  std::vector<char> hbuf(b_in_end);
  std::memcpy(hbuf.data() + b_fo, feat_offset, (size_t)(n_planes + 1) * 4);
  std::memcpy(hbuf.data() + b_mo, meas_offset, (size_t)(Ftot + 1) * 4);
  if (M > 0) {
    std::memcpy(hbuf.data() + b_mc, meas_clone, (size_t)M * 4);
    std::memcpy(hbuf.data() + b_uv, uv_norm, (size_t)M * 8);
  }
  std::memcpy(hbuf.data() + b_fx, fix_plane, (size_t)n_planes * 4);
  std::memcpy(hbuf.data() + b_p0, p_FinG, (size_t)Ftot * 24);
  std::memcpy(hbuf.data() + b_c0, cp_inG, (size_t)n_planes * 24);
  char *d = (char *)c->d_stage;
  OVP_CUDA(cudaMemcpyAsync(d, hbuf.data(), b_in_end, cudaMemcpyHostToDevice, c->stream));
  c->h2d_bytes += (int64_t)b_in_end;
  cam_pose_kernel<<<(nh + 127) / 128, 128, 0, c->stream>>>(nh, c->d_var_kind, c->d_var_id, c->d_val, c->h_calib, (double *)(d + b_R), (double *)(d + b_pc));
  A.feat_offset = (const int *)(d + b_fo);
  A.meas_offset = (const int *)(d + b_mo);
  A.meas_clone = (const int *)(d + b_mc);
  A.fix_plane = (const int *)(d + b_fx);
  A.uvn = (const float *)(d + b_uv);
  A.p0 = (const double *)(d + b_p0);
  A.cp0 = (const double *)(d + b_c0);
  A.Rc = (const double *)(d + b_R);
  A.pc = (const double *)(d + b_pc);
  A.sigma_px_norm = opt->sigma_px_norm;
  A.sigma_c = opt->sigma_c;
  A.max_iter = opt->max_num_iterations > 0 ? opt->max_num_iterations : 12; // PlaneFitting.cpp:396
  A.scratch = (double *)(d + b_sc);
  A.p_out = (double *)(d + b_po);
  A.cp_out = (double *)(d + b_co);
  A.info = (double *)(d + b_if);
  A.inlier = (int *)(d + b_il);
  A.status = (int *)(d + b_st);
  optimize_plane_kernel<<<n_planes, PO_THREADS, 0, c->stream>>>(A);
  c->launches += 2;
  OVP_CUDA(cudaGetLastError());
  OVP_CUDA(cudaMemcpyAsync(p_FinG_out, d + b_po, (size_t)Ftot * 24, cudaMemcpyDeviceToHost, c->stream));
  OVP_CUDA(cudaMemcpyAsync(cp_out, d + b_co, (size_t)n_planes * 24, cudaMemcpyDeviceToHost, c->stream));
  OVP_CUDA(cudaMemcpyAsync(inlier, d + b_il, (size_t)Ftot * 4, cudaMemcpyDeviceToHost, c->stream));
  OVP_CUDA(cudaMemcpyAsync(status, d + b_st, (size_t)n_planes * 4, cudaMemcpyDeviceToHost, c->stream));
  if (info)
    OVP_CUDA(cudaMemcpyAsync(info, d + b_if, (size_t)n_planes * 40, cudaMemcpyDeviceToHost, c->stream));
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  c->d2h_bytes += (int64_t)Ftot * 28 + (int64_t)n_planes * (28 + (info ? 40 : 0));
  return OVP_OK;
}

} // extern "C"

#include "plane_init_tracks.inc" // UpdaterPlane::init_vio_plane end to end on the stages above

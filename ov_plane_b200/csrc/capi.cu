// extern "C" surface of include/ovp.h: State construction, StateHelper entry points, the stateless UpdaterHelper /
// UpdaterPlane helpers, UpdaterMSCKF::update, the multi-GPU shard halves and the Propagator.
#include <cstdlib>
#include "jacobian_core.h"
#include "ovp_internal.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <set>

using namespace ovp;

namespace ovp {

// -------------------------------------------------------------------------------------------------------------------
// small state kernels
// -------------------------------------------------------------------------------------------------------------------
// StateHelper::marginalize (StateHelper.cpp:302-318): x1x1, x1x2 and x2x2 are copied; x2x1 is the transpose of the new x1x2 block
// (:311), not the stored x2x1, which differs from it wherever P is not exactly symmetric (EKFPropagation leaves it so, :103-105)
__global__ void marginalize_copy_kernel(const double *src, double *dst, int ld, int N, int mid, int ms) {
  int Nn = N - ms;
  size_t total = (size_t)Nn * Nn;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int i = (int)(idx % Nn), j = (int)(idx / Nn);
    int si = i < mid ? i : i + ms;
    int sj = j < mid ? j : j + ms;
    const bool x2x1 = i >= mid && j < mid;
    dst[(size_t)j * ld + i] = x2x1 ? src[(size_t)si * ld + sj] : src[(size_t)sj * ld + si];
  }
}
// append a copy of the rows / cols of [old, old+s) at [N, N+s)   (StateHelper::clone, StateHelper.cpp:376-378): the new x new block
// from the old x old block, the column block from the old columns, the row block from the old rows.  Thread (i, j) writes P(i, N+j)
// and, for i < N, P(N+j, i): every entry has one writer, and every read is of the first N rows and columns, which nothing writes.
__global__ void clone_kernel(double *P, int ld, int N, int old, int s) {
  int total = (N + s) * s;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int i = idx % (N + s), j = idx / (N + s);
    int si = i < N ? i : old + (i - N);
    P[(size_t)(N + j) * ld + i] = P[(size_t)(old + j) * ld + si];
    if (i < N)
      P[(size_t)i * ld + (N + j)] = P[(size_t)i * ld + (old + j)];
  }
}
// augment_clone time-offset terms (StateHelper.cpp:613-624), two passes (the second reads the updated dt row)
__global__ void dt_col_kernel(double *P, int ld, int rows, int newid, int dtid, const double *dnc) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * 6)
    return;
  int i = idx % rows, j = idx / rows;
  P[(size_t)(newid + j) * ld + i] += P[(size_t)dtid * ld + i] * dnc[j];
}
__global__ void dt_row_kernel(double *P, int ld, int rows, int newid, int dtid, const double *dnc) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * 6)
    return;
  int i = idx % rows, j = idx / rows;
  P[(size_t)i * ld + (newid + j)] += dnc[j] * P[(size_t)i * ld + dtid];
}
__global__ void gather_block_kernel(const double *P, int ld, const int *idx, int n, double *out) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * n)
    return;
  int i = t % n, j = t / n;
  out[(size_t)j * n + i] = P[(size_t)idx[j] * ld + idx[i]];
}
__global__ void scatter_block_kernel(double *P, int ld, const int *idx, int n, const double *in) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * n)
    return;
  int i = t % n, j = t / n;
  P[(size_t)idx[j] * ld + idx[i]] = in[(size_t)j * n + i];
}
__global__ void sym_from_upper_kernel(double *P, int ld, int N) {
  size_t total = (size_t)N * N;
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    int i = (int)(t % N), j = (int)(t / N);
    if (i > j)
      P[(size_t)j * ld + i] = P[(size_t)i * ld + j];
  }
}
// EKFPropagation write-back (StateHelper.cpp:100-105): P[start.., :] = C^T, P[:, start..] = C, P[start.., start..] = D
__global__ void prop_writeback_kernel(double *P, int ld, int N, int start, int kn, const double *C, int ldc, const double *D, int ldd) {
  int total = N * kn;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int i = idx % N, j = idx / N;
    double v;
    if (i >= start && i < start + kn)
      v = D[(size_t)j * ldd + (i - start)];
    else
      v = C[(size_t)j * ldc + i];
    P[(size_t)(start + j) * ld + i] = v;
    if (!(i >= start && i < start + kn))
      P[(size_t)i * ld + (start + j)] = v;
  }
}
// cross covariance of a newly initialised variable (StateHelper.cpp:568-573): P[0:N, N:N+s] = -M Hinv^T etc.
__global__ void init_grow_kernel(double *P, int ld, int N, int s, const double *Ma, int ldm, const double *HLinv, const double *PLL) {
  int total = (N + s) * s;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int i = idx % (N + s), j = idx / (N + s);
    double v;
    if (i < N) {
      v = 0.0;
      for (int k = 0; k < s; k++)
        v -= Ma[(size_t)k * ldm + i] * HLinv[(size_t)k * s + j]; // (-M_a * H_Linv^T)(i,j) = -sum_k M_a(i,k) H_Linv(j,k)
    } else { // P_LL from its lower triangle: the host product H_Linv M H_Linv^T is symmetric to rounding only, and the threads of
             // (r, j) and (j, r) both write both entries
      const int r = i - N;
      v = PLL[(size_t)min(r, j) * s + max(r, j)];
    }
    P[(size_t)(N + j) * ld + i] = v;
    P[(size_t)i * ld + (N + j)] = v;
  }
}

// UpdaterHelper::get_feature_jacobian_full as a stand-alone kernel: one thread per measurement, output in the reference's
// layout: H_f rows x (3|6), H_x rows x total_hx in x_order [extrinsics, intrinsics, clones (measurement order), plane]
struct JacArgs {
  int m;
  const int *clone_handles;
  const float *uv;
  double pf[3], pf_fej[3];
  int has_plane, plane_in_state;
  int plane_handle; // >= 0: linearisation points of the plane come from the device value / fej tables
  double cp[3], cp_fej[3];
  const double *val, *fej;
  int h_calib, h_intr;
  int do_fej, do_calib_pose, do_calib_intr;
  double white_px, white_c;
  double *Hf, *Hx, *res;
  int rows, hf_cols, hx_cols;
};
__global__ void jacobian_only_kernel(JacArgs a) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.m)
    return;
  const int hcl = a.clone_handles[k];
  const double *vc = a.val + (size_t)hcl * OVP_VAL_STRIDE;
  const double *fc = a.fej + (size_t)hcl * OVP_VAL_STRIDE;
  const double *vcal = a.val + (size_t)a.h_calib * OVP_VAL_STRIDE;
  const double *cam = a.val + (size_t)a.h_intr * OVP_VAL_STRIDE;
  double R_C[9];
  quat_to_rot(vcal, R_C);
  double res[2], Hf[6], Hcl[12], Hcal[12], Hin[16];
  bearing_rows(vc, vc + 4, fc, fc + 4, a.do_fej, R_C, vcal + 4, cam, a.pf, a.pf_fej, a.uv[2 * k], a.uv[2 * k + 1], a.white_px, res, Hf,
               Hcl, Hcal, Hin);
  const int ld = a.rows;
  for (int i = 0; i < 2; i++) {
    int r = 2 * k + i;
    for (int j = 0; j < 3; j++)
      a.Hf[(size_t)j * ld + r] = Hf[3 * i + j];
    int cb = 0;
    if (a.do_calib_pose) {
      for (int j = 0; j < 6; j++)
        a.Hx[(size_t)(cb + j) * ld + r] = Hcal[6 * i + j];
      cb += 6;
    }
    if (a.do_calib_intr) {
      for (int j = 0; j < 8; j++)
        a.Hx[(size_t)(cb + j) * ld + r] = Hin[8 * i + j];
      cb += 8;
    }
    for (int j = 0; j < 6; j++)
      a.Hx[(size_t)(cb + 6 * k + j) * ld + r] = Hcl[6 * i + j];
    a.res[r] = res[i];
  }
  if (a.has_plane) {
    double pr, pHf[3], pHcp[3];
    const double *cp = a.plane_handle >= 0 ? a.val + (size_t)a.plane_handle * OVP_VAL_STRIDE : a.cp;
    const double *cpf = a.plane_handle >= 0 ? a.fej + (size_t)a.plane_handle * OVP_VAL_STRIDE : a.cp_fej;
    plane_row(a.pf, a.pf_fej, cp, cpf, a.do_fej, a.white_c, pr, pHf, pHcp);
    int r = 2 * a.m + k;
    for (int j = 0; j < 3; j++) {
      a.Hf[(size_t)j * ld + r] = pHf[j];
      if (a.plane_in_state)
        a.Hx[(size_t)(a.hx_cols - 3 + j) * ld + r] = pHcp[j];
      else
        a.Hf[(size_t)(3 + j) * ld + r] = pHcp[j];
    }
    a.res[r] = pr;
  }
}

__global__ void dmma_selftest_fill(double *p, size_t n, double scale) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n)
    p[i] = scale * (double)((i * 2654435761u) % 1024) / 1024.0;
}

static int valid_handle(Ctx *c, int h) { return h >= 0 && h < (int)c->vars.size() && c->vars[h].alive; }

// device array of state column indices for a list of handles (into c->dcols + slot*Rcap)
static int upload_cols(Ctx *c, const int *handles, int k, int slot, int *n_out, bool require_in_state = true) {
  std::vector<int> cols;
  for (int i = 0; i < k; i++) {
    if (!valid_handle(c, handles[i]))
      return fail(c, OVP_ERR_BAD_ARGS, "invalid variable handle %d", handles[i]);
    const Var &v = c->vars[handles[i]];
    if (v.id < 0 && require_in_state)
      return fail(c, OVP_ERR_NOT_IN_STATE, "variable %d is not in the state", handles[i]);
    for (int j = 0; j < v.size; j++)
      cols.push_back(v.id + j);
  }
  if ((int)cols.size() > c->Rcap)
    return fail(c, OVP_ERR_CAPACITY, "%d columns exceed capacity %d", (int)cols.size(), c->Rcap);
  if (!cols.empty()) {
    int st = stage_copy_in(c, c->dcols + (size_t)slot * c->Rcap, cols.data(), cols.size() * sizeof(int));
    if (st)
      return st;
    OVP_CUDA(cudaStreamSynchronize(c->stream));
  }
  *n_out = (int)cols.size();
  return OVP_OK;
}

static int do_marginalize(Ctx *c, int h) {
  if (!valid_handle(c, h) || c->vars[h].id < 0)
    return fail(c, OVP_ERR_NOT_IN_STATE, "marginalize: variable %d not in the state (reference: std::exit, StateHelper.cpp:279-283)", h);
  Var &v = c->vars[h];
  if (v.kind == OVP_KIND_POSE) // a clone that still anchors a landmark: the reference asserts change_anchors ran first (UpdaterSLAM.cpp:699)
    for (auto &kv : c->slam)
      if (c->vars[kv.second].id >= 0 && c->vars[kv.second].rep >= 2 && c->vars[kv.second].anchor == h)
        return fail(c, OVP_ERR_BAD_ARGS, "marginalize: clone %d is the anchor of landmark %lld - call ovp_slam_change_anchors first", h, (long long)kv.first);
  int mid = v.id, ms = v.size, N = c->N;
  // compaction into the scratch covariance, then swap (StateHelper.cpp:302-318)
  double *dst = c->dM; // Nmax x Rcap >= Nmax x Nmax scratch
  int blocks = std::min(c->num_sms * 8, (int)(((size_t)(N - ms) * (N - ms) + 255) / 256) + 1);
  marginalize_copy_kernel<<<blocks, 256, 0, c->stream>>>(c->dP, dst, c->ldP, N, mid, ms);
  c->launches++;
  OVP_CUDA(cudaMemcpy2DAsync(c->dP, (size_t)c->ldP * sizeof(double), dst, (size_t)c->ldP * sizeof(double), (size_t)(N - ms) * sizeof(double),
                             N - ms, cudaMemcpyDeviceToDevice, c->stream));
  c->launches++;
  for (auto &o : c->vars)
    if (o.alive && o.id > mid)
      o.id -= ms;
  v.id = -1;
  v.alive = false;
  c->free_handles.push_back(h);
  c->order.erase(std::remove(c->order.begin(), c->order.end(), h), c->order.end());
  c->N = N - ms;
  c->var_table_dirty = true;
  for (auto it = c->clones.begin(); it != c->clones.end(); ++it)
    if (it->second == h) {
      c->clones.erase(it);
      break;
    }
  for (auto it = c->planes.begin(); it != c->planes.end(); ++it)
    if (it->second == h) {
      c->planes.erase(it);
      break;
    }
  for (auto it = c->slam.begin(); it != c->slam.end(); ++it)
    if (it->second == h) {
      c->slam_to_plane.erase(it->first);
      c->slam.erase(it);
      break;
    }
  return OVP_OK;
}

} // namespace ovp

extern "C" {

const char *ovp_status_string(int s) {
  switch (s) {
  case OVP_OK:
    return "ok";
  case OVP_ERR_BAD_ARGS:
    return "bad arguments";
  case OVP_ERR_NEGATIVE_DIAGONAL:
    return "negative covariance diagonal";
  case OVP_ERR_NON_CONTIGUOUS:
    return "non-contiguous NEW order";
  case OVP_ERR_NON_ISOTROPIC:
    return "noise not isotropic";
  case OVP_ERR_NOT_IN_STATE:
    return "variable not in the state";
  case OVP_ERR_ALREADY_IN_STATE:
    return "variable already in the state";
  case OVP_ERR_CAPACITY:
    return "capacity exceeded";
  case OVP_ERR_CUDA:
    return "CUDA error";
  case OVP_ERR_NOT_POSITIVE_DEFINITE:
    return "matrix not positive definite";
  case OVP_ERR_TIME:
    return "invalid timestamp";
  }
  return "unknown";
}

int ovp_create(const ovp_state_options *opt, int device, int max_state, int max_meas_rows, ovp_ctx **out) {
  if (!opt || !out || max_state < 32)
    return OVP_ERR_BAD_ARGS;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device >= ndev)
    return OVP_ERR_CUDA; // no CPU fallback: the path needs a CUDA device
  ovp_ctx *h = new ovp_ctx();
  h->c.device = device; // before enter: it makes this device current, and no other device gets a context
  Ctx *c = ovp::enter(h);
  c->opt = *opt;
  *out = h;
  OVP_CUDA(cudaSetDevice(device));
  OVP_CUDA(cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device));
  OVP_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  OVP_CUDA(cudaStreamCreateWithFlags(&c->stream2, cudaStreamNonBlocking));
  OVP_CUDA(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
  OVP_CUDA(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
  OVP_CUDA(cudaStreamCreateWithFlags(&c->stream3, cudaStreamNonBlocking));
  OVP_CUDA(cudaEventCreateWithFlags(&c->ev_dfork, cudaEventDisableTiming));
  OVP_CUDA(cudaEventCreateWithFlags(&c->ev_djoin, cudaEventDisableTiming));
  for (int i = 0; i < 8; i++)
    OVP_CUDA(cudaEventCreate(&c->ev[i]));
  c->Nmax = (max_state + 63) / 64 * 64;
  c->ldP = c->Nmax;
  c->Rcap = c->Nmax + 64;
  c->max_meas_rows = std::max(max_meas_rows, 64);
  c->max_handles = 8192; // live variables + reuse lag; slots are recycled (state_append_variable)
  OVP_CUDA(cudaMalloc(&c->dP, (size_t)c->ldP * c->Nmax * sizeof(double)));
  OVP_CUDA(cudaMemset(c->dP, 0, (size_t)c->ldP * c->Nmax * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->d_val, (size_t)c->max_handles * OVP_VAL_STRIDE * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->d_fej, (size_t)c->max_handles * OVP_VAL_STRIDE * sizeof(double)));
  OVP_CUDA(cudaMemset(c->d_val, 0, (size_t)c->max_handles * OVP_VAL_STRIDE * sizeof(double)));
  OVP_CUDA(cudaMemset(c->d_fej, 0, (size_t)c->max_handles * OVP_VAL_STRIDE * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->d_var_id, c->max_handles * sizeof(int)));
  OVP_CUDA(cudaMalloc(&c->d_var_size, c->max_handles * sizeof(int)));
  OVP_CUDA(cudaMalloc(&c->d_var_kind, c->max_handles * sizeof(int)));
  int st = ws_alloc(c, c->wsG, c->Rcap);
  if (st)
    return st;
  st = ws_alloc(c, c->wsS, c->Rcap);
  if (st)
    return st;
  c->cf_maxT = c->Rcap / 64 + 1;
  OVP_CUDA(cudaMalloc(&c->cf_linv, (size_t)c->cf_maxT * 4096 * sizeof(double)));
  // exchange slots of the fused Cholesky (cholfused.cu): T*T panel tiles + 2T hand-off tiles, 64 x 68 doubles each
  OVP_CUDA(cudaMalloc(&c->cf_xch, ((size_t)c->cf_maxT * c->cf_maxT + 2 * c->cf_maxT) * 64 * 68 * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->cf_diag0, (size_t)c->cf_maxT * 64 * sizeof(double)));
  OVP_CUDA(cudaMemset(c->cf_diag0, 0, (size_t)c->cf_maxT * 64 * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->cf_flags, (size_t)(3 * c->cf_maxT + c->cf_maxT * c->cf_maxT) * sizeof(int)));
  // epoch, finished CTAs, product queue head, M done per column block, z-row tiles stored, "S(i, j) stored" per lower tile
  const size_t nctrl = 5 + c->cf_maxT + (size_t)c->cf_maxT * (c->cf_maxT + 1) / 2;
  OVP_CUDA(cudaMalloc(&c->cf_ctrl, nctrl * sizeof(int)));
  OVP_CUDA(cudaMemset(c->cf_linv, 0, (size_t)c->cf_maxT * 4096 * sizeof(double)));
  OVP_CUDA(cudaMemset(c->cf_flags, 0, (size_t)(3 * c->cf_maxT + c->cf_maxT * c->cf_maxT) * sizeof(int)));
  OVP_CUDA(cudaMemset(c->cf_ctrl, 0, nctrl * sizeof(int)));
  // the second set, for the innovation factorisation of a pair (chol_fused_pair)
  OVP_CUDA(cudaMalloc(&c->cf_linv_s, (size_t)c->cf_maxT * 4096 * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->cf_xch_s, ((size_t)c->cf_maxT * c->cf_maxT + 2 * c->cf_maxT) * 64 * 68 * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->cf_diag0_s, (size_t)c->cf_maxT * 64 * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->cf_flags_s, (size_t)(3 * c->cf_maxT + c->cf_maxT * c->cf_maxT) * sizeof(int)));
  OVP_CUDA(cudaMemset(c->cf_linv_s, 0, (size_t)c->cf_maxT * 4096 * sizeof(double)));
  OVP_CUDA(cudaMemset(c->cf_diag0_s, 0, (size_t)c->cf_maxT * 64 * sizeof(double)));
  OVP_CUDA(cudaMemset(c->cf_flags_s, 0, (size_t)(3 * c->cf_maxT + c->cf_maxT * c->cf_maxT) * sizeof(int)));
  // systems wider than one launch (cholpanel.cu): original diagonal, z, chi2 per panel
  OVP_CUDA(cudaMalloc(&c->cf_panel, ((size_t)2 * c->Rcap + c->cf_maxT) * sizeof(double)));
  OVP_CUDA(cudaMemset(c->cf_panel, 0, ((size_t)2 * c->Rcap + c->cf_maxT) * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->dM, (size_t)c->Nmax * c->Rcap * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->dY, (size_t)c->Nmax * c->Rcap * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->dHT, (size_t)c->Rcap * c->Rcap * sizeof(double)));
  OVP_CUDA(cudaMemset(c->dM, 0, (size_t)c->Nmax * c->Rcap * sizeof(double)));
  OVP_CUDA(cudaMemset(c->dY, 0, (size_t)c->Nmax * c->Rcap * sizeof(double)));
  OVP_CUDA(cudaMemset(c->dHT, 0, (size_t)c->Rcap * c->Rcap * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->dvec, ((size_t)8 * c->Rcap + (2 + OVP_DX_SPLIT) * c->Nmax) * sizeof(double)));
  OVP_CUDA(cudaMemset(c->dvec, 0, ((size_t)8 * c->Rcap + (2 + OVP_DX_SPLIT) * c->Nmax) * sizeof(double)));
  OVP_CUDA(cudaMalloc(&c->dcols, (size_t)8 * c->Rcap * sizeof(int)));
  OVP_CUDA(cudaMalloc(&c->dflags, 256 * sizeof(int)));
  OVP_CUDA(cudaMemset(c->dflags, 0, 256 * sizeof(int)));
  OVP_CUDA(cudaMalloc(&c->dscal, 256 * sizeof(double)));
  OVP_CUDA(cudaMemset(c->dscal, 0, 256 * sizeof(double)));
  c->Hs_elems = (size_t)(c->max_meas_rows + 8) * c->Rcap;
  OVP_CUDA(cudaMalloc(&c->dHs, c->Hs_elems * sizeof(double)));
  OVP_CUDA(cudaMemset(c->dHs, 0, c->Hs_elems * sizeof(double)));
  c->part_elems = (size_t)64 * c->Rcap * c->Rcap;
  OVP_CUDA(cudaMalloc(&c->dPart, c->part_elems * sizeof(double)));
  OVP_CUDA(cudaMemset(c->dPart, 0, c->part_elems * sizeof(double)));
  OVP_CUDA(cudaDeviceSynchronize());
  // ---- State::State(options), State.cpp:33-102 ----
  Var imu;
  imu.kind = OVP_KIND_IMU;
  imu.size = 15;
  imu.nvalue = 16;
  double v16[16] = {0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  st = state_append_variable(c, imu, v16, v16, &c->h_imu);
  if (st)
    return st;
  c->vars[c->h_imu].id = 0;
  c->order.push_back(c->h_imu);
  int cur = 15;
  Var dt;
  dt.kind = OVP_KIND_VEC;
  dt.size = 1;
  dt.nvalue = 1;
  double z1[1] = {0};
  st = state_append_variable(c, dt, z1, z1, &c->h_dt);
  if (st)
    return st;
  if (opt->do_calib_camera_timeoffset) {
    c->vars[c->h_dt].id = cur;
    c->order.push_back(c->h_dt);
    cur += 1;
  }
  Var ext;
  ext.kind = OVP_KIND_POSE;
  ext.size = 6;
  ext.nvalue = 7;
  double v7[7] = {0, 0, 0, 1, 0, 0, 0};
  st = state_append_variable(c, ext, v7, v7, &c->h_calib);
  if (st)
    return st;
  Var intr;
  intr.kind = OVP_KIND_VEC;
  intr.size = 8;
  intr.nvalue = 8;
  double z8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  st = state_append_variable(c, intr, z8, z8, &c->h_intr);
  if (st)
    return st;
  if (opt->do_calib_camera_pose) {
    c->vars[c->h_calib].id = cur;
    c->order.push_back(c->h_calib);
    cur += 6;
  }
  if (opt->do_calib_camera_intrinsics) {
    c->vars[c->h_intr].id = cur;
    c->order.push_back(c->h_intr);
    cur += 8;
  }
  c->N = cur;
  std::vector<double> P0((size_t)cur * cur, 0.0);
  for (int i = 0; i < cur; i++)
    P0[(size_t)i * cur + i] = std::pow(1e-3, 2);
  if (opt->do_calib_camera_timeoffset) {
    int b = c->vars[c->h_dt].id;
    P0[(size_t)b * cur + b] = std::pow(0.01, 2);
  }
  if (opt->do_calib_camera_pose) {
    int b = c->vars[c->h_calib].id;
    for (int i = 0; i < 3; i++) {
      P0[(size_t)(b + i) * cur + b + i] = std::pow(0.005, 2);
      P0[(size_t)(b + 3 + i) * cur + b + 3 + i] = std::pow(0.01, 2);
    }
  }
  if (opt->do_calib_camera_intrinsics) {
    int b = c->vars[c->h_intr].id;
    for (int i = 0; i < 4; i++) {
      P0[(size_t)(b + i) * cur + b + i] = std::pow(1.0, 2);
      P0[(size_t)(b + 4 + i) * cur + b + 4 + i] = std::pow(0.005, 2);
    }
  }
  st = stage_copy2d_in(c, c->dP, (size_t)c->ldP * sizeof(double), P0.data(), (size_t)cur * sizeof(double), (size_t)cur * sizeof(double), cur);
  if (st)
    return st;
  return upload_var_table(c); // synchronises the stream
}

void ovp_destroy(ovp_ctx *h) {
  if (!h)
    return;
  Ctx *c = ovp::enter(h);
  if (c->stream)
    cudaStreamSynchronize(c->stream);
  cudaFree(c->dP);
  cudaFree(c->d_val);
  cudaFree(c->d_fej);
  cudaFree(c->d_var_id);
  cudaFree(c->d_var_size);
  cudaFree(c->d_var_kind);
  cudaFree(c->cf_linv);
  cudaFree(c->cf_xch);
  cudaFree(c->cf_diag0);
  cudaFree(c->cf_flags);
  cudaFree(c->cf_ctrl);
  cudaFree(c->cf_linv_s);
  cudaFree(c->cf_xch_s);
  cudaFree(c->cf_diag0_s);
  cudaFree(c->cf_flags_s);
  cudaFree(c->cf_panel);
  ws_free(c->wsG);
  ws_free(c->wsS);
  cudaFree(c->dM);
  cudaFree(c->dY);
  cudaFree(c->dHT);
  cudaFree(c->dvec);
  cudaFree(c->dcols);
  cudaFree(c->dflags);
  cudaFree(c->dscal);
  if (c->nccl_comm)
    ovp_nccl_finalize(h);
  cudaFree(c->d_gather);
  cudaFree(c->dHs);
  cudaFree(c->d_mw);
  cudaFree(c->dPart);
  cudaFree(c->d_chi2_table);
  cudaFree(c->d_batch);
  cudaFree(c->d_stage);
  cudaFree(c->snapP);
  cudaFree(c->snap_val);
  cudaFree(c->snap_fej);
  c->snapP = c->snap_val = c->snap_fej = nullptr;
  free_prepared(c);
  for (auto e : c->ev_pool)
    cudaEventDestroy(e);
  c->ev_pool.clear();
  c->ev_used = 0;
  if (c->h_pinned)
    cudaFreeHost(c->h_pinned);
  for (int i = 0; i < 8; i++)
    cudaEventDestroy(c->ev[i]);
  if (c->stream2)
    cudaStreamDestroy(c->stream2);
  if (c->ev_fork)
    cudaEventDestroy(c->ev_fork);
  if (c->ev_join)
    cudaEventDestroy(c->ev_join);
  if (c->stream3)
    cudaStreamDestroy(c->stream3);
  if (c->ev_dfork)
    cudaEventDestroy(c->ev_dfork);
  if (c->ev_djoin)
    cudaEventDestroy(c->ev_djoin);
  if (c->stream)
    cudaStreamDestroy(c->stream);
  delete h;
}

const char *ovp_last_error(ovp_ctx *h) { return h ? h->c.last_error.c_str() : "null ctx"; }

int ovp_set_chi2_table(ovp_ctx *h, const double *q, int n) {
  Ctx *c = ovp::enter(h);
  if (!q || n < 2)
    return fail(c, OVP_ERR_BAD_ARGS, "chi2 table needs >= 2 entries");
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  // a prepared batch (and its captured graph) holds the old table pointer and host-side thresholds by value: drop it
  free_prepared(c);
  c->chi2_table.assign(q, q + n);
  if (c->d_chi2_table)
    cudaFree(c->d_chi2_table);
  c->d_chi2_table = nullptr;
  OVP_CUDA(cudaMalloc(&c->d_chi2_table, n * sizeof(double)));
  int st = stage_copy_in(c, c->d_chi2_table, q, n * sizeof(double));
  if (st)
    return st;
  c->chi2_table_n = n;
  return OVP_OK;
}

int ovp_cov_rows(ovp_ctx *h) { return h->c.N; }
int ovp_cov_download(ovp_ctx *h, double *out, int ld) {
  Ctx *c = ovp::enter(h);
  if (ld < c->N)
    return fail(c, OVP_ERR_BAD_ARGS, "ld < rows");
  int st = stage_copy2d_out(c, out, (size_t)ld * sizeof(double), c->dP, (size_t)c->ldP * sizeof(double), (size_t)c->N * sizeof(double), c->N);
  if (st)
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  return OVP_OK;
}
int ovp_cov_upload(ovp_ctx *h, const double *in, int n, int ld) {
  Ctx *c = ovp::enter(h);
  if (n != c->N || ld < n)
    return fail(c, OVP_ERR_BAD_ARGS, "cov_upload: n=%d but the state has %d rows", n, c->N);
  int st = stage_copy2d_in(c, c->dP, (size_t)c->ldP * sizeof(double), in, (size_t)ld * sizeof(double), (size_t)n * sizeof(double), n);
  if (st)
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  return OVP_OK;
}
int ovp_handle_imu(ovp_ctx *h) { return h->c.h_imu; }
int ovp_handle_dt(ovp_ctx *h) { return h->c.h_dt; }
int ovp_handle_calib(ovp_ctx *h) { return h->c.h_calib; }
int ovp_handle_intrinsics(ovp_ctx *h) { return h->c.h_intr; }
int ovp_var_id(ovp_ctx *h, int v) { return valid_handle(&h->c, v) ? h->c.vars[v].id : -1; }
int ovp_var_size(ovp_ctx *h, int v) { return (v >= 0 && v < (int)h->c.vars.size()) ? h->c.vars[v].size : -1; }
int ovp_var_value_size(ovp_ctx *h, int v) { return (v >= 0 && v < (int)h->c.vars.size()) ? h->c.vars[v].nvalue : -1; }
int ovp_var_set(ovp_ctx *h, int v, const double *value, const double *fej) {
  Ctx *c = ovp::enter(h);
  if (v < 0 || v >= (int)c->vars.size())
    return fail(c, OVP_ERR_BAD_ARGS, "invalid handle %d", v);
  int st = sync_host_values(c);
  if (st)
    return st;
  for (int i = 0; i < c->vars[v].nvalue; i++) {
    if (value)
      c->h_val[(size_t)v * OVP_VAL_STRIDE + i] = value[i];
    if (fej)
      c->h_fej[(size_t)v * OVP_VAL_STRIDE + i] = fej[i];
  }
  return push_host_values(c, v);
}
int ovp_var_get(ovp_ctx *h, int v, double *value, double *fej) {
  Ctx *c = ovp::enter(h);
  if (v < 0 || v >= (int)c->vars.size())
    return fail(c, OVP_ERR_BAD_ARGS, "invalid handle %d", v);
  int st = sync_host_values(c);
  if (st)
    return st;
  for (int i = 0; i < c->vars[v].nvalue; i++) {
    if (value)
      value[i] = c->h_val[(size_t)v * OVP_VAL_STRIDE + i];
    if (fej)
      fej[i] = c->h_fej[(size_t)v * OVP_VAL_STRIDE + i];
  }
  return OVP_OK;
}
int ovp_num_variables(ovp_ctx *h) { return (int)h->c.order.size(); }
int ovp_variable_order(ovp_ctx *h, int *handles) {
  for (size_t i = 0; i < h->c.order.size(); i++)
    handles[i] = h->c.order[i];
  return OVP_OK;
}
int ovp_set_timestamp(ovp_ctx *h, double t) {
  h->c.timestamp = t;
  return OVP_OK;
}
double ovp_get_timestamp(ovp_ctx *h) { return h->c.timestamp; }
int ovp_plane_handle(ovp_ctx *h, int64_t planeid) {
  auto it = h->c.planes.find(planeid);
  return it == h->c.planes.end() ? -1 : it->second;
}
int ovp_clone_handle(ovp_ctx *h, double ts) {
  auto it = h->c.clones.find(ts);
  return it == h->c.clones.end() ? -1 : it->second;
}

static int add_raw(Ctx *c, Var v, const double *value, const double *fej, int *handle) {
  if (c->N + v.size > c->Nmax)
    return fail(c, OVP_ERR_CAPACITY, "state capacity %d exceeded", c->Nmax);
  int st = state_append_variable(c, v, value, fej, handle);
  if (st)
    return st;
  int blocks = ((c->N + v.size) * v.size + 255) / 256;
  ovp::zero_band_kernel<<<blocks, 256, 0, c->stream>>>(c->dP, c->ldP, c->N, v.size);
  c->launches++;
  c->vars[*handle].id = c->N;
  c->order.push_back(*handle);
  c->N += v.size;
  return OVP_OK;
}
int ovp_add_clone_raw(ovp_ctx *h, double timestamp, const double *value7, const double *fej7, int *handle) {
  Ctx *c = ovp::enter(h);
  if (c->clones.count(timestamp))
    return fail(c, OVP_ERR_TIME, "clone at this timestamp already exists");
  Var v;
  v.kind = OVP_KIND_POSE;
  v.size = 6;
  v.nvalue = 7;
  int st = add_raw(c, v, value7, fej7, handle);
  if (st)
    return st;
  c->clones[timestamp] = *handle;
  return OVP_OK;
}
int ovp_add_plane_raw(ovp_ctx *h, int64_t planeid, const double *cp, const double *cp_fej, int *handle) {
  Ctx *c = ovp::enter(h);
  if (c->planes.count(planeid))
    return fail(c, OVP_ERR_ALREADY_IN_STATE, "plane already in the state");
  Var v;
  v.kind = OVP_KIND_VEC;
  v.size = 3;
  v.nvalue = 3;
  v.tag = planeid;
  int st = add_raw(c, v, cp, cp_fej, handle);
  if (st)
    return st;
  c->planes[planeid] = *handle;
  return OVP_OK;
}
int ovp_add_slam_raw(ovp_ctx *h, int64_t featid, const double *p, const double *p_fej, int *handle) {
  Ctx *c = ovp::enter(h);
  if (c->slam.count(featid))
    return fail(c, OVP_ERR_ALREADY_IN_STATE, "landmark already in the state");
  Var v;
  v.kind = OVP_KIND_LANDMARK;
  v.size = 3;
  v.nvalue = 3;
  v.tag = featid;
  int st = add_raw(c, v, p, p_fej, handle);
  if (st)
    return st;
  c->slam[featid] = *handle;
  return OVP_OK;
}

// ---- StateHelper -----------------------------------------------------------------------------------------------------
int ovp_get_marginal_covariance(ovp_ctx *h, const int *handles, int k, double *out) {
  Ctx *c = ovp::enter(h);
  int n = 0;
  int st = upload_cols(c, handles, k, 0, &n);
  if (st)
    return st;
  if (n == 0)
    return OVP_OK;
  StageLayout L;
  const size_t b_blk = L.take((size_t)n * n * sizeof(double));
  if ((st = ensure_stage(c, L)))
    return st;
  double *blk = (double *)(c->d_stage + b_blk);
  gather_block_kernel<<<(n * n + 255) / 256, 256, 0, c->stream>>>(c->dP, c->ldP, c->dcols, n, blk);
  c->launches++;
  if ((st = stage_copy_out(c, out, blk, (size_t)n * n * sizeof(double))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  return OVP_OK;
}
int ovp_set_initial_covariance(ovp_ctx *h, const double *cov, int n_in, const int *handles, int k) {
  Ctx *c = ovp::enter(h);
  int n = 0;
  int st = upload_cols(c, handles, k, 0, &n);
  if (st)
    return st;
  if (n != n_in)
    return fail(c, OVP_ERR_BAD_ARGS, "set_initial_covariance: %d != sum of sizes %d", n_in, n);
  StageLayout L;
  const size_t b_blk = L.take((size_t)n * n * sizeof(double));
  if ((st = ensure_stage(c, L)))
    return st;
  double *blk = (double *)(c->d_stage + b_blk);
  if ((st = stage_copy_in(c, blk, cov, (size_t)n * n * sizeof(double))))
    return st;
  scatter_block_kernel<<<(n * n + 255) / 256, 256, 0, c->stream>>>(c->dP, c->ldP, c->dcols, n, blk);
  c->launches++;
  sym_from_upper_kernel<<<c->num_sms * 4, 256, 0, c->stream>>>(c->dP, c->ldP, c->N);
  c->launches++;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  return OVP_OK;
}

int ovp_ekf_propagation(ovp_ctx *h, const int *new_h, int kn, const int *old_h, int ko, const double *Phi, int phi_rows, int phi_cols,
                        const double *Q) {
  Ctx *c = ovp::enter(h);
  if (kn <= 0 || ko <= 0)
    return fail(c, OVP_ERR_BAD_ARGS, "EKFPropagation called with empty variable arrays (reference: std::exit, StateHelper.cpp:46-49)");
  for (int i = 0; i < kn; i++)
    if (!valid_handle(c, new_h[i]) || c->vars[new_h[i]].id < 0)
      return fail(c, OVP_ERR_NOT_IN_STATE, "EKFPropagation: NEW variable %d not in the state", new_h[i]);
  int size_new = c->vars[new_h[0]].size;
  for (int i = 0; i + 1 < kn; i++) {
    if (c->vars[new_h[i]].id + c->vars[new_h[i]].size != c->vars[new_h[i + 1]].id)
      return fail(c, OVP_ERR_NON_CONTIGUOUS, "EKFPropagation: non-contiguous state elements (StateHelper.cpp:52-61)");
    size_new += c->vars[new_h[i + 1]].size;
  }
  int size_old = 0;
  int st = upload_cols(c, old_h, ko, 0, &size_old);
  if (st)
    return st;
  if (size_new != phi_rows || size_old != phi_cols)
    return fail(c, OVP_ERR_BAD_ARGS, "EKFPropagation: Phi is %dx%d, variables give %dx%d", phi_rows, phi_cols, size_new, size_old);
  if (size_new > c->Rcap || size_old > c->Rcap)
    return fail(c, OVP_ERR_CAPACITY, "EKFPropagation: block too large");
  const int N = c->N, start = c->vars[new_h[0]].id;
  StageLayout L;
  const size_t phi_bytes = (size_t)phi_rows * phi_cols * sizeof(double), q_bytes = (size_t)phi_rows * phi_rows * sizeof(double);
  const size_t b_phi = L.take(phi_bytes), b_q = L.take(q_bytes);
  if ((st = ensure_stage(c, L)))
    return st;
  double *dPhi = (double *)(c->d_stage + b_phi), *dQ = (double *)(c->d_stage + b_q);
  if ((st = stage_copy_in(c, dPhi, Phi, phi_bytes)) || (st = stage_copy_in(c, dQ, Q, q_bytes)))
    return st;
  sym_from_upper_kernel<<<8, 256, 0, c->stream>>>(dQ, phi_rows, phi_rows); // Q.selfadjointView<Upper>() (:93)
  c->launches++;
  // Cov_PhiT = P[:, old] Phi^T   (N x kn)
  launch_gemm1(c, make_problem(N, phi_rows, phi_cols, mv(c->dP, c->ldP, 0, nullptr, c->dcols), mv(dPhi, phi_rows, 1), c->dM, c->Nmax));
  // Phi_Cov_PhiT = Qsym + Phi * Cov_PhiT[old rows, :]
  {
    GemmProblem p = make_problem(phi_rows, phi_rows, phi_cols, mv(dPhi, phi_rows), mv(c->dM, c->Nmax, 0, c->dcols, nullptr), dQ, phi_rows, 1.0, 1.0);
    launch_gemm1(c, p);
  }
  prop_writeback_kernel<<<std::min(c->num_sms * 4, (N * phi_rows + 255) / 256), 256, 0, c->stream>>>(c->dP, c->ldP, N, start, phi_rows, c->dM, c->Nmax,
                                                                                               dQ, phi_rows);
  c->launches++;
  diag_check_kernel<<<(N + 127) / 128, 128, 0, c->stream>>>(c->dP, c->ldP, N, c->dflags, nullptr);
  c->launches++;
  return check_status_flags(c);
}

} // extern "C"

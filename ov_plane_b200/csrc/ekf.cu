// Device-resident State (covariance + variable values) and the StateHelper algebra:
// EKFUpdate (StateHelper.cpp:121-202), EKFPropagation (:41-119), clone / augment_clone (:346-396, :588-625),
// marginalize (:276-344), get_marginal_covariance (:231-259), set_initial_covariance (:204-229),
// initialize_invertible's covariance growth (:568-573) and ov_type::*::update (the manifold update of every variable).
#include "ovp_internal.h"
#include "host_math.h"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace ovp {

// -------------------------------------------------------------------------------------------------------------------
// ov_type::Vec/JPLQuat/PoseJPL/IMU/Landmark::update on the device (JPL left-multiplicative quaternion update)
// -------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void quat_left_update(double *q, const double *dth) {
  // dq = quatnorm([0.5*dth; 1]); q <- quat_multiply(dq, q)   (ov_core quat_ops.h semantics, SURVEY §8(c))
  double a0 = 0.5 * dth[0], a1 = 0.5 * dth[1], a2 = 0.5 * dth[2], a3 = 1.0;
  double nrm = sqrt(a0 * a0 + a1 * a1 + a2 * a2 + a3 * a3);
  a0 /= nrm;
  a1 /= nrm;
  a2 /= nrm;
  a3 /= nrm;
  double p0 = q[0], p1 = q[1], p2 = q[2], p3 = q[3];
  // Qm = [a3*I - skew(av), av; -av^T, a3]
  double r0 = a3 * p0 + a2 * p1 - a1 * p2 + a0 * p3;
  double r1 = -a2 * p0 + a3 * p1 + a0 * p2 + a1 * p3;
  double r2 = a1 * p0 - a0 * p1 + a3 * p2 + a2 * p3;
  double r3 = -a0 * p0 - a1 * p1 - a2 * p2 + a3 * p3;
  if (r3 < 0) {
    r0 = -r0;
    r1 = -r1;
    r2 = -r2;
    r3 = -r3;
  }
  double n2 = sqrt(r0 * r0 + r1 * r1 + r2 * r2 + r3 * r3);
  q[0] = r0 / n2;
  q[1] = r1 / n2;
  q[2] = r2 / n2;
  q[3] = r3 / n2;
}

// dx = Y w, stage 1: OVP_DX_SPLIT partial sums per state row.  Y is column-major (row i of column k at Y[k * ldy + i]): 64 consecutive rows per
// CTA are one coalesced 512-byte segment per column; the CTA's 4 thread groups take every 4th column of the chunk, so a thread has <= 16
// independent loads (all in flight at once) and a fixed summation order.
__global__ void __launch_bounds__(256) dx_partial_kernel(const double *Y, int ldy, int N, const double *w, int rr, double *part, int ldpart,
                                                         const int *flag) {
  if (flag && *flag == 0)
    return;
  __shared__ double red[4][64];
  const int r = threadIdx.x & 63, kl = threadIdx.x >> 6;
  const int i = blockIdx.x * 64 + r;
  const int chunk = (rr + OVP_DX_SPLIT - 1) / OVP_DX_SPLIT;
  const int k0 = blockIdx.y * chunk, k1 = min(rr, k0 + chunk);
  double s = 0.0;
  if (i < N) {
    for (int kb = k0 + kl; kb < k1; kb += 64) { // 16 columns of this thread group per round
      double v[16], wk[16];
#pragma unroll
      for (int u = 0; u < 16; u++) {
        const int k = kb + 4 * u;
        const bool ok = k < k1;
        v[u] = ok ? Y[(size_t)k * ldy + i] : 0.0;
        wk[u] = ok ? w[k] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 16; u++)
        s = fma(v[u], wk[u], s);
    }
  }
  red[kl][r] = s;
  __syncthreads();
  if (kl == 0 && i < N)
    part[(size_t)blockIdx.y * ldpart + i] = ((red[0][r] + red[1][r]) + red[2][r]) + red[3][r];
}

// Tail of EKFUpdate, stage 2, one warp per variable: dx rows of the variable = sum of the partial sums (lane = row, fixed order),
// ov_type::update on the device (StateHelper.cpp:190-193), and optionally the negative-diagonal check of the variable's covariance rows
// (:176-187).  Skipped when the gate flag says the update was rejected.
__global__ void __launch_bounds__(128) finish_update_kernel(int nh, const int *var_id, const int *var_size, const int *var_kind, double *val,
                                                            const double *part, int ldpart, const double *P, int ldP, int *neg_flag,
                                                            const int *flag) {
  const int h = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (h >= nh)
    return;
  if (flag && *flag == 0)
    return;
  const int id = var_id[h];
  if (id < 0)
    return;
  const int s = var_size[h];
  double mine = 0.0;
  if (lane < s) {
    double pv[OVP_DX_SPLIT];
#pragma unroll
    for (int q = 0; q < OVP_DX_SPLIT; q++)
      pv[q] = part[(size_t)q * ldpart + id + lane];
#pragma unroll
    for (int q = 0; q < OVP_DX_SPLIT; q++)
      mine += pv[q];
  }
  double acc[15];
#pragma unroll
  for (int j = 0; j < 15; j++)
    acc[j] = __shfl_sync(0xffffffffu, mine, j); // dx of row j on every lane
  if (P && lane < s && P[(size_t)(id + lane) * ldP + id + lane] < 0.0)
    atomicExch(neg_flag, 1);
  if (lane != 0)
    return;
  double *v = val + (size_t)h * OVP_VAL_STRIDE;
  const int kind = var_kind[h];
  if (kind == OVP_KIND_VEC || kind == OVP_KIND_LANDMARK) {
#pragma unroll
    for (int i = 0; i < 15; i++)
      if (i < s)
        v[i] += acc[i];
    return;
  }
  quat_left_update(v, acc);
  v[4] += acc[3];
  v[5] += acc[4];
  v[6] += acc[5];
  if (kind == OVP_KIND_IMU)
#pragma unroll
    for (int i = 0; i < 9; i++)
      v[7 + i] += acc[6 + i];
}

__global__ void diag_check_kernel(const double *P, int ld, int N, int *flag_out, const int *flag) {
  if (flag && *flag == 0)
    return;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N && P[(size_t)i * ld + i] < 0.0)
    atomicExch(flag_out, 1);
}

int upload_var_table(Ctx *c) {
  int nh = (int)c->vars.size();
  if (nh > c->max_handles)
    return fail(c, OVP_ERR_CAPACITY, "variable handle capacity %d exceeded", c->max_handles);
  std::vector<int> id(nh), sz(nh), kd(nh);
  for (int h = 0; h < nh; h++) {
    id[h] = c->vars[h].alive ? c->vars[h].id : -1;
    sz[h] = c->vars[h].size;
    kd[h] = c->vars[h].kind;
  }
  OVP_CUDA(cudaMemcpyAsync(c->d_var_id, id.data(), nh * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  OVP_CUDA(cudaMemcpyAsync(c->d_var_size, sz.data(), nh * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  OVP_CUDA(cudaMemcpyAsync(c->d_var_kind, kd.data(), nh * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  OVP_CUDA(cudaStreamSynchronize(c->stream)); // host vectors go out of scope
  c->var_table_dirty = false;
  return OVP_OK;
}

int sync_host_values(Ctx *c) {
  if (!c->host_values_stale)
    return OVP_OK;
  size_t n = c->vars.size() * OVP_VAL_STRIDE;
  OVP_CUDA(cudaMemcpyAsync(c->h_val.data(), c->d_val, n * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  c->d2h_bytes += (int64_t)(n * sizeof(double));
  c->host_values_stale = false;
  return OVP_OK;
}

int push_host_values(Ctx *c, int h) {
  OVP_CUDA(cudaMemcpyAsync(c->d_val + (size_t)h * OVP_VAL_STRIDE, c->h_val.data() + (size_t)h * OVP_VAL_STRIDE,
                           OVP_VAL_STRIDE * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  OVP_CUDA(cudaMemcpyAsync(c->d_fej + (size_t)h * OVP_VAL_STRIDE, c->h_fej.data() + (size_t)h * OVP_VAL_STRIDE,
                           OVP_VAL_STRIDE * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  return OVP_OK;
}

// zero the new rows / cols [N, N+s) of P
__global__ void zero_band_kernel(double *P, int ld, int N, int s) {
  int total = (N + s) * s;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int i = idx % (N + s), j = idx / (N + s);
    P[(size_t)(N + j) * ld + i] = 0.0;
    P[(size_t)i * ld + (N + j)] = 0.0;
  }
}

// Handles are slots of the variable table.  A marginalised variable's slot goes to a FIFO free list and is handed out again once
// OVP_HANDLE_REUSE_LAG newer slots have been freed (a stale handle held by the caller keeps failing with NOT_IN_STATE for a while
// instead of silently naming a new variable), so the table - and every O(table) pass: finish_update_kernel, upload_var_table,
// sync_host_values, the plan signature - stays the size of the live state instead of growing by one clone per camera frame.
#define OVP_HANDLE_REUSE_LAG 64
int state_append_variable(Ctx *c, Var v, const double *value, const double *fej, int *handle) {
  int st = sync_host_values(c);
  if (st)
    return st;
  // `value` / `fej` may point INTO the host mirror (StateHelper::clone passes the cloned variable's own values): copy them out
  // before the mirror can be reallocated below
  double vbuf[OVP_VAL_STRIDE], fbuf[OVP_VAL_STRIDE];
  for (int i = 0; i < OVP_VAL_STRIDE; i++) {
    vbuf[i] = (i < v.nvalue && value) ? value[i] : 0.0;
    fbuf[i] = (i < v.nvalue) ? (fej ? fej[i] : (value ? value[i] : 0.0)) : 0.0;
  }
  int h;
  const bool table_full = (int)c->vars.size() >= c->max_handles;
  if (!c->free_handles.empty() && (table_full || (int)c->free_handles.size() > OVP_HANDLE_REUSE_LAG)) {
    h = c->free_handles.front();
    c->free_handles.pop_front();
    c->vars[h] = v;
  } else {
    if (table_full)
      return fail(c, OVP_ERR_CAPACITY, "variable handle capacity %d exceeded", c->max_handles);
    h = (int)c->vars.size();
    c->vars.push_back(v);
    c->h_val.resize((size_t)(h + 1) * OVP_VAL_STRIDE, 0.0);
    c->h_fej.resize((size_t)(h + 1) * OVP_VAL_STRIDE, 0.0);
  }
  for (int i = 0; i < OVP_VAL_STRIDE; i++) {
    c->h_val[(size_t)h * OVP_VAL_STRIDE + i] = vbuf[i];
    c->h_fej[(size_t)h * OVP_VAL_STRIDE + i] = fbuf[i];
  }
  c->var_table_dirty = true;
  *handle = h;
  return push_host_values(c, h);
}

double chi2_q95(Ctx *c, int dof) {
  if (dof < 1)
    dof = 1;
  if (dof < c->chi2_table_n)
    return c->chi2_table[dof];
  return hm::chi2_quantile95(dof);
}

int check_status_flags(Ctx *c) {
  int f[2] = {0, 0};
  OVP_CUDA(cudaMemcpyAsync(f, c->dflags, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  if (f[0] || f[1]) {
    OVP_CUDA(cudaMemsetAsync(c->dflags, 0, 2 * sizeof(int), c->stream));
    if (f[1])
      return fail(c, OVP_ERR_NOT_POSITIVE_DEFINITE, "innovation covariance not positive definite");
    return fail(c, OVP_ERR_NEGATIVE_DIAGONAL, "covariance has a negative diagonal entry (reference: std::exit, StateHelper.cpp:176-187)");
  }
  return OVP_OK;
}

// -------------------------------------------------------------------------------------------------------------------
// EKF update core (see ovp_internal.h).  K M^T = M S^-1 M^T is applied as (M L^-T)(M L^-T)^T and dx = (M L^-T)(L^-1 z):
// algebraically the reference's K = M S^-1, P -= K M^T, dx = K res (StateHelper.cpp:165-171,190).
// -------------------------------------------------------------------------------------------------------------------
int join_side_stream(Ctx *c) {
  if (c->join_pending) {
    OVP_CUDA(cudaStreamWaitEvent(c->stream, c->ev_join, 0));
    c->join_pending = false;
  }
  return OVP_OK;
}

int ekf_update_core(Ctx *c, const int *d_cols, int nc, MatView HT, int rr, const double *d_z, const double *d_Rdiag, double gate_thresh,
                    int *d_gate_flag, double *d_chi2, bool apply, int zstride, bool defer_join, bool ht_lower) {
  if (rr <= 0 || nc <= 0)
    return OVP_OK;
  {
    int stj = join_side_stream(c); // this update reads P
    if (stj)
      return stj;
  }
  if (rr > c->wsS.cap || nc > c->Rcap)
    return fail(c, OVP_ERR_CAPACITY, "ekf_update: system %d x %d exceeds capacity %d", rr, nc, c->Rcap);
  if (c->var_table_dirty) {
    int st = upload_var_table(c);
    if (st)
      return st;
  }
  const int N = c->N;
  // 1. M = P[:, cols] * HT        (N x rr)
  {
    GemmProblem p = make_problem(N, rr, nc, mv(c->dP, c->ldP, 0, nullptr, d_cols), HT, c->dM, c->Nmax);
    p.ktri = ht_lower ? 1 : 0; // H^T = L (the compression's Cholesky factor): column j is zero above row j
    launch_gemm1(c, p);
  }
  // 2. S = HT^T * M[cols, :] + R  (lower part)
  {
    MatView HTt = HT;
    HTt.trans ^= 1;
    GemmProblem p = make_problem(rr, rr, nc, HTt, mv(c->dM, c->Nmax, 0, d_cols, nullptr), c->wsS.S, c->wsS.cap);
    p.diag_add = d_Rdiag;
    p.diag_const = 1.0;
    p.tri = TRI_LOWER;
    p.ktri = ht_lower ? 2 : 0; // row i of H = L^T is zero left of column i
    launch_gemm1(c, p);
  }
  double *d_w = c->dvec; // [0, Rcap)
  double *chi2 = d_chi2 ? d_chi2 : c->dscal;
  int *flag = d_gate_flag ? d_gate_flag : (c->dflags + 2);
  // 3-5. S = L L^T, Y = M L^-T, w = L^-1 z, chi2 = |w|^2 and the gate flag in one launch (cholfused.cu)
  {
    int st = chol_fused(c, c->wsS.S, c->wsS.cap, rr, rr, 0.0, c->dM, c->Nmax, N, d_z, zstride, c->dY, c->Nmax, d_w, gate_thresh, chi2, flag);
    if (st)
      return st;
  }
  if (!apply)
    return OVP_OK;
  // 6. P -= Y Y^T (lower tiles, mirrored) and the negative-diagonal check (StateHelper.cpp:176-187)  [skipped on the device when the gate
  //    failed].  Nothing downstream needs the new P before the next update's M = P[:, ids] H^T (or a point-feature gate), so this branch
  //    runs on the side stream, in parallel with step 7 and with whatever the caller enqueues next on the main stream.
  const bool side = c->stream2 != nullptr && !c->profiling;
  cudaStream_t main_stream = c->stream;
  if (side) {
    OVP_CUDA(cudaEventRecord(c->ev_fork, main_stream));
    OVP_CUDA(cudaStreamWaitEvent(c->stream2, c->ev_fork, 0));
    c->stream = c->stream2; // the launch helpers below enqueue on c->stream
  }
  {
    GemmProblem p = make_problem(N, N, rr, mv(c->dY, c->Nmax), mv(c->dY, c->Nmax, 1), c->dP, c->ldP, -1.0, 1.0);
    p.tri = TRI_LOWER_MIRROR;
    p.nosplit = 1; // on the side stream it hides behind the next update's launches; unsplit it takes fewer SMs from them (DESIGN.md §9)
    launch_gemm1(c, p, flag);
  }
  diag_check_kernel<<<(N + 255) / 256, 256, 0, c->stream>>>(c->dP, c->ldP, N, c->dflags, flag);
  c->launches++;
  if (side) {
    c->stream = main_stream;
    OVP_CUDA(cudaEventRecord(c->ev_join, c->stream2));
    c->join_pending = true;
  }
  // 7. dx = Y w and the manifold update of every variable: one launch
  int nh = (int)c->vars.size();
  double *d_part = c->dvec + (size_t)8 * c->Rcap + 2 * (size_t)c->Nmax;
  dx_partial_kernel<<<dim3((N + 63) / 64, OVP_DX_SPLIT), 256, 0, c->stream>>>(c->dY, c->Nmax, N, d_w, rr, d_part, c->Nmax, flag);
  finish_update_kernel<<<(nh * 32 + 127) / 128, 128, 0, c->stream>>>(nh, c->d_var_id, c->d_var_size, c->d_var_kind, c->d_val, d_part, c->Nmax, nullptr,
                                                                      c->ldP, c->dflags, flag);
  c->launches += 2;
  c->host_values_stale = true;
  if (!defer_join)
    return join_side_stream(c);
  return OVP_OK;
}

} // namespace ovp

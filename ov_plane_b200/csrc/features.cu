// UpdaterMSCKF::update from "features triangulated, plane CPs known" onward (UpdaterMSCKF.cpp:407-828), device side:
//   feature kernel  : one CTA per tracked feature — Jacobian rows (UpdaterHelper.cpp:195-513) built in shared memory from
//                     the device-resident clone/calibration values, left-nullspace projection of H_f (UpdaterHelper.cpp:515-546,
//                     UpdaterPlane.cpp:483-517; 3 Householder reflectors instead of 3*(rows-2) sequential Givens rotations),
//                     per-feature Mahalanobis gate against P (UpdaterMSCKF.cpp:739-764) and scatter into the stacked system;
//   gram kernel     : G = [H_x H_cp r]^T [H_x H_cp r] on FP64 tensor cores (split-K, deterministic reduction);
//   compression     : partial Cholesky of G = the Q-less QR of the stacked system (UpdaterHelper.cpp:548-579,
//                     UpdaterPlane.cpp:519-552 incl. its "keep the first n rows" semantics), then ekf_update_core.
#include "jacobian_core.h"
#include "ovp_internal.h"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>

namespace ovp {

#ifdef OVP_DEBUG
// Raw whitened blocks of the feature kernels as they hold them (ovp_debug_msckf_gram, ovp_debug_slam_update; libovp_debug.so only).
// Measurement g of the batch owns 3 rows of OVP_RAW_ROW doubles from raw[g * 3 * OVP_RAW_ROW]: its two bearing rows, [0,3) H_f (SLAM: the
// landmark's columns), [3,9) H_clone, [9, 9 + ncal) calibration, [23] r; with a plane its point-on-plane row, [0,3) H_f, [9,12) H_cp,
// [23] r.  Entries not named are left.
#define OVP_RAW_ROW 24
#endif
struct FeatArgs {
  const int *meas_offset;
  const int *meas_clone;
  const float *uv;
  const double *pf;       // 3 per feature (position used for this pass); unused in SLAM mode
  const int *feat_sel;    // feature indices processed by this launch
  const int *row_off;     // per selected feature: first row in the stacked system
  const int *feat_plane_slot; // per feature (global index): slot of its plane in plane_pass[] or -1
  const int *plane_pass;  // device flags written by the plane updates (1 = passed => feature consumed)
  const int *feat_lm;     // SLAM mode: per feature, handle of its landmark variable
  const int *feat_ph;     // SLAM mode: per feature, handle of its in-state plane or -1
  const double *val;
  const double *fej;
  const int *var_id;
  int h_calib, h_intr;
  int do_fej, do_calib_pose, do_calib_intr;
  int mode;               // 0: MSCKF point (nullspace + per-feature gate), 1: MSCKF plane (nullspace, H_cp carried, no gate),
                          // 2: SLAM (landmark and plane are state columns, no nullspace, gate with plane -> no-plane fallback)
  int plane_handle;       // mode 1: >= 0: plane is in the state (cp from val/fej tables); -1: use plane_cp
  const double *plane_cp; // mode 1, plane not in the state: its 3 linearisation values in the batch staging buffer (read through
                          // the pointer so that a replayed CUDA graph sees the values of THIS call, not of the capture call)
  double white_px, white_c;
  const double *P;
  int ldP;
  const int *state2compact;
  int col_cp, col_res;    // stacked-system columns of H_cp (3, mode 1) and of the residual
  double *Hs;
  int ldHs;
#ifdef OVP_DEBUG
  double *raw; // ovp_debug_msckf_gram: the raw whitened blocks of every feature (layout OVP_RAW_* above), nullptr: none
#endif
  const double *chi2_table;
  int chi2_n;
  double chi2_mult;
  int *feat_flag;
  double *feat_chi2;
  int lda;   // smem column stride of the feature block (odd)
  int ldt;   // smem column stride of T / S (odd)
  int maxcols; // capacity of local columns
};

__device__ __forceinline__ double warp_sum(double s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// Mahalanobis gate on the sub-block rows [rb, rb+nr) x columns [cb, cb+ncg) of the feature block A:
// S = H P_marg H^T + I, chi2 = r^T S^-1 r (UpdaterMSCKF.cpp:739-742, UpdaterSLAM.cpp:528-532).  gid[c] = state index of local column c.
// Returns chi2 (NaN-safe: ok flag in *ok_out).  All 128 threads participate.
__device__ double gate_chi2(const double *A, int lda, double *T, double *S, int ldt, double *ybuf, double *Pp, int ldpp, int rb, int nr, int cb,
                            int ncg, const int *gid, const double *P, int ldP, int c_res, int tid, int *s_ok, double *s_chi2) {
  // S = I + sum over panels of 8 covariance columns of (H P_marg[:, panel]) H[:, panel]^T.  The panel P[gid[:], gid[b0 .. b0+7]] is
  // gathered into shared memory with all loads of a thread in flight at once (runs of 6-14 contiguous doubles per clone / calibration
  // block), T = H * panel (nr x 8) is formed out of shared memory and folded into the lower triangle of S right away: the full
  // nr x ncg product H P_marg is never stored (it was 40 % of the block's shared memory and capped the clone window at 30).
  for (int w = tid; w < nr * nr; w += 128) {
    const int i = w % nr, jj = w / nr;
    S[(size_t)jj * ldt + i] = (i == jj) ? 1.0 : 0.0;
  }
  for (int b0 = 0; b0 < ncg; b0 += 8) {
    const int nb = min(8, ncg - b0);
    for (int w = tid; w < nb * ncg; w += 128) {
      const int b = w / ncg, k = w - b * ncg;
      Pp[b * ldpp + k] = P[(size_t)gid[cb + b0 + b] * ldP + gid[cb + k]];
    }
    __syncthreads();
    for (int w = tid; w < nb * nr; w += 128) {
      const int b = w / nr, i = w - b * nr;
      const double *hc = A + (size_t)cb * lda + rb + i, *pc = Pp + b * ldpp;
      double acc = 0.0;
      for (int k = 0; k < ncg; k++)
        acc += hc[(size_t)k * lda] * pc[k];
      T[(size_t)b * ldt + i] = acc;
    }
    __syncthreads();
    for (int w = tid; w < nr * nr; w += 128) {
      const int i = w % nr, jj = w / nr;
      if (i < jj)
        continue;
      double s = S[(size_t)jj * ldt + i];
      for (int b = 0; b < nb; b++)
        s += T[(size_t)b * ldt + i] * A[(size_t)(cb + b0 + b) * lda + rb + jj];
      S[(size_t)jj * ldt + i] = s;
    }
    // (the next panel's gather only writes Pp; its T is written after the barrier that follows the gather)
  }
  __syncthreads();
  if (tid == 0)
    *s_ok = 1;
  for (int jj = 0; jj < nr; jj++) {
    __syncthreads();
    if (tid == 0) {
      double d = S[(size_t)jj * ldt + jj];
      if (!(d > 0.0)) {
        *s_ok = 0;
        d = 1.0;
      }
      S[(size_t)jj * ldt + jj] = sqrt(d);
    }
    __syncthreads();
    double piv = S[(size_t)jj * ldt + jj];
    for (int i = jj + 1 + tid; i < nr; i += 128)
      S[(size_t)jj * ldt + i] /= piv;
    __syncthreads();
    int nrem = nr - 1 - jj;
    for (int w = tid; w < nrem * nrem; w += 128) {
      int i = jj + 1 + w % nrem, k = jj + 1 + w / nrem;
      if (i >= k)
        S[(size_t)k * ldt + i] -= S[(size_t)jj * ldt + i] * S[(size_t)jj * ldt + k];
    }
  }
  __syncthreads();
  if (tid < 32) {
    double chi = 0.0;
    for (int i = 0; i < nr; i++) {
      double s = 0.0;
      for (int k = tid; k < i; k += 32)
        s += S[(size_t)k * ldt + i] * ybuf[k];
      s = warp_sum(s);
      double y = (A[(size_t)c_res * lda + rb + i] - s) / S[(size_t)i * ldt + i];
      if (tid == 0)
        ybuf[i] = y;
      __syncwarp();
      chi += y * y;
    }
    if (tid == 0)
      *s_chi2 = chi;
  }
  __syncthreads();
  return *s_chi2;
}

// Local column layout of the feature block A (col-major, stride lda):
//   [0,3) H_f | [3, 3+cf) H_x = [extrinsics 6][intrinsics 8][clone_0 6]...[clone_{m-1} 6] | [3+cf, 3+cf+3) H_cp | last: res
__global__ void __launch_bounds__(128) feature_kernel(FeatArgs a) {
  extern __shared__ double sm[];
  const int tid = threadIdx.x;
  const int f = a.feat_sel[blockIdx.x];
  const int m0 = a.meas_offset[f];
  const int m = a.meas_offset[f + 1] - m0;
  if (a.mode == 0) {
    int slot = a.feat_plane_slot[f];
    if (slot >= 0 && a.plane_pass[slot] == 1) { // consumed by a successful plane update (UpdaterMSCKF.cpp:640-644,659)
      if (tid == 0) {
        a.feat_flag[f] = 2;
        a.feat_chi2[f] = nan("");
      }
      return;
    }
  }
  const int lm = (a.mode == 2) ? a.feat_lm[f] : -1;
  const int ph = (a.mode == 2) ? a.feat_ph[f] : a.plane_handle;
  const bool has_plane = (a.mode == 1) || (a.mode == 2 && ph >= 0);
  const int ncal = (a.do_calib_pose ? 6 : 0) + (a.do_calib_intr ? 8 : 0);
  const int cf = ncal + 6 * m;
  const int rows = has_plane ? 3 * m : 2 * m;
  const int ncols = 3 + cf + 3 + 1;
  const int c_cp = 3 + cf, c_res = 3 + cf + 3;
  const int lda = a.lda;
  double *A = sm;                                   // lda * maxcols
  double *T = A + (size_t)lda * a.maxcols;          // ldt * 8: H * (8-column covariance panel)   (gate only)
  double *S = T + (size_t)a.ldt * 8;                // ldt * ldt         (gate only)
  double *vbuf = (a.mode == 1) ? T : S + (size_t)a.ldt * a.ldt; // reflector / forward-substitution vector
  double *Pp = vbuf + lda + 1;                                 // 8 x maxcols covariance panel (gate only)
  __shared__ int gid[3 + 14 + 6 * 64 + 3]; // state index of every local column except the residual
  __shared__ double s_beta, s_chi2;
  __shared__ int s_ok;

  for (int idx = tid; idx < lda * ncols; idx += 128)
    A[idx] = 0.0;
  __syncthreads();

  // ---- Jacobian rows: one thread per measurement ----
  if (tid < m) {
    const int k = tid;
    const int hcl = a.meas_clone[m0 + k];
    const double *vc = a.val + (size_t)hcl * OVP_VAL_STRIDE;
    const double *fc = a.fej + (size_t)hcl * OVP_VAL_STRIDE;
    const double *vcal = a.val + (size_t)a.h_calib * OVP_VAL_STRIDE;
    const double *cam = a.val + (size_t)a.h_intr * OVP_VAL_STRIDE;
    double R_C[9];
    quat_to_rot(vcal, R_C);
    const double *pf, *pff;
    if (a.mode == 2) { // landmark in the state: value and first-estimate (UpdaterSLAM.cpp:488-489)
      pf = a.val + (size_t)lm * OVP_VAL_STRIDE;
      pff = a.fej + (size_t)lm * OVP_VAL_STRIDE;
    } else { // MSCKF feature: both are the triangulated point (UpdaterMSCKF.cpp:721-722)
      pf = a.pf + 3 * (size_t)f;
      pff = pf;
    }
    double res[2], Hf[6], Hcl[12], Hcal[12], Hin[16];
    bearing_rows(vc, vc + 4, fc, fc + 4, a.do_fej, R_C, vcal + 4, cam, pf, pff, a.uv[2 * (m0 + k)], a.uv[2 * (m0 + k) + 1], a.white_px,
                 res, Hf, Hcl, Hcal, Hin);
    for (int i = 0; i < 2; i++) {
      int r = 2 * k + i;
      for (int j = 0; j < 3; j++)
        A[(size_t)j * lda + r] = Hf[3 * i + j];
      int cb = 3;
      if (a.do_calib_pose) {
        for (int j = 0; j < 6; j++)
          A[(size_t)(cb + j) * lda + r] = Hcal[6 * i + j];
        cb += 6;
      }
      if (a.do_calib_intr) {
        for (int j = 0; j < 8; j++)
          A[(size_t)(cb + j) * lda + r] = Hin[8 * i + j];
        cb += 8;
      }
      for (int j = 0; j < 6; j++)
        A[(size_t)(cb + 6 * k + j) * lda + r] = Hcl[6 * i + j];
      A[(size_t)c_res * lda + r] = res[i];
    }
#ifdef OVP_DEBUG
    if (a.raw) // the rows just written to A, in the layout of OVP_RAW_ROW (SLAM: [0,3) are the landmark's columns)
      for (int i = 0; i < 2; i++) {
        double *rw = a.raw + ((size_t)(m0 + k) * 3 + i) * OVP_RAW_ROW;
        for (int j = 0; j < 3 + cf; j++)
          if (j < 3 + ncal || (j >= 3 + ncal + 6 * k && j < 3 + ncal + 6 * k + 6))
            rw[j < 3 ? j : (j < 3 + ncal ? j + 6 : j - ncal - 6 * k)] = A[(size_t)j * lda + 2 * k + i];
        rw[OVP_RAW_ROW - 1] = A[(size_t)c_res * lda + 2 * k + i];
      }
#endif
    const int idc = a.var_id[hcl];
    for (int j = 0; j < 6; j++)
      gid[3 + ncal + 6 * k + j] = idc + j;
    if (has_plane) {
      const double *cp, *cpf;
      if (ph >= 0) {
        cp = a.val + (size_t)ph * OVP_VAL_STRIDE;
        cpf = a.fej + (size_t)ph * OVP_VAL_STRIDE;
      } else {
        cp = a.plane_cp;
        cpf = a.plane_cp;
      }
      double pr, pHf[3], pHcp[3];
      plane_row(pf, pff, cp, cpf, a.do_fej, a.white_c, pr, pHf, pHcp);
      int r = 2 * m + k;
      for (int j = 0; j < 3; j++) {
        A[(size_t)j * lda + r] = pHf[j];
        A[(size_t)(c_cp + j) * lda + r] = pHcp[j];
      }
      A[(size_t)c_res * lda + r] = pr;
#ifdef OVP_DEBUG
      if (a.raw) {
        double *rw = a.raw + ((size_t)(m0 + k) * 3 + 2) * OVP_RAW_ROW;
        for (int j = 0; j < 3; j++) {
          rw[j] = A[(size_t)j * lda + r];
          rw[9 + j] = A[(size_t)(c_cp + j) * lda + r];
        }
        rw[OVP_RAW_ROW - 1] = A[(size_t)c_res * lda + r];
      }
#endif
    }
  }
  if (tid == 0) {
    int cb = 3;
    if (a.do_calib_pose) {
      int idb = a.var_id[a.h_calib];
      for (int j = 0; j < 6; j++)
        gid[cb + j] = idb + j;
      cb += 6;
    }
    if (a.do_calib_intr) {
      int idb = a.var_id[a.h_intr];
      for (int j = 0; j < 8; j++)
        gid[cb + j] = idb + j;
    }
    for (int j = 0; j < 3; j++) {
      gid[j] = (lm >= 0) ? a.var_id[lm] + j : 0;
      gid[c_cp + j] = (ph >= 0) ? a.var_id[ph] + j : 0;
    }
  }
  __syncthreads();

  int accept = 1, rb = 0, nr = rows, cb0 = 0, ncs = 3 + cf + (has_plane ? 3 : 0); // accepted sub-block: rows [rb, rb+nr), cols [cb0, cb0+ncs)
  if (a.mode != 2) {
    // ---- left-nullspace projection of H_f: 3 Householder reflectors applied to [H_f H_x H_cp res] ----
    for (int j = 0; j < 3; j++) {
      if (tid < 32) {
        double s = 0.0;
        for (int i = j + tid; i < rows; i += 32) {
          double v = A[(size_t)j * lda + i];
          s += v * v;
        }
        s = warp_sum(s);
        double x0 = A[(size_t)j * lda + j];
        double nrm = sqrt(s);
        double alpha = (x0 > 0.0) ? -nrm : nrm;
        double v0 = x0 - alpha;
        double vtv = s - x0 * x0 + v0 * v0;
        for (int i = j + tid; i < rows; i += 32)
          vbuf[i] = (i == j) ? v0 : A[(size_t)j * lda + i];
        if (tid == 0)
          s_beta = (vtv > 0.0 && nrm > 0.0) ? 2.0 / vtv : 0.0;
      }
      __syncthreads();
      const double beta = s_beta;
      for (int cidx = j + 1 + tid; cidx < ncols; cidx += 128) {
        double *col = A + (size_t)cidx * lda;
        double s = 0.0;
        for (int i = j; i < rows; i++)
          s += vbuf[i] * col[i];
        s *= beta;
        if (s != 0.0)
          for (int i = j; i < rows; i++)
            col[i] -= s * vbuf[i];
      }
      __syncthreads();
    }
    rb = 3;
    nr = rows - 3;
    cb0 = 3;
    ncs = cf;
    if (a.mode == 0) {
      double chi2 = gate_chi2(A, lda, T, S, a.ldt, vbuf, Pp, a.maxcols, rb, nr, cb0, ncs, gid, a.P, a.ldP, c_res, tid, &s_ok, &s_chi2);
      double thr = a.chi2_mult * a.chi2_table[nr < a.chi2_n ? nr : a.chi2_n - 1];
      accept = (s_ok && !(chi2 > thr)) ? 1 : 0;
      if (tid == 0) {
        a.feat_flag[f] = accept;
        a.feat_chi2[f] = chi2;
      }
    }
  } else {
    // ---- SLAM landmark: no nullspace; gate with the plane constraint, on failure retry without it (UpdaterSLAM.cpp:528-622) ----
    double chi2 = gate_chi2(A, lda, T, S, a.ldt, vbuf, Pp, a.maxcols, 0, nr, 0, ncs, gid, a.P, a.ldP, c_res, tid, &s_ok, &s_chi2);
    double thr = a.chi2_mult * a.chi2_table[nr < a.chi2_n ? nr : a.chi2_n - 1];
    int st = (s_ok && !(chi2 > thr)) ? 1 : 0;
    if (!st && has_plane) {
      __syncthreads();
      nr = 2 * m;
      ncs = 3 + cf;
      chi2 = gate_chi2(A, lda, T, S, a.ldt, vbuf, Pp, a.maxcols, 0, nr, 0, ncs, gid, a.P, a.ldP, c_res, tid, &s_ok, &s_chi2);
      thr = a.chi2_mult * a.chi2_table[nr < a.chi2_n ? nr : a.chi2_n - 1];
      st = (s_ok && !(chi2 > thr)) ? 3 : 0;
    }
    accept = st;
    if (tid == 0) {
      a.feat_flag[f] = st;
      a.feat_chi2[f] = chi2;
    }
  }
  if (!accept)
    return;
  // ---- scatter the accepted block into the stacked system ----
  const int r0 = a.row_off[blockIdx.x];
  for (int w = tid; w < ncs * nr; w += 128) {
    int i = w % nr, b = w / nr;
    int gc = a.state2compact[gid[cb0 + b]];
    a.Hs[(size_t)gc * a.ldHs + r0 + i] = A[(size_t)(cb0 + b) * lda + rb + i];
  }
  if (a.mode == 1)
    for (int w = tid; w < 3 * nr; w += 128) {
      int i = w % nr, b = w / nr;
      a.Hs[(size_t)(a.col_cp + b) * a.ldHs + r0 + i] = A[(size_t)(c_cp + b) * lda + rb + i];
    }
  for (int i = tid; i < nr; i += 128)
    a.Hs[(size_t)a.col_res * a.ldHs + r0 + i] = A[(size_t)c_res * lda + rb + i];
}

// -------------------------------------------------------------------------------------------------------------------
// Gram kernel: partial[z] = Hs[k-chunk z, :]^T Hs[k-chunk z, :]  (lower 64x64 tiles), FP64 DMMA
// -------------------------------------------------------------------------------------------------------------------
// Operand tiles are 64 columns of Hs x 16 rows (k), k contiguous in global memory AND in shared memory ([col][k], stride 20
// doubles: 16-byte vector copies without bank conflicts, DMMA fragment reads (8 cols x 4 k) on 16 distinct 8-byte banks because
// 20 mod 16 == 4); the next k-step is prefetched into registers while the current one is in the tensor pipe; a diagonal tile
// loads its operand once.
#define GRAM_KS 20
__global__ void __launch_bounds__(128) gram_kernel(const double *Hs, int ld, int rows, int nc, int kchunk, double *part, int ldp) {
  const int tm = blockIdx.y, tn = blockIdx.x;
  if (tm < tn)
    return;
  __shared__ __align__(16) double As[OVP_GT][GRAM_KS];
  __shared__ __align__(16) double Bs[OVP_GT][GRAM_KS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1;
  const int g = lane >> 2, t = lane & 3;
  const int m0 = tm * OVP_GT, n0 = tn * OVP_GT;
  const bool diag = tm == tn;
  const int kbeg = blockIdx.z * kchunk;
  const int kend = min(rows, kbeg + kchunk);
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++)
      acc[i][j][0] = acc[i][j][1] = 0.0;
  // thread -> 4 chunks of 2 k per operand: chunk e = tid + 128 q: column e >> 3, k offset (e & 7) * 2
  double2 ra[4], rb[4];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int e = tid + 128 * q, col = e >> 3, k2 = k0 + (e & 7) * 2;
      const int gi = m0 + col, gj = n0 + col;
      double2 z = make_double2(0.0, 0.0);
      ra[q] = z;
      rb[q] = z;
      if (gi < nc) {
        const double *src = Hs + (size_t)gi * ld + k2;
        if (k2 + 1 < kend)
          ra[q] = *reinterpret_cast<const double2 *>(src);
        else if (k2 < kend)
          ra[q].x = src[0];
      }
      if (!diag && gj < nc) {
        const double *src = Hs + (size_t)gj * ld + k2;
        if (k2 + 1 < kend)
          rb[q] = *reinterpret_cast<const double2 *>(src);
        else if (k2 < kend)
          rb[q].x = src[0];
      }
    }
  };
  fetch(kbeg);
  const double(*Bt)[GRAM_KS] = diag ? As : Bs;
  for (int k0 = kbeg; k0 < kend; k0 += OVP_GK) {
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int e = tid + 128 * q, col = e >> 3, ko = (e & 7) * 2;
      *reinterpret_cast<double2 *>(&As[col][ko]) = ra[q];
      if (!diag)
        *reinterpret_cast<double2 *>(&Bs[col][ko]) = rb[q];
    }
    __syncthreads();
    if (k0 + OVP_GK < kend)
      fetch(k0 + OVP_GK);
#pragma unroll
    for (int kk = 0; kk < OVP_GK; kk += 4) {
      double av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; i++)
        av[i] = As[wm * 32 + i * 8 + g][kk + t];
#pragma unroll
      for (int j = 0; j < 4; j++)
        bv[j] = Bt[wn * 32 + j * 8 + g][kk + t];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
          dmma_m8n8k4(acc[i][j][0], acc[i][j][1], av[i], bv[j]);
    }
    __syncthreads();
  }
  double *out = part + (size_t)blockIdx.z * ldp * ldp;
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        int gi = m0 + wm * 32 + i * 8 + g;
        int gj = n0 + wn * 32 + j * 8 + t * 2 + h;
        if (gi < nc && gj < nc)
          out[(size_t)gj * ldp + gi] = acc[i][j][h];
      }
}

// G[i,j] (lower, i >= j) = sum_z part[z][i,j] in fixed order (deterministic)
__global__ void gram_reduce_kernel(const double *part, int ldp, int nsplit, int nc, double *G, int ldg) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nc * nc)
    return;
  int i = idx % nc, j = idx / nc;
  if (i < j) { // strictly-upper part must read as zero: the factor is later used as a dense H^T operand
    G[(size_t)j * ldg + i] = 0.0;
    return;
  }
  double s = 0.0;
  for (int z = 0; z < nsplit; z++)
    s += part[(size_t)z * ldp * ldp + (size_t)j * ldp + i];
  G[(size_t)j * ldg + i] = s;
}

#include "msckf_warp.inc"

// D part of the block-sparse Gram matrix (msckf_warp.inc), combined with the SYRK partials in gram_reduce_sparse_kernel
struct SparseD {
  int ncal, nslots, nd, nchunk;
  const double *Dcc, *Ddc, *Dddp;
};
// Gram + reduce of the stacked system Hs (rows x nc) into ws.S (lower).  With sp: Hs holds the 4-rows-per-feature SYRK operand Y and
// the result is G = D - Y^T Y; work = algorithmic flops reported for the launch.
static int gram_of_stacked(Ctx *c, int rows, int nc, int ldHs, const SparseD *sp = nullptr, double work = -1.0) {
  int tiles = (nc + OVP_GT - 1) / OVP_GT;
  int ldp = tiles * OVP_GT;
  int ntile_lower = tiles * (tiles + 1) / 2;
  int nsplit = std::max(1, std::min((rows + 255) / 256, std::max(1, (c->num_sms * 4) / std::max(1, ntile_lower))));
  size_t need = (size_t)nsplit * ldp * ldp;
  if (need > c->part_elems) {
    nsplit = (int)(c->part_elems / ((size_t)ldp * ldp));
    if (nsplit < 1)
      return fail(c, OVP_ERR_CAPACITY, "gram: partial buffer too small");
  }
  int kchunk = ((rows + nsplit - 1) / nsplit + OVP_GK - 1) / OVP_GK * OVP_GK;
  nsplit = (rows + kchunk - 1) / kchunk;
  dim3 grid(tiles, tiles, nsplit);
  prof_begin(c, PROF_GRAM, work >= 0.0 ? work : (double)nc * nc * rows); // algorithmic flops of the symmetric product: 2 * n^2 * r / 2
  gram_kernel<<<grid, 128, 0, c->stream>>>(c->dHs, ldHs, rows, nc, kchunk, c->dPart, ldp);
  c->launches++;
  prof_end(c);
  if (sp)
    gram_reduce_sparse_kernel<<<(nc * nc + 255) / 256, 256, 0, c->stream>>>(c->dPart, ldp, nsplit, nc, sp->ncal, sp->nslots, sp->nd, sp->Dcc, sp->Ddc,
                                                                              sp->Dddp, sp->nchunk, c->wsG.S, c->wsG.cap);
  else
    gram_reduce_kernel<<<(nc * nc + 255) / 256, 256, 0, c->stream>>>(c->dPart, ldp, nsplit, nc, c->wsG.S, c->wsG.cap);
  c->launches++;
  return OVP_OK;
}

#include "features_host.inc"
#include "slam_host.inc"

// Factorisations wider than one co-resident launch of chol_fused_kernel (DESIGN.md 4.1).  The tile CTAs of one launch wait on each other,
// so a launch holds at most chol_fused_width columns (960 on an H100).  A wider system is factored right-looking, in panels of at most
// that width; panel k = columns [k0, k1):
//   1. one chol_fused launch on the diagonal block A[k0:k1, k0:k1], with the rows below, A[k1:n, k0:k1], as its right-hand side solved
//      in place: they come out as L[k1:n, k0:k1] (a compressed update's z row, row nc of its Gram matrix, among them).  With a right-hand
//      side M, its panel columns Y[:, k0:k1] and z[k0:k1] are solved against the same factor by the prefactored row-block launch
//      (chol_fused_rows): Y_k, w_k and the chi2 part |w_k|^2, no gate.
//   2. one DMMA GEMM launch downdates what follows: A[k1:n, k1:npiv] -= L21 L21^T (lower tiles), Y[:, k1:npiv] -= Y_k L21^T and
//      z[k1:npiv] -= L21 w_k, with L21 = L[k1:n, k0:k1].
//   3. after the last panel one small kernel sums the chi2 parts in panel order and writes chi2 and the gate flag where chol_fused would.
// The zero-pivot rule compares every pivot with tol times its column's ORIGINAL diagonal, saved before the first panel, as one launch
// does with the diagonal its tile CTAs record: the panel launches read the saved one (CholFusedArgs::diag0_saved), since their own
// diagonal blocks have been downdated by the panels before them.  Y starts as a copy of M and z as a copy in cf_panel, so the caller's
// M and z are only read.  The panels are fused launches, not one launch per 64-column block: a 2048-wide system is three panels
// (960 + 960 + 128) of four launches each.
#include "ovp_internal.h"

namespace ovp {

// the reference diagonal of the zero-pivot rule (npiv entries) and a contiguous working copy of z (nz entries)
__global__ void panel_prep_kernel(const double *A, int ld, int npiv, double *diag, const double *z, int zstride, int nz, double *zw) {
  chain_wait();
  chain_release();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(npiv, nz); i += gridDim.x * blockDim.x) {
    if (i < npiv)
      diag[i] = A[(size_t)i * ld + i];
    if (i < nz)
      zw[i] = z[(size_t)i * zstride];
  }
}

// chi2 = the panels' parts summed in panel order, and the gate flag as chol_fused_kernel forms it
__global__ void panel_gate_kernel(const double *parts, int np, double gate_thresh, double *chi2, int *gate_flag) {
  chain_wait();
  chain_release();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < np; k++)
      s += parts[k];
    if (chi2)
      *chi2 = s;
    if (gate_flag)
      *gate_flag = (gate_thresh < 0.0 || !(s > gate_thresh)) ? 1 : 0;
  }
}

int update_width(Ctx *c, int *width) {
  if (c->max_update_width > 0) {
    *width = c->max_update_width;
    return OVP_OK;
  }
  return chol_fused_width(c, width);
}

int chol_needs_panels(Ctx *c, int n, int npiv, bool *panels) {
  *panels = false;
  if (npiv <= 0)
    return OVP_OK;
  int cap = 0, width = 0;
  int st = chol_fused_capacity(c, &cap);
  if (st)
    return st;
  if (chol_fused_tiles(n, npiv) <= cap)
    return OVP_OK;
  st = update_width(c, &width);
  if (st)
    return st;
  *panels = n <= width;
  return OVP_OK;
}

int chol_panels(Ctx *c, int width, double *A, int ld, int n, int npiv, double tol, const double *M, int ldm, int mrows, const double *z,
                int zstride, double *Y, int ldy, double *w, double gate_thresh, double *chi2, int *gate_flag) {
  if (npiv <= 0)
    return OVP_OK;
  int cw = 0;
  int st = chol_fused_width(c, &cw);
  if (st)
    return st;
  if (width < 64 || width % 64 || width > cw)
    return fail(c, OVP_ERR_BAD_ARGS, "chol_panels: panel width %d is not a multiple of 64 up to the co-resident width %d", width, cw);
  if (npiv > n || n > c->Rcap || (M && mrows > c->Nmax))
    return fail(c, OVP_ERR_CAPACITY, "chol_panels: system %d (%d pivots, %d right-hand-side rows) exceeds the workspace %d", n, npiv,
                M ? mrows : 0, c->Rcap);
  const bool rhs = M && mrows >= 0;
  const int nz = (rhs && z && w) ? npiv : 0;
  const int np = (npiv + width - 1) / width;
  double *diag = c->cf_panel, *zw = diag + c->Rcap, *parts = zw + c->Rcap;
  OVP_CUDA(chain_launch(c, panel_prep_kernel, dim3((std::max(npiv, nz) + 255) / 256), dim3(256), 0, (const double *)A, ld, npiv, diag, z,
                        zstride, nz, zw));
  if (rhs && mrows > 0 && Y != M) {
    OVP_CUDA(cudaMemcpy2DAsync(Y, (size_t)ldy * sizeof(double), M, (size_t)ldm * sizeof(double), (size_t)mrows * sizeof(double), npiv,
                               cudaMemcpyDeviceToDevice, c->stream));
    c->launches++;
  }
  for (int k = 0; k < np; k++) {
    const int k0 = k * width, k1 = std::min(npiv, k0 + width), wk = k1 - k0;
    double *Ak = A + (size_t)k0 * ld + k0, *L21 = Ak + wk; // L21: rows [k1, n) of the panel's columns
    double *Yk = rhs ? Y + (size_t)k0 * ldy : nullptr;
    st = chol_fused(c, Ak, ld, wk, wk, tol, k1 < n ? L21 : nullptr, ld, n - k1, nullptr, 1, L21, ld, nullptr, -1.0, nullptr, nullptr, nullptr,
                    nullptr, diag + k0);
    if (!st && rhs)
      st = chol_fused_rows(c, Ak, ld, wk, wk, Yk, ldy, mrows, nz ? zw + k0 : nullptr, 1, Yk, ldy, nz ? w + k0 : nullptr, nz ? parts + k : nullptr);
    if (st)
      return st;
    if (k1 == npiv)
      break;
    GemmBatch b;
    b.n = 0;
    b.flag = nullptr;
    GemmProblem pa = make_problem(n - k1, npiv - k1, wk, mv(L21, ld), mv(L21, ld, 1), A + (size_t)k1 * ld + k1, ld, -1.0, 1.0);
    pa.tri = TRI_LOWER;
    b.p[b.n++] = pa;
    if (rhs && mrows > 0)
      b.p[b.n++] = make_problem(mrows, npiv - k1, wk, mv(Yk, ldy), mv(L21, ld, 1), Y + (size_t)k1 * ldy, ldy, -1.0, 1.0);
    if (nz)
      b.p[b.n++] = make_problem(npiv - k1, 1, wk, mv(L21, ld), mv(w + k0, wk), zw + k1, c->Rcap, -1.0, 1.0);
    launch_gemm(c, b);
  }
  if (nz && (chi2 || gate_flag))
    OVP_CUDA(chain_launch(c, panel_gate_kernel, dim3(1), dim3(32), 0, (const double *)parts, np, gate_thresh, chi2, gate_flag));
  return OVP_OK;
}

int chol_factor(Ctx *c, double *A, int ld, int n, int npiv, double tol, const double *M, int ldm, int mrows, const double *z, int zstride,
                double *Y, int ldy, double *w, double gate_thresh, double *chi2, int *gate_flag) {
  bool panels = false;
  int st = chol_needs_panels(c, n, npiv, &panels);
  if (st)
    return st;
  if (!panels)
    return chol_fused(c, A, ld, n, npiv, tol, M, ldm, mrows, z, zstride, Y, ldy, w, gate_thresh, chi2, gate_flag);
  int width = 0;
  st = chol_fused_width(c, &width);
  if (st)
    return st;
  return chol_panels(c, width, A, ld, n, npiv, tol, M, ldm, mrows, z, zstride, Y, ldy, w, gate_thresh, chi2, gate_flag);
}

} // namespace ovp

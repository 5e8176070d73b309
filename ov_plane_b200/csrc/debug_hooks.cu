// TEST / TUNING HOOKS — compiled only into libovp_debug.so (-DOVP_DEBUG), never into the product library libovp.so.
// Declared in include/ovp_debug.h.  Used by tools/microbench_chol.py (phase timeline of the fused Cholesky), by
// tests/test_gpu_cholfused.py and tests/test_gpu_gemm.py (unit tests of chol_fused_kernel and the DMMA GEMM against NumPy), by
// tests/test_gpu_numerics.py (the block-sparse feature path against the dense stack on the same batch) and by tests/test_gpu_compression.py
// (the compressed update's Gram matrix, zero-pivot rule and innovation gate against long-double references) and by
// tests/test_gpu_feature_gate.py (the per-feature chi2 gates of the MSCKF point and SLAM feature kernels) and by
// tests/test_gpu_slam_reference.py (the SLAM update's Gram matrix against long double).
#include "ovp_internal.h"
using namespace ovp;

namespace ovp {
__global__ void spd_fill_kernel(double *A, int ld, int n) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * n)
    return;
  int i = idx % n, j = idx / n;
  double v = (i == j) ? 4.0 + 0.001 * i : 0.3 / (1.0 + abs(i - j)) + 0.01 * ((i * 7 + j * 3) % 5);
  if (i < j)
    v = 0.0;
  else if (i != j)
    v = 0.3 / (1.0 + (i - j)) * 0.1 + 0.001 * (((i + j) * 7) % 5);
  A[(size_t)j * ld + i] = v;
}
} // namespace ovp
// microbenchmark of the fused Cholesky on a synthetic SPD n x n system (+ optional mrows x n right-hand side):
// out[0] = us per (fill + factor), out[1] = us per fill alone, out[2..] = globaltimer stamps (ns, relative to the earliest) of the
// last run, 16 per CTA
extern "C" int ovp_debug_chol_fused(ovp_ctx *h, int n, int mrows, int iters, double *out, int out_cap) {
  Ctx *c = ovp::enter(h);
  if (n > c->wsS.cap || mrows > c->Nmax)
    return fail(c, OVP_ERR_CAPACITY, "debug_chol_fused: too large");
  const int T = (n + 63) / 64;
  const int ncta = T * (T + 1) / 2 + (mrows ? (mrows + 1 + 15) / 16 : 0);
  long long *dbg = nullptr;
  OVP_CUDA(cudaMalloc(&dbg, ((size_t)ncta * 16 + 128) * sizeof(long long))); // + the spine's per-step stamps, not reported here
  OVP_CUDA(cudaMemset(dbg, 0, ((size_t)ncta * 16 + 128) * sizeof(long long)));
  float ms;
  for (int variant = 0; variant < 2; variant++) {
    for (int rep = 0; rep < 2; rep++) {
      if (rep == 1)
        cudaEventRecord(c->ev[4], c->stream);
      for (int it = 0; it < iters; it++) {
        spd_fill_kernel<<<(n * n + 255) / 256, 256, 0, c->stream>>>(c->wsS.S, c->wsS.cap, n);
        if (variant == 0) {
          int st = chol_fused(c, c->wsS.S, c->wsS.cap, n, n, 0.0, mrows ? c->dM : nullptr, c->Nmax, mrows, mrows ? c->dvec + c->Rcap : nullptr, 1,
                              c->dY, c->Nmax, c->dvec, -1.0, nullptr, nullptr, dbg);
          if (st)
            return st;
        }
      }
      if (rep == 1)
        cudaEventRecord(c->ev[5], c->stream);
      OVP_CUDA(cudaStreamSynchronize(c->stream));
    }
    cudaEventElapsedTime(&ms, c->ev[4], c->ev[5]);
    out[variant] = 1e3 * ms / iters;
  }
  std::vector<long long> ts((size_t)ncta * 16 + 64);
  OVP_CUDA(cudaMemcpy(ts.data(), dbg, ts.size() * sizeof(long long), cudaMemcpyDeviceToHost));
  cudaFree(dbg);
  long long t0 = LLONG_MAX;
  const size_t nper = (size_t)ncta * 16;
  for (size_t i = 0; i < nper; i++)
    if (ts[i] > 0 && ((i & 15) < 8 || (i & 15) == 15)) // slots 8..14 are clock64 stamps, relative to slot 8 of the same CTA
      t0 = std::min(t0, ts[i]);
  out[2] = ncta;
  for (size_t i = 0; i < ts.size() && (int)(3 + i) < out_cap; i++) {
    if (i >= nper) { // spine phase stamps (clock64), relative to the first one
      out[3 + i] = ts[i] > 0 ? (double)(ts[i] - ts[nper]) : -1.0;
      continue;
    }
    const bool cyc = (i & 15) >= 8 && (i & 15) < 15;
    out[3 + i] = ts[i] > 0 ? (double)(ts[i] - (cyc ? ts[(i & ~(size_t)15) + 8] : t0)) : -1.0;
  }
  int info = 0;
  OVP_CUDA(cudaMemcpy(&info, c->dflags + 1, sizeof(int), cudaMemcpyDeviceToHost));
  if (info) {
    cudaMemset(c->dflags + 1, 0, sizeof(int));
    return fail(c, OVP_ERR_NOT_POSITIVE_DEFINITE, "debug_chol_fused: test matrix not positive definite");
  }
  return OVP_OK;
}

// Test hook for the DMMA GEMM (tests/test_gpu_gemm.py): one GemmProblem on host operands through launch_gemm, tile width forced or
// automatic.  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_gemm(ovp_ctx *h, int M, int N, int K, const double *A, int a_rows, int a_cols, int a_trans, const int *akidx,
                              const double *B, int b_rows, int b_cols, int b_trans, const int *bkidx, double *C, int ldc, double alpha,
                              double beta, const double *diag_add, double diag_const, int tri, int ktri, int flag, int tile, int *info) {
  Ctx *c = ovp::enter(h);
  if (M < 0 || N < 0 || K < 0 || ldc < M || a_rows < 1 || a_cols < 1 || b_rows < 1 || b_cols < 1 || (tile != 0 && tile != 32 && tile != 64))
    return fail(c, OVP_ERR_BAD_ARGS, "debug_gemm: bad sizes");
  const size_t na = (size_t)a_rows * a_cols, nb = (size_t)b_rows * b_cols, nc = (size_t)ldc * std::max(N, 1);
  const size_t nd = (size_t)std::max(1, std::min(M, N));
  const size_t bytes = (na + nb + nc + nd) * sizeof(double) + 2 * ((size_t)K + 1) * sizeof(int) + 16;
  char *buf = nullptr;
  OVP_CUDA(cudaMalloc(&buf, bytes));
  double *dA = (double *)buf, *dB = dA + na, *dC = dB + nb, *dD = dC + nc;
  int *dak = (int *)(dD + nd), *dbk = dak + K + 1, *dflag = dbk + K + 1;
  int st = OVP_OK;
  auto run = [&]() -> int {
    OVP_CUDA(cudaMemcpyAsync(dA, A, na * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpyAsync(dB, B, nb * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpyAsync(dC, C, nc * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    if (diag_add)
      OVP_CUDA(cudaMemcpyAsync(dD, diag_add, std::min(M, N) * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    if (akidx && K)
      OVP_CUDA(cudaMemcpyAsync(dak, akidx, K * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    if (bkidx && K)
      OVP_CUDA(cudaMemcpyAsync(dbk, bkidx, K * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpyAsync(dflag, &flag, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    // logical A (M x K): gathers index the physical column (plain) or row (transposed); logical B (K x N): the physical row or column
    MatView va = a_trans ? mv(dA, a_rows, 1, akidx ? dak : nullptr, nullptr) : mv(dA, a_rows, 0, nullptr, akidx ? dak : nullptr);
    MatView vb = b_trans ? mv(dB, b_rows, 1, nullptr, bkidx ? dbk : nullptr) : mv(dB, b_rows, 0, bkidx ? dbk : nullptr, nullptr);
    GemmProblem p = make_problem(M, N, K, va, vb, dC, ldc, alpha, beta);
    p.diag_add = diag_add ? dD : nullptr;
    p.diag_const = diag_const;
    p.tri = tri;
    p.ktri = ktri;
    GemmBatch b;
    b.n = 1;
    b.p[0] = p;
    b.flag = flag >= 0 ? dflag : nullptr;
    info[0] = launch_gemm(c, b, tile);
    info[1] = c->num_sms;
    OVP_CUDA(cudaGetLastError());
    OVP_CUDA(cudaMemcpyAsync(C, dC, nc * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaStreamSynchronize(c->stream));
    return OVP_OK;
  };
  st = run();
  cudaFree(buf);
  return st;
}

// Test hook for the DMMA GEMM's k split (tests/test_gpu_gemm_split.py): the tile width and the chunks launch_gemm takes for one product of
// these sizes.  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_gemm_split(ovp_ctx *h, int M, int N, int K, int tri, int ktri, int tile, int *info) {
  Ctx *c = ovp::enter(h);
  if (M < 0 || N < 0 || K < 0 || (tile != 0 && tile != 32 && tile != 64))
    return fail(c, OVP_ERR_BAD_ARGS, "debug_gemm_split: bad sizes");
  GemmProblem p = make_problem(M, N, K, mv(nullptr, 1), mv(nullptr, 1), nullptr, std::max(M, 1));
  p.tri = tri;
  p.ktri = ktri;
  GemmBatch b;
  b.n = 1;
  b.p[0] = p;
  b.flag = nullptr;
  info[0] = gemm_plan(c, b, tile, &info[1], &info[2]);
  return OVP_OK;
}

// Test hook for the innovation launch of the fused Cholesky (tests/test_gpu_compression.py): factor a host matrix (lower triangle of A,
// n x n, column-major) over its leading npiv columns with pivot tolerance tol and, when M is given, solve Y = M L^-T (mrows x npiv) and
// w = L^-1 z, and form chi2 = |w|^2 and the gate flag of gate_thresh in the same launch.  z (npiv values) is read on the device with
// stride zstride: 1 from a vector of its own, 0 in place in a column-major workspace of leading dimension wsG.cap, the layout of the
// compressed update (gram_factor_update reads z as the last row of the Gram factor); the rest of that workspace holds NaNs.  Not part of
// the ABI in include/ovp.h.
// panel = 0: one chol_fused launch; > 0: chol_panels with panels of that width
static int debug_chol_solve(ovp_ctx *h, int panel, const double *A, int n, int npiv, double tol, const double *M, int mrows, const double *z,
                            int zstride, double gate_thresh, double *L_out, double *Y_out, double *w_out, double *chi2_out, int *gate_out) {
  Ctx *c = ovp::enter(h);
  if (n > c->wsS.cap || mrows > c->Nmax || npiv > n || npiv > c->wsG.cap)
    return fail(c, OVP_ERR_CAPACITY, "debug_chol_solve: too large");
  if (zstride != 0 && zstride != 1)
    return fail(c, OVP_ERR_BAD_ARGS, "debug_chol_solve: zstride must be 0 or 1");
  const int ld = c->wsS.cap;
  OVP_CUDA(cudaMemsetAsync(c->wsS.S, 0, (size_t)ld * ld * sizeof(double), c->stream));
  OVP_CUDA(cudaMemcpy2DAsync(c->wsS.S, (size_t)ld * sizeof(double), A, (size_t)n * sizeof(double), (size_t)n * sizeof(double), n,
                             cudaMemcpyHostToDevice, c->stream));
  double *dz = nullptr;
  int zs = 1;
  if (M) {
    OVP_CUDA(cudaMemcpy2DAsync(c->dM, (size_t)c->Nmax * sizeof(double), M, (size_t)mrows * sizeof(double), (size_t)mrows * sizeof(double),
                               npiv, cudaMemcpyHostToDevice, c->stream));
    if (zstride == 1) {
      dz = c->dvec + c->Rcap;
      OVP_CUDA(cudaMemcpyAsync(dz, z, (size_t)npiv * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    } else { // row npiv - 1 of the Gram workspace, as row nc of the compressed update's factor (all-ones bytes: NaN everywhere else)
      zs = c->wsG.cap;
      dz = c->wsG.S + (npiv - 1);
      OVP_CUDA(cudaMemsetAsync(c->wsG.S, 0xff, (size_t)zs * zs * sizeof(double), c->stream));
      OVP_CUDA(cudaMemcpy2DAsync(dz, (size_t)zs * sizeof(double), z, sizeof(double), sizeof(double), npiv, cudaMemcpyHostToDevice, c->stream));
    }
  }
  int st = panel ? chol_panels(c, panel, c->wsS.S, ld, n, npiv, tol, M ? c->dM : nullptr, c->Nmax, mrows, dz, zs, c->dY, c->Nmax, c->dvec,
                               gate_thresh, c->dscal + 8, c->dflags + 3)
                 : chol_fused(c, c->wsS.S, ld, n, npiv, tol, M ? c->dM : nullptr, c->Nmax, mrows, dz, zs, c->dY, c->Nmax, c->dvec, gate_thresh,
                              c->dscal + 8, c->dflags + 3);
  if (st)
    return st;
  OVP_CUDA(cudaMemcpy2DAsync(L_out, (size_t)n * sizeof(double), c->wsS.S, (size_t)ld * sizeof(double), (size_t)n * sizeof(double), n,
                             cudaMemcpyDeviceToHost, c->stream));
  if (M) {
    OVP_CUDA(cudaMemcpy2DAsync(Y_out, (size_t)mrows * sizeof(double), c->dY, (size_t)c->Nmax * sizeof(double), (size_t)mrows * sizeof(double),
                               npiv, cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaMemcpyAsync(w_out, c->dvec, (size_t)npiv * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (chi2_out)
      OVP_CUDA(cudaMemcpyAsync(chi2_out, c->dscal + 8, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (gate_out)
      OVP_CUDA(cudaMemcpyAsync(gate_out, c->dflags + 3, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  }
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  int info = 0;
  OVP_CUDA(cudaMemcpy(&info, c->dflags + 1, sizeof(int), cudaMemcpyDeviceToHost));
  if (info) {
    cudaMemset(c->dflags + 1, 0, sizeof(int));
    return fail(c, OVP_ERR_NOT_POSITIVE_DEFINITE, "debug_chol_solve: matrix not positive definite (strict mode)");
  }
  return OVP_OK;
}
extern "C" int ovp_debug_chol_solve_gated(ovp_ctx *h, const double *A, int n, int npiv, double tol, const double *M, int mrows,
                                          const double *z, int zstride, double gate_thresh, double *L_out, double *Y_out, double *w_out,
                                          double *chi2_out, int *gate_out) {
  return debug_chol_solve(h, 0, A, n, npiv, tol, M, mrows, z, zstride, gate_thresh, L_out, Y_out, w_out, chi2_out, gate_out);
}

// Test hook for the panelled factorisation (tests/test_gpu_wide_updates.py): ovp_debug_chol_solve_gated through chol_panels with panels of
// `panel` columns (a multiple of 64 up to the co-resident width), so that narrow systems cross panel boundaries.  Not part of the ABI in
// include/ovp.h.
extern "C" int ovp_debug_chol_panels(ovp_ctx *h, int panel, const double *A, int n, int npiv, double tol, const double *M, int mrows,
                                     const double *z, int zstride, double gate_thresh, double *L_out, double *Y_out, double *w_out,
                                     double *chi2_out, int *gate_out) {
  if (panel <= 0)
    return fail(&h->c, OVP_ERR_BAD_ARGS, "debug_chol_panels: panel width %d", panel);
  return debug_chol_solve(h, panel, A, n, npiv, tol, M, mrows, z, zstride, gate_thresh, L_out, Y_out, w_out, chi2_out, gate_out);
}

// Test hook for the fused Cholesky (tests/test_gpu_cholfused.py, tests/test_gpu_fused_products.py): ovp_debug_chol_solve_gated with z
// read from a vector of its own and no gate.  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_chol_solve(ovp_ctx *h, const double *A, int n, int npiv, double tol, const double *M, int mrows, const double *z,
                                    double *L_out, double *Y_out, double *w_out) {
  return ovp_debug_chol_solve_gated(h, A, n, npiv, tol, M, mrows, z, 1, -1.0, L_out, Y_out, w_out, nullptr, nullptr);
}

// Test hook (tests/test_gpu_numerics.py): on != 0 sends every later MSCKF batch of this context through the one-block-per-feature kernel
// and the dense stacked system, whatever its longest track; the plan key includes the setting.  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_force_dense_features(ovp_ctx *h, int on) {
  h->c.force_dense_features = on != 0;
  return OVP_OK;
}

// Test hook (tests/test_gpu_fused_products.py): on != 0 sends every later compressed update of this context through the factorisation
// and two GEMM launches for M and S, instead of the factorisation that forms them; the plan key includes the setting.  Not part of
// the ABI in include/ovp.h.
extern "C" int ovp_debug_unfused_update_products(ovp_ctx *h, int on) {
  h->c.unfused_update_products = on != 0;
  return OVP_OK;
}

// Test / A-B hook (tests/test_gpu_pipelined_factor.py): with on != 0 every later compressed update of this context factors its Gram
// matrix and its innovation system one after the other, also when they would fit a pair (chol_fused_pair); the plan key includes
// the setting.  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_sequential_factorisations(ovp_ctx *h, int on) {
  h->c.sequential_factorisations = on != 0;
  return OVP_OK;
}

// Test / A-B hook (tests/test_gpu_pdl_chain.py): with on == 0 every later launch of the update chain waits for the whole of the launch
// before it instead of starting as its programmatic dependent (chain_launch).  A changed setting drops the prepared batch's captured
// graph, so the next launch of the same plan captures its kernels with the new setting.  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_programmatic_launches(ovp_ctx *h, int on) {
  if (h->c.programmatic != (on != 0))
    drop_prepared_graph(&h->c);
  h->c.programmatic = on != 0;
  return OVP_OK;
}

// Test hook (tests/test_gpu_pipelined_factor.py, tools/microbench_chol.py): ovp_debug_chol_products followed by the innovation
// factorisation of a compressed update, as gram_factor_update runs them (paired unless ovp_debug_sequential_factorisations or the pair does
// not fit).  z = row nc of the Gram factor.  Outputs as ovp_debug_chol_products, plus LS_out (npiv x npiv: S factored in place, lower tiles
// written, the rest left as passed in), Y_out (N x npiv), w_out (npiv), chi2_out / gate_out (gate_thresh < 0: always 1).  info[0] = 1 when
// the pair ran.  timeline (NULL, or 64 doubles): globaltimer stamps in us relative to the first, -1 where absent:
// [k] the Gram spine released D(k), [32 + k] the innovation spine started step k (k < 32).  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_chol_pair(ovp_ctx *h, const double *G, int nc, int npiv, double tol, const double *P, int N, const int *cols,
                                   double gate_thresh, double *L_out, double *M_out, double *LS_out, double *Y_out, double *w_out,
                                   double *chi2_out, int *gate_out, int *info, double *timeline) {
  Ctx *c = ovp::enter(h);
  const int n = nc + 1;
  if (n > c->wsG.cap || npiv > c->wsS.cap || N > c->Nmax || npiv > nc || N < 1 || npiv < 1)
    return fail(c, OVP_ERR_CAPACITY, "debug_chol_pair: too large");
  const int ldp = (N + 1) & ~1;
  // stamps of at most the paired grid (64 product-only CTAs is more than any launch takes) + the phase and step stamps
  const size_t ndbg = (size_t)16 * (chol_fused_tiles(n, npiv) + chol_fused_tiles(npiv, npiv) + 64 + (N + 16) / 16) + 192;
  char *buf = nullptr;
  OVP_CUDA(cudaMalloc(&buf, 2 * sizeof(double) + (size_t)ldp * N * sizeof(double) + ndbg * sizeof(long long) + (size_t)nc * sizeof(int)));
  double *dchi2 = (double *)buf;
  int *dgate = (int *)(dchi2 + 1);
  double *dP = dchi2 + 2;
  long long *dbg = (long long *)(dP + (size_t)ldp * N);
  int *dcols = (int *)(dbg + ndbg);
  auto run = [&]() -> int {
    const int ldg = c->wsG.cap, lds = c->wsS.cap;
    OVP_CUDA(cudaMemsetAsync(dbg, 0, ndbg * sizeof(long long), c->stream));
    OVP_CUDA(cudaMemsetAsync(c->wsG.S, 0, (size_t)ldg * ldg * sizeof(double), c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(c->wsG.S, (size_t)ldg * sizeof(double), G, (size_t)n * sizeof(double), (size_t)n * sizeof(double), n,
                               cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(dP, (size_t)ldp * sizeof(double), P, (size_t)N * sizeof(double), (size_t)N * sizeof(double), N,
                               cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpyAsync(dcols, cols, (size_t)nc * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(c->wsS.S, (size_t)lds * sizeof(double), LS_out, (size_t)npiv * sizeof(double), (size_t)npiv * sizeof(double),
                               npiv, cudaMemcpyHostToDevice, c->stream));
    const CholProducts pr{dP, dcols, c->dM, c->wsS.S, ldp, N, nc, c->Nmax, lds};
    const double *z = c->wsG.S + nc;
    bool paired = false;
    int s = chol_fused_pair(c, c->wsG.S, ldg, n, npiv, tol, pr, z, ldg, c->dY, c->Nmax, c->dvec, gate_thresh, dchi2, dgate, dbg, &paired);
    if (!s && !paired) {
      s = chol_fused(c, c->wsG.S, ldg, n, npiv, tol, nullptr, 0, 0, nullptr, 1, nullptr, 0, nullptr, -1.0, nullptr, nullptr, nullptr, &pr);
      if (!s)
        s = chol_fused(c, c->wsS.S, lds, npiv, npiv, 0.0, c->dM, c->Nmax, N, z, ldg, c->dY, c->Nmax, c->dvec, gate_thresh, dchi2, dgate);
    }
    if (s)
      return s;
    OVP_CUDA(cudaGetLastError());
    OVP_CUDA(cudaMemcpy2DAsync(L_out, (size_t)n * sizeof(double), c->wsG.S, (size_t)ldg * sizeof(double), (size_t)n * sizeof(double), npiv,
                               cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(M_out, (size_t)N * sizeof(double), c->dM, (size_t)c->Nmax * sizeof(double), (size_t)N * sizeof(double), npiv,
                               cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(LS_out, (size_t)npiv * sizeof(double), c->wsS.S, (size_t)lds * sizeof(double), (size_t)npiv * sizeof(double),
                               npiv, cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(Y_out, (size_t)N * sizeof(double), c->dY, (size_t)c->Nmax * sizeof(double), (size_t)N * sizeof(double), npiv,
                               cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaMemcpyAsync(w_out, c->dvec, (size_t)npiv * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    double chi2 = 0.0;
    int gate = 0;
    OVP_CUDA(cudaMemcpyAsync(&chi2, dchi2, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaMemcpyAsync(&gate, dgate, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    std::vector<long long> ts(ndbg);
    OVP_CUDA(cudaMemcpyAsync(ts.data(), dbg, ndbg * sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaStreamSynchronize(c->stream));
    if (chi2_out)
      *chi2_out = chi2;
    if (gate_out)
      *gate_out = gate;
    info[0] = paired ? 1 : 0;
    if (timeline) { // the pair's cooperative grid: its step stamps sit after 16 per CTA and 64 phase stamps (cholfused.cu, CF_STEP_TS)
      for (int k = 0; k < 64; k++)
        timeline[k] = -1.0;
      if (paired) {
        size_t grid = 0;
        while (grid * 16 + 192 <= ndbg && ts[grid * 16 + 15] != 0)
          grid++; // every CTA stamps its end (slot 15)
        const long long *st = ts.data() + grid * 16 + 64;
        long long t0 = LLONG_MAX;
        for (int k = 0; k < 32; k++) {
          if (st[32 + k])
            t0 = std::min(t0, st[32 + k]);
          if (st[64 + k])
            t0 = std::min(t0, st[64 + k]);
        }
        for (int k = 0; k < 32; k++) {
          timeline[k] = st[32 + k] ? 1e-3 * (double)(st[32 + k] - t0) : -1.0;
          timeline[32 + k] = st[64 + k] ? 1e-3 * (double)(st[64 + k] - t0) : -1.0;
        }
      }
    }
    return OVP_OK;
  };
  int st = run();
  cudaFree(buf);
  if (!st) {
    int pd = 0;
    OVP_CUDA(cudaMemcpy(&pd, c->dflags + 1, sizeof(int), cudaMemcpyDeviceToHost));
    if (pd) {
      cudaMemset(c->dflags + 1, 0, sizeof(int));
      return fail(c, OVP_ERR_NOT_POSITIVE_DEFINITE, "debug_chol_pair: innovation system not positive definite");
    }
  }
  return st;
}

// Test hook (tests/test_gpu_fused_products.py): one factorisation launch that also forms the update products.  G: (nc + 1) x (nc + 1)
// lower triangle, column-major, factored over its leading npiv columns with pivot tolerance tol; P: N x N, column-major; cols: nc state
// indices.  L_out: (nc + 1) x npiv, M_out: N x npiv, S_out: npiv x npiv (lower triangle written, the rest left as passed in).  Not part of
// the ABI in include/ovp.h.
extern "C" int ovp_debug_chol_products(ovp_ctx *h, const double *G, int nc, int npiv, double tol, const double *P, int N, const int *cols,
                                       double *L_out, double *M_out, double *S_out) {
  Ctx *c = ovp::enter(h);
  const int n = nc + 1;
  if (n > c->wsG.cap || npiv > c->wsS.cap || N > c->Nmax || npiv > nc || N < 1 || npiv < 1)
    return fail(c, OVP_ERR_CAPACITY, "debug_chol_products: too large");
  const int ldp = (N + 1) & ~1;
  char *buf = nullptr;
  OVP_CUDA(cudaMalloc(&buf, (size_t)ldp * N * sizeof(double) + (size_t)nc * sizeof(int)));
  double *dP = (double *)buf;
  int *dcols = (int *)(dP + (size_t)ldp * N);
  int st = OVP_OK;
  auto run = [&]() -> int {
    const int ldg = c->wsG.cap, lds = c->wsS.cap;
    OVP_CUDA(cudaMemsetAsync(c->wsG.S, 0, (size_t)ldg * ldg * sizeof(double), c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(c->wsG.S, (size_t)ldg * sizeof(double), G, (size_t)n * sizeof(double), (size_t)n * sizeof(double), n,
                               cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(dP, (size_t)ldp * sizeof(double), P, (size_t)N * sizeof(double), (size_t)N * sizeof(double), N,
                               cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpyAsync(dcols, cols, (size_t)nc * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(c->wsS.S, (size_t)lds * sizeof(double), S_out, (size_t)npiv * sizeof(double), (size_t)npiv * sizeof(double),
                               npiv, cudaMemcpyHostToDevice, c->stream));
    const CholProducts pr{dP, dcols, c->dM, c->wsS.S, ldp, N, nc, c->Nmax, lds};
    int s = chol_fused(c, c->wsG.S, ldg, n, npiv, tol, nullptr, 0, 0, nullptr, 1, nullptr, 0, nullptr, -1.0, nullptr, nullptr, nullptr, &pr);
    if (s)
      return s;
    OVP_CUDA(cudaGetLastError());
    OVP_CUDA(cudaMemcpy2DAsync(L_out, (size_t)n * sizeof(double), c->wsG.S, (size_t)ldg * sizeof(double), (size_t)n * sizeof(double), npiv,
                               cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(M_out, (size_t)N * sizeof(double), c->dM, (size_t)c->Nmax * sizeof(double), (size_t)N * sizeof(double), npiv,
                               cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaMemcpy2DAsync(S_out, (size_t)npiv * sizeof(double), c->wsS.S, (size_t)lds * sizeof(double), (size_t)npiv * sizeof(double),
                               npiv, cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaStreamSynchronize(c->stream));
    return OVP_OK;
  };
  st = run();
  cudaFree(buf);
  return st;
}

// Test hook (tests/test_gpu_compression.py): prepare a feature batch as ovp_msckf_update does and run the first non-empty plan of its
// launch order (a plane plan first if the batch has planes, otherwise the point plan) up to its Gram matrix G = D - Y^T Y; nothing after
// it runs, so the state is left as it was.  Eager launches.  G_out (gcap x gcap, column-major, leading dimension nc1) receives all of G.
// info: [0] nc1, [1] ncal, [2] ncx (x columns; H_cp, when present, sits at ncx .. ncx + 2 and the residual at nc1 - 1), [3] point plan,
// [4] selected features nsel, [5] CTA-per-feature path, [6] plane slot, [7] plane in the state.  cols_out (gcap): compact column -> state
// index of the x columns; sel_out (F): the plan's features; feat_status / feat_chi2 (F): the per-feature status words after the plan's
// feature kernel.  raw_out (optional, 3 * OVP_RAW_ROW doubles per measurement, OVP_RAW_ROW in features.cu): the raw whitened rows the
// feature kernel built.  A plan that goes straight into the update (no compression) has no Gram matrix: it stops after its feature
// kernel, without updating, with info[0] = 0, info[5] = 0 and G_out untouched; raw_out holds its rows (tests/test_gpu_plane_update_reference.py).
// Not part of the ABI in include/ovp.h.
// ovp_debug_msckf_gram_landmarks: the same with the landmark members of ovp_msckf_update_landmarks (their columns follow the x columns
// of the batch features, ncx counts them).
static int debug_msckf_gram(ovp_ctx *h, const ovp_feature_batch *b, const ovp_plane_landmarks *lm, const ovp_updater_options *opt, int gcap,
                            double *G_out, int *info, int *cols_out, int *sel_out, int *feat_status, double *feat_chi2, double *raw_out) {
  Ctx *c = ovp::enter(h);
  if (!b || !opt || b->F <= 0)
    return fail(c, OVP_ERR_BAD_ARGS, "debug_msckf_gram: empty batch");
  MsckfExtra ex;
  ex.landmarks = lm;
  int st = msckf_prepare(c, b, opt, lm && lm->n > 0 ? &ex : nullptr);
  if (st)
    return st;
  Prepared &P = *c->prep;
  const size_t nraw = (size_t)3 * OVP_RAW_ROW * std::max(P.M, 1);
  double *draw = nullptr;
  if (raw_out) {
    OVP_CUDA(cudaMalloc(&draw, nraw * sizeof(double)));
    OVP_CUDA(cudaMemsetAsync(draw, 0, nraw * sizeof(double), c->stream));
  }
  c->dbg_raw = draw;
  c->dbg_gram_stop = true;
  c->dbg_gram_plan = -1;
  st = msckf_launch_body(c, true);
  c->dbg_raw = nullptr;
  c->dbg_gram_stop = false;
  auto run = [&]() -> int {
    if (st)
      return st;
    OVP_CUDA(cudaStreamSynchronize(c->stream));
    if (c->dbg_gram_plan < 0)
      return fail(c, OVP_ERR_BAD_ARGS, "debug_msckf_gram: the batch has no plan with features");
    const UpdatePlan &pl = P.plans[c->dbg_gram_plan];
    const int ncx = pl.nx(), nc1 = pl.is_point ? ncx + 1 : ncx + 4;
    if (nc1 > gcap)
      return fail(c, OVP_ERR_CAPACITY, "debug_msckf_gram: %d columns, room for %d", nc1, gcap);
    const int ncal = (c->opt.do_calib_camera_pose ? 6 : 0) + (c->opt.do_calib_camera_intrinsics ? 8 : 0);
    // a plan that goes straight into the update has no Gram matrix: nc1 is reported as 0 and G_out is left as passed
    const int v[8] = {pl.direct ? 0 : nc1, ncal, ncx, pl.is_point ? 1 : 0, (int)pl.feats.size(), P.fast && !pl.direct ? 1 : 0, pl.plane_slot,
                      pl.in_state ? 1 : 0};
    std::memcpy(info, v, sizeof(v));
    std::memcpy(cols_out, pl.cols.data(), pl.cols.size() * sizeof(int));
    for (size_t k = 0; k < pl.lm_handle.size(); k++)
      for (int j = 0; j < 3; j++)
        cols_out[pl.cols.size() + 3 * k + j] = c->vars[pl.lm_handle[k]].id + j;
    std::memcpy(sel_out, pl.feats.data(), pl.feats.size() * sizeof(int));
    if (!pl.direct)
      OVP_CUDA(cudaMemcpy2DAsync(G_out, (size_t)nc1 * sizeof(double), c->wsG.S, (size_t)c->wsG.cap * sizeof(double), (size_t)nc1 * sizeof(double),
                               nc1, cudaMemcpyDeviceToHost, c->stream));
    if (raw_out)
      OVP_CUDA(cudaMemcpyAsync(raw_out, draw, nraw * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    std::vector<int> flag;
    std::vector<double> chi2;
    int s = read_feature_status(c, P.F, (const char *)c->d_batch, P.o_flag, P.o_chi, flag, chi2); // synchronises
    if (s)
      return s;
    std::memcpy(feat_status, flag.data(), P.F * sizeof(int));
    std::memcpy(feat_chi2, chi2.data(), P.F * sizeof(double));
    return OVP_OK;
  };
  st = run();
  free_prepared(c); // the next update prepares its batch again (this one stopped half way)
  if (draw)
    cudaFree(draw);
  return st;
}
extern "C" int ovp_debug_msckf_gram(ovp_ctx *h, const ovp_feature_batch *b, const ovp_updater_options *opt, int gcap, double *G_out,
                                    int *info, int *cols_out, int *sel_out, int *feat_status, double *feat_chi2, double *raw_out) {
  return debug_msckf_gram(h, b, nullptr, opt, gcap, G_out, info, cols_out, sel_out, feat_status, feat_chi2, raw_out);
}
extern "C" int ovp_debug_msckf_gram_landmarks(ovp_ctx *h, const ovp_feature_batch *b, const ovp_plane_landmarks *lm, const ovp_updater_options *opt,
                                              int gcap, double *G_out, int *info, int *cols_out, int *sel_out, int *feat_status, double *feat_chi2,
                                              double *raw_out) {
  return debug_msckf_gram(h, b, lm, opt, gcap, G_out, info, cols_out, sel_out, feat_status, feat_chi2, raw_out);
}

// Test hook (tests/test_gpu_feature_gate.py): ovp_slam_update, which also returns the raw whitened rows the SLAM feature kernel built
// (raw_out: 3 * OVP_RAW_ROW doubles per measurement of the batch, OVP_RAW_ROW in features.cu, [0,3) holding the landmark's columns).  The
// update itself runs as ovp_slam_update runs it.  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_slam_update(ovp_ctx *h, int F, const int *meas_offset, const int *meas_clone, const float *uv, const int64_t *featid,
                                     const int64_t *planeid, const ovp_updater_options *opt, int use_plane_constraint, int *feat_status,
                                     double *feat_chi2, double *raw_out) {
  Ctx *c = ovp::enter(h);
  if (F > 0 && (!meas_offset || !meas_clone || !uv || !featid || !opt))
    return fail(c, OVP_ERR_BAD_ARGS, "debug_slam_update: null argument");
  int M = 0;
  int st = check_offsets(c, "debug_slam_update", "meas_offset", F, meas_offset, &M);
  if (st)
    return st;
  const size_t nraw = (size_t)3 * OVP_RAW_ROW * std::max(M, 1);
  double *draw = nullptr;
  if (raw_out) {
    OVP_CUDA(cudaMalloc(&draw, nraw * sizeof(double)));
    OVP_CUDA(cudaMemsetAsync(draw, 0, nraw * sizeof(double), c->stream));
  }
  c->dbg_raw = draw;
  st = slam_update_impl(c, F, meas_offset, meas_clone, uv, featid, planeid, opt, use_plane_constraint, feat_status, feat_chi2);
  c->dbg_raw = nullptr;
  auto run = [&]() -> int {
    if (st || !raw_out)
      return st;
    OVP_CUDA(cudaMemcpyAsync(raw_out, draw, nraw * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaStreamSynchronize(c->stream));
    return OVP_OK;
  };
  st = run();
  if (draw)
    cudaFree(draw);
  return st;
}

// Test hook (tests/test_gpu_slam_reference.py): ovp_slam_update up to its Gram matrix, with the state and the bookkeeping left as they were
// (declared in include/ovp_debug.h).  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_slam_gram(ovp_ctx *h, int F, const int *meas_offset, const int *meas_clone, const float *uv, const int64_t *featid,
                                   const int64_t *planeid, const ovp_updater_options *opt, int use_plane_constraint, int gcap, double *G_out,
                                   int *info, int *cols_out, int *feat_status, double *feat_chi2, double *raw_out) {
  Ctx *c = ovp::enter(h);
  if (F <= 0 || !meas_offset || !meas_clone || !uv || !featid || !opt || !G_out || !info || !cols_out || !feat_status || !feat_chi2)
    return fail(c, OVP_ERR_BAD_ARGS, "debug_slam_gram: empty batch or null argument");
  int M = 0;
  int st = check_offsets(c, "debug_slam_gram", "meas_offset", F, meas_offset, &M);
  if (st)
    return st;
  const size_t nraw = (size_t)3 * OVP_RAW_ROW * std::max(M, 1);
  double *draw = nullptr;
  if (raw_out) {
    OVP_CUDA(cudaMalloc(&draw, nraw * sizeof(double)));
    OVP_CUDA(cudaMemsetAsync(draw, 0, nraw * sizeof(double), c->stream));
  }
  c->dbg_raw = draw;
  c->dbg_gram_stop = true;
  c->dbg_slam_cols.clear();
  c->dbg_slam_rows = 0;
  st = slam_update_impl(c, F, meas_offset, meas_clone, uv, featid, planeid, opt, use_plane_constraint, feat_status, feat_chi2);
  c->dbg_raw = nullptr;
  c->dbg_gram_stop = false;
  auto run = [&]() -> int {
    if (st)
      return st;
    const int nc = (int)c->dbg_slam_cols.size(), nc1 = nc + 1;
    if (nc1 > gcap)
      return fail(c, OVP_ERR_CAPACITY, "debug_slam_gram: %d columns, room for %d", nc1, gcap);
    info[0] = nc1;
    info[1] = c->dbg_slam_rows;
    std::memcpy(cols_out, c->dbg_slam_cols.data(), (size_t)nc * sizeof(int));
    OVP_CUDA(cudaMemcpy2DAsync(G_out, (size_t)nc1 * sizeof(double), c->wsG.S, (size_t)c->wsG.cap * sizeof(double), (size_t)nc1 * sizeof(double), nc1,
                               cudaMemcpyDeviceToHost, c->stream));
    if (raw_out)
      OVP_CUDA(cudaMemcpyAsync(raw_out, draw, nraw * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaStreamSynchronize(c->stream));
    return OVP_OK;
  };
  st = run();
  if (draw)
    cudaFree(draw);
  return st;
}

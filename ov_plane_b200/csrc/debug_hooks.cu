// TEST / TUNING HOOKS — compiled only into libovp_debug.so (-DOVP_DEBUG), never into the product library libovp.so.
// Declared in include/ovp_debug.h.  Used by tools/microbench_chol.py (phase timeline of the fused Cholesky), by
// tests/test_gpu_cholfused.py and tests/test_gpu_gemm.py (unit tests of chol_fused_kernel and the DMMA GEMM against NumPy) and by
// tests/test_gpu_numerics.py (the block-sparse feature path against the dense stack on the same batch).
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
  OVP_CUDA(cudaMalloc(&dbg, ((size_t)ncta * 16 + 64) * sizeof(long long)));
  OVP_CUDA(cudaMemset(dbg, 0, ((size_t)ncta * 16 + 64) * sizeof(long long)));
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

// Test hook for the fused Cholesky (tests/test_gpu_cholfused.py): factor a host matrix (lower triangle of A, n x n, column-major)
// over its leading npiv columns with pivot tolerance tol and, when M is given, solve Y = M L^-T (mrows x npiv) and w = L^-1 z.
// Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_chol_solve(ovp_ctx *h, const double *A, int n, int npiv, double tol, const double *M, int mrows, const double *z,
                                    double *L_out, double *Y_out, double *w_out) {
  Ctx *c = ovp::enter(h);
  if (n > c->wsS.cap || mrows > c->Nmax || npiv > n)
    return fail(c, OVP_ERR_CAPACITY, "debug_chol_solve: too large");
  const int ld = c->wsS.cap;
  OVP_CUDA(cudaMemsetAsync(c->wsS.S, 0, (size_t)ld * ld * sizeof(double), c->stream));
  OVP_CUDA(cudaMemcpy2DAsync(c->wsS.S, (size_t)ld * sizeof(double), A, (size_t)n * sizeof(double), (size_t)n * sizeof(double), n,
                             cudaMemcpyHostToDevice, c->stream));
  if (M) {
    OVP_CUDA(cudaMemcpy2DAsync(c->dM, (size_t)c->Nmax * sizeof(double), M, (size_t)mrows * sizeof(double), (size_t)mrows * sizeof(double),
                               npiv, cudaMemcpyHostToDevice, c->stream));
    OVP_CUDA(cudaMemcpyAsync(c->dvec + c->Rcap, z, (size_t)npiv * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  }
  int st = chol_fused(c, c->wsS.S, ld, n, npiv, tol, M ? c->dM : nullptr, c->Nmax, mrows, M ? c->dvec + c->Rcap : nullptr, 1, c->dY, c->Nmax, c->dvec, -1.0,
                      c->dscal + 8, nullptr);
  if (st)
    return st;
  OVP_CUDA(cudaMemcpy2DAsync(L_out, (size_t)n * sizeof(double), c->wsS.S, (size_t)ld * sizeof(double), (size_t)n * sizeof(double), n,
                             cudaMemcpyDeviceToHost, c->stream));
  if (M) {
    OVP_CUDA(cudaMemcpy2DAsync(Y_out, (size_t)mrows * sizeof(double), c->dY, (size_t)c->Nmax * sizeof(double), (size_t)mrows * sizeof(double),
                               npiv, cudaMemcpyDeviceToHost, c->stream));
    OVP_CUDA(cudaMemcpyAsync(w_out, c->dvec, (size_t)npiv * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
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

// Test hook (tests/test_gpu_numerics.py): on != 0 sends every later MSCKF batch of this context through the one-block-per-feature kernel
// and the dense stacked system, whatever its longest track; the plan signature includes the setting.  Not part of the ABI in include/ovp.h.
extern "C" int ovp_debug_force_dense_features(ovp_ctx *h, int on) {
  h->c.force_dense_features = on != 0;
  return OVP_OK;
}

// Dense fp64 building blocks: batched DMMA GEMM launcher, blocked (rank-tolerant) Cholesky with diagonal-block and full
// triangular inverses, gemv / reductions.  Replaces Eigen's LLT + solveInPlace(I) + dense products of
// StateHelper::EKFUpdate (StateHelper.cpp:156-171) and the Givens triangularisation of measurement_compress_inplace
// (UpdaterHelper.cpp:548-579) by a Q-less Cholesky-QR (DESIGN.md §kernels).
#include <cstdlib>
#include "ovp_internal.h"
#include <algorithm>
#include <cstdarg>
#include <cstdio>

namespace ovp {

int fail(Ctx *c, int status, const char *fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  c->last_error = buf;
  return status;
}

template <int TILE> static void launch_gemm_tile(Ctx *c, const GemmBatch &b, dim3 grid) {
  const bool ga = b.p[0].A.kidx != nullptr, gb = b.p[0].B.kidx != nullptr;
  if (ga && gb)
    gemm_f64_kernel<TILE, true, true><<<grid, 128, 0, c->stream>>>(b);
  else if (ga)
    gemm_f64_kernel<TILE, true, false><<<grid, 128, 0, c->stream>>>(b);
  else if (gb)
    gemm_f64_kernel<TILE, false, true><<<grid, 128, 0, c->stream>>>(b);
  else
    gemm_f64_kernel<TILE, false, false><<<grid, 128, 0, c->stream>>>(b);
}
int launch_gemm(Ctx *c, const GemmBatch &b, int tile) {
  int tm = 0, tn = 0;
  long long tiles64 = 0;
  double work = 0;
  for (int i = 0; i < b.n; i++) {
    int a = (b.p[i].M + 63) / 64, bb = (b.p[i].N + 63) / 64;
    tm = std::max(tm, a);
    tn = std::max(tn, bb);
    tiles64 += (b.p[i].tri == TRI_FULL) ? (long long)a * bb : (long long)a * (a + 1) / 2;
    work += (b.p[i].tri == TRI_FULL ? 2.0 : 1.0) * (double)b.p[i].M * b.p[i].N * b.p[i].K;
  }
  if (tm == 0 || tn == 0 || b.n == 0)
    return 0;
  if (tile != 32 && tile != 64) // below one wave of 64-wide tiles, 32-wide ones give more CTAs to hide the k-loop latency
    tile = tiles64 >= c->num_sms ? 64 : 32;
  prof_begin(c, PROF_GEMM, work);
  if (tile == 64) {
    launch_gemm_tile<64>(c, b, dim3(tn, tm, b.n));
  } else { // fewer 64-tiles than SMs: 32-tiles quadruple the CTA count and quarter the per-CTA tensor work
    int tm32 = 0, tn32 = 0;
    for (int i = 0; i < b.n; i++) {
      tm32 = std::max(tm32, (b.p[i].M + 31) / 32);
      tn32 = std::max(tn32, (b.p[i].N + 31) / 32);
    }
    launch_gemm_tile<32>(c, b, dim3(tn32, tm32, b.n));
  }
  c->launches++;
  prof_end(c);
  return tile;
}

static cudaEvent_t prof_event(Ctx *c) {
  if (c->ev_used == c->ev_pool.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    c->ev_pool.push_back(e);
  }
  return c->ev_pool[c->ev_used++];
}
void prof_begin(Ctx *c, int id, double work) {
  if (!c->profiling)
    return;
  c->prof_pending = prof_event(c);
  c->prof_pending_id = id;
  c->prof_pending_work = work;
  cudaEventRecord(c->prof_pending, c->stream);
}
void prof_end(Ctx *c) {
  if (!c->profiling || !c->prof_pending)
    return;
  Ctx::ProfRec r;
  r.id = c->prof_pending_id;
  r.e0 = c->prof_pending;
  r.e1 = prof_event(c);
  r.work = c->prof_pending_work;
  cudaEventRecord(r.e1, c->stream);
  c->prof_recs.push_back(r);
  c->prof_pending = nullptr;
}
void launch_gemm1(Ctx *c, const GemmProblem &p, const int *flag) {
  if (p.M <= 0 || p.N <= 0)
    return;
  GemmBatch b;
  b.n = 1;
  b.p[0] = p;
  b.flag = flag;
  launch_gemm(c, b);
}

// -------------------------------------------------------------------------------------------------------------------
__global__ void fill_kernel(double *p, size_t n, double v) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride)
    p[i] = v;
}
void launch_fill(Ctx *c, double *p, size_t n, double v) {
  if (n == 0)
    return;
  if (v == 0.0) {
    cudaMemsetAsync(p, 0, n * sizeof(double), c->stream);
    c->launches++;
    return;
  }
  int blocks = (int)std::min<size_t>((n + 255) / 256, c->num_sms * 8);
  fill_kernel<<<blocks, 256, 0, c->stream>>>(p, n, v);
  c->launches++;
}


int ws_alloc(Ctx *c, DenseWs &ws, int cap) {
  ws.cap = cap;
  size_t e = (size_t)cap * cap;
  OVP_CUDA(cudaMalloc(&ws.S, e * sizeof(double)));
  OVP_CUDA(cudaMemset(ws.S, 0, e * sizeof(double)));
  return OVP_OK;
}
void ws_free(DenseWs &ws) {
  cudaFree(ws.S);
  ws = DenseWs();
}

// Cholesky of the leading npiv columns of the n x n lower-stored matrix A in place (rows npiv..n-1 are solved along): one launch
// of the fused kernel (cholfused.cu).  Pivots <= tol * original diagonal are treated as exact zeros (rank-deficient Gram matrices).
int chol_partial(Ctx *c, double *A, int ld, int n, int npiv, double tol) {
  return chol_fused(c, A, ld, n, npiv, tol, nullptr, 0, 0, nullptr, 1, nullptr, 0, nullptr, -1.0, nullptr, nullptr);
}

// stand-alone Householder left-nullspace projection on a global-memory matrix (col-major, ld): reflectors from the first
// nref columns applied to all ncols columns.  One CTA.
__global__ void __launch_bounds__(256) householder_cols_kernel(double *A, int ld, int rows, int ncols, int nref) {
  extern __shared__ double vbuf[];
  __shared__ double s_beta;
  const int tid = threadIdx.x;
  for (int j = 0; j < nref; j++) {
    if (tid < 32) {
      double s = 0.0;
      for (int i = j + tid; i < rows; i += 32) {
        double v = A[(size_t)j * ld + i];
        s += v * v;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        s += __shfl_xor_sync(0xffffffffu, s, o);
      double x0 = A[(size_t)j * ld + j];
      double nrm = sqrt(s);
      double alpha = (x0 > 0.0) ? -nrm : nrm;
      double v0 = x0 - alpha;
      double vtv = s - x0 * x0 + v0 * v0;
      for (int i = j + tid; i < rows; i += 32) {
        vbuf[i] = (i == j) ? v0 : A[(size_t)j * ld + i];
        if (nrm > 0.0)
          A[(size_t)j * ld + i] = (i == j) ? alpha : 0.0; // the reflected column itself: [alpha; 0]
      }
      if (tid == 0)
        s_beta = (vtv > 0.0 && nrm > 0.0) ? 2.0 / vtv : 0.0;
    }
    __syncthreads();
    const double beta = s_beta;
    for (int cidx = j + 1 + tid; cidx < ncols; cidx += 256) {
      double *col = A + (size_t)cidx * ld;
      double s = 0.0;
      for (int i = j; i < rows; i++)
        s += vbuf[i] * col[i];
      s *= beta;
      for (int i = j; i < rows; i++)
        col[i] -= s * vbuf[i];
    }
    __syncthreads();
  }
}


} // namespace ovp

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

template <int TILE, bool GA, bool GB> static void launch_gemm_kernel(Ctx *c, const GemmBatch &b, dim3 grid, int nchunk, int kc) {
  const size_t smem = gemm_smem_bytes<TILE>(GA, GB, kc);
  if (smem > 48 * 1024) // the 64-wide tile's stages, or a long gather-index slice: opt in to more than the default 48 KB
    cudaFuncSetAttribute(gemm_f64_kernel<TILE, GA, GB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(128);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = c->stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 1;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = nchunk; // the chunks of one output tile
  cfg.attrs = &attr;
  cfg.numAttrs = nchunk > 1 ? 1 : 0;
  cudaLaunchKernelEx(&cfg, gemm_f64_kernel<TILE, GA, GB>, b, nchunk, kc);
}
template <int TILE> static void launch_gemm_tile(Ctx *c, const GemmBatch &b, dim3 grid, int nchunk, int kc) {
  const bool ga = b.p[0].A.kidx != nullptr, gb = b.p[0].B.kidx != nullptr;
  if (ga && gb)
    launch_gemm_kernel<TILE, true, true>(c, b, grid, nchunk, kc);
  else if (ga)
    launch_gemm_kernel<TILE, true, false>(c, b, grid, nchunk, kc);
  else if (gb)
    launch_gemm_kernel<TILE, false, true>(c, b, grid, nchunk, kc);
  else
    launch_gemm_kernel<TILE, false, false>(c, b, grid, nchunk, kc);
}

// Shortest k chunk of a split launch: 8 k-steps of 16.  On an H100, chunks of 64 (up to 8 per tile) made the benchmark step slower than
// chunks of 128 (up to 4): more CTAs, half of them dead under ktri, and twice the reduction traffic for the same k walk (DESIGN.md §9).
static constexpr int kGemmMinChunk = 128;

int gemm_plan(const Ctx *c, const GemmBatch &b, int tile, int *nchunk, int *kc) {
  long long tiles64 = 0, tiles = 0;
  int K = 0;
  bool nosplit = false;
  for (int i = 0; i < b.n; i++) {
    int a = (b.p[i].M + 63) / 64, bb = (b.p[i].N + 63) / 64;
    tiles64 += (b.p[i].tri == TRI_FULL) ? (long long)a * bb : (long long)a * (a + 1) / 2;
    K = std::max(K, b.p[i].K);
    nosplit |= b.p[i].nosplit != 0;
  }
  if (tile != 32 && tile != 64) // below one wave of 64-wide tiles, 32-wide ones give more CTAs to hide the k-loop latency
    tile = tiles64 >= c->num_sms ? 64 : 32;
  for (int i = 0; i < b.n; i++) {
    int a = (b.p[i].M + tile - 1) / tile, bb = (b.p[i].N + tile - 1) / tile;
    tiles += (b.p[i].tri == TRI_FULL) ? (long long)a * bb : (long long)a * (a + 1) / 2;
  }
  // Split k when the tiles alone are less than two waves and K is longer than one chunk: up to OVP_GSPLIT_MAX chunks of at least
  // kGemmMinChunk, kc rounded up to the k-step.  Only the shapes, the tile width and the SM count enter, so a product always sums
  // in the same order (auto and forced tile widths included).
  int n = 1;
  if (!nosplit && tiles < 2LL * c->num_sms && K > kGemmMinChunk)
    n = std::min(OVP_GSPLIT_MAX, (K + kGemmMinChunk - 1) / kGemmMinChunk);
  int len = ((K + n - 1) / n + OVP_GK - 1) / OVP_GK * OVP_GK;
  len = std::max(len, OVP_GK);
  *kc = len;
  *nchunk = std::max(1, (K + len - 1) / len);
  return tile;
}

int launch_gemm(Ctx *c, const GemmBatch &b, int tile) {
  int tm = 0, tn = 0;
  double work = 0;
  for (int i = 0; i < b.n; i++) {
    tm = std::max(tm, (b.p[i].M + 63) / 64);
    tn = std::max(tn, (b.p[i].N + 63) / 64);
    work += (b.p[i].tri == TRI_FULL ? 2.0 : 1.0) * (double)b.p[i].M * b.p[i].N * b.p[i].K;
  }
  if (tm == 0 || tn == 0 || b.n == 0)
    return 0;
  int nchunk = 1, kc = OVP_GK;
  tile = gemm_plan(c, b, tile, &nchunk, &kc);
  prof_begin(c, PROF_GEMM, work);
  if (tile == 64) {
    launch_gemm_tile<64>(c, b, dim3(tn, tm, b.n * nchunk), nchunk, kc);
  } else { // fewer 64-tiles than SMs: 32-tiles quadruple the CTA count and quarter the per-CTA tensor work
    int tm32 = 0, tn32 = 0;
    for (int i = 0; i < b.n; i++) {
      tm32 = std::max(tm32, (b.p[i].M + 31) / 32);
      tn32 = std::max(tn32, (b.p[i].N + 31) / 32);
    }
    launch_gemm_tile<32>(c, b, dim3(tn32, tm32, b.n * nchunk), nchunk, kc);
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
// of the fused kernel (cholfused.cu), or its panels when the system is wider (cholpanel.cu).  Pivots <= tol * original diagonal are
// treated as exact zeros (rank-deficient Gram matrices).
int chol_partial(Ctx *c, double *A, int ld, int n, int npiv, double tol) {
  return chol_factor(c, A, ld, n, npiv, tol, nullptr, 0, 0, nullptr, 1, nullptr, 0, nullptr, -1.0, nullptr, nullptr);
}

// stand-alone Householder left-nullspace projection on a global-memory matrix (col-major, ld): reflectors from the first
// nref columns applied to all ncols columns.  One CTA, any number of rows: the reflector v = [v0; A(j+1:, j)] is read from
// column j itself (only v0 is kept in shared memory), and column j becomes [alpha; 0] once every trailing column has been reflected.
__global__ void __launch_bounds__(256) householder_cols_kernel(double *A, int ld, int rows, int ncols, int nref) {
  __shared__ double s_v0, s_beta;
  const int tid = threadIdx.x;
  for (int j = 0; j < nref; j++) {
    double *vcol = A + (size_t)j * ld;
    double alpha = 0.0, nrm = 0.0;
    if (tid < 32) {
      double s = 0.0;
      for (int i = j + tid; i < rows; i += 32) {
        double v = vcol[i];
        s += v * v;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        s += __shfl_xor_sync(0xffffffffu, s, o);
      double x0 = vcol[j];
      nrm = sqrt(s);
      alpha = (x0 > 0.0) ? -nrm : nrm;
      double v0 = x0 - alpha;
      double vtv = s - x0 * x0 + v0 * v0;
      if (tid == 0) {
        s_v0 = v0;
        s_beta = (vtv > 0.0 && nrm > 0.0) ? 2.0 / vtv : 0.0;
      }
    }
    __syncthreads();
    const double beta = s_beta, v0 = s_v0;
    for (int cidx = j + 1 + tid; cidx < ncols; cidx += 256) {
      double *col = A + (size_t)cidx * ld;
      double s = 0.0;
      s += v0 * col[j];
      for (int i = j + 1; i < rows; i++)
        s += vcol[i] * col[i];
      s *= beta;
      col[j] -= s * v0;
      for (int i = j + 1; i < rows; i++)
        col[i] -= s * vcol[i];
    }
    __syncthreads(); // every trailing column has read v: the reflected column itself becomes [alpha; 0]
    if (tid < 32 && nrm > 0.0)
      for (int i = j + tid; i < rows; i += 32)
        vcol[i] = (i == j) ? alpha : 0.0;
  }
}


} // namespace ovp

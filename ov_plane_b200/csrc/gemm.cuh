// FP64 tensor-core (DMMA, mma.sync.m8n8k4.f64) tile GEMM used by every dense contraction of the path:
// M = P[:,ids] H^T, S = H M[ids,:] + R, the Cholesky trailing updates, the triangular-inverse merges, Y = M L^-T and
// P -= Y Y^T (StateHelper.cpp:142-171 restructured, see DESIGN.md).  wgmma has no f64 kind, and the path needs fp64
// (DESIGN.md "precision"), so the fp64 tensor-core work goes through warp-level mma.sync.  This kernel uses the m8n8k4 shape; sm_90
// also has the f64 shapes m16n8k4 / m16n8k8 / m16n8k16, each a single DMMA instruction.  Measured on an H100 80GB HBM3 at a 700 W
// power limit (tools/lab/dmma_lab.cu, one SM): m8n8k4 reaches 127 FP64 flops / cycle with 8 warps, every m16n8 shape 252-255, i.e.
// m8n8k4 runs at HALF the tensor rate; dependent-chain latency 30 / 34 / 50 / 82 cycles for m8n8k4 / k4 / k8 / k16 (7.5 / 8.5 / 6.3 /
// 5.1 cycles per unit of k).  The fused Cholesky (cholfused.cu) runs on m16n8k16; moving this kernel is open.
//
// Operands are strided views (element (i,k) = p[i*si + K(k)*sk], optional gather K(k) = kidx[k] along the contraction
// dimension) so that transposes and the P[:, ids] / M[ids, :] gathers of EKFUpdate need no copies and no divergent code.  A CTA
// stages its slice of each gather index in shared memory once, then streams the operand tiles through a 3-stage cp.async pipeline
// (16-byte copies along a contiguous direction, 8-byte copies for gathered elements), so no operand load waits on an index load.
// When the output tiles alone would leave the SMs idle, the launcher splits k into fixed chunks, one CTA per chunk; the CTAs of a
// tile form a thread-block cluster and reduce their partial tiles over distributed shared memory in chunk order (see the kernel).
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ovp {
namespace cg = cooperative_groups;

// Address of a shared-memory array, pinned in a register.  nvcc 12.9 may treat the address of every shared array (static, and
// the dynamic block) as a constant it may REMATERIALISE at each use as (SR_CgaCtaId << 24) + offset: one S2R (tens of cycles, and the
// consumer waits on it) in front of every inner loop that touches shared memory.  The opaque asm stops that; going through
// shared -> generic keeps the address space known, so accesses through the returned pointer are still LDS / STS.
template <typename T> __device__ __forceinline__ T *pin_shared(T *p) {
  unsigned a = (unsigned)__cvta_generic_to_shared(p);
  asm volatile("" : "+r"(a));
  return (T *)__cvta_shared_to_generic((size_t)a);
}

__device__ __forceinline__ void dmma_m8n8k4(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}
// c += A B, A 16 x 16, B 16 x 8 (one DMMA.16x8x16).  With g = lane / 4, t = lane % 4:
//   a[i] = A(g + 8 (i & 1), t + 4 (i >> 1)),   b[i] = B(t + 4 i, g),   c[i] = C(g + 8 (i >> 1), 2 t + (i & 1))
__device__ __forceinline__ void dmma_m16n8k16(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// Host-side logical matrix view: element (i,j) = p[row(i) + col(j)*ld] (after optional transpose), optional gather indices.
struct MatView {
  const double *p;
  int ld;
  const int *ridx; // physical row index per logical row (nullptr = identity)
  const int *cidx; // physical col index per logical col (nullptr = identity)
  int trans;       // 1: logical (i,j) reads physical (j,i)
  __device__ __forceinline__ double at(int i, int j) const {
    if (trans) {
      int t = i;
      i = j;
      j = t;
    }
    int r = ridx ? ridx[i] : i;
    int c = cidx ? cidx[j] : j;
    return p[(size_t)c * (size_t)ld + (size_t)r];
  }
};
inline MatView mv(const double *p, int ld, int trans = 0, const int *ridx = nullptr, const int *cidx = nullptr) {
  MatView v;
  v.p = p;
  v.ld = ld;
  v.ridx = ridx;
  v.cidx = cidx;
  v.trans = trans;
  return v;
}

// Device-side strided operand: element (x, k) = p[x * sx + K(k) * sk]   (x = row of A or column of B)
struct SView {
  const double *p;
  long long sx, sk;
  const int *kidx;
};

enum { TRI_FULL = 0, TRI_LOWER = 1, TRI_LOWER_MIRROR = 2 };

// C[i + j*ldc] = alpha * sum_k A(i,k) B(k,j) + beta * C + (i==j ? diag_add[i] or diag_const : 0)
struct GemmProblem {
  int M, N, K;
  SView A; // M x K
  SView B; // K x N (x = column j)
  double *C;
  int ldc;
  double alpha, beta;
  const double *diag_add; // optional, length >= min(M,N)
  double diag_const;
  int tri;     // TRI_*: LOWER computes tiles with tile_row >= tile_col only; MIRROR additionally writes C(j,i)
  int a_kfast; // 1: A is contiguous along k in memory (tile loader walks k fastest)
  int b_kfast;
  int ktri;    // structural zeros along k: 1 = B(k, j) == 0 for k < j (B lower trapezoidal: a Cholesky factor used as H^T), 2 = A(i, k) == 0
               // for k < i (its transpose on the left).  A tile starts its k loop at its own first column / row instead of 0: the skipped
               // products are exact zeros, so the result is bit-identical and M = P[:, ids] L, S = L^T M[ids, :] cost half / a third.
  int nosplit; // 1: the launcher never splits k for this product (one chunk), whatever its shape
};
#define OVP_GEMM_MAX_BATCH 8
struct GemmBatch {
  GemmProblem p[OVP_GEMM_MAX_BATCH];
  int n;
  const int *flag; // optional device flag: when non-null and *flag == 0 the whole launch is a no-op
};

#define OVP_GT 64  // large tile edge
#define OVP_GK 16  // k step
#define OVP_GLD 68 // smem leading dim of the 64-tile (68 mod 16 == 4: conflict-free DMMA fragment reads)
#define OVP_GSTAGES 3   // cp.async stages of the operand pipeline
#define OVP_GSPLIT_MAX 8 // k chunks per tile at most: one thread-block cluster of the portable size

// Staging layout in shared memory: element (k, x) at k * sk + x * sx.  An operand walked x-fastest is stored [k][x] (sk = TILE + 4,
// sx = 1); one walked k-fastest (k contiguous in global memory) is stored [x][k] with stride 20 (sk = 1, sx = 20): either way the
// DMMA fragment reads (8 x, 4 k) fall on 16 distinct 8-byte banks (TILE + 4 and 20 are 4 mod 16).
#define OVP_GKS 20
// doubles of one operand's stage buffer
template <int TILE> __host__ __device__ constexpr int gemm_stage_doubles() {
  return (OVP_GK * (TILE + 4) > TILE * OVP_GKS) ? OVP_GK * (TILE + 4) : TILE * OVP_GKS;
}
// dynamic shared memory of one CTA: the operand stages, then the CTA's slice of each gather index (kc ints per gathered operand).  The
// partial tile of a split launch (TILE x (TILE + 4) doubles) reuses the stages.
template <int TILE> inline size_t gemm_smem_bytes(bool ga, bool gb, int kc) {
  return (size_t)2 * OVP_GSTAGES * gemm_stage_doubles<TILE>() * sizeof(double) + ((ga ? 1 : 0) + (gb ? 1 : 0)) * (size_t)kc * sizeof(int);
}

// cp.async copies global -> shared that bypass the registers; a copy whose source size is 0 (or 8 of 16) zero-fills the rest
__device__ __forceinline__ void cp_async8(double *dst, const double *src, bool ok) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src), "r"(ok ? 8 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async16(double *dst, const double *src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// One operand's TILE x 16 block of the k-step [k0, k0 + 16) into a stage buffer: TILE / 16 element pairs per thread, each pair along
// the operand's contiguous direction (k for a k-fastest operand, x otherwise), so a warp reads whole 128- or 256-byte segments.  A
// pair is one 16-byte copy when it is contiguous and aligned in global memory (vec), else two 8-byte copies; a gathered k-fastest
// operand is always copied element by element.  Gather indices come from the CTA's slice in shared memory (sidx[k - klo]), so no
// copy waits on an index load.  Elements outside [0, X) x [k0, khi) are zero-filled.
template <int TILE, bool GATHER>
__device__ __forceinline__ void issue_tile(double *sm, const SView &v, const int *sidx, int x0, int X, int k0, int klo, int khi, int kfast,
                                           bool vec, int tid) {
#pragma unroll
  for (int t = 0; t < TILE / 16; t++) {
    const int q = tid + 128 * t;
    if (kfast) { // (x, k), (x, k + 1), stored [x][k]
      const int xx = q >> 3, kk = 2 * (q & 7);
      const int gx = x0 + xx, gk = k0 + kk;
      const bool ok0 = gx < X && gk < khi, ok1 = gx < X && gk + 1 < khi;
      double *d = sm + xx * OVP_GKS + kk;
      const double *row = v.p + (long long)gx * v.sx;
      if (GATHER) {
        cp_async8(d, ok0 ? row + (long long)sidx[gk - klo] * v.sk : v.p, ok0);
        cp_async8(d + 1, ok1 ? row + (long long)sidx[gk + 1 - klo] * v.sk : v.p, ok1);
      } else if (vec) {
        cp_async16(d, ok0 ? row + gk : v.p, ok0 ? (ok1 ? 16 : 8) : 0);
      } else {
        cp_async8(d, ok0 ? row + (long long)gk * v.sk : v.p, ok0);
        cp_async8(d + 1, ok1 ? row + (long long)(gk + 1) * v.sk : v.p, ok1);
      }
    } else { // (x, k), (x + 1, k), stored [k][x]
      const int xx = 2 * (q % (TILE / 2)), kk = q / (TILE / 2);
      const int gx = x0 + xx, gk = k0 + kk;
      const bool okk = gk < khi, ok0 = okk && gx < X, ok1 = okk && gx + 1 < X;
      double *d = sm + kk * (TILE + 4) + xx;
      const long long kp = GATHER ? (okk ? (long long)sidx[gk - klo] : 0) : gk;
      const double *col = v.p + kp * v.sk + (long long)gx * v.sx;
      if (vec) {
        cp_async16(d, ok0 ? col : v.p, ok0 ? (ok1 ? 16 : 8) : 0);
      } else {
        cp_async8(d, ok0 ? col : v.p, ok0);
        cp_async8(d + 1, ok1 ? col + v.sx : v.p, ok1);
      }
    }
  }
}
// 16-byte copies need the pair contiguous (unit stride along the copy direction) and every pair start 16-byte aligned
__device__ __forceinline__ bool gemm_vec_ok(const SView &v, int kfast, bool gather) {
  if (((unsigned long long)v.p & 15) != 0)
    return false;
  return kfast ? (!gather && v.sk == 1 && (v.sx & 1) == 0) : (v.sx == 1 && (v.sk & 1) == 0);
}

// one element of the result: v = alpha * sum + beta * C0, plus the diagonal term, stored as tri asks
__device__ __forceinline__ void gemm_store(const GemmProblem &pb, int gi, int gj, double v) {
  if (gi == gj)
    v += pb.diag_add ? pb.diag_add[gi] : pb.diag_const;
  double *Cp = pb.C;
  if (pb.tri == TRI_FULL) {
    Cp[(size_t)gj * pb.ldc + gi] = v;
  } else if (gi >= gj) { // lower part of the (diagonal) tile
    Cp[(size_t)gj * pb.ldc + gi] = v;
    if (pb.tri == TRI_LOWER_MIRROR && gi != gj && gi < pb.N && gj < pb.M)
      Cp[(size_t)gi * pb.ldc + gj] = v;
  }
}

// TILE = 64: 4 warps x (32x32) ; TILE = 32: 4 warps x (16x16) — the small tile spreads mid-size problems over all SMs.
//
// Split k.  The k range is cut into nchunk chunks at fixed, absolute boundaries: chunk c is [c kc, min(K, (c + 1) kc)), kc a multiple of
// 16.  blockIdx.z = problem * nchunk + c, and the nchunk CTAs of one output tile form one thread-block cluster (launched with cluster
// dims (1, 1, nchunk)).  Each CTA sums its chunk into a partial tile in its own shared memory; after a cluster barrier, CTA r reduces
// the r-th slice of the tile by reading every live chunk's partial over distributed shared memory in chunk order, and applies the
// epilogue (alpha, beta C, the diagonal, tri and the mirror) once.  A second cluster barrier keeps every CTA's shared memory alive until
// its peers have read it.  No global workspace, no counters: a launch leaves no state behind, so graph replays and concurrent contexts
// need nothing reset.  A chunk is live when it meets the tile's [kbeg, K) range (ktri); a CTA whose chunk is dead skips the k walk and
// only takes part in the barriers and the reduction.  Every accumulator starts at +0 and DMMA never turns +0 into -0, so a skipped chunk
// or k-step is exactly the +0 it would have added: ktri = 1 / 2 is bit-identical to ktri = 0, because the boundaries do not move with
// ktri.  nchunk = 1 (kc >= K) is the single-pass walk: no cluster, the epilogue straight from the registers.
template <int TILE, bool GA, bool GB> __global__ void __launch_bounds__(128) gemm_f64_kernel(GemmBatch batch, int nchunk, int kc) {
  if (batch.flag && *batch.flag == 0)
    return;
  const int chunk = blockIdx.z % nchunk;
  const GemmProblem &pb = batch.p[blockIdx.z / nchunk];
  const int tm = blockIdx.y, tn = blockIdx.x;
  // the tests below are the same for every CTA of a cluster: a cluster runs or returns as a whole
  if (tm * TILE >= pb.M || tn * TILE >= pb.N)
    return;
  if (pb.tri != TRI_FULL && tm < tn)
    return;
  constexpr int WT = TILE / 2; // warp tile edge
  constexpr int NM = WT / 8;   // mma tiles per warp per dimension
  constexpr int SMT = gemm_stage_doubles<TILE>();
  extern __shared__ __align__(16) double ovp_gemm_smem[];
  double *const sm = pin_shared(ovp_gemm_smem);
  int *const sidx_a = (int *)(sm + 2 * OVP_GSTAGES * SMT);
  int *const sidx_b = sidx_a + (GA ? kc : 0);
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1;
  const int m0 = tm * TILE, n0 = tn * TILE;
  const int M = pb.M, N = pb.N, K = pb.K;
  const SView va = pb.A, vb = pb.B;
  const int akf = pb.a_kfast, bkf = pb.b_kfast;
  const bool avec = gemm_vec_ok(va, akf, GA), bvec = gemm_vec_ok(vb, bkf, GB);
  const int ask = akf ? 1 : TILE + 4, asx = akf ? OVP_GKS : 1, bsk = bkf ? 1 : TILE + 4, bsx = bkf ? OVP_GKS : 1;
  const int kbeg = (pb.ktri == 1) ? (n0 & ~(OVP_GK - 1)) : ((pb.ktri == 2) ? (m0 & ~(OVP_GK - 1)) : 0);
  const int klo = max(chunk * kc, kbeg), khi = min(K, chunk * kc + kc);
  const int nsteps = klo < khi ? (khi - klo + OVP_GK - 1) / OVP_GK : 0;
  const double alpha = pb.alpha, beta = pb.beta;
  // the CTA's slice of the gather indices, once
  if (GA || GB) {
    for (int k = klo + tid; k < khi; k += 128) {
      if (GA)
        sidx_a[k - klo] = va.kidx[k];
      if (GB)
        sidx_b[k - klo] = vb.kidx[k];
    }
    __syncthreads();
  }
  double acc[NM][NM][2];
#pragma unroll
  for (int i = 0; i < NM; i++)
#pragma unroll
    for (int j = 0; j < NM; j++)
      acc[i][j][0] = acc[i][j][1] = 0.0;
  // OVP_GSTAGES-deep cp.async pipeline: k-step t + 2 is in flight while t is in the tensor pipe.  One group is committed per k-step
  // (empty past the end) so that wait_group counts stay uniform.
#pragma unroll
  for (int s = 0; s < OVP_GSTAGES - 1; s++) {
    if (s < nsteps) {
      double *st = sm + s * 2 * SMT;
      issue_tile<TILE, GA>(st, va, sidx_a, m0, M, klo + s * OVP_GK, klo, khi, akf, avec, tid);
      issue_tile<TILE, GB>(st + SMT, vb, sidx_b, n0, N, klo + s * OVP_GK, klo, khi, bkf, bvec, tid);
    }
    cp_async_commit();
  }
  int rd = 0, wr = OVP_GSTAGES - 1; // stage read at this k-step, stage written by its prefetch
  for (int t = 0; t < nsteps; t++) {
    cp_async_wait<OVP_GSTAGES - 2>();
    __syncthreads(); // stage rd has landed for every thread, and stage wr (read at t - 1) is free
    if (t + OVP_GSTAGES - 1 < nsteps) {
      double *st = sm + wr * 2 * SMT;
      const int k0 = klo + (t + OVP_GSTAGES - 1) * OVP_GK;
      issue_tile<TILE, GA>(st, va, sidx_a, m0, M, k0, klo, khi, akf, avec, tid);
      issue_tile<TILE, GB>(st + SMT, vb, sidx_b, n0, N, k0, klo, khi, bkf, bvec, tid);
    }
    cp_async_commit();
    const double *As = sm + rd * 2 * SMT, *Bs = As + SMT;
#pragma unroll
    for (int kk = 0; kk < OVP_GK; kk += 4) {
      double a[NM], b[NM];
#pragma unroll
      for (int i = 0; i < NM; i++)
        a[i] = As[(kk + (lane & 3)) * ask + (wm * WT + i * 8 + (lane >> 2)) * asx];
#pragma unroll
      for (int j = 0; j < NM; j++)
        b[j] = Bs[(kk + (lane & 3)) * bsk + (wn * WT + j * 8 + (lane >> 2)) * bsx];
#pragma unroll
      for (int i = 0; i < NM; i++)
#pragma unroll
        for (int j = 0; j < NM; j++)
          dmma_m8n8k4(acc[i][j][0], acc[i][j][1], a[i], b[j]);
    }
    rd = rd == OVP_GSTAGES - 1 ? 0 : rd + 1;
    wr = wr == OVP_GSTAGES - 1 ? 0 : wr + 1;
  }
  cp_async_wait<0>();
  if (nchunk == 1) {
#pragma unroll
    for (int i = 0; i < NM; i++)
#pragma unroll
      for (int j = 0; j < NM; j++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
          int gi = m0 + wm * WT + i * 8 + (lane >> 2);
          int gj = n0 + wn * WT + j * 8 + (lane & 3) * 2 + h;
          if (gi < M && gj < N) {
            const double c0 = (beta != 0.0) ? pb.C[(size_t)gj * pb.ldc + gi] : 0.0;
            gemm_store(pb, gi, gj, alpha * acc[i][j][h] + beta * c0);
          }
        }
    return;
  }
  // split: the partial tile, column-major with leading dimension TILE + 4 (4 mod 16: the fragment stores of a warp take 2 wavefronts)
  constexpr int PLD = TILE + 4;
  __syncthreads(); // every warp is done with the stages the partial overwrites
#pragma unroll
  for (int i = 0; i < NM; i++)
#pragma unroll
    for (int j = 0; j < NM; j++)
#pragma unroll
      for (int h = 0; h < 2; h++)
        sm[(wn * WT + j * 8 + (lane & 3) * 2 + h) * PLD + wm * WT + i * 8 + (lane >> 2)] = acc[i][j][h];
  cg::cluster_group cluster = cg::this_cluster();
  cluster.sync(); // partials written and visible cluster-wide
  constexpr int E = TILE * TILE;
  const int per = (E + nchunk - 1) / nchunk, e1 = min(E, (chunk + 1) * per);
  for (int e = chunk * per + tid; e < e1; e += 128) {
    const int ii = e % TILE, jj = e / TILE;
    const int gi = m0 + ii, gj = n0 + jj;
    const bool out = gi < M && gj < N && (pb.tri == TRI_FULL || gi >= gj);
    const double c0 = (out && beta != 0.0) ? pb.C[(size_t)gj * pb.ldc + gi] : 0.0;
    double s = 0.0;
    for (int c = 0; c < nchunk; c++)
      if (max(c * kc, kbeg) < min(K, c * kc + kc)) // live chunks only, in chunk order
        s += cluster.map_shared_rank(sm, c)[jj * PLD + ii];
    if (out)
      gemm_store(pb, gi, gj, alpha * s + beta * c0);
  }
  cluster.sync(); // no CTA leaves while a peer may still read its partial
}

// A: logical M x K view; gathers are supported along K only
inline SView sview_A(const MatView &v) {
  SView s;
  s.p = v.p;
  if (!v.trans) {
    s.sx = 1;
    s.sk = v.ld;
    s.kidx = v.cidx;
  } else {
    s.sx = v.ld;
    s.sk = 1;
    s.kidx = v.ridx;
  }
  return s;
}
// B: logical K x N view
inline SView sview_B(const MatView &v) {
  SView s;
  s.p = v.p;
  if (!v.trans) {
    s.sk = 1;
    s.sx = v.ld;
    s.kidx = v.ridx;
  } else {
    s.sx = 1;
    s.sk = v.ld;
    s.kidx = v.cidx;
  }
  return s;
}

inline GemmProblem make_problem(int M, int N, int K, MatView A, MatView B, double *C, int ldc, double alpha = 1.0, double beta = 0.0) {
  GemmProblem p;
  p.M = M;
  p.N = N;
  p.K = K;
  p.A = sview_A(A);
  p.B = sview_B(B);
  p.C = C;
  p.ldc = ldc;
  p.alpha = alpha;
  p.beta = beta;
  p.diag_add = nullptr;
  p.diag_const = 0.0;
  p.tri = TRI_FULL;
  p.ktri = 0;
  p.nosplit = 0;
  // loader walk: along whichever logical direction is contiguous in memory
  p.a_kfast = (p.A.sk == 1) ? 1 : 0;
  p.b_kfast = (p.B.sk == 1) ? 1 : 0;
  return p;
}

} // namespace ovp

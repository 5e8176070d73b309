// FP64 tensor-core shapes on one SM: mma.sync m8n8k4, m16n8k4, m16n8k8 and m16n8k16 (.f64), timed with clock64 inside the kernel.
//   layout     : one product per shape against a host reference (the fragment layouts below are the ones csrc/cholfused.cu uses)
//   latency    : one warp, a chain of dependent instructions (each accumulates onto the previous result): cycles per instruction,
//                and per unit of k (what a dependent k chain of one output tile costs)
//   throughput : 8 warps of one CTA, 8 independent accumulators each: FP64 flops per cycle per SM
//   fragments  : shared-memory reads of A fragments (row g [+8], column t [+4i]) from a column-major tile with a leading dimension of 68
//                (csrc/cholfused.cu CF_LD) against 64 (every quarter warp on the same banks)
// Prints the card name, its power limit and its SM clocks first.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dmma_lab dmma_lab.cu
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

// ---- the four shapes: A fragment a[NA], B fragment b[NB], accumulator c[NC] --------------------------------------------------------
// m8n8k4  : a (g, t)                          b (k t, col g)                         c (g, 2t + h)
// m16n8kK : a[i] (g + 8 (i & 1), t + 4 (i >> 1)) b[i] (k t + 4 i, col g)               c[i] (g + 8 (i >> 1), 2t + (i & 1))
template <int SH> struct Shape;
template <> struct Shape<0> {
  static constexpr int M = 8, N = 8, K = 4, NA = 1, NB = 1, NC = 2;
  static constexpr const char *name = "m8n8k4";
  static __device__ __forceinline__ void mma(double (&c)[NC], const double (&a)[NA], const double (&b)[NB]) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
  }
};
template <> struct Shape<1> {
  static constexpr int M = 16, N = 8, K = 4, NA = 2, NB = 1, NC = 4;
  static constexpr const char *name = "m16n8k4";
  static __device__ __forceinline__ void mma(double (&c)[NC], const double (&a)[NA], const double (&b)[NB]) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(b[0]));
  }
};
template <> struct Shape<2> {
  static constexpr int M = 16, N = 8, K = 8, NA = 4, NB = 2, NC = 4;
  static constexpr const char *name = "m16n8k8";
  static __device__ __forceinline__ void mma(double (&c)[NC], const double (&a)[NA], const double (&b)[NB]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
  }
};
template <> struct Shape<3> {
  static constexpr int M = 16, N = 8, K = 16, NA = 8, NB = 4, NC = 4;
  static constexpr const char *name = "m16n8k16";
  static __device__ __forceinline__ void mma(double (&c)[NC], const double (&a)[NA], const double (&b)[NB]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
                 "{%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]),
                   "d"(b[3]));
  }
};
template <int SH> __device__ __forceinline__ int a_row(int i, int g) { return Shape<SH>::M == 8 ? g : g + 8 * (i & 1); }
template <int SH> __device__ __forceinline__ int a_col(int i, int t) { return Shape<SH>::M == 8 ? t : t + 4 * (i >> 1); }
template <int SH> __device__ __forceinline__ int c_row(int i, int g) { return Shape<SH>::M == 8 ? g : g + 8 * (i >> 1); }

// C (M x N, row-major) = A (M x K, row-major) B (K x N, row-major), one warp
template <int SH> __global__ void layout(const double *A, const double *B, double *C) {
  using S = Shape<SH>;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  double a[S::NA], b[S::NB], c[S::NC];
  for (int i = 0; i < S::NA; i++)
    a[i] = A[a_row<SH>(i, g) * S::K + a_col<SH>(i, t)];
  for (int i = 0; i < S::NB; i++)
    b[i] = B[(t + 4 * i) * S::N + g];
  for (int i = 0; i < S::NC; i++)
    c[i] = 0.0;
  S::mma(c, a, b);
  for (int i = 0; i < S::NC; i++)
    C[c_row<SH>(i, g) * S::N + 2 * t + (i & 1)] = c[i];
}

// nacc independent accumulators per warp, iters instructions on each; the first nwarps warps run, clock64 around the loop
template <int SH, int NACC> __global__ void __launch_bounds__(256, 1) timed(double *out, long long *cyc, int iters, int nwarps) {
  using S = Shape<SH>;
  const int warp = threadIdx.x >> 5;
  double a[S::NA], b[S::NB], c[NACC][S::NC];
  for (int i = 0; i < S::NA; i++)
    a[i] = 1e-3 * (threadIdx.x + i);
  for (int i = 0; i < S::NB; i++)
    b[i] = 1e-3 * (threadIdx.x - i);
  for (int q = 0; q < NACC; q++)
    for (int i = 0; i < S::NC; i++)
      c[q][i] = q;
  __syncthreads();
  long long t0 = 0;
  if (warp < nwarps) {
    t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < iters; it++)
#pragma unroll
      for (int q = 0; q < NACC; q++)
        S::mma(c[q], a, b);
  }
  double s = 0.0;
  for (int q = 0; q < NACC; q++)
    for (int i = 0; i < S::NC; i++)
      s += c[q][i];
  const long long t1 = clock64();
  if (warp < nwarps && (threadIdx.x & 31) == 0)
    cyc[warp] = t1 - t0;
  out[threadIdx.x] = s;
}

// 8 warps read A fragments (row g [+8], column t [+4i]) of a column-major 64 x 64 tile with leading dimension LD, reps times
template <int LD> __global__ void __launch_bounds__(256, 1) frag(double *out, long long *cyc, int reps) {
  extern __shared__ double sm[];
  for (int i = threadIdx.x; i < 64 * LD; i += 256)
    sm[i] = 1e-3 * i;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  const unsigned base = (unsigned)__cvta_generic_to_shared(sm + t * LD + 8 * (warp & 1) + g);
  double s = 0.0;
  const long long t0 = clock64();
#pragma unroll 1
  for (int r = 0; r < reps; r++)
#pragma unroll
    for (int i = 0; i < 16; i++) { // 16 reads per lane: k = 0..63 in steps of 4
      double v;
      asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(base + 8u * (4 * i * LD + (unsigned)(r & 1) * 16)));
      s += v;
    }
  const long long t1 = clock64();
  if (lane == 0)
    cyc[warp] = t1 - t0;
  out[threadIdx.x] = s;
}

#define CK(x)                                                                                                                      \
  do {                                                                                                                             \
    cudaError_t e_ = (x);                                                                                                          \
    if (e_ != cudaSuccess) {                                                                                                       \
      printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__);                                                    \
      exit(1);                                                                                                                     \
    }                                                                                                                              \
  } while (0)

static double *d_out;
static long long *d_cyc;

template <int SH> bool check_layout() {
  using S = Shape<SH>;
  double hA[16 * 16], hB[16 * 8], hC[16 * 8], ref[16 * 8];
  for (int i = 0; i < S::M * S::K; i++)
    hA[i] = (double)((i * 37) % 101) / 7.0 - 5.0;
  for (int i = 0; i < S::K * S::N; i++)
    hB[i] = (double)((i * 53) % 89) / 11.0 - 3.0;
  double *dA, *dB, *dC;
  CK(cudaMalloc(&dA, sizeof hA));
  CK(cudaMalloc(&dB, sizeof hB));
  CK(cudaMalloc(&dC, sizeof hC));
  CK(cudaMemcpy(dA, hA, sizeof hA, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dB, hB, sizeof hB, cudaMemcpyHostToDevice));
  layout<SH><<<1, 32>>>(dA, dB, dC);
  CK(cudaMemcpy(hC, dC, sizeof hC, cudaMemcpyDeviceToHost));
  double err = 0.0;
  for (int r = 0; r < S::M; r++)
    for (int c = 0; c < S::N; c++) {
      long double s = 0.0L;
      for (int k = 0; k < S::K; k++)
        s += (long double)hA[r * S::K + k] * hB[k * S::N + c];
      ref[r * S::N + c] = (double)s;
      err = fmax(err, fabs(hC[r * S::N + c] - ref[r * S::N + c]) / (1.0 + fabs(ref[r * S::N + c])));
    }
  CK(cudaFree(dA));
  CK(cudaFree(dB));
  CK(cudaFree(dC));
  printf("layout   %-9s max rel. error vs long double %.2e  %s\n", S::name, err, err < 1e-14 ? "ok" : "WRONG");
  return err < 1e-14;
}

template <int SH> void measure() {
  using S = Shape<SH>;
  const double flops = 2.0 * S::M * S::N * S::K;
  long long h[8];
  // latency: one warp, one accumulator
  const int lat_iters = 4096;
  timed<SH, 1><<<1, 256>>>(d_out, d_cyc, 64, 1); // warm-up
  timed<SH, 1><<<1, 256>>>(d_out, d_cyc, lat_iters, 1);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(h, d_cyc, 8 * sizeof(long long), cudaMemcpyDeviceToHost));
  const double lat = (double)h[0] / lat_iters;
  // throughput: 8 warps x 8 independent accumulators
  const int thr_iters = 1024;
  timed<SH, 8><<<1, 256>>>(d_out, d_cyc, 64, 8);
  timed<SH, 8><<<1, 256>>>(d_out, d_cyc, thr_iters, 8);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(h, d_cyc, 8 * sizeof(long long), cudaMemcpyDeviceToHost));
  long long mx = 0;
  for (int w = 0; w < 8; w++)
    mx = h[w] > mx ? h[w] : mx;
  const double thr = 8.0 * 8.0 * thr_iters * flops / (double)mx;
  // 4 warps (one per SM sub-partition) x 8 accumulators
  timed<SH, 8><<<1, 256>>>(d_out, d_cyc, thr_iters, 4);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(h, d_cyc, 8 * sizeof(long long), cudaMemcpyDeviceToHost));
  mx = 0;
  for (int w = 0; w < 4; w++)
    mx = h[w] > mx ? h[w] : mx;
  const double thr4 = 4.0 * 8.0 * thr_iters * flops / (double)mx;
  printf("%-9s latency %6.1f cycles / instruction, %5.2f cycles per unit of k | throughput 8 warps %6.1f, 4 warps %6.1f "
         "FP64 flops / cycle / SM\n",
         S::name, lat, lat / S::K, thr, thr4);
}

template <int LD> void measure_frag() {
  const int reps = 1024;
  const size_t smem = 64 * LD * sizeof(double);
  CK(cudaFuncSetAttribute(frag<LD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  frag<LD><<<1, 256, smem>>>(d_out, d_cyc, 16);
  frag<LD><<<1, 256, smem>>>(d_out, d_cyc, reps);
  CK(cudaDeviceSynchronize());
  long long h[8];
  CK(cudaMemcpy(h, d_cyc, 8 * sizeof(long long), cudaMemcpyDeviceToHost));
  long long mx = 0;
  for (int w = 0; w < 8; w++)
    mx = h[w] > mx ? h[w] : mx;
  printf("fragment reads, leading dimension %d: %5.2f cycles per warp-wide 8-byte load (8 warps)\n", LD, (double)mx / (reps * 16));
}

int main() {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s, %d SMs\n", prop.name, prop.multiProcessorCount);
  fflush(stdout);
  if (system("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv") != 0)
    printf("(nvidia-smi query failed)\n");
  fflush(stdout);
  CK(cudaMalloc(&d_out, 256 * sizeof(double)));
  CK(cudaMalloc(&d_cyc, 8 * sizeof(long long)));
  bool ok = check_layout<0>() & check_layout<1>() & check_layout<2>() & check_layout<3>();
  measure<0>();
  measure<1>();
  measure<2>();
  measure<3>();
  measure_frag<68>();
  measure_frag<64>();
  CK(cudaFree(d_out));
  CK(cudaFree(d_cyc));
  return ok ? 0 : 1;
}

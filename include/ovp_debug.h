/* TEST / TUNING HOOKS of the H100-native ov_plane hot path — NOT part of the drop-in ABI (include/ovp.h).
 *
 * These entry points exist only in ov_plane_b200/lib/libovp_debug.so (the product sources compiled with -DOVP_DEBUG); the
 * product library libovp.so does not export them.  They let tools/microbench_chol.py time the fused Cholesky, let
 * tests/test_gpu_cholfused.py / tests/test_gpu_gemm.py / tests/test_gpu_gemm_split.py unit-test chol_fused_kernel and the DMMA GEMM against NumPy on arbitrary
 * matrices, and let tests/test_gpu_numerics.py run one batch through both MSCKF feature paths. */
#ifndef OVP_DEBUG_H
#define OVP_DEBUG_H
#include "ovp.h"
#ifdef __cplusplus
extern "C" {
#endif

/* fused Cholesky on a synthetic SPD n x n system (+ mrows x n right-hand side): out[0] = us per (fill + factor), out[1] = us per
 * fill, out[2..] = per-CTA globaltimer stamps of the last run */
int ovp_debug_chol_fused(ovp_ctx *ctx, int n, int mrows, int iters, double *out, int out_cap);
/* factor the lower triangle of a host matrix A (n x n, column-major) over its leading npiv columns with pivot tolerance tol and,
 * when M is given, solve Y = M L^-T (mrows x npiv) and w = L^-1 z */
int ovp_debug_chol_solve(ovp_ctx *ctx, const double *A, int n, int npiv, double tol, const double *M, int mrows, const double *z,
                         double *L_out, double *Y_out, double *w_out);
/* one product C = alpha * A B + beta * C (+ diagonal) through the DMMA GEMM (tests/test_gpu_gemm.py).  Host matrices are column-major:
 * A is a_rows x a_cols, logical A (M x K) = A, or A^T when a_trans; B is b_rows x b_cols, logical B (K x N) = B, or B^T when b_trans.
 * akidx / bkidx (length K, or NULL) gather the contraction index of A / B.  C is ldc x N, updated in place.  diag_add (length
 * min(M, N), or NULL) or diag_const is added on the diagonal.  tri: 0 full, 1 lower tiles, 2 lower mirrored; ktri as GemmProblem::ktri.
 * flag >= 0 places a device flag of that value (0: the launch is a no-op).  tile: 32 or 64 forces the tile width, 0 lets the launcher
 * choose.  info[0] = tile width launched, info[1] = SM count of the device. */
int ovp_debug_gemm(ovp_ctx *ctx, int M, int N, int K, const double *A, int a_rows, int a_cols, int a_trans, const int *akidx, const double *B,
                   int b_rows, int b_cols, int b_trans, const int *bkidx, double *C, int ldc, double alpha, double beta, const double *diag_add,
                   double diag_const, int tri, int ktri, int flag, int tile, int *info);
/* the k split the DMMA GEMM takes for one product of these sizes (tests/test_gpu_gemm_split.py): info[0] = tile width (tile 32 / 64 forces
 * it, 0 lets the launcher choose, as in ovp_debug_gemm), info[1] = chunk count, info[2] = chunk length kc.  Chunk c covers
 * [c kc, min(K, (c + 1) kc)); one chunk is the unsplit k walk. */
int ovp_debug_gemm_split(ovp_ctx *ctx, int M, int N, int K, int tri, int ktri, int tile, int *info);
/* on != 0: every later ovp_msckf_update of this context builds its point and plane systems with the one-block-per-feature kernel and
 * the dense stacked Gram matrix, also when all its tracks fit the warp-per-feature path (at most 32 measurements) */
int ovp_debug_force_dense_features(ovp_ctx *ctx, int on);

#ifdef __cplusplus
}
#endif
#endif

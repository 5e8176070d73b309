/* TEST / TUNING HOOKS of the H100-native ov_plane hot path — NOT part of the drop-in ABI (include/ovp.h).
 *
 * These entry points exist only in ov_plane_b200/lib/libovp_debug.so (the product sources compiled with -DOVP_DEBUG); the
 * product library libovp.so does not export them.  They let tools/microbench_chol.py time the fused Cholesky, let
 * tests/test_gpu_cholfused.py / tests/test_gpu_gemm.py / tests/test_gpu_gemm_split.py unit-test chol_fused_kernel and the DMMA GEMM against NumPy on arbitrary
 * matrices, let tests/test_gpu_numerics.py run one batch through both MSCKF feature paths, let tests/test_gpu_fused_products.py check the
 * update products formed inside the Gram factorisation and run the update both with and without them, let
 * tests/test_gpu_compression.py check the compressed update's Gram matrix, zero-pivot rule and innovation gate element by element, and
 * let tests/test_gpu_feature_gate.py check the per-feature chi2 gates of the MSCKF point and SLAM feature kernels against long-double
 * references on the raw rows those kernels built, and let tests/test_gpu_plane_update_reference.py check the plane updates and plane
 * initialisation, direct and compressed, against long-double references on the plan's raw rows or Gram matrix. */
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
/* ovp_debug_chol_solve with the innovation launch's gate (tests/test_gpu_compression.py): the same launch also forms chi2 = |w|^2
 * (chi2_out) and the gate flag (gate_out: 1 when gate_thresh < 0 or chi2 <= gate_thresh, else 0).  z holds npiv values; the launch
 * reads them with stride 1 (zstride = 1) or in place as a row of a column-major workspace, with the stride of the compressed update
 * (zstride = 0).  chi2_out and gate_out may be NULL. */
int ovp_debug_chol_solve_gated(ovp_ctx *ctx, const double *A, int n, int npiv, double tol, const double *M, int mrows, const double *z,
                               int zstride, double gate_thresh, double *L_out, double *Y_out, double *w_out, double *chi2_out, int *gate_out);
/* ovp_debug_chol_solve_gated through the panelled factorisation of systems wider than one co-resident launch (DESIGN.md 4.1), with a
 * forced panel width (a multiple of 64 up to the co-resident width; anything else: OVP_ERR_BAD_ARGS), so that narrow systems cross panel
 * boundaries (tests/test_gpu_wide_updates.py) */
int ovp_debug_chol_panels(ovp_ctx *ctx, int panel, const double *A, int n, int npiv, double tol, const double *M, int mrows, const double *z,
                          int zstride, double gate_thresh, double *L_out, double *Y_out, double *w_out, double *chi2_out, int *gate_out);
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
 * the dense stacked Gram matrix, also when all its tracks fit the block-sparse path (at most 32 measurements) */
int ovp_debug_force_dense_features(ovp_ctx *ctx, int on);
/* on != 0: every later compressed update of this context forms M = P[:, cols] L and S = L^T M[cols, :] + I with two GEMM launches after
 * the factorisation of its Gram matrix, instead of inside that factorisation launch */
int ovp_debug_unfused_update_products(ovp_ctx *ctx, int on);
/* on != 0: every later compressed update of this context factors its Gram matrix and its innovation system one after the other, also
 * when the two fit a pair (the innovation factorisation starting while the Gram factorisation runs) */
int ovp_debug_sequential_factorisations(ovp_ctx *ctx, int on);
/* on == 0: every later launch of the update chain (feature kernels, Gram, Gram reduction, the update's tail) waits for the whole of the
 * launch before it, instead of being placed while that launch runs as its programmatic dependent (the default, on != 0).  The results
 * are the same bit for bit.  A changed setting drops the captured graph of the prepared batch. */
int ovp_debug_programmatic_launches(ovp_ctx *ctx, int on);
/* one factorisation of the lower triangle of G ((nc + 1) x (nc + 1), column-major) over its leading npiv columns with pivot tolerance
 * tol, forming the update products in the same launch: with L = rows [0, nc) of the factor, M = P[:, cols] L (N x npiv) and the lower
 * tiles of S = L^T M[cols, :] + I (npiv x npiv; the 64 x 64 tiles on and below the diagonal are written, S_out's other entries are kept).  P is N x N, cols holds nc indices into it.
 * L_out receives the factor's (nc + 1) x npiv columns. */
int ovp_debug_chol_products(ovp_ctx *ctx, const double *G, int nc, int npiv, double tol, const double *P, int N, const int *cols,
                            double *L_out, double *M_out, double *S_out);
/* width > 0: every later factorisation of this context wider than width columns runs in panels of width (width: a multiple of 64 up
 * to the co-resident width of one fused launch; anything else: OVP_ERR_BAD_ARGS), the Gram matrix of a compressed update and its
 * innovation system alike, so that a compressed update forms M and S with two GEMM launches as one wider than a launch does
 * (tests/test_gpu_msckf_point_reference.py).  width = 0 (the default): off.  Whether an update is compressed is still decided on the
 * co-resident width.  A changed setting re-plans the prepared batch and drops its captured graph. */
int ovp_debug_update_panel_width(ovp_ctx *ctx, int width);
/* ovp_debug_chol_products followed by the innovation factorisation of the compressed update, as the update runs them (as a pair when
 * they fit co-resident together and ovp_debug_sequential_factorisations is off, else one after the other): with z = row nc of the Gram
 * factor, S = L_S L_S^T (LS_out: S's lower tiles on input as S_out above, the factor on output), Y = M L_S^-T (Y_out, N x npiv),
 * w = L_S^-1 z (w_out), chi2 = |w|^2 (chi2_out) and the gate (gate_out: 1 when gate_thresh < 0 or chi2 <= gate_thresh).  info[0] = 1 when
 * the pair ran.  timeline (NULL or 64 doubles, debug stamps of the pair, us from the first, -1 where absent): [k] the
 * Gram spine released its diagonal block k, [32 + k] the innovation spine started step k. */
int ovp_debug_chol_pair(ovp_ctx *ctx, const double *G, int nc, int npiv, double tol, const double *P, int N, const int *cols,
                        double gate_thresh, double *L_out, double *M_out, double *LS_out, double *Y_out, double *w_out, double *chi2_out,
                        int *gate_out, int *info, double *timeline);
/* prepare a feature batch as ovp_msckf_update does and run the first non-empty plan of its launch order (planes in ascending id, then the
 * point update) up to its Gram matrix G = [H_o r_o]^T [H_o r_o] of the nullspace-projected system; the state is left as it was.  G_out
 * (gcap * gcap doubles) receives all of G, nc1 x nc1 column-major: the ncx x columns (calibration, then 6 per clone), for a plane its
 * 3 H_cp columns, the residual last.  info[8] = {nc1, ncal, ncx, point plan, nsel, block-sparse path, plane slot, plane in the
 * state}.  cols_out (gcap): state index of every x column; sel_out (F): the nsel features of the plan; feat_status / feat_chi2 (F): the
 * per-feature status words after the plan's feature kernel (point plan: 1 accepted, 0 rejected by the gate).  raw_out (NULL, or 72
 * doubles per measurement of the batch): the raw whitened rows the feature kernel built, per measurement 3 rows of 24 doubles: the two
 * bearing rows [0,3) H_f, [3,9) H_clone, [9, 9 + ncal) calibration, [23] r, then (plane plans) the point-on-plane row [0,3) H_f,
 * [9,12) H_cp, [23] r.  A plan that updates without compression (the direct form) has no Gram matrix: the call stops after that plan's
 * feature kernel, before its update, and returns OVP_OK with info[0] = 0 and info[5] = 0 (the direct form always runs the
 * one-block-per-feature kernel); G_out is left as passed, and raw_out holds the rows the update would have stacked. */
int ovp_debug_msckf_gram(ovp_ctx *ctx, const ovp_feature_batch *b, const ovp_updater_options *opt, int gcap, double *G_out, int *info,
                         int *cols_out, int *sel_out, int *feat_status, double *feat_chi2, double *raw_out);
/* the same for ovp_msckf_update_landmarks: a plane plan's G also holds its landmark members' rows, their 3 columns each after the batch
 * features' x columns (counted in ncx; cols_out gives their state indices) and before H_cp. */
int ovp_debug_msckf_gram_landmarks(ovp_ctx *ctx, const ovp_feature_batch *b, const ovp_plane_landmarks *lm, const ovp_updater_options *opt,
                                   int gcap, double *G_out, int *info, int *cols_out, int *sel_out, int *feat_status, double *feat_chi2,
                                   double *raw_out);
/* ovp_slam_update, which also returns the raw whitened rows the SLAM feature kernel built (tests/test_gpu_feature_gate.py): raw_out (NULL,
 * or 72 doubles per measurement of the batch) in the layout of ovp_debug_msckf_gram, with [0,3) holding the landmark's columns in the
 * bearing rows and in the point-on-plane row.  The update runs as ovp_slam_update runs it. */
int ovp_debug_slam_update(ovp_ctx *ctx, int F, const int *meas_offset, const int *meas_clone, const float *uv, const int64_t *featid,
                          const int64_t *planeid, const ovp_updater_options *opt, int use_plane_constraint, int *feat_status, double *feat_chi2,
                          double *raw_out);
/* ovp_slam_update up to its Gram matrix G = [H r]^T [H r] of the stacked rows (tests/test_gpu_slam_reference.py); nothing after it runs, so
 * the state and its bookkeeping (should_marg, the landmark-to-plane map) are left as they were.  G_out (gcap x gcap doubles) receives G
 * column-major with leading dimension nc1 = nc + 1 (the residual last); info: [0] nc1, [1] the stacked rows the update laid out (its row
 * offsets: 3m per landmark on its plane, 2m otherwise, whatever its status); cols_out (gcap): the state index
 * of every compact column; feat_status / feat_chi2 (F): the per-landmark statuses and chi2; raw_out (NULL, or 72 doubles per measurement):
 * the raw rows, as ovp_debug_slam_update returns them. */
int ovp_debug_slam_gram(ovp_ctx *ctx, int F, const int *meas_offset, const int *meas_clone, const float *uv, const int64_t *featid,
                        const int64_t *planeid, const ovp_updater_options *opt, int use_plane_constraint, int gcap, double *G_out, int *info,
                        int *cols_out, int *feat_status, double *feat_chi2, double *raw_out);
/* the plane tracker's history of each feature of featid[n] (tests/test_gpu_plane_track.py), per feature: A (9, row-major), b (3), count
 * (as a double), has_inG (0 / 1), hist_feat_inG (3), the window length, then OVP_PLANE_TRACK_MAX_NORM_COUNT normals (3 each, oldest first,
 * zero past the length): 18 + 3 * OVP_PLANE_TRACK_MAX_NORM_COUNT doubles.  A feature the tracker does not hold reads as all zeros. */
int ovp_debug_plane_track_history(ovp_ctx *ctx, int n, const int64_t *featid, double *out);

#ifdef __cplusplus
}
#endif
#endif

// Internal declarations of the H100-native ov_plane hot path library (not part of the C ABI).
#pragma once
#include "../../include/ovp.h"
#include "gemm.cuh"
#include <cuda_runtime.h>
#include <deque>
#include <map>
#include <string>
#include <vector>

namespace ovp {

#define OVP_VAL_STRIDE 16 // doubles per variable in the value / fej tables (IMU has 16 values)

struct Var {
  int kind = OVP_KIND_VEC;
  int size = 0;   // error-state size
  int nvalue = 0; // value size
  int id = -1;    // covariance offset, -1 = not in the state
  int64_t tag = 0;
  bool should_marg = false;
  bool alive = true;
  int rep = 0;     // ov_type::LandmarkRepresentation of a SLAM landmark (0 = GLOBAL_3D)
  int anchor = -1; // handle of its anchor clone (anchored representations), anchors.cu
};

struct ImuSample {
  double t;
  double wm[3], am[3];
};

// Workspace for one dense system of up to `cap` rows/cols
struct DenseWs {
  int cap = 0;         // max system size (multiple of 64)
  double *S = nullptr; // cap x cap (Gram / S, factored in place to lower L)
};

struct Ctx {
  int device = 0;
  int num_sms = 0; // SMs of the device: grid sizes of the grid-stride kernels and the tile / split-K choices scale with it
  cudaStream_t stream = nullptr;
  // side stream of the update chain: the covariance downdate P -= Y Y^T (and its negative-diagonal check) of update k runs here while the
  // main stream already applies dx and builds the next update's Jacobians / Gram matrix (which do not read P); joined before the next
  // reader of P.  Fork / join through events, so the pattern is captured into the CUDA graph as parallel branches.
  cudaStream_t stream2 = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool join_pending = false;
  ovp_state_options opt;
  std::string last_error;
  int64_t launches = 0;
  bool use_graphs = true;    // replay the static launch sequence of a prepared batch as a CUDA graph
  double gram_tol = 1e-11;   // zero-pivot rule of the Gram Cholesky, relative to the column's original diagonal (ovp_set_rank_tolerance)
  bool force_dense_features = false; // MSCKF batches take the one-block-per-feature kernel and the dense stack (ovp_debug_force_dense_features)
  bool unfused_update_products = false; // compressed updates form M and S with two GEMM launches (ovp_debug_unfused_update_products)
#ifdef OVP_DEBUG
  // ovp_debug_msckf_gram: the feature kernels write their raw blocks to dbg_raw (when set), and with dbg_gram_stop the MSCKF launch
  // returns right after the first Gram matrix it forms, recording that plan's index in dbg_gram_plan
  double *dbg_raw = nullptr;
  bool dbg_gram_stop = false;
  int dbg_gram_plan = -1;
#endif

  // --- State mirror -------------------------------------------------------------------------------------------
  int Nmax = 0, ldP = 0, N = 0;
  double *dP = nullptr;
  std::vector<Var> vars;          // indexed by handle
  std::deque<int> free_handles;   // slots of marginalised variables, reused FIFO (ekf.cu state_append_variable)
  std::vector<int> order;         // State::_variables (handles)
  std::vector<double> h_val, h_fej; // host mirror, OVP_VAL_STRIDE per handle
  bool host_values_stale = false;   // device values are newer than the host mirror
  double *d_val = nullptr, *d_fej = nullptr;
  int *d_var_id = nullptr, *d_var_size = nullptr, *d_var_kind = nullptr;
  int max_handles = 0;
  bool var_table_dirty = true;
  int h_imu = -1, h_dt = -1, h_calib = -1, h_intr = -1;
  double timestamp = -1;
  std::map<double, int> clones;   // State::_clones_IMU
  std::map<int64_t, int> planes;  // State::_features_PLANE
  std::map<int64_t, int> slam;    // State::_features_SLAM
  std::map<int64_t, int64_t> slam_to_plane;
  std::vector<double> chi2_table;
  double *d_chi2_table = nullptr;
  int chi2_table_n = 0;

  // --- workspaces ---------------------------------------------------------------------------------------------
  int Rcap = 0;                // max dense system size
  DenseWs wsG, wsS;            // compress factor / innovation factor
  double *dM = nullptr, *dY = nullptr; // Nmax x Rcap
  double *dHT = nullptr;       // Rcap x Rcap (H^T operand for generic ekf_update)
  double *dvec = nullptr;      // misc vectors: z, w, dx ... (8 * Rcap), then 2 * Nmax, then the OVP_DX_SPLIT x Nmax partial sums of dx = Y w
  int *dcols = nullptr;        // gather index arrays (8 * Rcap ints)
  int *dflags = nullptr;       // device flags / status words (256 ints)
  double *dscal = nullptr;     // device scalars (256 doubles)
  // fused Cholesky (cholfused.cu): diagonal-block inverses, inter-CTA flags, epoch word
  double *cf_linv = nullptr, *cf_diag0 = nullptr, *cf_xch = nullptr;
  int *cf_flags = nullptr, *cf_ctrl = nullptr;
  int cf_maxT = 0;
  bool cf_attr_set = false;   // per context (= per device): >48 KB dynamic shared memory opt-in of chol_fused_kernel / feature kernels
  int cf_max_coresident = 0;  // co-resident CTA capacity of this device for chol_fused_kernel
  bool feat_smem_set = false;
  int max_meas_rows = 0;
  double *dHs = nullptr;       // stacked [H_x | H_cp | res], max_meas_rows x (Rcap) col-major
  size_t Hs_elems = 0;
  double *dPart = nullptr;     // split-K partials for the Gram kernel
  size_t part_elems = 0;
  // NCCL communicator owned by the context (capi_nccl.inc; libnccl is dlopen'ed on first use, no link-time dependency)
  void *nccl_comm = nullptr;
  int nccl_rank = 0, nccl_nranks = 1;
  double *d_gather = nullptr;  // nranks packed lower triangles
  size_t d_gather_elems = 0;
  double *d_mw = nullptr;      // warp-per-feature path: measurement blocks, per-feature dense blocks, D part (msckf_warp.inc)
  size_t d_mw_elems = 0;
  // feature batch staging
  void *d_batch = nullptr;
  size_t d_batch_bytes = 0;
  void *h_pinned = nullptr;
  size_t h_pinned_bytes = 0;
  // host staging for small dense transfers
  double *d_stage = nullptr;
  size_t d_stage_elems = 0;

  // Propagator
  double sigma_w = 1.6968e-04, sigma_wb = 1.9393e-05, sigma_a = 2.0000e-3, sigma_ab = 3.0000e-03;
  double gravity[3] = {0, 0, 9.81};
  std::vector<ImuSample> imu_data;
  // UpdaterZeroVelocity keeps its own IMU buffer and time-offset memory (UpdaterZeroVelocity.h)
  std::vector<ImuSample> zupt_imu;
  double zupt_last_offset = 0.0, zupt_last_state_timestamp = 0.0;
  bool zupt_have_offset = false;
  double last_prop_time_offset = 0.0;
  bool have_last_prop_time_offset = false;

  // timing
  cudaEvent_t ev[8];
  double last_ms[4] = {0, 0, 0, 0};
  // prepared feature batch (features_host.inc), byte counters of the host<->device copies this ctx issued
  void *prep = nullptr;
  int64_t h2d_bytes = 0, d2h_bytes = 0;
  // snapshot of (P, values, fej) for repeatable benchmarking
  double *snapP = nullptr, *snap_val = nullptr, *snap_fej = nullptr;
  int snapN = -1;
  // per-kernel profiling with CUDA events on the launch stream (bench.py's roofline leg)
  bool profiling = false;
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_used = 0;
  struct ProfRec {
    int id;
    cudaEvent_t e0, e1;
    double work;
  };
  std::vector<ProfRec> prof_recs;
  cudaEvent_t prof_pending = nullptr;
  int prof_pending_id = 0;
  double prof_pending_work = 0;
};
enum { PROF_GEMM = 0, PROF_GRAM = 1, PROF_POTRF = 2, PROF_FEATURE = 3, PROF_OTHER = 4, PROF_N = 5 };
void prof_begin(Ctx *c, int id, double work);
void prof_end(Ctx *c);
int msckf_prepare(Ctx *c, const ovp_feature_batch *b, const ovp_updater_options *opt, const struct MsckfExtra *extra);
int msckf_launch(Ctx *c);
int msckf_finish(Ctx *c, int *feat_status, double *feat_chi2, int *plane_status, double *plane_chi2, int *hx_order, int *hx_order_n);
void free_prepared(Ctx *c);

// error helpers
int fail(Ctx *c, int status, const char *fmt, ...);
#define OVP_CUDA(call)                                                                                                      \
  do {                                                                                                                       \
    cudaError_t e__ = (call);                                                                                                \
    if (e__ != cudaSuccess)                                                                                                  \
      return fail(c, OVP_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));                   \
  } while (0)

// ---- linalg.cu ---------------------------------------------------------------------------------------------------
// The two products of a compressed update, formed inside the factorisation of its Gram matrix (cholfused.cu): with L = rows [0, nc) of
// the factor, M = P[:, cols] L (N x npiv, ld ldm) and the lower tiles of S = L^T M[cols, :] + I (npiv x npiv, ld lds).  ldp is even.
struct CholProducts {
  const double *P;
  const int *cols;
  double *M, *S;
  int ldp, N, nc, ldm, lds;
};
int chol_fused(Ctx *c, double *A, int ld, int n, int npiv, double tol, const double *M, int ldm, int mrows, const double *z, int zstride,
               double *Y, int ldy, double *w, double gate_thresh, double *chi2, int *gate_flag, long long *dbg = nullptr,
               const CholProducts *prod = nullptr);
// every tile CTA of one chol_fused launch must be co-resident: the tile CTAs a factorisation of the leading npiv columns of an n x n
// system needs, how many the device holds, and the widest full factorisation (a multiple of 64) that fits
int chol_fused_tiles(int n, int npiv);
int chol_fused_capacity(Ctx *c, int *max_tiles);
int chol_fused_width(Ctx *c, int *width);
// tile = 0: 64-wide tiles when the batch has at least one 64-tile per SM, else 32-wide; 32 / 64 force the width (test hook).
// Returns the tile width launched (0: nothing to do).
int launch_gemm(Ctx *c, const GemmBatch &b, int tile = 0);
// the tile width (returned) and the k split (chunk count, chunk length) launch_gemm uses for b; tile 32 / 64 forces the width
int gemm_plan(const Ctx *c, const GemmBatch &b, int tile, int *nchunk, int *kc);
void launch_gemm1(Ctx *c, const GemmProblem &p, const int *flag = nullptr);
// In-place blocked Cholesky of the leading `npiv` pivots of the symmetric (lower-stored) matrix A (size n x n, ld):
int chol_partial(Ctx *c, double *A, int ld, int n, int npiv, double tol); // one launch of chol_fused
int ws_alloc(Ctx *c, DenseWs &ws, int cap);
void ws_free(DenseWs &ws);
// y = alpha * A(m x k view) * x  (one warp per row)
// sum of squares of x[0:n] -> out[0]
void launch_fill(Ctx *c, double *p, size_t n, double v);

// ---- ekf.cu ------------------------------------------------------------------------------------------------------
// Generic EKF update core.  HT: nc x rr (column-major, ld ldHT) = H^T in the column order given by d_cols (device array of
// nc state indices).  z: rr.  Rdiag: rr or nullptr (identity).  If gate_thresh >= 0, chi2 = z^T S^-1 z is compared with
// it on the device and the update is skipped when larger (flag written to d_gate_flag, chi2 to d_chi2).  ht_lower: HT(k, j) == 0 for k < j
// (HT is the lower Cholesky factor of the compression) - the two products skip the structural zeros.
// products_done: M = P[:, cols] HT (in dM) and S = HT^T M[cols, :] + R (in wsS) are already formed; steps 1-2 are skipped.
int ekf_update_core(Ctx *c, const int *d_cols, int nc, MatView HT, int rr, const double *d_z, const double *d_Rdiag, double gate_thresh,
                    int *d_gate_flag, double *d_chi2, bool apply = true, int zstride = 1, bool defer_join = false, bool ht_lower = false,
                    bool products_done = false);
// The compressed update: factor the Gram matrix in wsG (nc + 1 columns, z last; pivots on the leading npiv) and update with H^T = L
// (rows [0, nc)), z = row nc of the factor, R = I.  The factorisation launch also forms M and S.
int gram_factor_update(Ctx *c, const int *d_cols, int nc, int npiv, double tol, double gate_thresh, int *d_gate_flag, double *d_chi2,
                       bool defer_join);
int join_side_stream(Ctx *c); // make the main stream wait for the side stream's covariance downdate (no-op when nothing is pending)
int upload_var_table(Ctx *c);
int sync_host_values(Ctx *c);
int push_host_values(Ctx *c, int handle);
int state_append_variable(Ctx *c, Var v, const double *value, const double *fej, int *handle);
int check_status_flags(Ctx *c);
// chi-squared 0.95 quantile: the injected table (ovp_set_chi2_table) below its length, computed exactly beyond it - never clamped
double chi2_q95(Ctx *c, int dof);

// ---- features.cu -------------------------------------------------------------------------------------------------
// extra: forced_cols != nullptr => point features only, x columns fixed to this list of state indices (multi-GPU shard
// half); d_export != nullptr => write the (n+1)x(n+1) factor block [R^T ; z^T] there and skip the EKF update.
#define OVP_DX_SPLIT 8 // dx = Y w is summed in this many fixed chunks of the compressed rows (dx_partial_kernel, ekf.cu)
struct MsckfExtra {
  const std::vector<int> *forced_cols = nullptr;
  double *d_export = nullptr;
  bool allgather_gram = false; // sharded update: all-gather the rank-local packed Gram matrices over the ctx's NCCL communicator, sum them
                               // in rank order on every rank, then the ordinary compression + EKF update (replicated)
  int64_t only_plane_id = 0;   // init_vio_plane: build the W system of this (out-of-state) plane only and stop
  double sigma_c_scale = 0.0;  // > 0: multiply sigma_constraint (const_init_multi)
};
int msckf_last_W(Ctx *c, int *rowsW, int *ncx, int *rows_ref, const int **d_cols);
int allgather_gram(Ctx *c, int nc1); // capi_nccl.inc: wsG.S (rank-local Gram, lower) -> sum over the ranks of the ctx's communicator
int msckf_update_impl(Ctx *c, const ovp_feature_batch *batch, const ovp_updater_options *opt, int *feat_status, double *feat_chi2,
                      int *plane_status, double *plane_chi2, int *hx_order, int *hx_order_n, const MsckfExtra *extra = nullptr);

} // namespace ovp

struct ovp_ctx {
  ovp::Ctx c;
};
namespace ovp {
// every ABI entry point that touches the device starts here: allocations, attribute settings and launches must land on the
// context's own device when one process drives several GPUs (one ctx per device)
static inline Ctx *enter(ovp_ctx *h) {
  int cur = -1;
  if (cudaGetDevice(&cur) != cudaSuccess || cur != h->c.device)
    cudaSetDevice(h->c.device);
  return &h->c;
}
} // namespace ovp

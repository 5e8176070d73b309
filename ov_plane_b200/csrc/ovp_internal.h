// Internal declarations of the H100-native ov_plane hot path library (not part of the C ABI).
#pragma once
#include "../../include/ovp.h"
#include "gemm.cuh"
#include <cuda_runtime.h>
#include <deque>
#include <map>
#include <string>
#include <utility>
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

struct Prepared; // the plan of the last prepared MSCKF batch (features_host.inc)

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
  // D-part stream of a block-sparse Gram matrix: gram_dpart_kernel runs here beside the SYRK of the same update (both read only the
  // feature kernel's output, the reduction needs both); forked after the feature kernel, joined before the reduction (features_host.inc)
  cudaStream_t stream3 = nullptr;
  cudaEvent_t ev_dfork = nullptr, ev_djoin = nullptr;
  ovp_state_options opt;
  std::string last_error;
  int64_t launches = 0;
  bool use_graphs = true;    // replay the static launch sequence of a prepared batch as a CUDA graph
  double gram_tol = 1e-11;   // zero-pivot rule of the Gram Cholesky, relative to the column's original diagonal (ovp_set_rank_tolerance)
  bool force_dense_features = false; // MSCKF batches take the one-block-per-feature kernel and the dense stack (ovp_debug_force_dense_features)
  bool unfused_update_products = false; // compressed updates form M and S with two GEMM launches (ovp_debug_unfused_update_products)
  bool sequential_factorisations = false; // compressed updates never pair their two factorisations (ovp_debug_sequential_factorisations)
  bool programmatic = true; // chain_launch makes each update-chain kernel a programmatic dependent (ovp_debug_programmatic_launches)
#ifdef OVP_DEBUG
  // ovp_debug_msckf_gram: the feature kernels write their raw blocks to dbg_raw (when set), and with dbg_gram_stop the MSCKF launch
  // returns right after the first Gram matrix it forms, recording that plan's index in dbg_gram_plan
  double *dbg_raw = nullptr;
  bool dbg_gram_stop = false;
  int dbg_gram_plan = -1;
  // ovp_debug_slam_gram: with dbg_gram_stop the SLAM update returns right after its Gram matrix, leaving the compact columns' state
  // indices and the stacked rows it laid out here
  std::vector<int> dbg_slam_cols;
  int dbg_slam_rows = 0;
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
  // UpdaterSLAM's options_aruco (ovp_set_aruco_options): with has_aruco, the SLAM entry points whiten and gate every feature with
  // featid < opt.max_aruco_features with these instead of the call's options (aruco_options_of)
  bool has_aruco = false;
  ovp_updater_options aruco = {1.0, 1.0};
  // StateOptions::feat_rep_slam / feat_rep_aruco (ovp_set_landmark_options): with has_lm_rep, ovp_slam_update takes landmarks in any
  // representation 0..4 and ovp_slam_delayed_init_tracks creates each landmark in its feature's (landmark_rep_of)
  bool has_lm_rep = false;
  ovp_landmark_options lm_rep = {0, 0};
  // FeatureInitializerOptions::triangulate_1d / refine_features (ovp_set_triangulation_mode): the triangulation kernel every entry point
  // launches (launch_triangulate); {0, 1} is ov_core's default
  ovp_triangulation_mode tri_mode = {0, 1};
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
  double *cf_linv_s = nullptr, *cf_diag0_s = nullptr, *cf_xch_s = nullptr; // the innovation factorisation's set in a pair
  int *cf_flags_s = nullptr;
  int cf_maxT = 0;
  bool cf_attr_set = false;   // per context (= per device): >48 KB dynamic shared memory opt-in of chol_fused_kernel / feature kernels
  int cf_max_coresident = 0;  // co-resident CTA capacity of this device for chol_fused_kernel
  int max_update_width = 0;   // ovp_set_max_update_width (0: the co-resident width of one fused launch)
  double *cf_panel = nullptr; // panelled factorisation (cholpanel.cu): original diagonal (Rcap), z (Rcap), chi2 per panel (cf_maxT)
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
  double *d_mw = nullptr;      // CTA-per-feature path: measurement blocks, per-feature dense blocks, D part (msckf_warp.inc)
  size_t d_mw_elems = 0;
  // feature batch staging
  void *d_batch = nullptr;
  size_t d_batch_bytes = 0;
  void *h_pinned = nullptr;
  size_t h_pinned_bytes = 0;
  // device side of the host <-> device transfers of the ABI entry points, laid out by a StageLayout (ensure_stage)
  char *d_stage = nullptr;
  size_t d_stage_bytes = 0;

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
  Prepared *prep = nullptr;
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
void drop_prepared_graph(Ctx *c); // the prepared batch's captured graph: its next launch captures the plan again

// error helpers
int fail(Ctx *c, int status, const char *fmt, ...);
#define OVP_CUDA(call)                                                                                                      \
  do {                                                                                                                       \
    cudaError_t e__ = (call);                                                                                                \
    if (e__ != cudaSuccess)                                                                                                  \
      return fail(c, OVP_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));                   \
  } while (0)

// ---- programmatic dependent launches of the update chain ---------------------------------------------------------
// A kernel launched through chain_launch may be placed on the SMs while the kernel before it on the stream still runs: its launch
// latency and CTA set-up hide behind that kernel's tail.  Every such kernel calls chain_wait() in every CTA before it touches global
// memory, so nothing it reads or writes races with an earlier kernel, and - because every CTA waits on every path - its completion
// still implies its predecessor's, which keeps stream order transitive for the launches after it.  chain_release() right after the
// wait lets the next dependent be placed; it takes effect once every CTA of the grid has issued it or exited, so in a multi-wave grid
// not before the last wave is resident.  Both are no-ops in a kernel not launched as a programmatic dependent.
__device__ __forceinline__ void chain_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void chain_release() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// kernel<<<grid, block, smem, c->stream>>>(args...) as a programmatic dependent of the previous kernel on c->stream (unless
// c->programmatic is off), counted in c->launches.  Returns the launch's error.
template <class... KArgs, class... Args>
static inline cudaError_t chain_launch(Ctx *c, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, Args &&...args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = c->stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = c->programmatic ? 1 : 0;
  c->launches++;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// ---- linalg.cu ---------------------------------------------------------------------------------------------------
// The two products of a compressed update, formed inside the factorisation of its Gram matrix (cholfused.cu): with L = rows [0, nc) of
// the factor, M = P[:, cols] L (N x npiv, ld ldm) and the lower tiles of S = L^T M[cols, :] + I (npiv x npiv, ld lds).  ldp is even.
struct CholProducts {
  const double *P;
  const int *cols;
  double *M, *S;
  int ldp, N, nc, ldm, lds;
};
// diag0 (optional): the reference diagonal of the zero-pivot rule for the npiv pivots, in place of the diagonal the launch loads (a panel
// of chol_panels, whose diagonal the panels before it have downdated)
int chol_fused(Ctx *c, double *A, int ld, int n, int npiv, double tol, const double *M, int ldm, int mrows, const double *z, int zstride,
               double *Y, int ldy, double *w, double gate_thresh, double *chi2, int *gate_flag, long long *dbg = nullptr,
               const CholProducts *prod = nullptr, double *diag0 = nullptr);
// Y = M L^-T, w = L^-1 z and chi2 = |w|^2 (no gate) against the factor the chol_fused launch before it on the stream left in the exchange
// slots (a factorisation of the same n, npiv): the second launch of chol_fused's two-launch fallback, on a right-hand side of its own.
// Y may be M (each row block reads its rows whole before it writes them).
int chol_fused_rows(Ctx *c, double *A, int ld, int n, int npiv, const double *M, int ldm, int mrows, const double *z, int zstride, double *Y,
                    int ldy, double *w, double *chi2);
// every tile CTA of one chol_fused launch must be co-resident: the tile CTAs a factorisation of the leading npiv columns of an n x n
// system needs, how many the device holds, and the widest full factorisation (a multiple of 64) that fits
int chol_fused_tiles(int n, int npiv);
// The two factorisations of a compressed update overlapped when they fit co-resident together: the Gram matrix A (n x n, leading npiv
// columns) with the products `prod` and S = prod.S (npiv x npiv) in one cooperative launch, S's tiles starting as their products are
// stored, then Y = prod.M L_S^-T, w = L_S^-1 z, chi2 and the gate (M rows: prod.N) in a launch that starts while the first runs.  Two
// launches, bit for bit what chol_fused produces for the two one after the other.  *paired = false: nothing was launched (the pair does
// not fit, or c->sequential_factorisations), the caller runs the two factorisations.
int chol_fused_pair(Ctx *c, double *A, int ld, int n, int npiv, double tol, const CholProducts &prod, const double *z, int zstride, double *Y,
                    int ldy, double *w, double gate_thresh, double *chi2, int *gate_flag, long long *dbg, bool *paired);
int chol_fused_capacity(Ctx *c, int *max_tiles);
int chol_fused_width(Ctx *c, int *width);
// ---- cholpanel.cu: systems wider than one co-resident launch ----
// the widest system one update may factor (ovp_set_max_update_width; 0 declared: chol_fused_width)
int update_width(Ctx *c, int *width);
// *panels: the factorisation of the leading npiv columns of an n x n system runs in panels (chol_panels) - it does not fit one
// co-resident launch and n is within the declared width
int chol_needs_panels(Ctx *c, int n, int npiv, bool *panels);
// The contract of chol_fused without products, for a system of any width up to the workspaces: the columns are factored in panels of
// `width` (a multiple of 64, at most chol_fused_width), each one chol_fused launch on its diagonal block, its rows below solved against it,
// and the trailing blocks downdated with the DMMA GEMM; chi2 and the gate flag are formed from the panels' parts at the end.  Every pivot
// is compared with its column's original diagonal.  Y receives M's columns and is worked in place; M and z are only read.
int chol_panels(Ctx *c, int width, double *A, int ld, int n, int npiv, double tol, const double *M, int ldm, int mrows, const double *z,
                int zstride, double *Y, int ldy, double *w, double gate_thresh, double *chi2, int *gate_flag);
// The one entry of every update's factorisation: chol_fused when the system fits co-resident, chol_panels (panels of chol_fused_width)
// when it does not and the declared width allows it; otherwise chol_fused's refusal.
int chol_factor(Ctx *c, double *A, int ld, int n, int npiv, double tol, const double *M, int ldm, int mrows, const double *z, int zstride,
                double *Y, int ldy, double *w, double gate_thresh, double *chi2, int *gate_flag);
// tile = 0: 64-wide tiles when the batch has at least one 64-tile per SM, else 32-wide; 32 / 64 force the width (test hook).
// Returns the tile width launched (0: nothing to do).
int launch_gemm(Ctx *c, const GemmBatch &b, int tile = 0);
// the tile width (returned) and the k split (chunk count, chunk length) launch_gemm uses for b; tile 32 / 64 forces the width
int gemm_plan(const Ctx *c, const GemmBatch &b, int tile, int *nchunk, int *kc);
void launch_gemm1(Ctx *c, const GemmProblem &p, const int *flag = nullptr);
// In-place blocked Cholesky of the leading `npiv` pivots of the symmetric (lower-stored) matrix A (size n x n, ld):
int chol_partial(Ctx *c, double *A, int ld, int n, int npiv, double tol); // chol_factor without a right-hand side
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
// done: 1 - M = P[:, cols] HT (in dM) and S = HT^T M[cols, :] + R (in wsS) are already formed, steps 1-2 are skipped; 2 - S is also
// factored and Y, w, chi2 and the gate flag are formed (chol_fused_pair), steps 1-5 are skipped.
// feat_flag (nfeat status words, or nullptr): the update is also skipped on the device when none of them is in the accepted set
// accept_mask (bit s set: status s accepted).  A point update none of whose features passed its gate (status 1) leaves the state
// untouched (UpdaterMSCKF.cpp:796-807), and so does a SLAM update none of whose landmarks has status 1 or 3 (UpdaterSLAM.cpp:663-664).
#define OVP_ACCEPT_POINT (1u << 1)
#define OVP_ACCEPT_SLAM ((1u << 1) | (1u << 3))
int ekf_update_core(Ctx *c, const int *d_cols, int nc, MatView HT, int rr, const double *d_z, const double *d_Rdiag, double gate_thresh,
                    int *d_gate_flag, double *d_chi2, bool apply = true, int zstride = 1, bool defer_join = false, bool ht_lower = false,
                    int done = 0, const int *feat_flag = nullptr, int nfeat = 0, unsigned accept_mask = OVP_ACCEPT_POINT);
// The compressed update: factor the Gram matrix in wsG (nc + 1 columns, z last; pivots on the leading npiv) and update with H^T = L
// (rows [0, nc)), z = row nc of the factor, R = I.  The factorisation launch also forms M and S.
int gram_factor_update(Ctx *c, const int *d_cols, int nc, int npiv, double tol, double gate_thresh, int *d_gate_flag, double *d_chi2,
                       bool defer_join, const int *feat_flag = nullptr, int nfeat = 0, unsigned accept_mask = OVP_ACCEPT_POINT);
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
  const ovp_plane_landmarks *landmarks = nullptr; // use_plane_constraint_slamu: candidate landmark members of the out-of-state planes
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

// h names a clone (State::_clones_IMU): a live pose other than the camera extrinsics, which with need_slot must also have covariance
// columns.  A measurement's clone, an anchor and a shard's clone list are checked with this.
static inline bool is_clone(const Ctx *c, int h, bool need_slot) {
  return h >= 0 && h < (int)c->vars.size() && c->vars[h].alive && c->vars[h].kind == OVP_KIND_POSE && h != c->h_calib &&
         (!need_slot || c->vars[h].id >= 0);
}

// an ArUco tag corner of UpdaterSLAM ((int)featid < max_aruco_features, UpdaterSLAM.cpp:164, 257, 303, 500, 546) while ArUco options are set
static inline bool is_aruco_tag(const Ctx *c, int64_t featid) { return c->has_aruco && (int)featid < c->opt.max_aruco_features; }
// the options UpdaterSLAM whitens and gates feature featid with: options_aruco for a tag, the call's own (options_slam) otherwise
static inline const ovp_updater_options &slam_options_of(const Ctx *c, int64_t featid, const ovp_updater_options &opt) {
  return is_aruco_tag(c, featid) ? c->aruco : opt;
}
// the representation UpdaterSLAM creates the landmark of feature featid in (UpdaterSLAM.cpp:231-232): feat_rep_aruco for an ArUco id,
// feat_rep_slam otherwise; GLOBAL_3D (0) while no landmark options are set
static inline int landmark_rep_of(const Ctx *c, int64_t featid) {
  if (!c->has_lm_rep)
    return 0;
  return (int)featid < c->opt.max_aruco_features ? c->lm_rep.feat_rep_aruco : c->lm_rep.feat_rep_slam;
}

// bump allocator of a staging buffer: consecutive slices, each starting 16-byte aligned
struct StageLayout {
  size_t top = 0;
  size_t take(size_t bytes) {
    const size_t at = top;
    top = (top + bytes + 15) & ~(size_t)15;
    return at;
  }
};
// c->d_stage grown to hold L's slices (its base is 16-byte aligned, like every slice)
int ensure_stage(Ctx *c, const StageLayout &L);
// Every host <-> device copy of the library goes through these: asynchronous on c->stream, counted in c->h2d_bytes / c->d2h_bytes
// (ovp_transfer_bytes).  The 2D forms copy `cols` columns of col_bytes each between buffers with the given column pitches.  Nothing to
// copy: no call.
int stage_copy_in(Ctx *c, void *dst, const void *src, size_t bytes);
int stage_copy_out(Ctx *c, void *dst, const void *src, size_t bytes);
int stage_copy2d_in(Ctx *c, void *dst, size_t dpitch, const void *src, size_t spitch, size_t col_bytes, size_t cols);
int stage_copy2d_out(Ctx *c, void *dst, size_t dpitch, const void *src, size_t spitch, size_t col_bytes, size_t cols);
} // namespace ovp

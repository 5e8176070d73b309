/*
 * ovp.h — C ABI of the H100-native ov_plane hot path (MSCKF / point-on-plane EKF update + IMU covariance propagation).
 *
 * Drop-in boundary (SURVEY.md §8(b)): the reference has no FFI seam — its updaters are C++ classes calling the all-static
 * `StateHelper` (ov_plane/src/state/StateHelper.h) on a `State` whose covariance is private (State.h:123-133).  This library
 * replaces what sits behind that seam.  An `ovp_ctx` owns, on ONE GPU, the covariance `_Cov` (fp64, column-major, symmetric,
 * full storage), the variable table `_variables` (id / size / kind, same id semantics as ov_type::Type::id()) and the
 * mean + first-estimate values of every variable (so that a chain of dependent updates never returns to the host).
 * Every entry point below cites the reference function it replaces.  INTEGRATION.md shows the adapter a maintainer adds on
 * the reference side (thin C++ shims with the reference's own signatures).
 *
 * Conventions: all matrices are column-major IEEE double; `handle` = stable integer naming one variable (what a
 * std::shared_ptr<ov_type::Type> is in the reference); `id` = its offset in the covariance (-1 when not in the state).
 * All functions return an ovp_status (0 = OK).  The reference prints and calls std::exit(EXIT_FAILURE) on the conditions
 * mapped to OVP_ERR_* (StateHelper.cpp:46-49,55-59,116-118,185-187,279-283,387-391,403-407); an adapter maps non-zero
 * status to the same print + exit.  One in-flight call per ctx; distinct ctxs are independent (State is unsynchronised in
 * the reference too, SURVEY §8(b) "Threading").  There is NO CPU fallback: every entry point needs a CUDA device.
 */
#ifndef OVP_H
#define OVP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ovp_ctx ovp_ctx;

typedef enum ovp_status {
  OVP_OK = 0,
  OVP_ERR_BAD_ARGS = 1,          /* shape / handle errors (reference: assert, StateHelper.cpp:70-73,127-128) */
  OVP_ERR_NEGATIVE_DIAGONAL = 2, /* StateHelper.cpp:107-118,176-187 */
  OVP_ERR_NON_CONTIGUOUS = 3,    /* StateHelper.cpp:52-61 */
  OVP_ERR_NON_ISOTROPIC = 4,     /* StateHelper.cpp:413-425 */
  OVP_ERR_NOT_IN_STATE = 5,      /* StateHelper.cpp:279-283,387-391 */
  OVP_ERR_ALREADY_IN_STATE = 6,  /* StateHelper.cpp:403-407 */
  OVP_ERR_CAPACITY = 7,          /* state / measurement capacity given to ovp_create exceeded, or a dense system wider than the
                                    declared update width (ovp_set_max_update_width; by default the widest system the device
                                    factors in one co-resident launch, 64 x T columns with T(T+1)/2 <= SMs: 960 on an H100,
                                    DESIGN.md 4.1) */
  OVP_ERR_CUDA = 8,              /* CUDA runtime failure; see ovp_last_error */
  OVP_ERR_NOT_POSITIVE_DEFINITE = 9,
  OVP_ERR_TIME = 10              /* Propagator.cpp:41-51 (same / backwards timestamp), StateHelper.cpp:591-594 */
} ovp_status;

/* ov_type kinds the path needs (error-state size / value size): Vec(n/n), PoseJPL(6/7: q_xyzw,p), IMU(15/16: q,p,v,bg,ba),
 * Landmark GLOBAL_3D (3/3).  JPL quaternion, left-multiplicative update (ov_type::JPLQuat::update). */
typedef enum ovp_kind { OVP_KIND_VEC = 0, OVP_KIND_POSE = 1, OVP_KIND_IMU = 2, OVP_KIND_LANDMARK = 3 } ovp_kind;

/* Subset of ov_plane::StateOptions (state/StateOptions.h:41-153) the path reads. */
typedef struct ovp_state_options {
  int do_fej;
  int imu_avg;
  int use_rk4_integration;
  int do_calib_camera_pose;
  int do_calib_camera_intrinsics;
  int do_calib_camera_timeoffset;
  int max_clone_size;
  int max_aruco_features;
  double sigma_constraint;
  double const_init_multi;
  double const_init_chi2;
  double sigma_plane_merge;
  double plane_merge_chi2;
  double plane_merge_deg_max;
} ovp_state_options;

/* ---- context / State (state/State.h, State.cpp:33-102) ------------------------------------------------------------ */
/* Builds the State exactly like State::State(options): imu, [dt], [extrinsics], [intrinsics] and the prior diagonal.
 * max_state: covariance capacity (rows); max_meas_rows: capacity of one stacked measurement system (rows of Hx_big). */
int ovp_create(const ovp_state_options *opt, int device, int max_state, int max_meas_rows, ovp_ctx **out);
void ovp_destroy(ovp_ctx *ctx);
const char *ovp_last_error(ovp_ctx *ctx);
const char *ovp_status_string(int status);
int ovp_set_chi2_table(ovp_ctx *ctx, const double *quantile95, int n); /* chi_squared_table, UpdaterMSCKF.cpp:59-62 */

int ovp_cov_rows(ovp_ctx *ctx);                                       /* State::max_covariance_size(), State.h:87 */
int ovp_cov_download(ovp_ctx *ctx, double *out, int ld);              /* StateHelper::get_full_covariance, :261-274 */
int ovp_cov_upload(ovp_ctx *ctx, const double *in, int n, int ld);    /* raw overwrite, n must equal ovp_cov_rows */
int ovp_handle_imu(ovp_ctx *ctx);
int ovp_handle_dt(ovp_ctx *ctx);
int ovp_handle_calib(ovp_ctx *ctx);
int ovp_handle_intrinsics(ovp_ctx *ctx);
int ovp_var_id(ovp_ctx *ctx, int handle);                             /* Type::id() */
int ovp_var_size(ovp_ctx *ctx, int handle);                           /* Type::size() */
int ovp_var_value_size(ovp_ctx *ctx, int handle);
int ovp_var_set(ovp_ctx *ctx, int handle, const double *value, const double *fej); /* Type::set_value / set_fej */
int ovp_var_get(ovp_ctx *ctx, int handle, double *value, double *fej);             /* Type::value / fej */
int ovp_num_variables(ovp_ctx *ctx);
int ovp_variable_order(ovp_ctx *ctx, int *handles);                   /* State::_variables order */
int ovp_set_timestamp(ovp_ctx *ctx, double t);
double ovp_get_timestamp(ovp_ctx *ctx);
/* Append a variable with zero covariance (used by initialize_with_gt-style set-up and by tests; the covariance is then
 * written with ovp_set_initial_covariance / ovp_cov_upload). */
int ovp_add_clone_raw(ovp_ctx *ctx, double timestamp, const double *value7, const double *fej7, int *handle);
int ovp_add_plane_raw(ovp_ctx *ctx, int64_t planeid, const double *cp, const double *cp_fej, int *handle);
int ovp_add_slam_raw(ovp_ctx *ctx, int64_t featid, const double *p, const double *p_fej, int *handle);
int ovp_plane_handle(ovp_ctx *ctx, int64_t planeid); /* State::_features_PLANE lookup, -1 when absent */
int ovp_clone_handle(ovp_ctx *ctx, double timestamp); /* State::_clones_IMU lookup, -1 when absent */

/* ---- StateHelper (state/StateHelper.cpp) ---------------------------------------------------------------------------- */
int ovp_set_initial_covariance(ovp_ctx *ctx, const double *cov, int n, const int *handles, int k);      /* :204-229 */
int ovp_get_marginal_covariance(ovp_ctx *ctx, const int *handles, int k, double *out);                   /* :231-259 */
int ovp_ekf_propagation(ovp_ctx *ctx, const int *new_handles, int k_new, const int *old_handles, int k_old, const double *Phi,
                        int phi_rows, int phi_cols, const double *Q);                                     /* :41-119 */
/* H: rows x n (n = sum of sizes of `handles`), ld = rows; Rdiag NULL => identity (every caller on the path, SURVEY §8(a)) */
int ovp_ekf_update(ovp_ctx *ctx, const int *handles, int k, const double *H, int rows, const double *res,
                   const double *Rdiag);                                                                  /* :121-202 */
int ovp_marginalize(ovp_ctx *ctx, int handle);                                                            /* :276-344 */
int ovp_clone(ovp_ctx *ctx, int handle, int *new_handle);                                                 /* :346-396 */
int ovp_augment_clone(ovp_ctx *ctx, double timestamp, const double last_w[3], int *new_handle);           /* :588-625 */
int ovp_marginalize_old_clone(ovp_ctx *ctx);                                                              /* :627-636 */
int ovp_marginalize_slam(ovp_ctx *ctx);                                                                   /* :638-652 */
/* initialize a new Vec (plane CP, tag = plane id) or Landmark (tag = feature id) of size s; R = sigma2 * I (isotropic is
 * required, :413-425).  H_R rows x n, H_L rows x s, col-major.  *accepted = 0 on chi2 failure (state untouched). */
int ovp_initialize(ovp_ctx *ctx, int kind, int s, const double *value, const double *fej, int64_t tag, const int *handles, int k,
                   const double *H_R, const double *H_L, const double *res, int rows, double sigma2, double chi2_mult,
                   int do_update, int *accepted, int *new_handle);                                        /* :398-487 */
int ovp_initialize_invertible(ovp_ctx *ctx, int kind, int s, const double *value, const double *fej, int64_t tag,
                              const int *handles, int k, const double *H_R, const double *H_L, const double *res, double sigma2,
                              int *new_handle);                                                           /* :489-586 */
int ovp_merge_planes_and_marginalize(ovp_ctx *ctx, const int64_t *f2p_feat, const int64_t *f2p_plane, int nf,
                                     const int64_t *merge_new, const int64_t *merge_old, int nm);         /* :654-758 */

/* ---- UpdaterHelper / UpdaterPlane static helpers (stateless, host buffers in / out, computed on the GPU) ------------ */
/* UpdaterHelper::get_feature_jacobian_full (UpdaterHelper.cpp:195-513), mono, GLOBAL_3D.  Outputs col-major with
 * ld = *rows_out; buffers sized for 3*m(+1) rows and (14 + 6*m + 3) columns; x_order receives variable handles. */
/* UpdaterHelper::get_feature_jacobian_representation (UpdaterHelper.cpp:35-193), context-free host helper.  representation follows
 * ov_type::LandmarkRepresentation (0 GLOBAL_3D, 1 GLOBAL_FULL_INVERSE_DEPTH, 2 ANCHORED_3D, 3 ANCHORED_FULL_INVERSE_DEPTH,
 * 4 ANCHORED_MSCKF_INVERSE_DEPTH, 5 ANCHORED_INVERSE_DEPTH_SINGLE); poses are [q (JPL xyzw), p]: anchor = [q_GtoI, p_IinG],
 * calib = [q_ItoC, p_IinC].  Outputs column-major: H_f 3 x hf_cols (3, or 1 for the single-depth form), and for anchored forms
 * (has_anchor = 1) H_anc 3 x 6 w.r.t. the anchor clone [theta, p] and H_calib 3 x 6 w.r.t. the extrinsics [theta, p]. */
int ovp_feature_jacobian_representation(int representation, int do_fej, const double *p_FinG, const double *p_FinG_fej,
                                        const double *p_FinA, const double *anchor_pose7, const double *anchor_pose_fej7,
                                        const double *calib7, double *H_f, int *hf_cols, double *H_anc, double *H_calib, int *has_anchor);
int ovp_feature_jacobian_full(ovp_ctx *ctx, int m, const int *clone_handles, const float *uv, const double *p_FinG,
                              const double *p_FinG_fej, int64_t planeid, const double *cp, const double *cp_fej, double sigma_px,
                              double sigma_c, double *H_f, int *hf_cols, double *H_x, int *hx_cols, double *res, int *rows_out,
                              int *x_order, int *x_order_n);
/* UpdaterHelper::nullspace_project_inplace (:515-546) / UpdaterPlane::nullspace_project_inplace (UpdaterPlane.cpp:483-517).
 * Result is an orthogonal-equivalent left-nullspace projection (Householder instead of the reference's Givens order):
 * identical H_o^T H_o, H_o^T r and chi2; rows of H_o differ by an orthogonal transform (SURVEY §7 hazard list).
 * Any rows >= hf_cols are projected (rows == hf_cols returns *rows_out = 0); an exactly zero column of H_f is skipped. */
int ovp_nullspace_project_inplace(ovp_ctx *ctx, double *H_f, int hf_cols, double *H_x, int hx_cols, double *res, int rows,
                                  int *rows_out);
int ovp_plane_nullspace_project_inplace(ovp_ctx *ctx, double *H_f, int hf_cols, double *H_x, int hx_cols, double *H_cp,
                                        double *res, int rows, int *rows_out);
/* UpdaterHelper::measurement_compress_inplace (:548-579) / UpdaterPlane::measurement_compress_inplace
 * (UpdaterPlane.cpp:519-552).  Q-less Cholesky-QR on tensor cores: returns upper-trapezoidal R with R^T R = H^T H and
 * z = R^-T H^T res (equal to the Givens result up to row signs when H has full column rank; rank-deficient pivots give
 * zero rows).  The plane variant carries H_cp and keeps only the first min(rows, cols) rows like the reference. */
int ovp_measurement_compress_inplace(ovp_ctx *ctx, double *H_x, int cols, double *res, int rows, int *rows_out);
int ovp_plane_measurement_compress_inplace(ovp_ctx *ctx, double *H_x, int cols, double *H_cp, double *res, int rows,
                                           int *rows_out);

/* ---- UpdaterMSCKF::update from "features triangulated, plane CPs known" on (UpdaterMSCKF.cpp:407-828) --------------- */
/* Feature tracks, as every entry point that takes them reads them (this batch, ovp_slam_update, ovp_slam_delayed_init, ovp_feature_tracks,
 * ovp_triangulate_features, ovp_optimize_plane): meas_offset holds F + 1 prefix offsets that start at 0 and never decrease, so feature f's
 * measurements are meas_offset[f] .. meas_offset[f + 1] - 1 of the meas_offset[F] in the measurement arrays; each measurement's handle is a
 * clone in the state (a live pose other than the camera extrinsics); and, mono camera, a track observes each clone at most once (the
 * triangulation and the refinement take a clone twice).  The arrays an entry point reads are non-null when F > 0 (the measurement arrays
 * when there are measurements).  A batch that breaks this is refused with OVP_ERR_BAD_ARGS before any of it is copied or launched, with
 * the state untouched; each entry point below states its own track-length limits.
 * Track length: every feature of a batch has 2..39 measurements, or 2..37 when the batch runs a plane update (an in-state plane,
 * a plane not in the state with >= 4 features, or ovp_plane_init).  Tracks of up to 32 run on the block-sparse feature kernel; one
 * longer track puts the whole batch on the dense stacked one, whose per-feature system must fit the CTA's shared memory.  A longer track
 * is refused with OVP_ERR_CAPACITY before anything is launched, and the message names the limit.  Every other capacity check
 * of the update (rows, columns, factorisation width) also runs before the first launch, so a refused batch leaves the state as
 * it was.  The factorisation width is the declared update width (ovp_set_max_update_width: by default 960 compressed columns on an
 * H100, about 157 clones). */
typedef struct ovp_feature_batch {
  int F;                         /* number of features (feature_vec after triangulation, caller's order)               */
  const int *meas_offset;        /* F+1 prefix offsets into the measurement arrays (feature tracks, above)             */
  const int *meas_clone;         /* per measurement: handle of the clone it was taken at (Feature::timestamps)          */
  const float *uv;               /* per measurement: raw pixel (u,v) as float, like Feature::uvs (Eigen::VectorXf)       */
  const double *p_FinG;          /* 3F: triangulated (and, for on-plane features, plane-refined) position               */
  const double *p_FinG_original; /* 3F: position before plane refinement (UpdaterMSCKF.cpp:160,663); may alias p_FinG   */
  const int64_t *featid;         /* F                                                                                   */
  const int64_t *planeid;        /* F: feat2plane value, 0 = not on a plane                                             */
  int nplanes;                   /* planes that obtained a linearisation point (plane_estimates_cp_inG, :198-404)       */
  const int64_t *plane_ids;      /* nplanes, any order (visited ascending like the std::map)                            */
  const double *plane_cp;        /* 3*nplanes: CP estimate for planes NOT in the state (in-state planes use the state)  */
} ovp_feature_batch;

typedef struct ovp_updater_options { /* UpdaterOptions.h:38-54 */
  double sigma_pix;
  double chi2_multipler;
} ovp_updater_options;

/* Outputs: feat_status[F]: 1 accepted in the point update, 0 chi2-rejected, 2 consumed by a passed plane update;
 * feat_chi2[F] (NaN when not gated individually); plane_status[nplanes]: 1 pass, 0 chi2 fail, -1 not visited;
 * plane_chi2[nplanes]; hx_order: Hx_order_big of the final point update as variable handles (first-seen order over the
 * accepted features, UpdaterMSCKF.cpp:768-775).  Any output pointer may be NULL. */
int ovp_msckf_update(ovp_ctx *ctx, const ovp_feature_batch *batch, const ovp_updater_options *opt, int *feat_status,
                     double *feat_chi2, int *plane_status, double *plane_chi2, int *hx_order, int *hx_order_n);

/* The same update with the in-state SLAM landmarks of use_plane_constraint_slamu (UpdaterMSCKF.cpp:231-254, 454-560, 626-639).
 * The caller passes the feat2plane entries of its landmarks (n = 0: slamu off, the result is bit-identical to ovp_msckf_update);
 * the library keeps the ones that join a plane: featid is in State::_features_SLAM, planeid names a plane of the batch that is NOT
 * in the state, and _features_SLAM_to_PLANE[featid] is absent or non-zero.  Each member counts towards its plane's 4-feature
 * rule (the plane still needs one batch feature) and adds one point-on-plane row with its 3 landmark columns as state columns
 * (residual at the landmark's value, Jacobians at its first estimate when do_fej).  After the plane's gate the library sets
 * _features_SLAM_to_PLANE[featid] to the plane id (pass) or 0 (fail).  Refused with OVP_ERR_BAD_ARGS before anything is
 * launched: a member that is not GLOBAL_3D, a featid listed twice, a featid that is also a feature of the batch. */
typedef struct ovp_plane_landmarks {
  int n;
  const int64_t *featid;  /* n */
  const int64_t *planeid; /* n: feat2plane entry, 0 = not on a plane */
} ovp_plane_landmarks;
int ovp_msckf_update_landmarks(ovp_ctx *ctx, const ovp_feature_batch *batch, const ovp_plane_landmarks *landmarks,
                               const ovp_updater_options *opt, int *feat_status, double *feat_chi2, int *plane_status,
                               double *plane_chi2, int *hx_order, int *hx_order_n);

/* UpdaterPlane::init_vio_plane from "plane linearisation points known" on (UpdaterPlane.cpp:297-481): every plane of the batch
 * that is NOT in the state (ascending id) and has >= 3 features is stacked (Jacobians with sigma_c * const_init_multi),
 * compressed and handed to StateHelper::initialize with const_init_chi2.  plane_status[i]: 1 initialised, 0 chi2-rejected,
 * -1 not attempted; new_handles[i]: handle of the new plane variable (or -1).  Features are NOT consumed here: the caller
 * removes the features of initialised planes from its MSCKF list like UpdaterPlane.cpp:459-475. */
int ovp_plane_init(ovp_ctx *ctx, const ovp_feature_batch *batch, const ovp_updater_options *opt, int *plane_status, int *new_handles);

/* ---- UpdaterSLAM (update/UpdaterSLAM.cpp) — GLOBAL_3D landmarks, and with ovp_set_landmark_representations the other five
 * representations, mono camera ---------------------------------------------------------------------------------------------------------- */
/* UpdaterSLAM::update from "calculate the max possible measurement size" on (:389-735): per landmark feature
 * get_feature_jacobian_full with the landmark (and its in-state plane, when use_plane_constraint and
 * _features_SLAM_to_PLANE allows it) as state columns, chi2 gate against the marginal covariance, on failure WITH a plane
 * one retry without it (:547-609), then ONE EKF update with the stack of the accepted blocks (R = I).
 * planeid[f]: the feat2plane entry of the feature (0 = none).  feat_status[f]: 1 accepted (plane constraint included when the
 * feature had one), 3 accepted after dropping the plane constraint, 0 rejected (landmark flagged should_marg), -1 not updated: an
 * ANCHORED_INVERSE_DEPTH_SINGLE landmark with one measurement, which the projection of its bearing needs two of (:410-417); feat_chi2 is NaN,
 * nothing is launched or copied for it, the state and its flags (should_marg, _features_SLAM_to_PLANE) are unchanged, and the rest of the
 * batch runs exactly as it would without it.  A landmark whose size does not match its representation (1 for ANCHORED_INVERSE_DEPTH_SINGLE, 3
 * otherwise, e.g. a variable of size 1 that ovp_initialize registered as a landmark) is refused with OVP_ERR_BAD_ARGS before anything is
 * copied or launched.
 * Every landmark has 1..29 measurements; a longer track is refused with OVP_ERR_CAPACITY before anything is launched.  So is a batch
 * whose compressed width (3 per landmark, 6 per involved clone, plus the calibration) exceeds the declared update width
 * (ovp_set_max_update_width: by default 960 on an H100, about 300 landmarks). */
int ovp_slam_update(ovp_ctx *ctx, int F, const int *meas_offset, const int *meas_clone, const float *uv, const int64_t *featid,
                    const int64_t *planeid, const ovp_updater_options *opt, int use_plane_constraint, int *feat_status,
                    double *feat_chi2);
/* UpdaterSLAM::delayed_init from "8. Finally, initialize" on (:225-372): per feature, in order, Jacobians at p_FinG (FEJ =
 * value), StateHelper::initialize(Landmark, ..., chi2_multipler); a failure WITH a plane retries without it from
 * p_FinG_original (:310-359).  feat_status[f]: 1 / 3 as above, 0 not initialised; new_handles[f]: landmark handle or -1.
 * Every track has 1..64 measurements, from clones with or without covariance columns; every track is checked before the first landmark is
 * initialised, and a malformed one is refused with OVP_ERR_BAD_ARGS with the state untouched.  A featid that already has a landmark
 * (OVP_ERR_ALREADY_IN_STATE), a clone without covariance columns (OVP_ERR_NOT_IN_STATE) and the state's capacity are checked per feature,
 * in order: such a refusal keeps the landmarks initialised before it. */
int ovp_slam_delayed_init(ovp_ctx *ctx, int F, const int *meas_offset, const int *meas_clone, const float *uv, const double *p_FinG,
                          const double *p_FinG_original, const int64_t *featid, const int64_t *planeid,
                          const ovp_updater_options *opt, int use_plane_constraint, int *feat_status, int *new_handles);
int ovp_slam_handle(ovp_ctx *ctx, int64_t featid);       /* State::_features_SLAM lookup; -1 = absent */
int ovp_slam_should_marg(ovp_ctx *ctx, int64_t featid);  /* Landmark::should_marg (1/0), -1 = absent */
int64_t ovp_slam_plane_of(ovp_ctx *ctx, int64_t featid); /* State::_features_SLAM_to_PLANE entry, -1 = no entry */
/* UpdaterSLAM's options_aruco (UpdaterSLAM.h; UpdaterSLAM.cpp:164, 257, 302-304, 500, 545-547): once set, ovp_slam_update,
 * ovp_slam_delayed_init and ovp_slam_delayed_init_tracks whiten and gate every feature with featid < max_aruco_features (an ArUco tag
 * corner) with these instead of the call's own options: its bearing rows (not its point-on-plane rows, which keep sigma_constraint), its
 * chi2 gates with and without the plane, and in ovp_slam_delayed_init_tracks its single-feature refinement (sigma_pix / fx).  NULL clears
 * them (the default: every feature takes the call's options, and ovp_slam_delayed_init_tracks refuses ArUco ids).  sigma_pix <= 0 or
 * chi2_multipler <= 0: OVP_ERR_BAD_ARGS, the options held before are kept.  Host-only: nothing is copied to the device. */
int ovp_set_aruco_options(ovp_ctx *ctx, const ovp_updater_options *aruco);
/* StateOptions::feat_rep_slam / feat_rep_aruco (state/StateOptions.h; UpdaterSLAM.cpp:231-232), numbered as in
 * ovp_feature_jacobian_representation.  A feature takes feat_rep_aruco when featid < max_aruco_features, feat_rep_slam otherwise.
 * Two setters take them: ovp_set_landmark_representations takes every representation, 0..5; ovp_set_landmark_options is the same setter
 * restricted to 0..4, which it had been before the single-depth form was supported, and keeps refusing 5, so that a host built against that
 * contract keeps getting the refusal it handles.  Once set:
 *  - ovp_slam_update takes landmarks in any of the six representations, each with its own anchor (ovp_slam_get_representation), in one
 *    batch (:476-522, UpdaterHelper.cpp:243-303, 411-420).  A landmark outside GLOBAL_3D that would take its in-state plane
 *    (use_plane_constraint, plane in the state, _features_SLAM_to_PLANE not 0) is refused with OVP_ERR_BAD_ARGS before anything is copied or
 *    launched: the reference's plane constraint asserts GLOBAL_3D (UpdaterHelper.cpp:455-456).  The track limit of such a batch is the
 *    same 29 measurements, the anchor's 6 columns included (a longer track: OVP_ERR_CAPACITY before anything is launched).
 *    ANCHORED_INVERSE_DEPTH_SINGLE (5) is updated as ANCHORED_MSCKF_INVERSE_DEPTH at its p_FinA with H_f's last column as its one state
 *    column and the two bearing columns projected out: 2m - 2 rows, gated with chi2(2m - 2) (:475-479, 503-516, 558-571).
 *  - ovp_slam_delayed_init_tracks creates each landmark in its feature's representation, anchored (2..5) in the clone of the track's last
 *    measurement (camera 0), from the triangulation's p_FinA (:230-304).  A feature outside GLOBAL_3D that would be a plane candidate is
 *    refused up front, as above.
 *  - ovp_slam_delayed_init, which takes p_FinG only, refuses a batch in which any feature takes another representation than GLOBAL_3D.
 * Options {0, 0} behave exactly as none.  NULL clears them (the default: only GLOBAL_3D landmarks are created, and ovp_slam_update refuses
 * any other).  A value outside the setter's range is OVP_ERR_BAD_ARGS, the options held before are kept.  Host-only: nothing is copied to
 * the device. */
typedef struct ovp_landmark_options {
  int feat_rep_slam;
  int feat_rep_aruco;
} ovp_landmark_options;
int ovp_set_landmark_representations(ovp_ctx *ctx, const ovp_landmark_options *o);
int ovp_set_landmark_options(ovp_ctx *ctx, const ovp_landmark_options *o);
/* Landmark::get_xyz(getfej) of a landmark in the state, in any representation: p_FinG for 0 / 1, p_FinA in its anchor's camera for 2..5.
 * A single-depth landmark's value (ovp_var_get) is [rho] alone, as Landmark::value() is; its bearing is p_FinA * rho.  getfej reads the
 * first-estimate row (for 5: uv_norm_zero_fej / rho_fej). */
int ovp_slam_get_xyz(ovp_ctx *ctx, int64_t featid, int getfej, double *p_F);
/* ov_type::Landmark::get_xyz / set_from_xyz as context-free host helpers (no device work), for any representation 0..5: value holds 3
 * doubles (0 / 2 the position, 1 / 3 [theta, phi, rho], 4 [x/z, y/z, 1/z]) or, for 5, [rho, uv_norm_zero] (4 doubles); p_F is p_FinG for 0 / 1
 * and p_FinA for 2..5.  These are the functions the library applies to the rows of its value tables. */
int ovp_landmark_get_xyz(int representation, const double *value, double *p_F);
int ovp_landmark_set_from_xyz(int representation, const double *p_F, double *value);

/* ---- Anchored landmark representations (UpdaterHelper.cpp:35-193, UpdaterSLAM.cpp:684-850) -------------------------------------------- */
/* get_feature_jacobian_full (UpdaterHelper.cpp:195-449) for any ov_type::LandmarkRepresentation (numbering as in
 * ovp_feature_jacobian_representation).  p_F / p_F_fej: p_FinG and its first estimate for the global forms (0, 1), p_FinA for the anchored
 * forms (the first-estimate argument is then unused, :297-301).  The anchor clone is appended to x_order when no measurement was taken
 * from it (:245-264).  No plane rows: the reference's plane constraint asserts GLOBAL_3D (:455-456).  Same output layout as
 * ovp_feature_jacobian_full; H_f has 3 columns (1 for ANCHORED_INVERSE_DEPTH_SINGLE). */
int ovp_feature_jacobian_full_rep(ovp_ctx *ctx, int m, const int *clone_handles, const float *uv, int representation, int anchor_clone_handle,
                                  const double *p_F, const double *p_F_fej, double sigma_px, double *H_f, int *hf_cols, double *H_x, int *hx_cols,
                                  double *res, int *rows_out, int *x_order, int *x_order_n);
/* Landmark::_feat_representation / _anchor_clone_timestamp of a landmark that is in the state: declares how its 3-vector value is read
 * (0 / 2 position, 1 / 3 [theta, phi, rho], 4 [x/z, y/z, 1/z]).  ovp_slam_update takes landmarks declared otherwise once landmark options
 * are set (ovp_set_landmark_options) and refuses them before; ovp_msckf_update_landmarks takes GLOBAL_3D landmarks only.  The setter refuses
 * 5: a landmark of size 3 cannot become one of size 1, and the call carries no bearing; single-depth landmarks come from
 * ovp_slam_delayed_init_tracks, and the getter reports 5 for them. */
int ovp_slam_set_representation(ovp_ctx *ctx, int64_t featid, int representation, int anchor_clone_handle);
int ovp_slam_get_representation(ovp_ctx *ctx, int64_t featid, int *representation, int *anchor_clone_handle);
/* UpdaterSLAM::perform_anchor_change (:706-850): re-express an anchored landmark in another clone's camera frame; covariance through
 * StateHelper::EKFPropagation with the anchor-change Jacobian, value and first estimate re-anchored.  For ANCHORED_INVERSE_DEPTH_SINGLE the
 * Jacobian has one row and takes H_f_new's pseudo-inverse H_f_new^T / |H_f_new|^2 (:802-824); rho and the bearing are both reset from the
 * re-anchored point, in the value and in the first estimate. */
int ovp_slam_perform_anchor_change(ovp_ctx *ctx, int64_t featid, int new_anchor_clone_handle);
/* The host algebra of ovp_slam_perform_anchor_change as a context-free helper (no device work): for a landmark of anchored representation
 * 2..5 with value / first estimate as in ovp_landmark_get_xyz, anchored in the clone [q_GtoI, p_IinG] old7 (first estimate old_fej7), moving to
 * new7 / new_fej7 (same_anchor = 1: the same clone) with extrinsics calib7: Phi (column-major, *phi_rows = the landmark's size, 3 or 1, by
 * *phi_cols) over [old anchor 6][extrinsics 6 when calib_pose][new anchor 6 unless same_anchor][landmark], and the new value / first estimate
 * (set_from_xyz of the re-anchored points).  Phi holds up to 3 x 21 doubles. */
int ovp_anchor_change_jacobian(int representation, int do_fej, int calib_pose, int same_anchor, const double *value, const double *fej,
                               const double *old7, const double *old_fej7, const double *new7, const double *new_fej7, const double *calib7,
                               double *Phi, int *phi_rows, int *phi_cols, double *value_new, double *fej_new);
/* UpdaterSLAM::change_anchors (:684-704): when the clone window is over its limit, every landmark anchored in the clone about to be
 * marginalised (the oldest) moves to the clone at the state time.  *n_changed (optional): how many landmarks moved. */
int ovp_slam_change_anchors(ovp_ctx *ctx, int *n_changed);

/* ---- Multi-GPU sharding of one large update (SURVEY §8(e)) ----------------------------------------------------------- */
/* Rank-local half: Jacobians, nullspace, chi2 gates and compression of THIS rank's point features against the replicated
 * state; writes the (n+1) x (n+1) lower-triangular factor block [R^T ; z^T] in the canonical column order of the FULL batch
 * described by all_clone_handles (every rank passes the same list) to d_out (DEVICE pointer, (n+1)*(n+1) doubles).
 * Global half: stacks G gathered blocks (device pointer, G*(n+1)*(n+1) doubles, e.g. the output of ncclAllGather),
 * re-compresses and runs the EKF update on this ctx. */
int ovp_msckf_shard_columns(ovp_ctx *ctx, const int *all_clone_handles, int n_clones, int *n_cols);
int ovp_msckf_shard_compress(ovp_ctx *ctx, const ovp_feature_batch *batch, const ovp_updater_options *opt,
                             const int *all_clone_handles, int n_clones, double *d_out, int *feat_status, double *feat_chi2);
int ovp_msckf_update_gathered(ovp_ctx *ctx, const double *d_blocks, int G, const int *all_clone_handles, int n_clones);

/* The same update with the collective INSIDE the library (what a C++ host such as VioManager calls): the context owns an NCCL
 * communicator (libnccl.so.2 is dlopen'ed on first use).  Rank 0 obtains a 128-byte id with ovp_nccl_unique_id and hands it to its
 * peers by any means (MPI, a file, a socket); every rank then calls ovp_nccl_init(id, nranks, rank).  ovp_msckf_update_sharded is
 * collective: every rank passes ITS features (F may be 0) and the same all_clone_handles; rank-local Jacobians, gates and Gram
 * matrix, ONE ncclAllGather of the packed lower triangles ((n+1)(n+2)/2 doubles per rank) over NVLink, the sum in rank order
 * (bit-identical on every rank), one compression + EKF update replicated on every rank.  feat_status / feat_chi2: this rank's
 * features. */
int ovp_nccl_unique_id(ovp_ctx *ctx, char id128[128]);
int ovp_nccl_init(ovp_ctx *ctx, const char id128[128], int nranks, int rank);
int ovp_nccl_finalize(ovp_ctx *ctx);
int ovp_msckf_update_sharded(ovp_ctx *ctx, const ovp_feature_batch *local_batch, const ovp_updater_options *opt, const int *all_clone_handles,
                             int n_clones, int *feat_status, double *feat_chi2);

/* ---- Propagator (state/Propagator.cpp) ------------------------------------------------------------------------------- */
int ovp_propagator_set_noise(ovp_ctx *ctx, double sigma_w, double sigma_wb, double sigma_a, double sigma_ab,
                             double gravity_mag);                       /* NoiseManager.h:41-63, Propagator.h:57-64 */
int ovp_propagator_feed_imu(ovp_ctx *ctx, double timestamp, const double wm[3], const double am[3]); /* Propagator.h:71-88 */
/* propagate_and_clone (:37-126): IMU selection + mean (RK4 / discrete) + summed Phi, Qd on the host, then ONE device pass:
 * EKFPropagation + augment_clone.  Phi15 / Q15 (optional, 15x15 col-major) return the summed transition for parity tests. */
int ovp_propagate_and_clone(ovp_ctx *ctx, double timestamp, double *Phi15, double *Q15, int *new_handle);
/* fast_state_propagate (:128-224): IMU-rate odometry prediction on a copy of the IMU marginal; the state is not touched.
 * state_plus13 = [q_GtoI(4) p_IinG(3) v_IinI(3) w_IinI(3)], cov144 = 12 x 12 column-major over [theta p v_local w];
 * *ok = 0 when fewer than two IMU samples cover [state time, timestamp] (the reference returns false). */
int ovp_fast_state_propagate(ovp_ctx *ctx, double timestamp, double *state_plus13, double *cov144, int *ok);

/* ---- Triangulation on the device: the step right before the path (UpdaterMSCKF.cpp:142-194, UpdaterSLAM.cpp:118-160) ---- */
/* ov_core FeatureInitializerOptions (defaults of OpenVINS @74a63cf when opt == NULL) */
typedef struct ovp_triangulation_options {
  int max_runs;
  double init_lamda, max_lamda, min_dx, min_dcost, lam_mult, min_dist, max_dist, max_baseline, max_cond_number;
} ovp_triangulation_options;
/* FeatureInitializer::single_triangulation + single_gaussnewton for F features at once, against the clone and extrinsics values
 * that live in the context: meas_offset / meas_clone as in ovp_feature_batch (measurements in time order: the anchor is the last
 * one), uv_norm = Feature::uvs_norm (undistorted normalised coordinates, 2 floats per measurement).  status[f] = 1: p_FinG[3f..]
 * is the refined position; 0: the reference would drop the feature (condition number, depth range, baseline ratio, NaN).
 * opt == NULL runs the defaults.  Tracks of any length, a clone observed twice included; malformed tracks and a null pointer are refused
 * with OVP_ERR_BAD_ARGS before anything is copied or launched.  The linear stage and whether Gauss-Newton follows are the context's
 * triangulation mode (ovp_set_triangulation_mode): with triangulate_1d, single_triangulation_1d (rejects on depth range and NaN only) instead
 * of single_triangulation; without refine_features, p_FinG is the linear stage's position after that stage's own rules (no baseline-ratio
 * rule, no second depth check).  A feature that fails has status 0 and a zero position in every mode. */
int ovp_triangulate_features(ovp_ctx *ctx, int F, const int *meas_offset, const int *meas_clone, const float *uv_norm,
                             const ovp_triangulation_options *opt, double *p_FinG, int *status);

/* FeatureInitializerOptions::triangulate_1d / refine_features (feat/FeatureInitializerOptions.h), which every updater tests before it
 * triangulates (UpdaterMSCKF.cpp:147-166, UpdaterSLAM.cpp:128-145, UpdaterPlane.cpp:139-160).  ovp_triangulate_features,
 * ovp_plane_init_tracks and ovp_slam_delayed_init_tracks read the mode when they launch.  NULL restores ov_core's defaults {0, 1}, which
 * behave exactly as a context that never called this.  A value other than 0 or 1 is OVP_ERR_BAD_ARGS, the mode held before is kept.
 * Host-only: nothing is copied to the device. */
typedef struct ovp_triangulation_mode {
  int triangulate_1d;  /* single_triangulation_1d instead of single_triangulation */
  int refine_features; /* single_gaussnewton after the linear stage */
} ovp_triangulation_mode;
int ovp_set_triangulation_mode(ovp_ctx *ctx, const ovp_triangulation_mode *m);

/* ---- PlaneFitting (track_plane/PlaneFitting.cpp): plane hypothesis + refinement, the step right before the plane Jacobians ----------- */
/* Call sites: UpdaterMSCKF.cpp:267-360, UpdaterPlane.cpp:230-267, UpdaterSLAM.cpp:171.  Both entry points take a BATCH of candidate planes
 * (feat_offset: n_planes + 1 prefix offsets into the per-feature arrays, starting at 0 and never decreasing, else OVP_ERR_BAD_ARGS) and run
 * them concurrently. */
typedef struct ovp_plane_fit_options {
  int min_inlier_num;     /* StateOptions::plane_msckf_min_feat / plane_init_min_feat */
  double max_cond_number; /* StateOptions::plane_msckf_max_cond / plane_init_max_cond */
  int shuffle_kind;       /* draws of std::shuffle(std::mt19937(8888)) as produced by 0: libstdc++ of GCC 7..10 (the reference's Docker
                             images), 1: libstdc++ of GCC >= 11 (std::uniform_int_distribution changed) */
} ovp_plane_fit_options;
/* PlaneFitting::plane_fitting (:83-195): RANSAC over 200 five-point sets (points >= 0.05 m apart, condition number of the 5 x 3 system
 * <= max_cond_number), inliers within 0.05 m, winner = most inliers then smallest mean error, refit on its inliers.  status[p] = 1:
 * abcd[4p..] is the plane (unit normal, offset) and inlier[f] flags the features the reference keeps in `feats`; 0: the reference returns
 * false (too few points, a draw with fewer than five separated points, no valid set). */
int ovp_plane_fitting(ovp_ctx *ctx, int n_planes, const int *feat_offset, const double *p_FinG, const ovp_plane_fit_options *opt, int *status,
                      double *abcd, int *inlier);
/* The n_shuffles successive permutations of 0..n-1 the reference's RANSAC loop draws (context-free host helper; needs no GPU). */
int ovp_plane_shuffle(int n, int n_shuffles, int shuffle_kind, int *out);
typedef struct ovp_plane_refine_options {
  double sigma_px_norm;   /* sigma_pix / focal length (UpdaterMSCKF.cpp:271-272) */
  double sigma_c;         /* StateOptions::sigma_constraint */
  int max_num_iterations; /* 0 = the reference's 12 (PlaneFitting.cpp:396) */
} ovp_plane_refine_options;
/* PlaneFitting::optimize_plane (:197-514): joint refinement of the features of each plane (and of the plane unless fix_plane[p]) over
 * reprojection + point-on-plane factors with the Cauchy loss, Ceres' dogleg trust-region iteration restated on the device (one launch for
 * the whole batch).  Measurements as in ovp_triangulate_features (clone handles, undistorted normalised coordinates); a feature without
 * measurements is a SLAM feature: constant, one constraint with 2 sigma_c.  Camera poses, the current IMU pose and the extrinsics come from
 * the context.  status[p] = 1: success; p_FinG_out holds the refined positions of the inliers (others unchanged), cp_out the refined plane,
 * inlier[f] the kept features.  status[p] = 0 with cp_out == cp_inG: the solver did not converge within the iteration limit (nothing
 * changed); status[p] = 0 otherwise: too few inliers (positions / plane were already updated, like the reference's side effects).
 * info (optional, 5 doubles per plane): converged, iterations, initial cost, final cost, termination reason (1 gradient, 2 parameter,
 * 3 function tolerance, 4 no free parameter, -1 iteration limit, -2 invalid steps). */
int ovp_optimize_plane(ovp_ctx *ctx, int n_planes, const int *feat_offset, const int *meas_offset, const int *meas_clone, const float *uv_norm,
                       const double *p_FinG, const double *cp_inG, const int *fix_plane, const ovp_plane_refine_options *opt, double *p_FinG_out,
                       double *cp_out, int *inlier, int *status, double *info);

/* ---- UpdaterPlane::init_vio_plane end to end (UpdaterPlane.cpp:61-481): new planes from raw feature tracks ------------------------------ */
/* The caller's Feature objects after clean_old_measurements against the clone times, flattened: measurements in time order, clone handles,
 * raw pixels (for the Jacobians) and undistorted normalised coordinates (for triangulation and refinement). */
typedef struct ovp_feature_tracks {
  int F;
  const int *meas_offset; /* F+1 prefix offsets into the measurement arrays */
  const int *meas_clone;  /* clone handle per measurement */
  const float *uv;        /* Feature::uvs (raw pixels), 2 per measurement */
  const float *uv_norm;   /* Feature::uvs_norm, 2 per measurement */
  const int64_t *featid;  /* F, distinct */
  const int64_t *planeid; /* F: feat2plane entry, 0 = none */
} ovp_feature_tracks;
typedef struct ovp_plane_init_options {
  double sigma_pix;                     /* UpdaterOptions::sigma_pix of the MSCKF updater */
  int max_msckf_plane;                  /* StateOptions: a plane keeps its max_msckf_plane + 1 shortest tracks (UpdaterPlane.cpp:189) */
  int plane_init_min_feat;              /* StateOptions: RANSAC's inlier minimum */
  double plane_init_max_cond;           /* StateOptions: RANSAC's condition-number limit */
  int shuffle_kind;                     /* as ovp_plane_fit_options */
  const ovp_triangulation_options *tri; /* NULL = OpenVINS defaults */
} ovp_plane_init_options;
/* Candidates are the features on a plane that is not in the state; those with fewer than two measurements are dropped, the others are
 * triangulated, sorted by track length with std::sort (ascending, not stable), grouped per plane under the cap, fitted by RANSAC
 * (plane_init_min_feat / plane_init_max_cond) and refined jointly with the plane free (sigma_pix / fx of the current intrinsics,
 * sigma_constraint); every plane that obtained a linearisation point is then initialised like ovp_plane_init, ascending id.
 * The measurements cross to the device once; between stages only statuses, inlier flags and the refined plane come back.
 * The triangulation runs in the context's mode (ovp_set_triangulation_mode): the linear stage it selects, then Gauss-Newton when
 * refine_features.  feat_status[F]: -1 fewer than 2 measurements (erase it from feature_vec), -2 the selected triangulation stage failed
 * (keep it), 0 not a candidate, 2 candidate not consumed, 1 consumed by an initialised plane (to_delete, moved to feature_vec_used).
 * p_FinG_out[3F]: triangulated position (for -2, whatever the failed triangulation produced, as the reference leaves it in the Feature), or
 * the refinement's output for the features that went into a refinement; zero for features with status 0 or -1.  Plane outputs, sized F entries by the caller (at most one plane per feature): *n_planes planes, every plane
 * with a candidate after triangulation, ascending id; plane_status 1 initialised, 0 rejected by initialize's chi2, -2 RANSAC returned false,
 * -3 optimize_plane returned false, -1 not attempted (fewer than 3 features left); new_handles (or -1); cp_out[3 * n_planes] the
 * linearisation point handed to initialize (the refinement's plane, zero when RANSAC failed).
 * Refused before anything is copied or launched, with the state untouched: a null pointer, malformed tracks (a candidate's per-track rules
 * only), a duplicate featid, OVP_ERR_CAPACITY for a candidate
 * track longer than the plane-system limit (37, see ovp_msckf_update) or max_msckf_plane + 1 above RANSAC's 1900 points.  The capacities of
 * the initialisation stage itself (rows of one plane's stacked system against max_meas_rows, three more state rows per new plane against
 * max_state) depend on RANSAC's and the refinement's outcome and are checked by that stage as in ovp_plane_init: such a refusal comes after
 * the plane-fitting launches, leaves the plane it concerns (and the later ones) uninitialised, and keeps the planes initialised before it. */
int ovp_plane_init_tracks(ovp_ctx *ctx, const ovp_feature_tracks *t, const ovp_plane_init_options *opt, int *feat_status, double *p_FinG_out,
                          int *n_planes, int64_t *plane_ids, int *plane_status, int *new_handles, double *cp_out);

/* ---- UpdaterSLAM::delayed_init end to end (UpdaterSLAM.cpp:66-374): new SLAM landmarks from raw feature tracks ---------------------------- */
typedef struct ovp_slam_init_options {
  double sigma_pix;                     /* UpdaterOptions::sigma_pix of the SLAM updater */
  double chi2_multipler;                /* UpdaterOptions::chi2_multipler of the SLAM updater */
  int use_plane_constraint;             /* StateOptions::use_plane_constraint && use_plane_constraint_slamd */
  int use_refine_plane_feat;            /* StateOptions::use_refine_plane_feat */
  const ovp_triangulation_options *tri; /* NULL = OpenVINS defaults */
} ovp_slam_init_options;
/* Longest track ovp_slam_delayed_init_tracks takes: the limit of a single feature's Jacobian (triangulation and refinement have none) */
#define OVP_SLAM_INIT_MAX_TRACK 64
/* Tracks as ovp_plane_init_tracks takes them (cleaned against the clone times; uv for the Jacobians, uv_norm for triangulation and
 * refinement).  In the reference's order: a track with fewer than two measurements is erased; the others are triangulated in one launch;
 * a feature whose plane is in the state, with use_plane_constraint and use_refine_plane_feat set and _features_SLAM_to_PLANE[featid] absent
 * or non-zero, is a refinement candidate: every candidate is refined onto its plane (plane fixed at its current value, sigma_pix / fx of
 * the current intrinsics) in one launch, whether or not its triangulation succeeded (the reference refines first, :147-193).  A successful
 * refinement sets _features_SLAM_to_PLANE[featid] to the plane id; a failed one sets it to 0 when the triangulation succeeded (:195-200).
 * Then, per triangulated feature in input order, the initialisation of ovp_slam_delayed_init: with the plane from the refined position,
 * or without it from the triangulated position when the refinement failed; after a chi2 rejection with the plane, once more without it
 * from the triangulated position.  The measurements cross to the device once and the Jacobians read them there; statuses and positions
 * come back once before the initialisations.
 * feat_status[F]: -1 fewer than 2 measurements, -2 triangulation failed, 0 not initialised, 1 initialised (with its plane constraint when it
 * had one), 3 initialised after its plane was dropped for chi2.  plane_status[F] (may be NULL): -1 not a refinement candidate, 1 refined
 * onto its plane, 0 refinement failed.  p_FinG_out[3F]: what the reference leaves in Feature::p_FinG (the refined position for a refined
 * feature, also for status 3, whose landmark holds the triangulated one; zero for -1).  new_handles[F]: the landmark's handle, or -1.
 * The triangulation runs in the context's mode (ovp_set_triangulation_mode); -2 means that the selected stage failed.
 * Without landmark options only GLOBAL_3D landmarks are created.  With them (ovp_set_landmark_options / ovp_set_landmark_representations)
 * each landmark is created in its feature's representation: 2..5 anchored in the clone of the track's last measurement with the value and
 * first estimate set_from_xyz of the triangulation's p_FinA (the mode's: the linear stage's p_FinA without refine_features, the refined one
 * with it), 1 from p_FinG, with the Jacobians of ovp_feature_jacobian_full_rep (ovp_slam_get_representation reads both).
 * ANCHORED_INVERSE_DEPTH_SINGLE (5) takes the Jacobians of ANCHORED_MSCKF_INVERSE_DEPTH, projects H_f's two bearing columns out of
 * [H_x | H_rho | r] and initialises a landmark of size 1 from the remaining 2m - 2 rows, chi2 with 2m - 2 dof (UpdaterSLAM.cpp:260-283);
 * its value is rho = 1/z and it keeps its initial bearing (ovp_slam_get_xyz).
 * Refused before anything is copied or launched, with the state untouched: a null pointer, malformed tracks (the per-track rules for the
 * tracks of two or more measurements), a duplicate featid, a featid that already has a landmark (OVP_ERR_ALREADY_IN_STATE), a featid below
 * max_aruco_features while no ArUco options are set (ovp_set_aruco_options; with them tags are accepted), a feature outside GLOBAL_3D that
 * would be a refinement or plane candidate (use_plane_constraint, its plane in the state, _features_SLAM_to_PLANE absent or not 0: the
 * reference asserts GLOBAL_3D there, UpdaterHelper.cpp:455-456), a chi2 table too short for the
 * rows of a feature (3 per measurement with a plane, 2 without), sigma_pix <= 0, and OVP_ERR_CAPACITY for a track longer than
 * OVP_SLAM_INIT_MAX_TRACK (64).  The state and row capacities of an initialisation depend on which features pass and are checked per
 * feature as in ovp_slam_delayed_init: such a refusal comes after the launches and keeps the landmarks initialised before it. */
int ovp_slam_delayed_init_tracks(ovp_ctx *ctx, const ovp_feature_tracks *t, const ovp_slam_init_options *opt, int *feat_status, int *plane_status,
                                 double *p_FinG_out, int *new_handles);

/* ---- UpdaterZeroVelocity (update/UpdaterZeroVelocity.cpp:68-318) ------------------------------------------------------- */
typedef struct ovp_zupt_options {
  double gravity_mag;           /* VioManagerOptions.h:206 */
  double zupt_max_velocity;     /* reject when |v_IinG| is above (unless the disparity check passes) */
  double zupt_noise_multiplier; /* R *= multiplier (:176-178) */
  double zupt_max_disparity;    /* average pixel disparity below which the platform counts as stationary (:219) */
  double chi2_multipler;        /* UpdaterOptions::chi2_multipler */
} ovp_zupt_options;
/* UpdaterZeroVelocity::feed_imu: the ZUPT updater keeps its own IMU buffer (noises: ovp_propagator_set_noise) */
int ovp_zupt_feed_imu(ovp_ctx *ctx, double timestamp, const double wm[3], const double am[3]);
/* try_update: average_disparity / num_features are the outputs of FeatureHelper::compute_disparity between the state time and
 * `timestamp` (front end, upstream).  *accepted = 1: the zero-velocity update was applied (bias propagation + EKFUpdate with the
 * diagonal R) and the state time moved to `timestamp`; 0: nothing was touched, do the normal propagate + clone. */
int ovp_zupt_try_update(ovp_ctx *ctx, const ovp_zupt_options *opt, double timestamp, double average_disparity, int num_features,
                        int *accepted, double *chi2);

/* Split form of ovp_msckf_update for callers that keep one feature batch resident on the device: prepare = validation,
 * planning and the single host->device copy; launch = kernels only (asynchronous, repeatable: the state changes, the plan
 * does not); finish = device->host read of the gates and Hx_order.  ovp_msckf_update == prepare + launch + finish. */
int ovp_msckf_prepare(ovp_ctx *ctx, const ovp_feature_batch *batch, const ovp_updater_options *opt);
/* prepare of ovp_msckf_update_landmarks; the member list is part of the plan, and members' values are read on the device */
int ovp_msckf_prepare_landmarks(ovp_ctx *ctx, const ovp_feature_batch *batch, const ovp_plane_landmarks *landmarks,
                                const ovp_updater_options *opt);
int ovp_msckf_launch(ovp_ctx *ctx);
int ovp_msckf_finish(ovp_ctx *ctx, int *feat_status, double *feat_chi2, int *plane_status, double *plane_chi2, int *hx_order,
                     int *hx_order_n);
/* device-side copy of (covariance, values, first-estimates) and its restore; the variable table must be unchanged */
int ovp_snapshot(ovp_ctx *ctx);
int ovp_restore(ovp_ctx *ctx);

/* ---- instrumentation -------------------------------------------------------------------------------------------------- */
/* number of kernel launches issued by this ctx since creation (bench.py's gpu_launches) */
int64_t ovp_launch_count(ovp_ctx *ctx);
/* CUDA stream the ctx launches on (as an opaque pointer) so that callers can time with events on the right stream */
void *ovp_stream(ovp_ctx *ctx);
/* device-resident timing of the last ovp_msckf_update, ms: [0] total, [1] feature kernels, [2] gram+compress, [3] ekf update */
int ovp_last_timing(ovp_ctx *ctx, double *ms4);
int ovp_synchronize(ovp_ctx *ctx);
/* per-kernel timing with CUDA events on the launch stream: classes [0] DMMA gemm, [1] gram, [2] diagonal-block Cholesky,
 * [3] feature kernel, [4] other; report = total ms, launch count and algorithmic work (flops; bytes for [3]) since enabled */
int ovp_set_profiling(ovp_ctx *ctx, int on);
int ovp_profile_report(ovp_ctx *ctx, double *ms5, int64_t *count5, double *work5);
/* 1 (default): the static launch sequence of a prepared batch is captured into a CUDA graph and replayed */
int ovp_set_use_graphs(ovp_ctx *ctx, int on);
/* Zero-pivot rule of the measurement compression (Cholesky of the stacked Gram matrix, DESIGN.md §4): a pivot <= tol * (the
 * column's original diagonal entry) marks a rank-deficient (gauge) direction and is dropped.  Default 1e-11; the posterior is
 * invariant over 1e-9 .. 1e-13 on every scenario in tests/ (tests/test_gpu_numerics.py). */
int ovp_set_rank_tolerance(ovp_ctx *ctx, double tol);
/* Widest system (columns of a compressed update's Gram matrix, rows of an innovation system) one update may factor.  0 (the default):
 * the co-resident width of one fused launch on this device (T(T+1)/2 <= co-resident CTAs: 960 on an H100), and wider systems are refused
 * exactly as before.  A larger width, up to the context's column capacity (max_state rounded up to 64, plus 64), lets wider systems run:
 * they are factored in panels (DESIGN.md 4.1).  Systems within the co-resident width run the same launches and give the same bits
 * whatever is declared.  Out of range: OVP_ERR_BAD_ARGS, the width held before is kept.  Changing it drops a prepared batch's graph. */
int ovp_set_max_update_width(ovp_ctx *ctx, int width);
/* the declared width (after 0 is resolved) and the co-resident width of one fused launch on this device */
int ovp_max_update_width(ovp_ctx *ctx, int *width, int *coresident_width);
/* bytes this ctx copied host->device / device->host since creation: every host<->device copy the library issues for the ctx (operands,
 * results, column indices, variable tables and values, status words) is counted */
int ovp_transfer_bytes(ovp_ctx *ctx, int64_t *h2d, int64_t *d2h);
/* measured FP64 tensor-core (DMMA) throughput of this device with the library's own GEMM kernel: returns TFLOP/s */
int ovp_selftest_dgemm_tflops(ovp_ctx *ctx, int n, int iters, double *tflops);

#ifdef __cplusplus
}
#endif
#endif /* OVP_H */

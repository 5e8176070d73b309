// Anchored landmark representations on the path (reference: update/UpdaterHelper.cpp:35-193 get_feature_jacobian_representation, :195-449 the
// chain rule inside get_feature_jacobian_full; update/UpdaterSLAM.cpp:684-704 change_anchors, :706-850 perform_anchor_change).
//
//   ovp_feature_jacobian_full_rep : get_feature_jacobian_full for any of the six ov_type::LandmarkRepresentation values.  The bearing rows
//       (w dz/dp_FinG, clone / extrinsics / intrinsics blocks) come from the same device kernel as the GLOBAL_3D path; one more launch applies the
//       chain rule per row: H_f = (w dz/dp_FinG) dpfg_dlambda, H_x[anchor] += (w dz/dp_FinG) dpfg_danchor, H_x[calib] += (w dz/dp_FinG) dpfg_dcalib
//       (UpdaterHelper.cpp:411-420).  The three small matrices are per-feature constants (3x3 host algebra, ovp_feature_jacobian_representation).
//   ovp_slam_set_representation / ovp_slam_get_representation : Landmark::_feat_representation + _anchor_clone_timestamp of a landmark in the state.
//   ovp_slam_perform_anchor_change / ovp_slam_change_anchors : the anchor-change Jacobian Phi (3 x [old anchor, extrinsics, new anchor, landmark]) on
//       the host, StateHelper::EKFPropagation on the device (ovp_ekf_propagation), new value / first estimate of the landmark.
//   ovp_set_landmark_representations (0..5) / ovp_set_landmark_options (0..4) : StateOptions::feat_rep_slam / feat_rep_aruco.  Once set,
//       ovp_slam_update takes landmarks in those representations (feature_kernel<true, true>, features.cu: the same chain rule on the device,
//       its terms from the device value table) and ovp_slam_delayed_init_tracks creates them (slam_delayed_init_core, through
//       stage_feature_jacobian_rep below).  ANCHORED_INVERSE_DEPTH_SINGLE is a landmark of size 1 that keeps its initial bearing in slots 1..3
//       of its value / first-estimate rows (landmark_get_xyz below); the update and the initialisation take it as ANCHORED_MSCKF_INVERSE_DEPTH
//       with H_f's two bearing columns projected out, the anchor change with a one-row Phi.
//   ovp_slam_get_xyz : Landmark::get_xyz of a landmark in any representation.
// Out of scope: the MSCKF entry points (ovp_msckf_update, ovp_msckf_update_landmarks) stay GLOBAL_3D as the reference asserts
// (UpdaterMSCKF.cpp:250, 662), and so does any landmark on an in-state plane (the plane constraint asserts it, UpdaterHelper.cpp:455-456).
namespace ovp {

// per row r of the 2m bearing rows: raw = Hf[r, 0:3] (= w dz/dp_FinG); Hf[r, 0:k] = raw L; Hx[r, anchor cols] += raw Ha; Hx[r, calib cols] += raw Hc
struct RepChainArgs {
  double *Hf, *Hx;
  int rows, k, anchor_col, calib_col; // column offsets in Hx (-1: none)
  double L[9], Ha[18], Hc[18];        // column-major 3 x k, 3 x 6, 3 x 6
};
__global__ void representation_chain_kernel(RepChainArgs a) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.rows)
    return;
  const int ld = a.rows;
  const double raw[3] = {a.Hf[r], a.Hf[(size_t)ld + r], a.Hf[2 * (size_t)ld + r]};
  for (int j = 0; j < 3; j++)
    a.Hf[(size_t)j * ld + r] = (j < a.k) ? raw[0] * a.L[3 * j] + raw[1] * a.L[3 * j + 1] + raw[2] * a.L[3 * j + 2] : 0.0;
  if (a.anchor_col >= 0)
    for (int j = 0; j < 6; j++)
      a.Hx[(size_t)(a.anchor_col + j) * ld + r] += raw[0] * a.Ha[3 * j] + raw[1] * a.Ha[3 * j + 1] + raw[2] * a.Ha[3 * j + 2];
  if (a.calib_col >= 0)
    for (int j = 0; j < 6; j++)
      a.Hx[(size_t)(a.calib_col + j) * ld + r] += raw[0] * a.Hc[3 * j] + raw[1] * a.Hc[3 * j + 1] + raw[2] * a.Hc[3 * j + 2];
}

// ov_type::Landmark::get_xyz / set_from_xyz (ov_core @74a63cf, not in the tree): how the value a landmark stores maps to a position.
// Representations 0 / 2 store the position, 1 / 3 [theta, phi, rho] (spherical, rho = 1 / range), 4 [x/z, y/z, 1/z].  Representation 5 is a
// Landmark of size 1: its value is rho = 1/z in the anchor camera, and it carries the bearing it was set from, uv_norm_zero = rho p_FinA =
// [x/z, y/z, 1], in slots 1..3 of its value row (the first-estimate copy uv_norm_zero_fej in those of its first-estimate row); get_xyz is
// uv_norm_zero / rho, and set_from_xyz resets rho and the bearing.  The EKF update moves slot 0 only (its size is 1), so the bearing stays.
static bool landmark_get_xyz(int rep, const double *v, double *p) {
  if (rep == 5) {
    p[0] = v[1] / v[0], p[1] = v[2] / v[0], p[2] = v[3] / v[0];
  } else if (rep == 0 || rep == 2) {
    p[0] = v[0], p[1] = v[1], p[2] = v[2];
  } else if (rep == 4) {
    p[0] = v[0] / v[2], p[1] = v[1] / v[2], p[2] = 1.0 / v[2];
  } else if (rep == 1 || rep == 3) {
    p[0] = (1.0 / v[2]) * std::cos(v[0]) * std::sin(v[1]);
    p[1] = (1.0 / v[2]) * std::sin(v[0]) * std::sin(v[1]);
    p[2] = (1.0 / v[2]) * std::cos(v[1]);
  } else {
    return false;
  }
  return true;
}
static bool landmark_set_from_xyz(int rep, const double *p, double *v) {
  if (rep == 5) {
    const double rho = 1.0 / p[2];
    v[0] = rho, v[1] = rho * p[0], v[2] = rho * p[1], v[3] = rho * p[2];
  } else if (rep == 0 || rep == 2) {
    v[0] = p[0], v[1] = p[1], v[2] = p[2];
  } else if (rep == 4) {
    v[0] = p[0] / p[2], v[1] = p[1] / p[2], v[2] = 1.0 / p[2];
  } else if (rep == 1 || rep == 3) {
    const double g_rho = 1.0 / std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    v[0] = std::atan2(p[1], p[0]);
    v[1] = std::acos(g_rho * p[2]);
    v[2] = g_rho;
  } else {
    return false;
  }
  return true;
}
static void inverse3(const double *A, double *Ai) { // column-major 3x3, Gauss-Jordan with partial pivoting (stand-in for colPivHouseholderQr().solve(I))
  double M[3][6];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      M[i][j] = A[3 * j + i];
      M[i][3 + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int k = 0; k < 3; k++) {
    int p = k;
    for (int i = k + 1; i < 3; i++)
      if (std::fabs(M[i][k]) > std::fabs(M[p][k]))
        p = i;
    if (p != k)
      for (int j = 0; j < 6; j++)
        std::swap(M[k][j], M[p][j]);
    const double d = M[k][k];
    for (int j = 0; j < 6; j++)
      M[k][j] /= d;
    for (int i = 0; i < 3; i++)
      if (i != k) {
        const double f = M[i][k];
        for (int j = 0; j < 6; j++)
          M[i][j] -= f * M[k][j];
      }
  }
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      Ai[3 * j + i] = M[i][3 + j];
}
static bool is_relative(int rep) { return rep >= 2 && rep <= 5; }
// slots 1..3 of landmark h's value and first-estimate rows := b, the bearing of a single-depth landmark (slot 0, rho, is kept): written into
// the host mirror and copied to the same three slots of each device row, so that nothing else of either table is read back or rewritten
static int landmark_store_bearing(Ctx *c, int h, const double *b) {
  const size_t at = (size_t)h * OVP_VAL_STRIDE + 1;
  for (int i = 0; i < 3; i++)
    c->h_val[at + i] = c->h_fej[at + i] = b[i];
  int st;
  if ((st = stage_copy_in(c, c->d_val + at, c->h_val.data() + at, 3 * sizeof(double))) ||
      (st = stage_copy_in(c, c->d_fej + at, c->h_fej.data() + at, 3 * sizeof(double))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream)); // the copies read the host mirror, which a later append may reallocate
  return OVP_OK;
}

// get_feature_jacobian_full of one feature in representation rep on the staging buffer (FeatureJacobianStage layout, H_f with *k columns):
// the bearing rows of stage_feature_jacobian at p_FinG, then representation_chain_kernel (UpdaterHelper.cpp:411-420) with the 3x3 terms of
// ovp_feature_jacobian_representation on the host values.  p_F / p_F_fej: p_FinG and its first estimate for reps 0 / 1, p_FinA for the
// anchored ones.  *extra = 6 when no measurement was taken from the anchor: its columns follow the clones' in H_x.  dev: as for
// stage_feature_jacobian.  Shared by ovp_feature_jacobian_full_rep and the initialisations of slam_delayed_init_core.
static int stage_feature_jacobian_rep(Ctx *c, int m, const int *clone_handles, const float *uv, int representation, int anchor_clone_handle,
                                      const double *p_F, const double *p_F_fej, double sigma_px, FeatureJacobianStage *jo, int *k_out,
                                      int *extra_out, const DeviceTrack *dev) {
  const bool rel = is_relative(representation);
  int st = sync_host_values(c);
  if (st)
    return st;
  double pG[3] = {p_F[0], p_F[1], p_F[2]}, pGf[3] = {p_F_fej[0], p_F_fej[1], p_F_fej[2]};
  const double *cal = c->h_val.data() + (size_t)c->h_calib * OVP_VAL_STRIDE;
  const double *anc = rel ? c->h_val.data() + (size_t)anchor_clone_handle * OVP_VAL_STRIDE : nullptr;
  const double *ancf = rel ? c->h_fej.data() + (size_t)anchor_clone_handle * OVP_VAL_STRIDE : nullptr;
  if (rel) { // p_FinG = R_GtoI^T R_ItoC^T (p_FinA - p_IinC) + p_IinG; the FEJ copy is the same point (UpdaterHelper.cpp:281-301)
    double RC[9], RI[9], t[3], u[3];
    quat_to_rot(cal, RC);
    quat_to_rot(anc, RI);
    for (int i = 0; i < 3; i++)
      t[i] = p_F[i] - cal[4 + i];
    for (int i = 0; i < 3; i++)
      u[i] = RC[i] * t[0] + RC[3 + i] * t[1] + RC[6 + i] * t[2]; // R_ItoC^T t
    for (int i = 0; i < 3; i++)
      pG[i] = RI[i] * u[0] + RI[3 + i] * u[1] + RI[6 + i] * u[2] + anc[4 + i];
    for (int i = 0; i < 3; i++)
      pGf[i] = pG[i];
  }
  RepChainArgs a;
  int k = 3, has_anchor = 0;
  st = ovp_feature_jacobian_representation(representation, c->opt.do_fej, pG, pGf, rel ? p_F : nullptr, anc, ancf, cal, a.L, &k, a.Ha, a.Hc, &has_anchor);
  if (st)
    return fail(c, st, "feature_jacobian_full_rep: representation Jacobian failed");
  int anchor_k = -1; // measurement index whose clone is the anchor
  for (int i = 0; i < m && rel; i++)
    if (clone_handles[i] == anchor_clone_handle)
      anchor_k = i;
  const int extra = (rel && anchor_k < 0) ? 6 : 0;
  FeatureJacobianStage &j = *jo;
  st = stage_feature_jacobian(c, m, clone_handles, uv, pG, pGf, false, -1, nullptr, nullptr, sigma_px, 1.0, &j, extra, dev);
  if (st)
    return st;
  const int ncal_pose = c->opt.do_calib_camera_pose ? 6 : 0, ncal = ncal_pose + (c->opt.do_calib_camera_intrinsics ? 8 : 0);
  a.Hf = j.W(c);
  a.Hx = j.Hx(c);
  a.rows = j.rows;
  a.k = k;
  a.anchor_col = rel ? (anchor_k >= 0 ? ncal + 6 * anchor_k : ncal + 6 * m) : -1;
  a.calib_col = (rel && ncal_pose) ? 0 : -1;
  if (!rel)
    for (int i = 0; i < 18; i++)
      a.Ha[i] = a.Hc[i] = 0.0;
  representation_chain_kernel<<<(j.rows + 63) / 64, 64, 0, c->stream>>>(a);
  c->launches++;
  OVP_CUDA(cudaGetLastError());
  *k_out = k;
  *extra_out = extra;
  return OVP_OK;
}

} // namespace ovp

extern "C" {

int ovp_feature_jacobian_full_rep(ovp_ctx *h, int m, const int *clone_handles, const float *uv, int representation, int anchor_clone_handle,
                                  const double *p_F, const double *p_F_fej, double sigma_px, double *H_f, int *hf_cols, double *H_x, int *hx_cols,
                                  double *res, int *rows_out, int *x_order, int *x_order_n) {
  using namespace ovp;
  Ctx *c = ovp::enter(h);
  if (representation < 0 || representation > 5 || !p_F || !p_F_fej || !H_f || !H_x || !res)
    return fail(c, OVP_ERR_BAD_ARGS, "feature_jacobian_full_rep: bad representation / null argument");
  const bool rel = is_relative(representation);
  if (rel && !is_clone(c, anchor_clone_handle, true))
    return fail(c, OVP_ERR_BAD_ARGS, "feature_jacobian_full_rep: anchor handle %d is not a clone in the state", anchor_clone_handle);
  int st = check_jacobian_track(c, "feature_jacobian_full_rep", m, clone_handles);
  if (st)
    return st;
  FeatureJacobianStage j;
  int k = 3, extra = 0;
  if ((st = stage_feature_jacobian_rep(c, m, clone_handles, uv, representation, anchor_clone_handle, p_F, p_F_fej, sigma_px, &j, &k, &extra)))
    return st;
  if ((st = read_feature_jacobian(c, j, k, H_f, H_x, res)))
    return st;
  *hf_cols = k;
  *hx_cols = j.hxc;
  *rows_out = j.rows;
  int no = 0;
  if (c->opt.do_calib_camera_pose)
    x_order[no++] = c->h_calib;
  if (c->opt.do_calib_camera_intrinsics)
    x_order[no++] = c->h_intr;
  for (int i = 0; i < m; i++)
    x_order[no++] = clone_handles[i];
  if (extra)
    x_order[no++] = anchor_clone_handle;
  *x_order_n = no;
  return OVP_OK;
}

int ovp_set_landmark_representations(ovp_ctx *h, const ovp_landmark_options *o) {
  using namespace ovp;
  Ctx *c = &h->c; // host-only: the update reads each landmark's representation from the host table when it stages a batch
  if (!o) {
    c->has_lm_rep = false;
    return OVP_OK;
  }
  const int r[2] = {o->feat_rep_slam, o->feat_rep_aruco};
  for (int i = 0; i < 2; i++)
    if (r[i] < 0 || r[i] > 5)
      return fail(c, OVP_ERR_BAD_ARGS, "set_landmark_representations: %s = %d is not a representation (0..5)", i ? "feat_rep_aruco" : "feat_rep_slam",
                  r[i]);
  c->lm_rep = *o;
  c->has_lm_rep = true;
  return OVP_OK;
}

int ovp_set_landmark_options(ovp_ctx *h, const ovp_landmark_options *o) {
  using namespace ovp;
  Ctx *c = &h->c;
  const int r[2] = {o ? o->feat_rep_slam : 0, o ? o->feat_rep_aruco : 0};
  for (int i = 0; i < 2; i++) {
    if (r[i] == 5)
      return fail(c, OVP_ERR_BAD_ARGS, "set_landmark_options: %s = 5 (ANCHORED_INVERSE_DEPTH_SINGLE) is not supported: the landmark would have to "
                  "carry the bearing it was initialised with", i ? "feat_rep_aruco" : "feat_rep_slam");
    if (r[i] < 0 || r[i] > 4)
      return fail(c, OVP_ERR_BAD_ARGS, "set_landmark_options: %s = %d is not a representation (0..4)", i ? "feat_rep_aruco" : "feat_rep_slam", r[i]);
  }
  return ovp_set_landmark_representations(h, o);
}

int ovp_slam_get_xyz(ovp_ctx *h, int64_t featid, int getfej, double *p_F) {
  using namespace ovp;
  Ctx *c = ovp::enter(h);
  auto it = c->slam.find(featid);
  if (it == c->slam.end() || c->vars[it->second].id < 0)
    return fail(c, OVP_ERR_NOT_IN_STATE, "slam_get_xyz: feature %lld has no landmark in the state", (long long)featid);
  if (!p_F)
    return fail(c, OVP_ERR_BAD_ARGS, "slam_get_xyz: null argument");
  int st = sync_host_values(c);
  if (st)
    return st;
  const std::vector<double> &t = getfej ? c->h_fej : c->h_val;
  landmark_get_xyz(c->vars[it->second].rep, t.data() + (size_t)it->second * OVP_VAL_STRIDE, p_F);
  return OVP_OK;
}

int ovp_slam_set_representation(ovp_ctx *h, int64_t featid, int representation, int anchor_clone_handle) {
  using namespace ovp;
  Ctx *c = ovp::enter(h);
  auto it = c->slam.find(featid);
  if (it == c->slam.end() || c->vars[it->second].id < 0)
    return fail(c, OVP_ERR_NOT_IN_STATE, "slam_set_representation: feature %lld has no landmark in the state", (long long)featid);
  if (representation < 0 || representation > 4)
    return fail(c, OVP_ERR_BAD_ARGS, "slam_set_representation: representation %d (0..4; a single-depth landmark is created with its bearing by "
                                     "ovp_slam_delayed_init_tracks)", representation);
  if (c->vars[it->second].size != 3) // a single-depth landmark (size 1) cannot take a 3-vector form
    return fail(c, OVP_ERR_BAD_ARGS, "slam_set_representation: landmark %lld has size %d; representations 0..4 hold 3 values",
                (long long)featid, c->vars[it->second].size);
  if (is_relative(representation) && !is_clone(c, anchor_clone_handle, true))
    return fail(c, OVP_ERR_BAD_ARGS, "slam_set_representation: anchor handle %d is not a clone in the state", anchor_clone_handle);
  c->vars[it->second].rep = representation;
  c->vars[it->second].anchor = is_relative(representation) ? anchor_clone_handle : -1;
  return OVP_OK;
}
int ovp_slam_get_representation(ovp_ctx *h, int64_t featid, int *representation, int *anchor_clone_handle) {
  using namespace ovp;
  Ctx *c = &h->c;
  auto it = c->slam.find(featid);
  if (it == c->slam.end())
    return fail(c, OVP_ERR_NOT_IN_STATE, "slam_get_representation: feature %lld has no landmark", (long long)featid);
  if (representation)
    *representation = c->vars[it->second].rep;
  if (anchor_clone_handle)
    *anchor_clone_handle = c->vars[it->second].anchor;
  return OVP_OK;
}

int ovp_landmark_get_xyz(int representation, const double *value, double *p_F) {
  if (!value || !p_F)
    return OVP_ERR_BAD_ARGS;
  return ovp::landmark_get_xyz(representation, value, p_F) ? OVP_OK : OVP_ERR_BAD_ARGS;
}
int ovp_landmark_set_from_xyz(int representation, const double *p_F, double *value) {
  if (!value || !p_F)
    return OVP_ERR_BAD_ARGS;
  return ovp::landmark_set_from_xyz(representation, p_F, value) ? OVP_OK : OVP_ERR_BAD_ARGS;
}

int ovp_anchor_change_jacobian(int representation, int do_fej, int calib_pose, int same_anchor, const double *value, const double *fej,
                               const double *old7, const double *old_fej7, const double *new7, const double *new_fej7, const double *calib7,
                               double *Phi, int *phi_rows, int *phi_cols, double *value_new, double *fej_new) {
  using namespace ovp;
  const int rep = representation;
  if (!is_relative(rep) || !value || !fej || !old7 || !old_fej7 || !new7 || !new_fej7 || !calib7 || !Phi || !phi_rows || !phi_cols || !value_new ||
      !fej_new)
    return OVP_ERR_BAD_ARGS;
  const double *cal = calib7;
  double pA[3], pAf[3];
  landmark_get_xyz(rep, value, pA);
  landmark_get_xyz(rep, fej, pAf);
  // Jacobians of p_FinG w.r.t. the old representation (:723-727)
  double Hf_old[9], Ha_old[18], Hc_old[18], Hf_new[9], Ha_new[18], Hc_new[18], dummy[3] = {0, 0, 0};
  int k = 3, has = 0;
  int st = ovp_feature_jacobian_representation(rep, do_fej, dummy, dummy, pA, old7, old_fej7, cal, Hf_old, &k, Ha_old, Hc_old, &has);
  if (st)
    return st;
  // the landmark seen from the new anchor camera, best estimates and first estimates (:739-777; the extrinsics have no first estimate)
  auto reanchor = [&](const double *oldp, const double *newp, const double *p_in, double *p_out) {
    double RC[9], Ro[9], Rn[9], RGo[9], RGn[9], po[3], pn[3];
    quat_to_rot(cal, RC);
    quat_to_rot(oldp, Ro);
    quat_to_rot(newp, Rn);
    mat3_mul(RC, Ro, RGo); // R_GtoOLD
    mat3_mul(RC, Rn, RGn);
    for (int i = 0; i < 3; i++) {
      po[i] = oldp[4 + i] - (RGo[i] * cal[4] + RGo[3 + i] * cal[5] + RGo[6 + i] * cal[6]); // p_OLDinG
      pn[i] = newp[4 + i] - (RGn[i] * cal[4] + RGn[3 + i] * cal[5] + RGn[6 + i] * cal[6]);
    }
    double g[3]; // feature in the global frame through the old anchor, then into the new one: R_OLDtoNEW p + p_OLDinNEW
    for (int i = 0; i < 3; i++)
      g[i] = RGo[i] * p_in[0] + RGo[3 + i] * p_in[1] + RGo[6 + i] * p_in[2] + po[i];
    for (int i = 0; i < 3; i++)
      p_out[i] = RGn[3 * i] * (g[0] - pn[0]) + RGn[3 * i + 1] * (g[1] - pn[1]) + RGn[3 * i + 2] * (g[2] - pn[2]);
  };
  double pA_new[3], pAf_new[3];
  reanchor(old7, new7, pA, pA_new);
  reanchor(old_fej7, new_fej7, pAf, pAf_new);
  st = ovp_feature_jacobian_representation(rep, do_fej, dummy, dummy, pA_new, new7, new_fej7, cal, Hf_new, &k, Ha_new, Hc_new, &has);
  if (st)
    return st;
  // Phi over [old anchor, extrinsics (when calibrated), new anchor (when different), landmark] (:783-838)
  int col_old = 0, col_cal = -1, col_new = -1, col_lm = 0, cols = 6;
  if (calib_pose) {
    col_cal = cols;
    cols += 6;
  }
  if (!same_anchor) {
    col_new = cols;
    cols += 6;
  } else {
    col_new = col_old;
  }
  col_lm = cols;
  const int ps = (rep == 5) ? 1 : 3; // Phi's rows: the landmark's size (:802-803)
  cols += ps;
  double Hinv[9]; // ps x 3, column-major
  if (ps == 1) { // the single-depth form's H_f_new is 3 x 1: its pseudo-inverse H_f_new^T / |H_f_new|^2 (:807-808)
    const double n2 = Hf_new[0] * Hf_new[0] + Hf_new[1] * Hf_new[1] + Hf_new[2] * Hf_new[2];
    for (int i = 0; i < 3; i++)
      Hinv[i] = 1.0 / n2 * Hf_new[i];
  } else {
    inverse3(Hf_new, Hinv);
  }
  for (int i = 0; i < ps * cols; i++)
    Phi[i] = 0.0;
  auto add = [&](int col0, const double *B, int nb, double sign) { // Phi[:, col0 : col0 + nb] += sign * Hinv * B (column-major ps x nb)
    for (int j = 0; j < nb; j++)
      for (int i = 0; i < ps; i++)
        Phi[(size_t)(col0 + j) * ps + i] += sign * (Hinv[i] * B[3 * j] + Hinv[ps + i] * B[3 * j + 1] + Hinv[2 * ps + i] * B[3 * j + 2]);
  };
  add(col_old, Ha_old, 6, 1.0);
  if (calib_pose)
    add(col_cal, Hc_old, 6, 1.0);
  add(col_lm, Hf_old, ps, 1.0);
  add(col_new, Ha_new, 6, -1.0);
  if (calib_pose)
    add(col_cal, Hc_new, 6, -1.0);
  *phi_rows = ps;
  *phi_cols = cols;
  landmark_set_from_xyz(rep, pA_new, value_new);
  landmark_set_from_xyz(rep, pAf_new, fej_new);
  return OVP_OK;
}

int ovp_slam_perform_anchor_change(ovp_ctx *h, int64_t featid, int new_anchor_clone_handle) {
  using namespace ovp;
  Ctx *c = ovp::enter(h);
  auto it = c->slam.find(featid);
  if (it == c->slam.end() || c->vars[it->second].id < 0)
    return fail(c, OVP_ERR_NOT_IN_STATE, "perform_anchor_change: feature %lld has no landmark in the state", (long long)featid);
  const int hl = it->second, rep = c->vars[hl].rep, h_old = c->vars[hl].anchor;
  if (!is_relative(rep) || h_old < 0)
    return fail(c, OVP_ERR_BAD_ARGS, "perform_anchor_change: landmark %lld is not in an anchored representation (assert, UpdaterSLAM.cpp:710-711)",
                (long long)featid);
  if (!is_clone(c, h_old, true) || !is_clone(c, new_anchor_clone_handle, true))
    return fail(c, OVP_ERR_BAD_ARGS, "perform_anchor_change: old / new anchor is not a clone in the state");
  int st = sync_host_values(c);
  if (st)
    return st;
  const int h_new = new_anchor_clone_handle;
  const bool calib = c->opt.do_calib_camera_pose != 0;
  double *lv = c->h_val.data() + (size_t)hl * OVP_VAL_STRIDE, *lf = c->h_fej.data() + (size_t)hl * OVP_VAL_STRIDE;
  auto row = [&](const std::vector<double> &t, int hh) { return t.data() + (size_t)hh * OVP_VAL_STRIDE; };
  double Phi[3 * 21], vn[4], fn[4];
  int ps = 0, cols = 0;
  st = ovp_anchor_change_jacobian(rep, c->opt.do_fej, calib, h_new == h_old, lv, lf, row(c->h_val, h_old), row(c->h_fej, h_old), row(c->h_val, h_new),
                                  row(c->h_fej, h_new), row(c->h_val, c->h_calib), Phi, &ps, &cols, vn, fn);
  if (st)
    return fail(c, st, "perform_anchor_change: representation Jacobian failed");
  int old_h[4], no = 0; // Phi's column order
  old_h[no++] = h_old;
  if (calib)
    old_h[no++] = c->h_calib;
  if (h_new != h_old)
    old_h[no++] = h_new;
  old_h[no++] = hl;
  const double Q[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  st = ovp_ekf_propagation(h, &hl, 1, old_h, no, Phi, ps, cols, Q);
  if (st)
    return st;
  for (int i = 0; i < (rep == 5 ? 4 : 3); i++) { // Landmark::set_from_xyz of the re-anchored point, value and first estimate
    lv[i] = vn[i];
    lf[i] = fn[i];
  }
  c->vars[hl].anchor = h_new;
  return push_host_values(c, hl);
}

int ovp_slam_change_anchors(ovp_ctx *h, int *n_changed) {
  using namespace ovp;
  Ctx *c = ovp::enter(h);
  if (n_changed)
    *n_changed = 0;
  if ((int)c->clones.size() <= c->opt.max_clone_size) // :687-689
    return OVP_OK;
  const int h_marg = c->clones.begin()->second; // State::margtimestep(): the oldest clone
  auto cur = c->clones.find(c->timestamp);
  if (cur == c->clones.end())
    return fail(c, OVP_ERR_BAD_ARGS, "change_anchors: no clone at the state time %.9f", c->timestamp);
  std::vector<int64_t> todo;
  for (auto &kv : c->slam) { // ascending feature id (the reference iterates an unordered_map: the changes are independent of each other
    const Var &v = c->vars[kv.second]; // except through the covariance entries of the shared anchors, which a Phi with Q = 0 does not alter)
    if (v.id >= 0 && is_relative(v.rep) && v.anchor == h_marg)
      todo.push_back(kv.first);
  }
  for (int64_t fid : todo) {
    int st = ovp_slam_perform_anchor_change(h, fid, cur->second);
    if (st)
      return st;
    if (n_changed)
      (*n_changed)++;
  }
  return OVP_OK;
}

} // extern "C"

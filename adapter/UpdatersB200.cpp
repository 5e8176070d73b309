// Reference-side adapters for the remaining classes of the call surface, reference signatures, bodies forwarding to include/ovp.h:
//   UpdaterSLAM::update / delayed_init / change_anchors   (update/UpdaterSLAM.h:76-96;  UpdaterSLAM.cpp:376-682, 53-372, 684-704)
//   UpdaterPlane::init_vio_plane                          (update/UpdaterPlane.h:80-81;  UpdaterPlane.cpp:56-481)
//   Propagator::feed_imu / propagate_and_clone / fast_state_propagate (state/Propagator.h:71-118; Propagator.cpp:37-224)
// Built instead of UpdaterSLAM.cpp / UpdaterPlane.cpp / Propagator.cpp and linked with -lovp.  Host bookkeeping (track cleaning, triangulation
// failures, which features become landmarks) stays as in the reference; it is abbreviated here to the parts that touch the C ABI.
#include <cstdio>
#include <cstdlib>

#include "feat/Feature.h"
#include "ovp.h"
#include "state/Propagator.h"
#include "state/State.h"
#include "update/UpdaterPlane.h"
#include "update/UpdaterSLAM.h"

using namespace ov_plane;

static void ck(ovp_ctx *ctx, int st) {
  if (st) {
    std::fprintf(stderr, "%s\n", ovp_last_error(ctx));
    std::exit(EXIT_FAILURE);
  }
}
namespace {
struct Flat { // SoA view of a feature list (mono camera)
  std::vector<int> meas_offset{0}, meas_clone;
  std::vector<float> uv, uvn;
  std::vector<double> p;
  std::vector<int64_t> featid, planeid;
  void append(const std::shared_ptr<State> &state, const ov_core::Feature &f, const std::map<size_t, size_t> &feat2plane) {
    for (auto const &pair : f.timestamps)
      for (size_t m = 0; m < pair.second.size(); m++) {
        meas_clone.push_back(ovp_clone_handle(state->ctx, pair.second[m]));
        uv.push_back(f.uvs.at(pair.first)[m](0));
        uv.push_back(f.uvs.at(pair.first)[m](1));
        uvn.push_back(f.uvs_norm.at(pair.first)[m](0));
        uvn.push_back(f.uvs_norm.at(pair.first)[m](1));
      }
    meas_offset.push_back((int)meas_clone.size());
    for (int k = 0; k < 3; k++)
      p.push_back(f.p_FinG(k));
    featid.push_back((int64_t)f.featid);
    auto it = feat2plane.find(f.featid);
    planeid.push_back(it != feat2plane.end() ? (int64_t)it->second : 0);
  }
};
} // namespace

// ---- UpdaterSLAM ----------------------------------------------------------------------------------------------------------------------
namespace {
// StateOptions::feat_rep_slam / feat_rep_aruco, host-only: the representation every new landmark is created in (UpdaterSLAM.cpp:231-232)
// FeatureInitializerOptions to the library before a triangulating call: the mode (triangulate_1d / refine_features, which every updater tests
// before it triangulates) on the context, the ten numbers returned for the call
ovp_triangulation_options triangulation_options(const std::shared_ptr<State> &state, const ov_core::FeatureInitializerOptions &fi) {
  const ovp_triangulation_mode mode = {fi.triangulate_1d ? 1 : 0, fi.refine_features ? 1 : 0};
  ck(state->ctx, ovp_set_triangulation_mode(state->ctx, &mode));
  return {fi.max_runs, fi.init_lamda, fi.max_lamda, fi.min_dx, fi.min_dcost, fi.lam_mult, fi.min_dist, fi.max_dist, fi.max_baseline,
          fi.max_cond_number};
}

void set_landmark_options(const std::shared_ptr<State> &state) {
  const ovp_landmark_options lo = {(int)state->_options.feat_rep_slam, (int)state->_options.feat_rep_aruco};
  ck(state->ctx, ovp_set_landmark_representations(state->ctx, &lo)); // 0..5, ANCHORED_INVERSE_DEPTH_SINGLE included
}
// Landmark::_feat_representation, _anchor_cam_id and _anchor_clone_timestamp, value and first estimate of the landmark of featid as the
// library holds them (the anchor's timestamp is the one of the clone whose handle the library names)
void refresh_landmark(const std::shared_ptr<State> &state, ov_type::Landmark &landmark) {
  int rep = 0, anchor = -1;
  ck(state->ctx, ovp_slam_get_representation(state->ctx, (int64_t)landmark._featid, &rep, &anchor));
  landmark._feat_representation = (ov_type::LandmarkRepresentation::Representation)rep;
  landmark._anchor_cam_id = anchor >= 0 ? 0 : -1; // mono
  landmark._anchor_clone_timestamp = -1;
  for (const auto &clone : state->_clones_IMU)
    if (anchor >= 0 && state->handle.at(clone.second.get()) == anchor)
      landmark._anchor_clone_timestamp = clone.first;
  const int h = state->handle.at(&landmark), n = ovp_var_size(state->ctx, h); // 1 for the single-depth form, as Landmark::value() is
  Eigen::MatrixXd value(n, 1), fej(n, 1);
  ck(state->ctx, ovp_var_get(state->ctx, h, value.data(), fej.data()));
  landmark.set_value(value);
  landmark.set_fej(fej);
  if (rep == ov_type::LandmarkRepresentation::Representation::ANCHORED_INVERSE_DEPTH_SINGLE) { // the bearings it carries: rho p_FinA
    Eigen::Vector3d p, pf;
    ck(state->ctx, ovp_slam_get_xyz(state->ctx, (int64_t)landmark._featid, 0, p.data()));
    ck(state->ctx, ovp_slam_get_xyz(state->ctx, (int64_t)landmark._featid, 1, pf.data()));
    for (int k = 0; k < 3; k++) {
      landmark.uv_norm_zero(k) = value(0, 0) * p(k);
      landmark.uv_norm_zero_fej(k) = fej(0, 0) * pf(k);
    }
  }
}
} // namespace

UpdaterSLAM::UpdaterSLAM(UpdaterOptions &options_slam, UpdaterOptions &options_aruco, ov_core::FeatureInitializerOptions &feat_init_options)
    : _options_slam(options_slam), _options_aruco(options_aruco) {
  initializer_feat = std::shared_ptr<ov_core::FeatureInitializer>(new ov_core::FeatureInitializer(feat_init_options));
}

void UpdaterSLAM::update(std::shared_ptr<State> state, std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec,
                         const std::map<size_t, size_t> &feat2plane) {
  if (feature_vec.empty())
    return;
  Flat fl;
  for (auto &f : feature_vec)
    fl.append(state, *f, feat2plane);
  // the ArUco tags among them whiten and gate with _options_aruco (:500, :545-547); host-only, set on every call since the constructor has
  // no state to hand them to
  const ovp_updater_options ua = {_options_aruco.sigma_pix, _options_aruco.chi2_multipler};
  ck(state->ctx, ovp_set_aruco_options(state->ctx, &ua));
  set_landmark_options(state); // each landmark is updated in its own representation and anchor (:476-522)
  ovp_updater_options uo = {_options_slam.sigma_pix, _options_slam.chi2_multipler};
  std::vector<int> st(feature_vec.size());
  std::vector<double> chi(feature_vec.size());
  ck(state->ctx, ovp_slam_update(state->ctx, (int)feature_vec.size(), fl.meas_offset.data(), fl.meas_clone.data(), fl.uv.data(), fl.featid.data(),
                                 fl.planeid.data(), &uo, state->_options.use_plane_constraint_slamu ? 1 : 0, st.data(), chi.data()));
  for (size_t i = 0; i < feature_vec.size(); i++) { // 0: rejected -> the landmark is flagged for marginalisation unless a tag (:596-618)
    if (st[i] == -1)
      continue; // a single-depth landmark with one measurement: erased from feature_vec untouched (:410-417)
    feature_vec[i]->to_delete = true;
    if (st[i] == 0 && (int)feature_vec[i]->featid >= state->_options.max_aruco_features)
      state->_features_SLAM.at(feature_vec[i]->featid)->should_marg = true;
    if (st[i] == 3)
      state->_features_SLAM_to_PLANE[feature_vec[i]->featid] = 0; // accepted only without its plane (:594-609)
  }
}

void UpdaterSLAM::delayed_init(std::shared_ptr<State> state, std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec,
                               const std::map<size_t, size_t> &feat2plane) {
  if (feature_vec.empty())
    return;
  // ArUco features (featid < max_aruco_features) are initialised with _options_aruco (:164, :257, :302-304), in the same call as the rest
  const ovp_updater_options ua = {_options_aruco.sigma_pix, _options_aruco.chi2_multipler};
  ck(state->ctx, ovp_set_aruco_options(state->ctx, &ua));
  set_landmark_options(state); // anchored landmarks are created from the triangulation's p_FinA (:230-304)
  // :77-103 clean every track against the clone times
  std::vector<double> clonetimes;
  for (const auto &clone_imu : state->_clones_IMU)
    clonetimes.emplace_back(clone_imu.first);
  for (auto &f : feature_vec)
    f->clean_old_measurements(clonetimes);
  // :106-364 in one call: triangulation, the refinement onto in-state planes, the initialisation with its chi2 fallback
  Flat fl;
  for (auto &f : feature_vec)
    fl.append(state, *f, feat2plane);
  ovp_feature_tracks t;
  t.F = (int)feature_vec.size();
  t.meas_offset = fl.meas_offset.data();
  t.meas_clone = fl.meas_clone.data();
  t.uv = fl.uv.data();
  t.uv_norm = fl.uvn.data();
  t.featid = fl.featid.data();
  t.planeid = fl.planeid.data();
  ovp_slam_init_options o;
  o.sigma_pix = _options_slam.sigma_pix;
  o.chi2_multipler = _options_slam.chi2_multipler;
  o.use_plane_constraint = (state->_options.use_plane_constraint && state->_options.use_plane_constraint_slamd) ? 1 : 0;
  o.use_refine_plane_feat = state->_options.use_refine_plane_feat ? 1 : 0;
  const ovp_triangulation_options tri = triangulation_options(state, initializer_feat->config());
  o.tri = &tri;
  const size_t F = feature_vec.size();
  std::vector<int> feat_status(F), new_handles(F);
  std::vector<double> p_FinG(3 * F);
  ck(state->ctx, ovp_slam_delayed_init_tracks(state->ctx, &t, &o, feat_status.data(), nullptr, p_FinG.data(), new_handles.data()));
  std::vector<std::shared_ptr<ov_core::Feature>> kept;
  for (size_t i = 0; i < F; i++) {
    auto &f = feature_vec[i];
    f->to_delete = true; // every feature of the call (:98, :190, :306-361)
    for (int k = 0; k < 3; k++)
      f->p_FinG(k) = p_FinG[3 * i + k];
    const int64_t s2p = ovp_slam_plane_of(state->ctx, (int64_t)f->featid); // written by the refinement and the initialisation
    if (s2p >= 0)
      state->_features_SLAM_to_PLANE[f->featid] = (size_t)s2p;
    if (feat_status[i] <= 0)
      continue; // erased from feature_vec
    // :283-305, :352 register the landmark with its representation, anchor, value and first estimate as the library holds them
    auto landmark = std::make_shared<ov_type::Landmark>(ovp_var_size(state->ctx, new_handles[i])); // 1 for the single-depth form
    landmark->_featid = f->featid;
    landmark->_unique_camera_id = 0;
    state->handle[landmark.get()] = new_handles[i];
    refresh_landmark(state, *landmark);
    state->_features_SLAM.insert({f->featid, landmark});
    state->by_handle[new_handles[i]] = landmark;
    kept.push_back(f);
  }
  feature_vec.swap(kept);
}

void UpdaterSLAM::change_anchors(std::shared_ptr<State> state) {
  // :684-704; the landmarks the library moved get their new anchor, value and first estimate (perform_anchor_change, :840-848).  Refreshing
  // every anchored landmark reads back, for one that did not move, what it already holds.
  int n_changed = 0;
  ck(state->ctx, ovp_slam_change_anchors(state->ctx, &n_changed));
  if (n_changed == 0)
    return;
  for (auto &kv : state->_features_SLAM)
    if (ov_type::LandmarkRepresentation::is_relative_representation(kv.second->_feat_representation))
      refresh_landmark(state, *kv.second);
}

// ---- UpdaterPlane ---------------------------------------------------------------------------------------------------------------------
UpdaterPlane::UpdaterPlane(UpdaterOptions &options, ov_core::FeatureInitializerOptions &feat_init_options) : _options(options) {
  initializer_feat = std::shared_ptr<ov_core::FeatureInitializer>(new ov_core::FeatureInitializer(feat_init_options));
}

void UpdaterPlane::init_vio_plane(std::shared_ptr<State> state, std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec,
                                  std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec_used, const std::map<size_t, size_t> &feat2plane) {
  // :66-69 (the SLAM part of the reference's first test feeds a block that is commented out there, :200-215)
  if (feature_vec.empty() || feat2plane.empty())
    return;
  // :75-116 clean the tracks of the candidates against the clone times (non-candidates are left untouched, as in the reference)
  std::vector<double> clonetimes;
  for (const auto &clone_imu : state->_clones_IMU)
    clonetimes.emplace_back(clone_imu.first);
  for (auto &f : feature_vec) {
    auto it = feat2plane.find(f->featid);
    if (it != feat2plane.end() && state->_features_PLANE.find(it->second) == state->_features_PLANE.end())
      f->clean_old_measurements(clonetimes);
  }
  // :119-481 in one call: triangulation, track-length sort, per-plane cap, RANSAC, refinement, initialisation
  Flat fl;
  for (auto &f : feature_vec)
    fl.append(state, *f, feat2plane);
  ovp_feature_tracks t;
  t.F = (int)feature_vec.size();
  t.meas_offset = fl.meas_offset.data();
  t.meas_clone = fl.meas_clone.data();
  t.uv = fl.uv.data();
  t.uv_norm = fl.uvn.data();
  t.featid = fl.featid.data();
  t.planeid = fl.planeid.data();
  ovp_plane_init_options o;
  o.sigma_pix = _options.sigma_pix;
  o.max_msckf_plane = state->_options.max_msckf_plane;
  o.plane_init_min_feat = state->_options.plane_init_min_feat;
  o.plane_init_max_cond = state->_options.plane_init_max_cond;
  o.shuffle_kind = 0; // std::shuffle draws of the reference's GCC 7..10 images
  const ovp_triangulation_options tri = triangulation_options(state, initializer_feat->config());
  o.tri = &tri;
  const size_t F = feature_vec.size();
  std::vector<int> feat_status(F), plane_status(F), new_handles(F);
  std::vector<double> p_FinG(3 * F), cp(3 * F);
  std::vector<int64_t> plane_ids(F);
  int n_planes = 0;
  ck(state->ctx, ovp_plane_init_tracks(state->ctx, &t, &o, feat_status.data(), p_FinG.data(), &n_planes, plane_ids.data(), plane_status.data(),
                                       new_handles.data(), cp.data()));
  // :446-455 register every new plane with the value and first estimate the device holds
  for (int q = 0; q < n_planes; q++) {
    if (plane_status[q] != 1)
      continue;
    auto plane = std::make_shared<ov_type::Vec>(3);
    Eigen::MatrixXd value(3, 1), fej(3, 1);
    ck(state->ctx, ovp_var_get(state->ctx, new_handles[q], value.data(), fej.data()));
    plane->set_value(value);
    plane->set_fej(fej);
    state->_features_PLANE.insert({(size_t)plane_ids[q], plane});
    state->handle[plane.get()] = new_handles[q];
    state->by_handle[new_handles[q]] = plane;
  }
  // feat_status -> feature_vec / feature_vec_used / to_delete (:109-111, :158-161, :459-475); p_FinG written back like the reference's stages
  std::vector<std::shared_ptr<ov_core::Feature>> kept;
  for (size_t i = 0; i < F; i++) {
    auto &f = feature_vec[i];
    if (feat_status[i] == -2 || feat_status[i] >= 1)
      for (int k = 0; k < 3; k++)
        f->p_FinG(k) = p_FinG[3 * i + k];
    if (feat_status[i] == -1)
      continue; // fewer than two measurements: erased, not deleted
    if (feat_status[i] == 1) {
      f->to_delete = true;
      feature_vec_used.push_back(f);
      continue;
    }
    kept.push_back(f);
  }
  feature_vec.swap(kept);
}

// ---- Propagator -----------------------------------------------------------------------------------------------------------------------
ovp_ctx *Propagator::ctx = nullptr;

Propagator::Propagator(NoiseManager noises, double gravity_mag) : _noises(noises), _gravity_mag(gravity_mag) {
  if (ctx)
    ck(ctx, ovp_propagator_set_noise(ctx, noises.sigma_w, noises.sigma_wb, noises.sigma_a, noises.sigma_ab, gravity_mag));
}

void Propagator::feed_imu(const ov_core::ImuData &message, double oldest_time) {
  (void)oldest_time; // the library prunes its own buffer against the state time
  ck(ctx, ovp_propagator_feed_imu(ctx, message.timestamp, message.wm.data(), message.am.data()));
}

void Propagator::propagate_and_clone(std::shared_ptr<State> state, double timestamp) {
  int h = -1;
  ck(state->ctx, ovp_propagate_and_clone(state->ctx, timestamp, nullptr, nullptr, &h)); // OVP_ERR_TIME: same / backwards time (Propagator.cpp:41-51)
  auto pose = std::make_shared<ov_type::PoseJPL>();
  state->_clones_IMU[timestamp] = pose;
  state->handle[pose.get()] = h;
  state->by_handle[h] = pose;
  state->_timestamp = timestamp;
}

bool Propagator::fast_state_propagate(std::shared_ptr<State> state, double timestamp, Eigen::Matrix<double, 13, 1> &state_plus,
                                      Eigen::Matrix<double, 12, 12> &covariance) {
  int ok = 0;
  ck(state->ctx, ovp_fast_state_propagate(state->ctx, timestamp, state_plus.data(), covariance.data(), &ok));
  return ok != 0;
}

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
UpdaterSLAM::UpdaterSLAM(UpdaterOptions &options_slam, UpdaterOptions &options_aruco, ov_core::FeatureInitializerOptions &feat_init_options)
    : _options_slam(options_slam), _options_aruco(options_aruco) {
  (void)feat_init_options;
}

void UpdaterSLAM::update(std::shared_ptr<State> state, std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec,
                         const std::map<size_t, size_t> &feat2plane) {
  if (feature_vec.empty())
    return;
  Flat fl;
  for (auto &f : feature_vec)
    fl.append(state, *f, feat2plane);
  ovp_updater_options uo = {_options_slam.sigma_pix, _options_slam.chi2_multipler};
  std::vector<int> st(feature_vec.size());
  std::vector<double> chi(feature_vec.size());
  ck(state->ctx, ovp_slam_update(state->ctx, (int)feature_vec.size(), fl.meas_offset.data(), fl.meas_clone.data(), fl.uv.data(), fl.featid.data(),
                                 fl.planeid.data(), &uo, state->_options.use_plane_constraint_slamu ? 1 : 0, st.data(), chi.data()));
  for (size_t i = 0; i < feature_vec.size(); i++) { // 0: rejected -> the landmark is flagged for marginalisation (:659-668)
    feature_vec[i]->to_delete = true;
    if (st[i] == 0)
      state->_features_SLAM.at(feature_vec[i]->featid)->should_marg = true;
    if (st[i] == 3)
      state->_features_SLAM_to_PLANE[feature_vec[i]->featid] = 0; // accepted only without its plane (:594-609)
  }
}

void UpdaterSLAM::delayed_init(std::shared_ptr<State> state, std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec,
                               const std::map<size_t, size_t> &feat2plane) {
  if (feature_vec.empty())
    return;
  // triangulation on the device (:118-160), failures leave
  Flat tri;
  for (auto &f : feature_vec)
    tri.append(state, *f, feat2plane);
  std::vector<double> p(3 * feature_vec.size());
  std::vector<int> ok(feature_vec.size());
  ck(state->ctx, ovp_triangulate_features(state->ctx, (int)feature_vec.size(), tri.meas_offset.data(), tri.meas_clone.data(), tri.uvn.data(), nullptr,
                                          p.data(), ok.data()));
  Flat fl;
  std::vector<std::shared_ptr<ov_core::Feature>> kept;
  for (size_t i = 0; i < feature_vec.size(); i++) {
    if (!ok[i]) {
      feature_vec[i]->to_delete = true;
      continue;
    }
    for (int k = 0; k < 3; k++)
      feature_vec[i]->p_FinG(k) = p[3 * i + k];
    fl.append(state, *feature_vec[i], feat2plane);
    kept.push_back(feature_vec[i]);
  }
  if (kept.empty())
    return;
  ovp_updater_options uo = {_options_slam.sigma_pix, _options_slam.chi2_multipler};
  std::vector<int> st(kept.size()), nh(kept.size());
  ck(state->ctx, ovp_slam_delayed_init(state->ctx, (int)kept.size(), fl.meas_offset.data(), fl.meas_clone.data(), fl.uv.data(), fl.p.data(), fl.p.data(),
                                       fl.featid.data(), fl.planeid.data(), &uo, state->_options.use_plane_constraint_slamu ? 1 : 0, st.data(), nh.data()));
  for (size_t i = 0; i < kept.size(); i++) {
    kept[i]->to_delete = true;
    if (st[i] == 0)
      continue;
    auto landmark = std::make_shared<ov_type::Landmark>(3); // _features_SLAM.insert (:338-339); values are refreshed from the device
    landmark->_featid = kept[i]->featid;
    state->_features_SLAM.insert({kept[i]->featid, landmark});
    state->handle[landmark.get()] = nh[i];
    state->by_handle[nh[i]] = landmark;
  }
}

void UpdaterSLAM::change_anchors(std::shared_ptr<State> state) { ck(state->ctx, ovp_slam_change_anchors(state->ctx, nullptr)); }

// ---- UpdaterPlane ---------------------------------------------------------------------------------------------------------------------
UpdaterPlane::UpdaterPlane(UpdaterOptions &options, ov_core::FeatureInitializerOptions &feat_init_options) : _options(options) { (void)feat_init_options; }

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
  o.tri = nullptr;    // FeatureInitializerOptions defaults
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

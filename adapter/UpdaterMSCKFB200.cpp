// Reference-side adapter for ov_plane/src/update/UpdaterMSCKF.cpp: UpdaterMSCKF::update with the reference's own signature
// (update/UpdaterMSCKF.h:77-79), built instead of UpdaterMSCKF.cpp and linked with -lovp.  The host keeps what is bookkeeping in the reference
// (cleaning the tracks, grouping the features by plane, flagging what was consumed); every numerical stage is one call into the C ABI:
//   UpdaterMSCKF.cpp:142-194  triangulation                      -> ovp_triangulate_features
//   :262-360                  plane hypotheses + refinement       -> ovp_plane_fitting, ovp_optimize_plane (all planes of the frame in one batch)
//   :407-828                  plane updates, gates, compression,  -> ovp_msckf_update_landmarks (one call; the chain of dependent updates stays
//                             StateHelper::EKFUpdate, with the        on the device; the library keeps _features_SLAM_to_PLANE of the members)
//                             SLAM landmarks of out-of-state planes (:231-254)
// The chi2 table (:57-62) is handed to the library once (ovp_set_chi2_table) by the code that creates the context.
#include "update/UpdaterMSCKF.h"

#include <cstdio>
#include <cstdlib>
#include <memory>
#include <set>

#include "feat/Feature.h"
#include "ovp.h"
#include "state/State.h"

using namespace ov_plane;

static void ck(std::shared_ptr<State> state, int st) {
  if (st) {
    std::fprintf(stderr, "[MSCKF-UP]: %s\n", ovp_last_error(state->ctx));
    std::exit(EXIT_FAILURE);
  }
}

// FeatureInitializerOptions to the library before a triangulating call: the mode (triangulate_1d / refine_features, which every updater tests
// before it triangulates) on the context, the ten numbers returned for the call
static ovp_triangulation_options triangulation_options(const std::shared_ptr<State> &state, const ov_core::FeatureInitializerOptions &fi) {
  const ovp_triangulation_mode mode = {fi.triangulate_1d ? 1 : 0, fi.refine_features ? 1 : 0};
  ck(state, ovp_set_triangulation_mode(state->ctx, &mode));
  return {fi.max_runs, fi.init_lamda, fi.max_lamda, fi.min_dx, fi.min_dcost, fi.lam_mult, fi.min_dist, fi.max_dist, fi.max_baseline,
          fi.max_cond_number};
}

UpdaterMSCKF::UpdaterMSCKF(UpdaterOptions &options, ov_core::FeatureInitializerOptions &feat_init_options) : _options(options) {
  initializer_feat = std::shared_ptr<ov_core::FeatureInitializer>(new ov_core::FeatureInitializer(feat_init_options));
  _options.sigma_pix_sq = _options.sigma_pix * _options.sigma_pix;
}

namespace {
// SoA view of a feature list in the layout of ovp_feature_batch / ovp_triangulate_features (mono camera: one camera id per feature)
struct Flat {
  std::vector<int> meas_offset{0}, meas_clone;
  std::vector<float> uv, uvn;
  void append(const std::shared_ptr<State> &state, const ov_core::Feature &f) {
    for (auto const &pair : f.timestamps)
      for (size_t m = 0; m < pair.second.size(); m++) {
        meas_clone.push_back(ovp_clone_handle(state->ctx, pair.second[m]));
        uv.push_back(f.uvs.at(pair.first)[m](0));
        uv.push_back(f.uvs.at(pair.first)[m](1));
        uvn.push_back(f.uvs_norm.at(pair.first)[m](0));
        uvn.push_back(f.uvs_norm.at(pair.first)[m](1));
      }
    meas_offset.push_back((int)meas_clone.size());
  }
};
int count_meas(const ov_core::Feature &f) {
  int ct = 0;
  for (auto const &pair : f.timestamps)
    ct += (int)pair.second.size();
  return ct;
}
} // namespace

void UpdaterMSCKF::update(std::shared_ptr<State> state, std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec,
                          std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec_extra,
                          std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec_used, const std::map<size_t, size_t> &feat2plane) {
  if (feature_vec.empty())
    return;
  // 0-1. valid measurement times = clone times; features with fewer than two measurements leave (:72-118)
  std::vector<double> clonetimes;
  for (const auto &clone_imu : state->_clones_IMU)
    clonetimes.emplace_back(clone_imu.first);
  for (auto it = feature_vec.begin(); it != feature_vec.end();) {
    (*it)->clean_old_measurements(clonetimes);
    if (count_meas(**it) < 2) {
      (*it)->to_delete = true;
      it = feature_vec.erase(it);
    } else {
      ++it;
    }
  }
  for (auto it = feature_vec_extra.begin(); it != feature_vec_extra.end();) {
    (*it)->clean_old_measurements(clonetimes);
    it = (count_meas(**it) < 2) ? feature_vec_extra.erase(it) : it + 1;
  }
  // 3. triangulation of both lists on the device (:142-194): failures leave like in the reference
  auto triangulate = [&](std::vector<std::shared_ptr<ov_core::Feature>> &vec, bool flag_delete) {
    if (vec.empty())
      return;
    Flat fl;
    for (auto &f : vec)
      fl.append(state, *f);
    std::vector<double> p(3 * vec.size());
    std::vector<int> ok(vec.size());
    const ovp_triangulation_options tri = triangulation_options(state, initializer_feat->config());
    ck(state, ovp_triangulate_features(state->ctx, (int)vec.size(), fl.meas_offset.data(), fl.meas_clone.data(), fl.uvn.data(), &tri, p.data(), ok.data()));
    std::vector<std::shared_ptr<ov_core::Feature>> keep;
    for (size_t i = 0; i < vec.size(); i++) {
      if (!ok[i]) {
        if (flag_delete)
          vec[i]->to_delete = true;
        continue;
      }
      for (int k = 0; k < 3; k++)
        vec[i]->p_FinG(k) = p[3 * i + k];
      keep.push_back(vec[i]);
    }
    vec.swap(keep);
  };
  triangulate(feature_vec, true);
  triangulate(feature_vec_extra, false);
  std::vector<double> p_original; // positions before the plane refinement (:160,663)
  for (auto &f : feature_vec)
    for (int k = 0; k < 3; k++)
      p_original.push_back(f->p_FinG(k));

  // 4. planes of this frame (:198-404): features grouped by plane id, in-state planes refine their features against the state's estimate,
  //    new planes get a RANSAC hypothesis and a joint refinement - all candidates of the frame in ONE batch per stage
  std::map<size_t, std::vector<std::shared_ptr<ov_core::Feature>>> plane_feats;
  std::set<ov_core::Feature *> slam_members; // SLAM landmarks as measurement-free features of their plane (:231-254)
  if (state->_options.use_plane_constraint && (state->_options.use_plane_constraint_msckf || state->_options.use_plane_constraint_slamu)) {
    if (state->_options.use_plane_constraint_msckf)
      for (auto *vec : {&feature_vec, &feature_vec_extra})
        for (auto &feat : *vec)
          if (feat2plane.find(feat->featid) != feat2plane.end())
            plane_feats[feat2plane.at(feat->featid)].push_back(feat);
    if (state->_options.use_plane_constraint_slamu) {
      std::set<size_t> slam_ids; // ascending featid, the std::map order of the reference's _features_SLAM
      for (auto &kv : state->_features_SLAM)
        slam_ids.insert(kv.first);
      for (size_t featid : slam_ids) {
        auto it = feat2plane.find(featid);
        if (it == feat2plane.end() || state->_features_PLANE.count(it->second) || ovp_slam_plane_of(state->ctx, (int64_t)featid) == 0)
          continue;
        double value[16], fej[16]; // the device holds the current estimate
        ck(state, ovp_var_get(state->ctx, ovp_slam_handle(state->ctx, (int64_t)featid), value, fej));
        auto lm = std::make_shared<ov_core::Feature>();
        lm->featid = featid;
        for (int k = 0; k < 3; k++)
          lm->p_FinG(k) = value[k];
        slam_members.insert(lm.get());
        plane_feats[it->second].push_back(lm);
      }
    }
  }
  std::map<size_t, Eigen::Vector3d> plane_estimates_cp_inG;
  std::vector<size_t> cand; // plane ids that go through the refinement, in std::map order
  std::vector<int> feat_offset{0}, fix_plane;
  std::vector<double> p_all, cp_all;
  Flat fl_planes;
  {
    // RANSAC for the planes that are not in the state and have at least four features (:314-325)
    std::vector<size_t> fresh;
    std::vector<int> fo{0};
    std::vector<double> pts;
    for (auto &kv : plane_feats) {
      if (state->_features_PLANE.count(kv.first) || kv.second.size() < 4)
        continue;
      fresh.push_back(kv.first);
      for (auto &f : kv.second)
        for (int k = 0; k < 3; k++)
          pts.push_back(f->p_FinG(k));
      fo.push_back(fo.back() + (int)kv.second.size());
    }
    std::vector<int> st(fresh.size() + 1), inl(pts.size() / 3 + 1);
    std::vector<double> abcd(4 * fresh.size() + 4);
    if (!fresh.empty()) {
      ovp_plane_fit_options po = {state->_options.plane_msckf_min_feat, state->_options.plane_msckf_max_cond, 0};
      ck(state, ovp_plane_fitting(state->ctx, (int)fresh.size(), fo.data(), pts.data(), &po, st.data(), abcd.data(), inl.data()));
    }
    std::map<size_t, Eigen::Vector3d> cp_fresh;
    for (size_t q = 0; q < fresh.size(); q++) {
      auto &vec = plane_feats[fresh[q]];
      if (!st[q]) { // `continue` in the reference: the plane gets no linearisation point this frame
        vec.clear();
        continue;
      }
      std::vector<std::shared_ptr<ov_core::Feature>> keep; // feats = best_inliers
      for (size_t i = 0; i < vec.size(); i++)
        if (inl[fo[q] + i])
          keep.push_back(vec[i]);
      vec.swap(keep);
      Eigen::Vector3d cp;
      for (int k = 0; k < 3; k++)
        cp(k) = -abcd[4 * q + k] * abcd[4 * q + 3];
      cp_fresh[fresh[q]] = cp;
    }
    // refinement batch: in-state planes with the plane fixed (:267-280), fresh planes free (:345-354)
    for (auto &kv : plane_feats) {
      const bool in_state = state->_features_PLANE.count(kv.first) != 0;
      if (kv.second.empty() || (!in_state && !cp_fresh.count(kv.first)))
        continue;
      cand.push_back(kv.first);
      fix_plane.push_back(in_state ? 1 : 0);
      for (int k = 0; k < 3; k++)
        cp_all.push_back(in_state ? state->_features_PLANE.at(kv.first)->value()(k) : cp_fresh[kv.first](k));
      for (auto &f : kv.second) {
        fl_planes.append(state, *f);
        for (int k = 0; k < 3; k++)
          p_all.push_back(f->p_FinG(k));
      }
      feat_offset.push_back(feat_offset.back() + (int)kv.second.size());
    }
  }
  if (!cand.empty()) {
    std::vector<int> st(cand.size()), inl(p_all.size() / 3);
    std::vector<double> p_ref(p_all.size()), cp_ref(cp_all.size());
    if (state->_options.use_refine_plane_feat) {
      const double focal_length = state->_cam_intrinsics.at(0)->value()(0);
      ovp_plane_refine_options ro = {_options.sigma_pix / focal_length, state->_options.sigma_constraint, 0};
      ck(state, ovp_optimize_plane(state->ctx, (int)cand.size(), feat_offset.data(), fl_planes.meas_offset.data(), fl_planes.meas_clone.data(),
                                   fl_planes.uvn.data(), p_all.data(), cp_all.data(), fix_plane.data(), &ro, p_ref.data(), cp_ref.data(), inl.data(),
                                   st.data(), nullptr));
    } else {
      p_ref = p_all;
      cp_ref = cp_all;
      std::fill(st.begin(), st.end(), 1);
      std::fill(inl.begin(), inl.end(), 1);
    }
    for (size_t q = 0; q < cand.size(); q++) {
      auto &vec = plane_feats[cand[q]];
      std::vector<std::shared_ptr<ov_core::Feature>> keep;
      for (size_t i = 0; i < vec.size(); i++) {
        if (!inl[feat_offset[q] + i])
          continue;
        for (int k = 0; k < 3; k++)
          vec[i]->p_FinG(k) = p_ref[3 * (feat_offset[q] + i) + k]; // side effect of optimize_plane, also when it returns false (:476)
        keep.push_back(vec[i]);
      }
      if (!st[q])
        continue; // no linearisation point for this plane (:279-280, :353-354)
      vec.swap(keep);
      if (!fix_plane[q] && vec.size() < 4)
        continue; // :396-397
      Eigen::Vector3d cp;
      for (int k = 0; k < 3; k++)
        cp(k) = cp_ref[3 * q + k];
      plane_estimates_cp_inG[cand[q]] = cp;
    }
  }

  // 5-6. everything from "plane CPs known" on is ONE call (:407-828): plane updates in ascending plane id, per-feature gates, compression, EKFUpdate
  std::vector<std::shared_ptr<ov_core::Feature>> all = feature_vec;
  std::set<ov_core::Feature *> in_main;
  for (auto &f : feature_vec)
    in_main.insert(f.get());
  // features of feature_vec_extra that lie on a plane with an estimate take part in its update only; landmarks that stayed on such a
  // plane are members of its update
  std::vector<int64_t> lm_featid, lm_planeid;
  for (auto &kv : plane_feats) {
    if (!plane_estimates_cp_inG.count(kv.first))
      continue;
    for (auto &f : kv.second) {
      if (slam_members.count(f.get())) {
        lm_featid.push_back((int64_t)f->featid);
        lm_planeid.push_back((int64_t)kv.first);
      } else if (!in_main.count(f.get())) {
        all.push_back(f);
        for (int k = 0; k < 3; k++)
          p_original.push_back(f->p_FinG(k));
      }
    }
  }
  Flat fl;
  std::vector<double> p;
  std::vector<int64_t> featid, planeid, plane_ids;
  std::vector<double> plane_cp;
  for (auto &f : all) {
    fl.append(state, *f);
    for (int k = 0; k < 3; k++)
      p.push_back(f->p_FinG(k));
    featid.push_back((int64_t)f->featid);
    auto it = feat2plane.find(f->featid);
    planeid.push_back((it != feat2plane.end() && plane_estimates_cp_inG.count(it->second)) ? (int64_t)it->second : 0);
  }
  for (auto &kv : plane_estimates_cp_inG) {
    plane_ids.push_back((int64_t)kv.first);
    for (int k = 0; k < 3; k++)
      plane_cp.push_back(kv.second(k));
  }
  ovp_feature_batch b;
  b.F = (int)all.size();
  b.meas_offset = fl.meas_offset.data();
  b.meas_clone = fl.meas_clone.data();
  b.uv = fl.uv.data();
  b.p_FinG = p.data();
  b.p_FinG_original = p_original.data();
  b.featid = featid.data();
  b.planeid = planeid.data();
  b.nplanes = (int)plane_ids.size();
  b.plane_ids = plane_ids.data();
  b.plane_cp = plane_cp.data();
  ovp_updater_options uo = {_options.sigma_pix, _options.chi2_multipler};
  std::vector<int> feat_status(all.size()), plane_status(plane_ids.size() + 1);
  const ovp_plane_landmarks lm = {(int)lm_featid.size(), lm_featid.data(), lm_planeid.data()};
  ck(state, ovp_msckf_update_landmarks(state->ctx, &b, &lm, &uo, feat_status.data(), nullptr, plane_status.data(), nullptr, nullptr, nullptr));
  // bookkeeping of the outcome: rejected features are deleted, features consumed by a passed plane update are reported as used (:640-659, :745-764)
  for (size_t i = 0; i < all.size(); i++) {
    if (feat_status[i] == 0)
      all[i]->to_delete = true;
    if (feat_status[i] == 2)
      feature_vec_used.push_back(all[i]);
  }
  // the ov_type objects are refreshed from the device by StateHelperB200's refresh() (the state lives in the context)
}

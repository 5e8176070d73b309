// TEST INFRASTRUCTURE: UpdaterSLAM::delayed_init (UpdaterSLAM.cpp:66-374) restated on the CPU oracle's own stages: triangulation,
// PlaneFitting::optimize_plane with a single feature and the plane fixed, then the oracle's existing initialisation (orc_slam_delayed_init,
// :205-364).  The refinement writes State::_features_SLAM_to_PLANE between the stages (:175, :199), which the oracle's C API does not expose,
// so this file includes the oracle's header and reaches the state of the context it is handed (checked on every use, see slam_to_plane).
// Built by __graft_entry__.build() against liboracle.so and driven from tests/oracle_slam_init.py on the same oracle context.
#include "../oracle/oracle.hpp"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

extern "C" {
int orc_plane_handle(void *p, long long planeid);
int orc_slam_handle(void *p, long long featid);
int orc_handle_intr(void *p);
int orc_handle_imu(void *p);
int orc_cov_rows(void *p);
int orc_num_variables(void *p);
void orc_var_get(void *p, int h, double *value, double *fej);
int orc_var_nvalue(void *p, int h);
int orc_triangulate_features(void *p, int F, const int *meas_offset, const int *meas_clone, const float *uv_norm, double *p_FinG, int *status);
int orc_optimize_plane(void *p, int F, const int *meas_offset, const int *meas_clone, const float *uv_norm, const double *p_FinG, const double *cp_inG,
                       double sigma_px_norm, double sigma_c, int fix_plane, int max_num_iterations, double *p_out, double *cp_out, int *inlier, int *ok,
                       double *info);
int orc_slam_delayed_init(void *p, int F, const int *meas_offset, const int *meas_clone, const float *uv, const double *p_FinG,
                          const double *p_FinG_original, const long long *featid, const long long *planeid, double sigma_pix, double chi2_mult,
                          int *feat_status, int *new_handles);
}

namespace {
// The oracle context (oracle_capi.cpp) starts with the shared pointer to its State.  Nothing in the oracle's C API states that, so every use
// first checks the State found there against what the API reports about the same context, and stops the process when they disagree.
std::map<size_t, size_t> &slam_to_plane(void *h) {
  const orc::StateP &s = *static_cast<orc::StateP *>(h);
  if (!s || s->_Cov.rows() != orc_cov_rows(h) || (int)s->_variables.size() != orc_num_variables(h) ||
      (int)s->_features_SLAM.size() < 0 || s->_imu->handle != orc_handle_imu(h) || s->_cam_intrinsics->handle != orc_handle_intr(h)) {
    std::fprintf(stderr, "oracle_slam_init: the oracle context no longer starts with its State pointer; rebuild this file against oracle_capi.cpp\n");
    std::abort();
  }
  return s->_features_SLAM_to_PLANE;
}
} // namespace

// State::_features_SLAM_to_PLANE of the oracle context: the entry of featid, -1 = none; and a write of one entry (the hand chain's stand-in for
// the refinement's side effect)
extern "C" long long orc_slam_plane_of(void *h, long long featid) {
  auto &m = slam_to_plane(h);
  auto it = m.find((size_t)featid);
  return it == m.end() ? -1 : (long long)it->second;
}
extern "C" void orc_slam_set_plane_of(void *h, long long featid, long long planeid) { slam_to_plane(h)[(size_t)featid] = (size_t)planeid; }

// Outputs as ovp_slam_delayed_init_tracks.  use_plane: StateOptions::use_plane_constraint && use_plane_constraint_slamd.  tri_p / tri_status
// (may be NULL): the triangulation of the tracks with >= 2 measurements, in input order, used instead of the oracle's own.
extern "C" int orcsi_slam_delayed_init_tracks(void *h, int F, const int *meas_offset, const int *meas_clone, const float *uv, const float *uv_norm,
                                              const long long *featid, const long long *planeid, double sigma_pix, double chi2_mult, double sigma_c,
                                              int use_plane, int use_refine, const double *tri_p, const int *tri_status, int *feat_status,
                                              int *plane_status, double *p_out, int *new_handles) {
  std::vector<int> trk; // :84-103 tracks with at least two measurements
  for (int f = 0; f < F; f++) {
    feat_status[f] = meas_offset[f + 1] - meas_offset[f] < 2 ? -1 : 0;
    plane_status[f] = -1;
    new_handles[f] = -1;
    p_out[3 * f] = p_out[3 * f + 1] = p_out[3 * f + 2] = 0.0;
    if (feat_status[f] == 0)
      trk.push_back(f);
  }
  const int T = (int)trk.size();
  if (T == 0)
    return 0;
  auto sub = [&](const std::vector<int> &idx, const float *src, std::vector<int> &mo, std::vector<int> &mc, std::vector<float> &u) {
    mo.assign(1, 0);
    mc.clear();
    u.clear();
    for (int f : idx) {
      mc.insert(mc.end(), meas_clone + meas_offset[f], meas_clone + meas_offset[f + 1]);
      u.insert(u.end(), src + 2 * meas_offset[f], src + 2 * meas_offset[f + 1]);
      mo.push_back((int)mc.size());
    }
  };
  // :126-145 triangulation + Gauss-Newton
  std::vector<double> pt(3 * (size_t)T);
  std::vector<int> ok(T);
  if (tri_p && tri_status) {
    std::memcpy(pt.data(), tri_p, pt.size() * sizeof(double));
    std::memcpy(ok.data(), tri_status, ok.size() * sizeof(int));
  } else {
    std::vector<int> mo, mc;
    std::vector<float> un;
    sub(trk, uv_norm, mo, mc, un);
    if (int e = orc_triangulate_features(h, T, mo.data(), mc.data(), un.data(), pt.data(), ok.data()))
      return e;
  }
  const double fx = [&] {
    const int hi = orc_handle_intr(h);
    std::vector<double> v(orc_var_nvalue(h, hi));
    orc_var_get(h, hi, v.data(), nullptr);
    return v[0];
  }();
  // :147-202 per feature, in order: the refinement onto an in-state plane first, then the triangulation's verdict
  std::vector<int> init;
  for (int i = 0; i < T; i++) {
    const int f = trk[i];
    std::memcpy(p_out + 3 * f, &pt[3 * (size_t)i], 3 * sizeof(double));
    const int ph = planeid[f] != 0 ? orc_plane_handle(h, planeid[f]) : -1;
    bool success_plane = true;
    if (use_plane && ph >= 0 && orc_slam_plane_of(h, featid[f]) != 0 && use_refine) {
      std::vector<double> cp(orc_var_nvalue(h, ph));
      orc_var_get(h, ph, cp.data(), nullptr);
      std::vector<int> mo, mc;
      std::vector<float> un;
      sub({f}, uv_norm, mo, mc, un);
      double po[3], cpo[3];
      int inl = 0, pok = 0;
      if (int e = orc_optimize_plane(h, 1, mo.data(), mc.data(), un.data(), p_out + 3 * f, cp.data(), sigma_pix / fx, sigma_c, 1, 0, po, cpo, &inl, &pok,
                                     nullptr))
        return e;
      std::memcpy(p_out + 3 * f, po, sizeof(po)); // optimize_plane writes the feature back (unchanged when it fails)
      success_plane = pok != 0;
      plane_status[f] = pok ? 1 : 0;
      if (success_plane)
        orc_slam_set_plane_of(h, featid[f], planeid[f]);
    }
    if (!ok[i]) {
      feat_status[f] = -2;
      continue;
    }
    if (!success_plane) {
      std::memcpy(p_out + 3 * f, &pt[3 * (size_t)i], 3 * sizeof(double));
      orc_slam_set_plane_of(h, featid[f], 0);
    }
    init.push_back(i);
  }
  if (init.empty())
    return 0;
  // :205-364 on the oracle, from the positions above; the fallback starts from the triangulated one
  std::vector<int> idx;
  std::vector<long long> fid, pid;
  std::vector<double> pf, po;
  for (int i : init) {
    const int f = trk[i];
    idx.push_back(f);
    fid.push_back(featid[f]);
    pid.push_back(use_plane ? planeid[f] : 0);
    pf.insert(pf.end(), p_out + 3 * f, p_out + 3 * f + 3);
    po.insert(po.end(), &pt[3 * (size_t)i], &pt[3 * (size_t)i] + 3);
  }
  std::vector<int> mo, mc, fs(idx.size()), nh(idx.size());
  std::vector<float> u;
  sub(idx, uv, mo, mc, u);
  if (int e = orc_slam_delayed_init(h, (int)idx.size(), mo.data(), mc.data(), u.data(), pf.data(), po.data(), fid.data(), pid.data(), sigma_pix, chi2_mult,
                                    fs.data(), nh.data()))
    return e;
  for (size_t k = 0; k < idx.size(); k++) {
    feat_status[idx[k]] = fs[k];
    new_handles[idx[k]] = nh[k];
  }
  return 0;
}

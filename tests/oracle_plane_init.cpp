// TEST INFRASTRUCTURE: UpdaterPlane::init_vio_plane up to "plane linearisation points known" (UpdaterPlane.cpp:61-294), restated on the CPU
// oracle's own stages (triangulation, PlaneFitting::plane_fitting, PlaneFitting::optimize_plane), followed by the oracle's existing
// initialisation (orc_plane_init, :297-481).  Built by __graft_entry__.build() against liboracle.so and driven from tests/oracle_plane_init.py
// on the same oracle context.  The track-length sort is the real std::sort of the compiler that builds it, so this is also the independent
// check of the sort order the library and ov_plane_b200.plane_init_chain produce.
#include <algorithm>
#include <cstring>
#include <map>
#include <vector>

extern "C" {
int orc_plane_handle(void *p, long long planeid);
int orc_handle_intr(void *p);
void orc_var_get(void *p, int h, double *value, double *fej);
int orc_var_nvalue(void *p, int h);
int orc_triangulate_features(void *p, int F, const int *meas_offset, const int *meas_clone, const float *uv_norm, double *p_FinG, int *status);
int orc_plane_fitting(int F, const double *pts, int min_inlier_num, double max_cond, int shuffle_kind, double *abcd, int *inlier, int *ok);
int orc_optimize_plane(void *p, int F, const int *meas_offset, const int *meas_clone, const float *uv_norm, const double *p_FinG, const double *cp_inG,
                       double sigma_px_norm, double sigma_c, int fix_plane, int max_num_iterations, double *p_out, double *cp_out, int *inlier, int *ok,
                       double *info);
int orc_plane_init(void *p, int F, const int *meas_offset, const int *meas_clone, const float *uv, const double *p_FinG, const long long *featid,
                   const long long *planeid, int nplanes, const long long *plane_est_ids, const double *plane_est_cp, double sigma_pix, int *plane_status,
                   int *new_handles);
}

namespace {
struct Feat { // the parts of ov_core::Feature the function reads and writes
  int index;  // position in the caller's arrays
  long long featid, planeid;
  std::vector<int> clone;
  std::vector<float> uv, uvn;
  double p[3];
};

// measurement arrays of a feature list (meas_offset / clones / one of the coordinate arrays)
void flatten(const std::vector<Feat *> &fs, bool norm, std::vector<int> &mo, std::vector<int> &mc, std::vector<float> &uv) {
  mo.assign(1, 0);
  mc.clear();
  uv.clear();
  for (const Feat *f : fs) {
    mc.insert(mc.end(), f->clone.begin(), f->clone.end());
    const std::vector<float> &src = norm ? f->uvn : f->uv;
    uv.insert(uv.end(), src.begin(), src.end());
    mo.push_back((int)mc.size());
  }
}
} // namespace

// stage[f]: 1 grouped for a plane, 2 RANSAC inlier, 3 refinement inlier.  Other outputs as ovp_plane_init_tracks.  tri_p / tri_status (may be
// NULL): the triangulation of the candidates with >= 2 measurements, in input order, used instead of the oracle's own.
extern "C" int orcpi_plane_init_tracks(void *h, int F, const int *meas_offset, const int *meas_clone, const float *uv, const float *uv_norm,
                                       const long long *featid, const long long *planeid, double sigma_pix, double sigma_c, int max_msckf_plane,
                                       int plane_init_min_feat, double plane_init_max_cond, int shuffle_kind, const double *tri_p,
                                       const int *tri_status, int *feat_status, double *p_out, int *stage, int *n_planes, long long *plane_ids,
                                       int *plane_status, int *new_handles, double *cp_out) {
  *n_planes = 0;
  std::vector<Feat> store(F);
  for (int f = 0; f < F; f++) {
    Feat &x = store[f];
    x.index = f;
    x.featid = featid[f];
    x.planeid = planeid[f];
    x.clone.assign(meas_clone + meas_offset[f], meas_clone + meas_offset[f + 1]);
    x.uv.assign(uv + 2 * meas_offset[f], uv + 2 * meas_offset[f + 1]);
    x.uvn.assign(uv_norm + 2 * meas_offset[f], uv_norm + 2 * meas_offset[f + 1]);
    x.p[0] = x.p[1] = x.p[2] = 0.0;
    feat_status[f] = 0;
    stage[f] = 0;
  }
  // :86-116 a feature with no plane, or whose plane is in the state, is skipped before its measurements are counted
  std::vector<Feat *> valid;
  for (Feat &x : store) {
    if (x.planeid == 0 || orc_plane_handle(h, x.planeid) >= 0)
      continue;
    if (x.clone.size() < 2) {
      feat_status[x.index] = -1; // erased from feature_vec, not deleted
      continue;
    }
    valid.push_back(&x);
  }
  if (valid.empty())
    return 0;
  // :139-165 triangulate + Gauss-Newton, drop the failures
  {
    std::vector<int> mo, mc, st(valid.size());
    std::vector<float> un;
    std::vector<double> pt(3 * valid.size());
    flatten(valid, true, mo, mc, un);
    if (tri_p && tri_status) {
      std::memcpy(pt.data(), tri_p, pt.size() * sizeof(double));
      std::memcpy(st.data(), tri_status, st.size() * sizeof(int));
    } else if (int e = orc_triangulate_features(h, (int)valid.size(), mo.data(), mc.data(), un.data(), pt.data(), st.data())) {
      return e;
    }
    std::vector<Feat *> kept;
    for (size_t i = 0; i < valid.size(); i++) {
      std::memcpy(valid[i]->p, &pt[3 * i], sizeof(valid[i]->p));
      if (st[i])
        kept.push_back(valid[i]);
      else
        feat_status[valid[i]->index] = -2;
    }
    valid.swap(kept);
  }
  // :168-177 ascending track length, std::sort (not stable)
  std::sort(valid.begin(), valid.end(), [](const Feat *a, const Feat *b) { return a->clone.size() < b->clone.size(); });
  // :179-198 group per plane; a plane stops taking features once its count is above max_msckf_plane
  std::map<long long, size_t> count;
  std::map<long long, std::vector<Feat *>> plane_feats;
  for (Feat *x : valid) {
    feat_status[x->index] = 2;
    if ((int)count[x->planeid] > max_msckf_plane)
      continue;
    count[x->planeid]++;
    plane_feats[x->planeid].push_back(x);
    stage[x->index] = 1;
  }
  const double fx = [&] {
    const int hi = orc_handle_intr(h);
    std::vector<double> v(orc_var_nvalue(h, hi));
    orc_var_get(h, hi, v.data(), nullptr);
    return v[0];
  }();
  // :223-293 a linearisation point for every plane: RANSAC with the init thresholds, then the refinement with the plane free
  std::map<long long, std::vector<double>> estimates;
  std::map<long long, int> status;
  std::map<long long, std::vector<double>> cps;
  for (auto &kv : plane_feats) {
    std::vector<Feat *> &feats = kv.second;
    status[kv.first] = -2;
    cps[kv.first] = std::vector<double>(3, 0.0);
    std::vector<double> pts;
    for (Feat *x : feats)
      pts.insert(pts.end(), x->p, x->p + 3);
    double abcd[4];
    std::vector<int> inl(feats.size());
    int ok = 0;
    if (int e = orc_plane_fitting((int)feats.size(), pts.data(), plane_init_min_feat, plane_init_max_cond, shuffle_kind, abcd, inl.data(), &ok))
      return e;
    if (!ok)
      continue;
    std::vector<Feat *> in;
    for (size_t i = 0; i < feats.size(); i++)
      if (inl[i]) {
        in.push_back(feats[i]);
        stage[feats[i]->index] = 2;
      }
    feats.swap(in); // PlaneFitting.cpp:186
    double cp[3] = {-abcd[0] * abcd[3], -abcd[1] * abcd[3], -abcd[2] * abcd[3]};
    std::vector<int> mo, mc;
    std::vector<float> un;
    flatten(feats, true, mo, mc, un);
    pts.clear();
    for (Feat *x : feats)
      pts.insert(pts.end(), x->p, x->p + 3);
    std::vector<double> po(pts.size());
    double cpo[3];
    inl.assign(feats.size(), 0);
    if (int e = orc_optimize_plane(h, (int)feats.size(), mo.data(), mc.data(), un.data(), pts.data(), cp, sigma_pix / fx, sigma_c, 0, 0, po.data(), cpo,
                                   inl.data(), &ok, nullptr))
      return e;
    for (size_t i = 0; i < feats.size(); i++) // optimize_plane writes every feature back
      std::memcpy(feats[i]->p, &po[3 * i], sizeof(feats[i]->p));
    cps[kv.first].assign(cpo, cpo + 3);
    if (!ok) {
      status[kv.first] = -3;
      continue;
    }
    in.clear();
    for (size_t i = 0; i < feats.size(); i++)
      if (inl[i]) {
        in.push_back(feats[i]);
        stage[feats[i]->index] = 3;
      }
    feats.swap(in); // PlaneFitting.cpp:511
    status[kv.first] = -1;
    estimates[kv.first] = cps[kv.first];
  }
  // :297-481 on the oracle: the planes with a linearisation point, ascending id
  std::vector<Feat *> batch;
  std::vector<long long> est_ids, fid, fpid;
  std::vector<double> est_cp, bp;
  for (auto &kv : estimates) {
    est_ids.push_back(kv.first);
    est_cp.insert(est_cp.end(), kv.second.begin(), kv.second.end());
    for (Feat *x : plane_feats[kv.first]) {
      batch.push_back(x);
      fid.push_back(x->featid);
      fpid.push_back(x->planeid);
      bp.insert(bp.end(), x->p, x->p + 3);
    }
  }
  std::vector<int> ps(est_ids.size(), -1), nh(est_ids.size(), -1);
  if (!est_ids.empty()) {
    std::vector<int> mo, mc;
    std::vector<float> buv;
    flatten(batch, false, mo, mc, buv);
    if (int e = orc_plane_init(h, (int)batch.size(), mo.data(), mc.data(), buv.data(), bp.data(), fid.data(), fpid.data(), (int)est_ids.size(),
                               est_ids.data(), est_cp.data(), sigma_pix, ps.data(), nh.data()))
      return e;
  }
  int k = 0;
  for (auto &kv : plane_feats) {
    plane_ids[k] = kv.first;
    plane_status[k] = status[kv.first];
    new_handles[k] = -1;
    std::memcpy(cp_out + 3 * k, cps[kv.first].data(), 3 * sizeof(double));
    for (size_t j = 0; j < est_ids.size(); j++)
      if (est_ids[j] == kv.first) {
        plane_status[k] = ps[j];
        new_handles[k] = nh[j];
        if (ps[j] == 1)
          for (Feat *x : kv.second)
            feat_status[x->index] = 1; // to_delete, feature_vec_used (:459-475)
      }
    k++;
  }
  *n_planes = k;
  for (const Feat &x : store)
    std::memcpy(p_out + 3 * x.index, x.p, sizeof(x.p));
  return 0;
}

// Reference-side adapter for TrackPlane::perform_plane_detection_monocular (track_plane/TrackPlane.cpp:580-1121): the reference's locks and
// early returns, undistort_cv per point on the host, then one ovp_plane_track_frame; hist_feat_to_plane, hist_plane_to_oldplanes and the
// tri_* display members are filled from the readbacks, so get_feature2plane, get_plane2oldplane, get_tracking_info and the display
// functions run unchanged.  The per-feature normal windows (hist_feat_norms_inG) stay on the device: the display draws no vertex-normal
// markers.  Built in place of that method's definition and linked with -lovp.
#include "track_plane/TrackPlane.h"

#include <cstdio>
#include <cstdlib>

using namespace ov_plane;

ovp_ctx *TrackPlane::ctx = nullptr;

static void ck(int st) {
  if (st) {
    std::fprintf(stderr, "[PLANE-TRACK]: %s\n", ovp_last_error(TrackPlane::ctx));
    std::exit(EXIT_FAILURE);
  }
}

void TrackPlane::perform_plane_detection_monocular(size_t cam_id) {
  const auto t0 = std::chrono::steady_clock::now();
  std::lock_guard<std::mutex> lckv1(mtx_last_vars);
  std::lock_guard<std::mutex> lckv2(mtx_hist_vars);
  cv::Mat img = img_last[cam_id].clone(), mask = img_mask_last[cam_id].clone();
  const double time = time_last[cam_id];
  std::vector<cv::KeyPoint> pts_left = pts_last[cam_id];
  std::vector<size_t> ids_left = ids_last[cam_id];
  if (pts_left.empty() || ids_left.empty())
    return;
  if (hist_state.find(time) == hist_state.end() || hist_calib.find(cam_id) == hist_calib.end())
    return;
  if (!options_sent) { // TrackPlane takes its options once, at construction
    const ovp_plane_track_options o = {options.max_tri_side_px,  options.max_norm_count,    options.max_norm_avg_max, options.max_norm_avg_var,
                                       options.max_norm_deg,     options.max_dist_between_z, options.max_pairwise_px, options.min_norms,
                                       options.check_old_feats,  options.filter_num_feat,   options.filter_z_thresh,  options.feat_init_min_obs,
                                       options.min_dist,         options.max_dist,          options.max_cond_number};
    ck(ovp_plane_track_set_options(ctx, &o));
    options_sent = true;
  }
  const int n = (int)pts_left.size();
  std::vector<int64_t> fid(n);
  std::vector<float> uv(2 * (size_t)n), uvn(2 * (size_t)n);
  for (int i = 0; i < n; i++) {
    fid[i] = (int64_t)ids_left[i];
    uv[2 * i] = pts_left[i].pt.x;
    uv[2 * i + 1] = pts_left[i].pt.y;
    const cv::Point2f pn = camera_calib.at(cam_id)->undistort_cv(pts_left[i].pt);
    uvn[2 * i] = pn.x;
    uvn[2 * i + 1] = pn.y;
  }
  const Eigen::VectorXd &state = hist_state.at(time), &calib = hist_calib.at(cam_id);
  double pose7[7], calib7[7];
  for (int k = 0; k < 7; k++) {
    pose7[k] = state(k);
    calib7[k] = calib(k);
  }
  ck(ovp_plane_track_frame(ctx, pose7, calib7, n, fid.data(), uv.data(), uvn.data()));

  // readbacks: the maps, then the mesh over the features that triangulated (the surviving order)
  std::vector<int64_t> f(n), p(n);
  int nf = 0;
  ck(ovp_plane_track_feature2plane(ctx, n, f.data(), p.data(), &nf));
  hist_feat_to_plane.clear();
  for (int i = 0; i < nf; i++)
    hist_feat_to_plane[(size_t)f[i]] = (size_t)p[i];
  std::vector<int64_t> pp(OVP_PLANE_TRACK_MAX_MERGES), po(OVP_PLANE_TRACK_MAX_MERGES);
  int np = 0;
  ck(ovp_plane_track_plane2oldplane(ctx, OVP_PLANE_TRACK_MAX_MERGES, pp.data(), po.data(), &np));
  hist_plane_to_oldplanes.clear();
  for (int i = 0; i < np; i++)
    hist_plane_to_oldplanes[(size_t)pp[i]].insert((size_t)po[i]);
  int nt = 0;
  ck(ovp_plane_track_mesh(ctx, 0, nullptr, nullptr, &nt));
  std::vector<int> tri(3 * (size_t)nt + 3);
  std::vector<double> nrm(3 * (size_t)nt + 3);
  ck(ovp_plane_track_mesh(ctx, nt, tri.data(), nrm.data(), &nt));
  // the mesh's vertices: the features that had a 3D estimate, in the frame's order
  std::vector<int64_t> vid(n);
  std::vector<float> vuv(2 * (size_t)n);
  int nv = 0;
  ck(ovp_plane_track_vertices(ctx, n, vid.data(), vuv.data(), &nv));
  std::vector<CDT::V2d<float>> verts((size_t)nv);
  std::vector<size_t> vert_ids((size_t)nv);
  std::vector<cv::KeyPoint> vert_pts((size_t)nv);
  for (int k = 0; k < nv; k++) {
    verts[k] = CDT::V2d<float>::make(vuv[2 * k], vuv[2 * k + 1]);
    vert_ids[k] = (size_t)vid[k];
    vert_pts[k].pt.x = vuv[2 * k];
    vert_pts[k].pt.y = vuv[2 * k + 1];
  }
  std::vector<CDT::Triangle> tris((size_t)nt);
  std::vector<Eigen::Vector3d> norms((size_t)nt);
  for (int t = 0; t < nt; t++)
    for (int j = 0; j < 3; j++) {
      tris[t].vertices[j] = (unsigned int)tri[3 * t + j];
      norms[t](j) = nrm[3 * t + j];
    }
  tri_img_last[cam_id] = img;
  tri_time_last[cam_id] = time;
  tri_mask_last[cam_id] = mask;
  tri_cdt_tri[cam_id] = tris;
  tri_cdt_tri_norms[cam_id] = norms;
  tri_cdt_verts[cam_id] = verts;
  tri_cdt_vert_ids[cam_id] = vert_ids;
  tri_cdt_vert_pts[cam_id] = vert_pts;
  // one device call: the split into triangulation / Delaunay / matching is not timed separately
  _tracking_time_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// STAND-IN for ov_plane/src/track_plane/TrackPlane.h:252-263 and the members perform_plane_detection_monocular reads and fills, with minimal
// stand-ins of the OpenCV / CDT / ov_core types they use.
#pragma once
#include <Eigen/Dense>
#include <chrono>
#include <cstddef>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <unordered_map>
#include <vector>

#include "ovp.h"

namespace cv {
struct Point2f {
  float x = 0, y = 0;
};
struct KeyPoint {
  Point2f pt;
};
struct Mat {
  Mat clone() const { return *this; }
};
} // namespace cv
namespace CDT {
struct Triangle {
  unsigned int vertices[3];
};
template <typename T> struct V2d {
  T x, y;
  static V2d make(T x, T y) { return V2d{x, y}; }
};
} // namespace CDT
namespace ov_core {
struct CamBase {
  virtual ~CamBase() {}
  virtual cv::Point2f undistort_cv(const cv::Point2f &uv_dist) = 0;
};
} // namespace ov_core
namespace ov_plane {
struct TrackPlaneOptions {
  int max_tri_side_px = 200, max_norm_count = 5;
  double max_norm_avg_max = 25.0, max_norm_avg_var = 25.0, max_norm_deg = 25.0, max_dist_between_z = 0.10;
  int max_pairwise_px = 100, min_norms = 3;
  bool check_old_feats = true;
  int filter_num_feat = 4;
  double filter_z_thresh = 1.2;
  int feat_init_min_obs = 4;
  double min_dist = 0.10, max_dist = 60, max_cond_number = 8000;
};
class TrackPlane {
public:
  void perform_plane_detection_monocular(size_t cam_id);
  // added by the integration: the filter context the tracker lives in (set once by VioManager after ovp_create)
  static ovp_ctx *ctx;

protected:
  TrackPlaneOptions options;
  std::unordered_map<size_t, std::shared_ptr<ov_core::CamBase>> camera_calib;
  std::mutex mtx_last_vars, mtx_hist_vars;
  std::map<size_t, cv::Mat> img_last, img_mask_last;
  std::unordered_map<size_t, double> time_last;
  std::unordered_map<size_t, std::vector<cv::KeyPoint>> pts_last;
  std::unordered_map<size_t, std::vector<size_t>> ids_last;
  std::map<double, Eigen::VectorXd> hist_state;
  std::map<size_t, Eigen::VectorXd> hist_calib;
  std::map<size_t, size_t> hist_feat_to_plane;
  std::map<size_t, std::set<size_t>> hist_plane_to_oldplanes;
  std::map<size_t, cv::Mat> tri_img_last, tri_mask_last;
  std::map<size_t, double> tri_time_last;
  std::map<size_t, std::vector<CDT::Triangle>> tri_cdt_tri;
  std::map<size_t, std::vector<Eigen::Vector3d>> tri_cdt_tri_norms;
  std::map<size_t, std::vector<CDT::V2d<float>>> tri_cdt_verts;
  std::map<size_t, std::vector<size_t>> tri_cdt_vert_ids;
  std::map<size_t, std::vector<cv::KeyPoint>> tri_cdt_vert_pts;
  std::map<size_t, std::vector<Eigen::Vector3d>> hist_feat_norms_inG;
  double _tracking_time_triangulation = 0, _tracking_time_delaunay = 0, _tracking_time_matching = 0, _tracking_time_total = 0;
  bool options_sent = false; // added by the integration: ovp_plane_track_set_options ran
};
} // namespace ov_plane

// MINIMAL STAND-IN for ov_plane/src/state/State.h (public members the adapter touches, State.h:53-134) PLUS the members the
// integration adds to it (adapter/README.md): the device context and the Type* <-> handle map.
#pragma once
#include "ovp.h"
#include "types/Type.h"
#include <map>
#include <memory>
#include <unordered_map>
#include <vector>
namespace ov_plane {
struct StateOptions {
  int max_clone_size = 11;
  int max_aruco_features = 1024;
  bool do_calib_camera_timeoffset = false;
  ov_type::LandmarkRepresentation::Representation feat_rep_slam = ov_type::LandmarkRepresentation::GLOBAL_3D; // StateOptions.h:82-88
  ov_type::LandmarkRepresentation::Representation feat_rep_aruco = ov_type::LandmarkRepresentation::GLOBAL_3D;
  // StateOptions.h:96-150 (plane options the updaters read)
  bool use_plane_constraint = true, use_plane_constraint_msckf = true, use_plane_constraint_slamu = true,
       use_plane_constraint_slamd = true, use_refine_plane_feat = true;
  double sigma_constraint = 0.01;
  int plane_msckf_min_feat = 20;
  double plane_msckf_max_cond = 100.0;
  int max_msckf_plane = 20; // StateOptions.h: per-plane feature cap of init_vio_plane
  int plane_init_min_feat = 8;
  double plane_init_max_cond = 200.0;
};
class State {
public:
  double margtimestep();
  int max_covariance_size();
  double _timestamp = -1;
  StateOptions _options;
  std::shared_ptr<ov_type::IMU> _imu;
  std::map<double, std::shared_ptr<ov_type::PoseJPL>> _clones_IMU;
  std::unordered_map<size_t, std::shared_ptr<ov_type::Landmark>> _features_SLAM;
  std::shared_ptr<ov_type::Vec> _calib_dt_CAMtoIMU;
  std::unordered_map<size_t, std::shared_ptr<ov_type::PoseJPL>> _calib_IMUtoCAM;
  std::unordered_map<size_t, std::shared_ptr<ov_type::Vec>> _cam_intrinsics;
  std::unordered_map<size_t, std::shared_ptr<ov_type::Vec>> _features_PLANE;
  std::unordered_map<size_t, size_t> _features_SLAM_to_PLANE;

  // ---- added by the integration (the covariance and the variable table live on the device) ----
  ovp_ctx *ctx = nullptr;
  std::unordered_map<ov_type::Type *, int> handle;                  // variable -> ovp handle
  std::unordered_map<int, std::shared_ptr<ov_type::Type>> by_handle; // ovp handle -> variable

private:
  friend class StateHelper;
  std::vector<std::shared_ptr<ov_type::Type>> _variables;
};
} // namespace ov_plane

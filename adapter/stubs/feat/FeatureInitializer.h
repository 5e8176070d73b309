// MINIMAL STAND-IN for ov_core feat/FeatureInitializer.h: ClonePose as used by PlaneFitting::optimize_plane, and the options the updaters
// read through config().  Syntax check only.
#pragma once
#include <Eigen/Dense>
#include "update/UpdaterOptions.h"
namespace ov_core {
class FeatureInitializer {
public:
  explicit FeatureInitializer(FeatureInitializerOptions &options) : _options(options) {}
  const FeatureInitializerOptions config() { return _options; }
  FeatureInitializerOptions _options;
  struct ClonePose {
    Eigen::Matrix3d _Rot;
    Eigen::Vector3d _pos;
    const Eigen::Matrix3d &Rot() { return _Rot; }
    const Eigen::Vector3d &pos() { return _pos; }
  };
};
} // namespace ov_core

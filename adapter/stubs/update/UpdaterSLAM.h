// STAND-IN for ov_plane/src/update/UpdaterSLAM.h:53-125 (the public call surface; same signatures).  Syntax check only.
#pragma once
#include <Eigen/Dense>
#include <map>
#include <memory>
#include <vector>

#include "feat/FeatureInitializer.h"
#include "update/UpdaterOptions.h"

namespace ov_core {
class Feature;
}
namespace ov_plane {
class State;
class UpdaterSLAM {
public:
  UpdaterSLAM(UpdaterOptions &options_slam, UpdaterOptions &options_aruco, ov_core::FeatureInitializerOptions &feat_init_options);
  void update(std::shared_ptr<State> state, std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec, const std::map<size_t, size_t> &feat2plane);
  void delayed_init(std::shared_ptr<State> state, std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec,
                    const std::map<size_t, size_t> &feat2plane);
  void change_anchors(std::shared_ptr<State> state);

protected:
  std::shared_ptr<ov_core::FeatureInitializer> initializer_feat;
  UpdaterOptions _options_slam;
  UpdaterOptions _options_aruco;
};
} // namespace ov_plane

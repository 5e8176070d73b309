// STAND-IN for ov_plane/src/update/UpdaterPlane.h:59-115 (init_vio_plane; the two static helpers are declared for completeness).
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
class UpdaterPlane {
public:
  UpdaterPlane(UpdaterOptions &options, ov_core::FeatureInitializerOptions &feat_init_options);
  void init_vio_plane(std::shared_ptr<State> state, std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec,
                      std::vector<std::shared_ptr<ov_core::Feature>> &feature_vec_used, const std::map<size_t, size_t> &feat2plane);

protected:
  std::shared_ptr<ov_core::FeatureInitializer> initializer_feat;
  UpdaterOptions _options;
};
} // namespace ov_plane

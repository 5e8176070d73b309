// STAND-IN for ov_plane/src/update/UpdaterOptions.h:38-54.  Syntax check only.
#pragma once
namespace ov_plane {
struct UpdaterOptions {
  double chi2_multipler = 5;
  double sigma_pix = 1;
  double sigma_pix_sq = 1;
};
} // namespace ov_plane
namespace ov_core {
// feat/FeatureInitializerOptions.h (OpenVINS @74a63cf): its twelve fields and defaults
struct FeatureInitializerOptions {
  bool triangulate_1d = false;
  bool refine_features = true;
  int max_runs = 5;
  double init_lamda = 1e-3;
  double max_lamda = 1e10;
  double min_dx = 1e-6;
  double min_dcost = 1e-6;
  double lam_mult = 10;
  double min_dist = 0.10;
  double max_dist = 60;
  double max_baseline = 40;
  double max_cond_number = 10000;
};
} // namespace ov_core

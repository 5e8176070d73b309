// Per-feature triangulation, the step immediately before the update path (UpdaterMSCKF.cpp:142-194, UpdaterSLAM.cpp:118-160):
// ov_core::FeatureInitializer::single_triangulation (linear, in the anchor camera frame) followed by single_gaussnewton
// (Levenberg-Marquardt on the inverse-depth parameters alpha, beta, rho).  ov_core is not part of /root/reference (OpenVINS
// @74a63cf, ReadMe.md:39): this restates the published algorithm of that commit with its default FeatureInitializerOptions
// (max_runs 5, init_lamda 1e-3, max_lamda 1e10, min_dx 1e-6, min_dcost 1e-6, lam_mult 10, min_dist 0.10, max_dist 60,
// max_baseline 40, max_cond_number 10000).  Camera poses: R_GtoCi = R_ItoC R_GtoIi, p_CiinG = p_IiinG - R_GtoCi^T p_IinC
// (UpdaterMSCKF.cpp:122-140).  The anchor is the LAST measurement's camera.  Normalised coordinates are single precision and the
// residuals are formed in single precision like ov_core (Feature::uvs_norm is an Eigen::VectorXf).
//
// FeatureInitializerOptions::triangulate_1d selects FeatureInitializer::single_triangulation_1d as the linear stage instead: the depth d
// of the anchor measurement's bearing b_A = normalize([u_A, v_A, 1]) that minimises sum_k |skew(b_k) (d b_A - p_CkinA)|^2 over every
// other measurement k (another observation from the anchor's clone included; only the anchor measurement itself is skipped), with
// b_k = normalize(R_AtoCk^T [u_k, v_k, 1]), R_AtoCk = R_GtoCk R_GtoA^T, p_CkinA = R_GtoA (p_CkinG - p_AinG):
//   a_k = skew(b_k) b_A,  A = sum a_k . a_k,  b = sum a_k . (skew(b_k) p_CkinA),  d = b / A,  p_FinA = d b_A.
// It rejects when p_FinA.z < min_dist, p_FinA.z > max_dist or |p_FinA| is NaN (A = 0 gives NaN or +-inf, and one of these catches it);
// there is no condition-number rule.  FeatureInitializerOptions::refine_features = false skips single_gaussnewton: the linear stage's
// p_FinA, after that stage's own rules, is the result (no baseline-ratio rule, no second depth check).
#pragma once
#include "jacobian_core.h"

namespace ovp {

struct TriOptions {
  int max_runs;
  double init_lamda, max_lamda, min_dx, min_dcost, lam_mult, min_dist, max_dist, max_baseline, max_cond_number;
};

// 3x3 symmetric solve A x = b (A positive definite here) by Cholesky; returns false when a pivot is not positive
OVP_HD bool tri_solve3(const double *A, const double *b, double *x) {
  double l00 = A[0];
  if (!(l00 > 0.0))
    return false;
  l00 = sqrt(l00);
  const double l10 = A[3] / l00, l20 = A[6] / l00;
  double l11 = A[4] - l10 * l10;
  if (!(l11 > 0.0))
    return false;
  l11 = sqrt(l11);
  const double l21 = (A[7] - l20 * l10) / l11;
  double l22 = A[8] - l20 * l20 - l21 * l21;
  if (!(l22 > 0.0))
    return false;
  l22 = sqrt(l22);
  const double y0 = b[0] / l00, y1 = (b[1] - l10 * y0) / l11, y2 = (b[2] - l20 * y0 - l21 * y1) / l22;
  x[2] = y2 / l22;
  x[1] = (y1 - l21 * x[2]) / l11;
  x[0] = (y0 - l10 * x[1] - l20 * x[2]) / l00;
  return true;
}
// extreme eigenvalues of a symmetric 3x3 matrix (trigonometric closed form): the singular values of the normal matrix
OVP_HD void tri_eig_minmax(const double *A, double &emin, double &emax) {
  const double p1 = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
  const double q = (A[0] + A[4] + A[8]) / 3.0;
  const double p2 = (A[0] - q) * (A[0] - q) + (A[4] - q) * (A[4] - q) + (A[8] - q) * (A[8] - q) + 2.0 * p1;
  const double p = sqrt(p2 / 6.0);
  if (!(p > 0.0)) {
    emin = emax = q;
    return;
  }
  double B[9];
  for (int i = 0; i < 9; i++)
    B[i] = (A[i] - ((i % 4 == 0) ? q : 0.0)) / p;
  double r = 0.5 * (B[0] * (B[4] * B[8] - B[5] * B[7]) - B[1] * (B[3] * B[8] - B[5] * B[6]) + B[2] * (B[3] * B[7] - B[4] * B[6]));
  r = r < -1.0 ? -1.0 : (r > 1.0 ? 1.0 : r);
  const double phi = acos(r) / 3.0;
  emax = q + 2.0 * p * cos(phi);
  emin = q + 2.0 * p * cos(phi + 2.0943951023931953);
}

// Camera poses come from a table indexed by idx[k] for measurement k: Rc (9 each, R_GtoCi row-major) and pc (3 each, p_CiinG);
// uvn: 2 floats per measurement.  Returns 1 and p_FinG on success; 0 when single_triangulation or single_gaussnewton would return false.
// p_FinA (optional): the position in the anchor camera frame, written on success (FeatureInitializer's Feature::p_FinA).
// single_triangulation_1d: p_FinA (3) of the track; false when the reference would return false
OVP_HD bool triangulate_linear_1d(int m, const int *idx, const double *Rc, const double *pc, const float *uvn, const TriOptions &o, const double *RA,
                                  const double *pA, double *pf) {
  double bA[3] = {(double)uvn[2 * (m - 1)], (double)uvn[2 * (m - 1) + 1], 1.0};
  const double nA = sqrt(bA[0] * bA[0] + bA[1] * bA[1] + bA[2] * bA[2]);
  bA[0] /= nA;
  bA[1] /= nA;
  bA[2] /= nA;
  double A = 0.0, b = 0.0;
  for (int k = 0; k < m - 1; k++) { // every measurement but the anchor's (the last)
    const double *R = Rc + 9 * idx[k], *p = pc + 3 * idx[k];
    double RAt[9]; // R_AtoCk = R_GtoCk R_GtoA^T
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        RAt[3 * i + j] = R[3 * i] * RA[3 * j] + R[3 * i + 1] * RA[3 * j + 1] + R[3 * i + 2] * RA[3 * j + 2];
    double d[3] = {p[0] - pA[0], p[1] - pA[1], p[2] - pA[2]}, pCA[3];
    mat3_vec(RA, d, pCA); // p_CkinA
    const double u = (double)uvn[2 * k], v = (double)uvn[2 * k + 1];
    double bk[3] = {RAt[0] * u + RAt[3] * v + RAt[6], RAt[1] * u + RAt[4] * v + RAt[7], RAt[2] * u + RAt[5] * v + RAt[8]}; // R_AtoCk^T [u v 1]
    const double nb = sqrt(bk[0] * bk[0] + bk[1] * bk[1] + bk[2] * bk[2]);
    bk[0] /= nb;
    bk[1] /= nb;
    bk[2] /= nb;
    // skew(b_k) x = b_k x x
    const double a[3] = {bk[1] * bA[2] - bk[2] * bA[1], bk[2] * bA[0] - bk[0] * bA[2], bk[0] * bA[1] - bk[1] * bA[0]};
    const double w[3] = {bk[1] * pCA[2] - bk[2] * pCA[1], bk[2] * pCA[0] - bk[0] * pCA[2], bk[0] * pCA[1] - bk[1] * pCA[0]};
    A += a[0] * a[0] + a[1] * a[1] + a[2] * a[2];
    b += a[0] * w[0] + a[1] * w[1] + a[2] * w[2];
  }
  const double depth = b / A;
  for (int i = 0; i < 3; i++)
    pf[i] = depth * bA[i];
  const double nrm = sqrt(pf[0] * pf[0] + pf[1] * pf[1] + pf[2] * pf[2]);
  return !(pf[2] < o.min_dist || pf[2] > o.max_dist || nrm != nrm);
}

// OneD: FeatureInitializerOptions::triangulate_1d, Refine: refine_features.  <false, true> is ov_core's default.
template <bool OneD, bool Refine>
OVP_HD int triangulate_feature(int m, const int *idx, const double *Rc, const double *pc, const float *uvn, const TriOptions &o, double *p_FinG,
                               double *p_FinA = nullptr) {
  const double *RA = Rc + 9 * idx[m - 1], *pA = pc + 3 * idx[m - 1]; // anchor = last measurement
  // ---- single_triangulation ----  (A, b, then pf: the declaration order of the 3-D-only kernel, whose SASS <false, true> keeps)
  double A[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
  if (!OneD)
    for (int k = 0; k < m; k++) {
      const double *R = Rc + 9 * idx[k], *p = pc + 3 * idx[k];
      double RAt[9]; // R_AtoCi = R_GtoCi R_GtoA^T
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
          RAt[3 * i + j] = R[3 * i] * RA[3 * j] + R[3 * i + 1] * RA[3 * j + 1] + R[3 * i + 2] * RA[3 * j + 2];
      double d[3] = {p[0] - pA[0], p[1] - pA[1], p[2] - pA[2]}, pCA[3];
      mat3_vec(RA, d, pCA); // p_CiinA
      const double u = (double)uvn[2 * k], v = (double)uvn[2 * k + 1];
      double bi[3] = {RAt[0] * u + RAt[3] * v + RAt[6], RAt[1] * u + RAt[4] * v + RAt[7], RAt[2] * u + RAt[5] * v + RAt[8]}; // R_AtoCi^T [u v 1]
      const double nb = sqrt(bi[0] * bi[0] + bi[1] * bi[1] + bi[2] * bi[2]);
      bi[0] /= nb;
      bi[1] /= nb;
      bi[2] /= nb;
      // Ai = skew(b)^T skew(b) = |b|^2 I - b b^T
      const double bb = bi[0] * bi[0] + bi[1] * bi[1] + bi[2] * bi[2];
      double Ai[9];
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
          Ai[3 * i + j] = ((i == j) ? bb : 0.0) - bi[i] * bi[j];
      for (int i = 0; i < 9; i++)
        A[i] += Ai[i];
      for (int i = 0; i < 3; i++)
        b[i] += Ai[3 * i] * pCA[0] + Ai[3 * i + 1] * pCA[1] + Ai[3 * i + 2] * pCA[2];
    }
  double pf[3];
  if (OneD) {
    if (!triangulate_linear_1d(m, idx, Rc, pc, uvn, o, RA, pA, pf))
      return 0;
  } else {
    if (!tri_solve3(A, b, pf))
      return 0;
    double emin, emax;
    tri_eig_minmax(A, emin, emax);
    const double condA = emax / emin;
    const double nrm = sqrt(pf[0] * pf[0] + pf[1] * pf[1] + pf[2] * pf[2]);
    if (!(fabs(condA) <= o.max_cond_number) || pf[2] < o.min_dist || pf[2] > o.max_dist || nrm != nrm)
      return 0;
  }
  if (!Refine) { // the linear stage's result, after its own rules only
    for (int i = 0; i < 3; i++)
      p_FinG[i] = RA[i] * pf[0] + RA[3 + i] * pf[1] + RA[6 + i] * pf[2] + pA[i];
    if (p_FinA)
      for (int i = 0; i < 3; i++)
        p_FinA[i] = pf[i];
    return 1;
  }
  // ---- single_gaussnewton ----
  double rho = 1.0 / pf[2], alpha = pf[0] / pf[2], beta = pf[1] / pf[2];
  double lam = o.init_lamda, eps = 10000.0;
  int runs = 0;
  bool recompute = true;
  double Hess[9], grad[3];
  // cost at (al, be, rh); when hg != 0 also accumulates Hess / grad
  auto accumulate = [&](double al, double be, double rh, bool hg) {
    double err = 0.0;
    if (hg)
      for (int i = 0; i < 9; i++) {
        Hess[i] = 0.0;
        if (i < 3)
          grad[i] = 0.0;
      }
    for (int k = 0; k < m; k++) {
      const double *R = Rc + 9 * idx[k], *p = pc + 3 * idx[k];
      double RAt[9];
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
          RAt[3 * i + j] = R[3 * i] * RA[3 * j] + R[3 * i + 1] * RA[3 * j + 1] + R[3 * i + 2] * RA[3 * j + 2];
      double d[3] = {p[0] - pA[0], p[1] - pA[1], p[2] - pA[2]}, pCA[3], pAC[3];
      mat3_vec(RA, d, pCA);
      mat3_vec(RAt, pCA, pAC);
      pAC[0] = -pAC[0];
      pAC[1] = -pAC[1];
      pAC[2] = -pAC[2]; // p_AinCi = -R_AtoCi p_CiinA
      const double hi1 = RAt[0] * al + RAt[1] * be + RAt[2] + rh * pAC[0];
      const double hi2 = RAt[3] * al + RAt[4] * be + RAt[5] + rh * pAC[1];
      const double hi3 = RAt[6] * al + RAt[7] * be + RAt[8] + rh * pAC[2];
      const float z0 = (float)(hi1 / hi3), z1 = (float)(hi2 / hi3);
      const float r0 = uvn[2 * k] - z0, r1 = uvn[2 * k + 1] - z1;
      const float rn = sqrtf(r0 * r0 + r1 * r1);
      err += (double)rn * (double)rn;
      if (hg) {
        const double h32 = hi3 * hi3;
        const double H[6] = {(RAt[0] * hi3 - hi1 * RAt[6]) / h32, (RAt[1] * hi3 - hi1 * RAt[7]) / h32, (pAC[0] * hi3 - hi1 * pAC[2]) / h32,
                             (RAt[3] * hi3 - hi2 * RAt[6]) / h32, (RAt[4] * hi3 - hi2 * RAt[7]) / h32, (pAC[1] * hi3 - hi2 * pAC[2]) / h32};
        for (int i = 0; i < 3; i++) {
          grad[i] += H[i] * (double)r0 + H[3 + i] * (double)r1;
          for (int j = 0; j < 3; j++)
            Hess[3 * i + j] += H[i] * H[j] + H[3 + i] * H[3 + j];
        }
      }
    }
    return err;
  };
  double cost_old = accumulate(alpha, beta, rho, false);
  while (runs < o.max_runs && lam < o.max_lamda && eps > o.min_dx) {
    if (recompute)
      accumulate(alpha, beta, rho, true);
    double Hl[9];
    for (int i = 0; i < 9; i++)
      Hl[i] = Hess[i];
    Hl[0] *= (1.0 + lam);
    Hl[4] *= (1.0 + lam);
    Hl[8] *= (1.0 + lam);
    double dx[3];
    if (!tri_solve3(Hl, grad, dx))
      return 0;
    const double cost = accumulate(alpha + dx[0], beta + dx[1], rho + dx[2], false);
    if (cost <= cost_old && (cost_old - cost) / cost_old < o.min_dcost) {
      alpha += dx[0];
      beta += dx[1];
      rho += dx[2];
      eps = 0;
      break;
    }
    if (cost <= cost_old) {
      recompute = true;
      cost_old = cost;
      alpha += dx[0];
      beta += dx[1];
      rho += dx[2];
      runs++;
      lam = lam / o.lam_mult;
      eps = sqrt(dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2]);
    } else {
      recompute = false;
      lam = lam * o.lam_mult;
    }
  }
  const double pfa[3] = {alpha / rho, beta / rho, 1.0 / rho};
  const double nf = sqrt(pfa[0] * pfa[0] + pfa[1] * pfa[1] + pfa[2] * pfa[2]);
  // largest baseline orthogonal to the bearing of the feature (the two tangent-plane directions of ov_core's Householder Q)
  double base_line_max = 0.0;
  for (int k = 0; k < m; k++) {
    const double *p = pc + 3 * idx[k];
    double d[3] = {p[0] - pA[0], p[1] - pA[1], p[2] - pA[2]}, pCA[3];
    mat3_vec(RA, d, pCA);
    const double along = (pCA[0] * pfa[0] + pCA[1] * pfa[1] + pCA[2] * pfa[2]) / nf;
    const double bl2 = pCA[0] * pCA[0] + pCA[1] * pCA[1] + pCA[2] * pCA[2] - along * along;
    const double bl = bl2 > 0.0 ? sqrt(bl2) : 0.0;
    if (bl > base_line_max)
      base_line_max = bl;
  }
  if (pfa[2] < o.min_dist || pfa[2] > o.max_dist || (nf / base_line_max) > o.max_baseline || nf != nf)
    return 0;
  // p_FinG = R_GtoA^T p_FinA + p_AinG
  for (int i = 0; i < 3; i++)
    p_FinG[i] = RA[i] * pfa[0] + RA[3 + i] * pfa[1] + RA[6 + i] * pfa[2] + pA[i];
  if (p_FinA)
    for (int i = 0; i < 3; i++)
      p_FinA[i] = pfa[i];
  return 1;
}

} // namespace ovp

// Per-measurement arithmetic of UpdaterHelper::get_feature_jacobian_full (UpdaterHelper.cpp:350-441, :447-512), mono camera,
// GLOBAL_3D representation, radtan distortion (ov_core::CamRadtan — every shipped config, config/*/kalibr_imucam_chain.yaml); at the end,
// the terms that chain the bearing rows onto a landmark held in one of the other representations (landmark_rep_terms).
// Shared by the CUDA feature kernels and by host code of the library (camera poses in planefit.cu / anchors.cu), hence __host__ __device__.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define OVP_HD __host__ __device__ __forceinline__
#else
#define OVP_HD inline
#endif

namespace ovp {

// JPL quaternion [x y z w] -> rotation, R = (2w^2-1) I - 2w [v x] + 2 v v^T   (row-major R[3*i+j])
OVP_HD void quat_to_rot(const double *q, double *R) {
  double x = q[0], y = q[1], z = q[2], w = q[3];
  double s = 2.0 * w * w - 1.0;
  R[0] = s + 2.0 * x * x;
  R[1] = 2.0 * w * z + 2.0 * x * y;
  R[2] = -2.0 * w * y + 2.0 * x * z;
  R[3] = -2.0 * w * z + 2.0 * y * x;
  R[4] = s + 2.0 * y * y;
  R[5] = 2.0 * w * x + 2.0 * y * z;
  R[6] = 2.0 * w * y + 2.0 * z * x;
  R[7] = -2.0 * w * x + 2.0 * z * y;
  R[8] = s + 2.0 * z * z;
}

OVP_HD void mat3_vec(const double *R, const double *v, double *o) {
  o[0] = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
  o[1] = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
  o[2] = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
}
OVP_HD void mat3_mul(const double *A, const double *B, double *C) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
// skew(v) row-major
OVP_HD void skew3(const double *v, double *S) {
  S[0] = 0;
  S[1] = -v[2];
  S[2] = v[1];
  S[3] = v[2];
  S[4] = 0;
  S[5] = -v[0];
  S[6] = -v[1];
  S[7] = v[0];
  S[8] = 0;
}

// cam = [fx fy cx cy k1 k2 p1 p2]
OVP_HD void radtan_distort(const double *cam, double x, double y, double &u, double &v) {
  double r = sqrt(x * x + y * y);
  double r_2 = r * r;
  double r_4 = r_2 * r_2;
  double x1 = x * (1 + cam[4] * r_2 + cam[5] * r_4) + 2 * cam[6] * x * y + cam[7] * (r_2 + 2 * x * x);
  double y1 = y * (1 + cam[4] * r_2 + cam[5] * r_4) + cam[6] * (r_2 + 2 * y * y) + 2 * cam[7] * x * y;
  u = cam[0] * x1 + cam[2];
  v = cam[1] * y1 + cam[3];
}
// dzn: 2x2 row-major d(uv)/d(uv_norm); dzeta: 2x8 row-major d(uv)/d(cam)
OVP_HD void radtan_jacobian(const double *cam, double x, double y, double *dzn, double *dzeta) {
  double r = sqrt(x * x + y * y);
  double r_2 = r * r;
  double r_4 = r_2 * r_2;
  double x_2 = x * x, y_2 = y * y, x_y = x * y;
  double rad = 1 + cam[4] * r_2 + cam[5] * r_4;
  dzn[0] = cam[0] * (rad + (2 * cam[4] * x_2 + 4 * cam[5] * x_2 * (x_2 + y_2)) + 2 * cam[6] * y + (2 * cam[7] * x + 4 * cam[7] * x));
  dzn[1] = cam[0] * (2 * cam[4] * x_y + 4 * cam[5] * x_y * (x_2 + y_2) + 2 * cam[6] * x + 2 * cam[7] * y);
  dzn[2] = cam[1] * (2 * cam[4] * x_y + 4 * cam[5] * x_y * (x_2 + y_2) + 2 * cam[6] * x + 2 * cam[7] * y);
  dzn[3] = cam[1] * (rad + (2 * cam[4] * y_2 + 4 * cam[5] * y_2 * (x_2 + y_2)) + 2 * cam[7] * x + (2 * cam[6] * y + 4 * cam[6] * y));
  double x1 = x * rad + 2 * cam[6] * x_y + cam[7] * (r_2 + 2 * x_2);
  double y1 = y * rad + cam[6] * (r_2 + 2 * y_2) + 2 * cam[7] * x_y;
  for (int i = 0; i < 16; i++)
    dzeta[i] = 0.0;
  dzeta[0] = x1;
  dzeta[2] = 1;
  dzeta[4] = cam[0] * x * r_2;
  dzeta[5] = cam[0] * x * r_4;
  dzeta[6] = 2 * cam[0] * x_y;
  dzeta[7] = cam[0] * (r_2 + 2 * x_2);
  dzeta[8 + 1] = y1;
  dzeta[8 + 3] = 1;
  dzeta[8 + 4] = cam[1] * y * r_2;
  dzeta[8 + 5] = cam[1] * y * r_4;
  dzeta[8 + 6] = cam[1] * (r_2 + 2 * y_2);
  dzeta[8 + 7] = 2 * cam[1] * x_y;
}

// One bearing measurement (UpdaterHelper.cpp:350-441).  All small matrices row-major.
//   q_cl/p_cl   : clone estimate (JPL quat xyzw, position)      q_cf/p_cf : clone first-estimate
//   R_C, p_C    : extrinsics R_ItoC (row-major), p_IinC (never FEJ'd, :379-380)
//   pf / pf_fej : feature position (best / first-estimate)
// Outputs: res[2], Hf[2x3], Hcl[2x6], Hcal[2x6], Hin[2x8]
OVP_HD void bearing_rows(const double *q_cl, const double *p_cl, const double *q_cf, const double *p_cf, int do_fej, const double *R_C,
                         const double *p_C, const double *cam, const double *pf, const double *pf_fej, float u_meas, float v_meas,
                         double white_px, double *res, double *Hf, double *Hcl, double *Hcal, double *Hin) {
  double R_i[9], d[3], p_I[3], p_Cm[3];
  quat_to_rot(q_cl, R_i);
  d[0] = pf[0] - p_cl[0];
  d[1] = pf[1] - p_cl[1];
  d[2] = pf[2] - p_cl[2];
  mat3_vec(R_i, d, p_I);
  mat3_vec(R_C, p_I, p_Cm);
  p_Cm[0] += p_C[0];
  p_Cm[1] += p_C[1];
  p_Cm[2] += p_C[2];
  double xn = p_Cm[0] / p_Cm[2], yn = p_Cm[1] / p_Cm[2];
  double ud, vd;
  radtan_distort(cam, xn, yn, ud, vd);
  res[0] = white_px * ((double)u_meas - ud);
  res[1] = white_px * ((double)v_meas - vd);
  if (do_fej) {
    quat_to_rot(q_cf, R_i);
    d[0] = pf_fej[0] - p_cf[0];
    d[1] = pf_fej[1] - p_cf[1];
    d[2] = pf_fej[2] - p_cf[2];
    mat3_vec(R_i, d, p_I);
    mat3_vec(R_C, p_I, p_Cm);
    p_Cm[0] += p_C[0];
    p_Cm[1] += p_C[1];
    p_Cm[2] += p_C[2];
    // uv_norm is NOT recomputed (UpdaterHelper.cpp:383)
  }
  double dzn[4], dzeta[16];
  radtan_jacobian(cam, xn, yn, dzn, dzeta);
  double X = p_Cm[0], Y = p_Cm[1], Z = p_Cm[2];
  double dp[6] = {1 / Z, 0, -X / (Z * Z), 0, 1 / Z, -Y / (Z * Z)};
  // A = white * dz_dzn * dzn_dpfc  (2x3)
  double A[6];
  for (int i = 0; i < 2; i++)
    for (int j = 0; j < 3; j++)
      A[3 * i + j] = white_px * (dzn[2 * i] * dp[j] + dzn[2 * i + 1] * dp[3 + j]);
  double B[9];
  mat3_mul(R_C, R_i, B); // dpfc_dpfg = R_ItoC * R_GtoIi
  for (int i = 0; i < 2; i++)
    for (int j = 0; j < 3; j++)
      Hf[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
  double Sk[9], RS[9];
  skew3(p_I, Sk);
  mat3_mul(R_C, Sk, RS); // R_ItoC * skew(p_FinIi)
  for (int i = 0; i < 2; i++)
    for (int j = 0; j < 3; j++) {
      Hcl[6 * i + j] = A[3 * i] * RS[j] + A[3 * i + 1] * RS[3 + j] + A[3 * i + 2] * RS[6 + j];
      Hcl[6 * i + 3 + j] = -Hf[3 * i + j];
    }
  double e[3] = {p_Cm[0] - p_C[0], p_Cm[1] - p_C[1], p_Cm[2] - p_C[2]};
  skew3(e, Sk);
  for (int i = 0; i < 2; i++)
    for (int j = 0; j < 3; j++) {
      Hcal[6 * i + j] = A[3 * i] * Sk[j] + A[3 * i + 1] * Sk[3 + j] + A[3 * i + 2] * Sk[6 + j];
      Hcal[6 * i + 3 + j] = A[3 * i + j];
    }
  for (int i = 0; i < 16; i++)
    Hin[i] = white_px * dzeta[i];
}

// Point-on-plane row (UpdaterHelper.cpp:450-497): res, H_f (1x3) and H_cp (1x3)
OVP_HD void plane_row(const double *pf, const double *pf_fej, const double *cp, const double *cp_fej, int do_fej, double white_c,
                      double &res, double *Hf, double *Hcp) {
  double d = sqrt(cp[0] * cp[0] + cp[1] * cp[1] + cp[2] * cp[2]);
  double n[3] = {cp[0] / d, cp[1] / d, cp[2] / d};
  res = white_c * (0.0 - ((n[0] * pf[0] + n[1] * pf[1] + n[2] * pf[2]) - d));
  const double *p = pf;
  if (do_fej) {
    p = pf_fej;
    d = sqrt(cp_fej[0] * cp_fej[0] + cp_fej[1] * cp_fej[1] + cp_fej[2] * cp_fej[2]);
    n[0] = cp_fej[0] / d;
    n[1] = cp_fej[1] / d;
    n[2] = cp_fej[2] / d;
  }
  double ntp = n[0] * p[0] + n[1] * p[1] + n[2] * p[2];
  double s = white_c * 1.0 / d;
  for (int j = 0; j < 3; j++) {
    Hcp[j] = s * (p[j] - ntp * n[j] - d * n[j]);
    Hf[j] = white_c * n[j];
  }
}

// ---- A landmark in the state in representation rep 1..5 (ov_type::LandmarkRepresentation; rep 0 needs none of this) ----
// ov_type::Landmark::get_xyz: 1 / 3 store [theta, phi, rho] (rho = 1 / range), 4 [x/z, y/z, 1/z], 2 the position itself, 5 rho = 1/z in
// slot 0 and the bearing it was created with, [x/z, y/z, 1], in slots 1..3 (p = bearing / rho)
OVP_HD void landmark_xyz(int rep, const double *v, double *p) {
  if (rep == 5) {
    p[0] = v[1] / v[0], p[1] = v[2] / v[0], p[2] = v[3] / v[0];
  } else if (rep == 4) {
    p[0] = v[0] / v[2], p[1] = v[1] / v[2], p[2] = 1.0 / v[2];
  } else if (rep == 1 || rep == 3) {
    p[0] = (1.0 / v[2]) * cos(v[0]) * sin(v[1]);
    p[1] = (1.0 / v[2]) * sin(v[0]) * sin(v[1]);
    p[2] = (1.0 / v[2]) * cos(v[1]);
  } else {
    p[0] = v[0], p[1] = v[1], p[2] = v[2];
  }
}
// d p / d (theta, phi, rho) of p = (1 / rho) [cos(theta) sin(phi), sin(theta) sin(phi), cos(phi)], evaluated at p (row-major)
OVP_HD void landmark_d_spherical(const double *p, double *D) {
  const double r = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
  const double rho = 1.0 / r, phi = acos(rho * p[2]), th = atan2(p[1], p[0]);
  const double st = sin(th), ct = cos(th), sp = sin(phi), cp = cos(phi), ir = 1.0 / rho, ir2 = 1.0 / (rho * rho);
  const double d[9] = {-ir * st * sp, ir * ct * cp, -ir2 * ct * sp, ir * ct * sp, ir * st * cp, -ir2 * st * sp, 0.0, -ir * sp, -ir2 * cp};
  for (int i = 0; i < 9; i++)
    D[i] = d[i];
}
// The terms get_feature_jacobian_full chains onto the bearing rows of a landmark in representation rep (UpdaterHelper.cpp:35-193, 281-303,
// 411-420), from the landmark's value lv / first estimate lf, the anchor clone's pose anc / first-estimate pose ancf (rep 2..5) and the
// extrinsics cal (7 each, JPL quaternion then position).  Rep 5 gets the terms of rep 4 at its p_FinA: the update takes its Jacobians as
// ANCHORED_MSCKF_INVERSE_DEPTH and keeps the third column (UpdaterSLAM.cpp:475-479, 503-516):
//   out[0:3]   p_FinG (rep 2..5: R_GtoI^T R_ItoC^T (p_FinA - p_IinC) + p_IinG at the anchor's current pose), out[3:6] its first estimate
//              (the same point for rep 2..5, :301-303);
//   out[6:15]  dpfg_dlambda, column-major 3 x 3;
//   out[15:33] dpfg_danchor and out[33:51] dpfg_dcalib, column-major 3 x 6 (rep 2..5 only), taken at the first-estimate anchor when do_fej.
// The same algebra as ovp_feature_jacobian_representation, written for one device thread.
OVP_HD void landmark_rep_terms(int rep, int do_fej, const double *lv, const double *lf, const double *anc, const double *ancf,
                               const double *cal, double *out) {
  double *pG = out, *pGf = out + 3, *L = out + 6, *Ha = out + 15, *Hc = out + 33;
  double D[9], M[9];
  if (rep == 1) {
    landmark_xyz(1, lv, pG);
    landmark_xyz(1, lf, pGf);
    landmark_d_spherical(do_fej ? pGf : pG, D);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        L[3 * j + i] = D[3 * i + j];
    return;
  }
  double RC[9], RI[9], pA[3], t[3], u[3];
  landmark_xyz(rep, lv, pA);
  quat_to_rot(cal, RC);
  quat_to_rot(anc, RI);
  for (int i = 0; i < 3; i++)
    t[i] = pA[i] - cal[4 + i];
  for (int i = 0; i < 3; i++)
    u[i] = RC[i] * t[0] + RC[3 + i] * t[1] + RC[6 + i] * t[2]; // R_ItoC^T t
  for (int i = 0; i < 3; i++)
    pG[i] = RI[i] * u[0] + RI[3 + i] * u[1] + RI[6 + i] * u[2] + anc[4 + i];
  for (int i = 0; i < 3; i++)
    pGf[i] = pG[i];
  const double *pI = anc + 4;
  if (do_fej) { // the best global estimate seen from the first-estimate anchor frame: pA = R_ItoC R_GtoI (p_FinG - p_IinG) + p_IinC
    quat_to_rot(ancf, RI);
    pI = ancf + 4;
    double g[3], w[3];
    for (int i = 0; i < 3; i++)
      g[i] = pG[i] - pI[i];
    mat3_vec(RI, g, w);
    mat3_vec(RC, w, pA);
    for (int i = 0; i < 3; i++)
      pA[i] += cal[4 + i];
  }
  double RCtoG[9], dA[3], v[3], S[9], T[9]; // R_CtoG = R_GtoI^T R_ItoC^T (row-major), dA = p_FinA - p_IinC
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      RCtoG[3 * i + j] = RI[i] * RC[3 * j] + RI[3 + i] * RC[3 * j + 1] + RI[6 + i] * RC[3 * j + 2];
  for (int i = 0; i < 3; i++)
    dA[i] = pA[i] - cal[4 + i];
  for (int i = 0; i < 3; i++)
    v[i] = RC[i] * dA[0] + RC[3 + i] * dA[1] + RC[6 + i] * dA[2]; // R_ItoC^T dA
  skew3(v, S);
  for (int i = 0; i < 3; i++) // dpfg_danchor[:, 0:3] = -R_GtoI^T skew(R_ItoC^T dA), [:, 3:6] = I
    for (int j = 0; j < 3; j++) {
      Ha[3 * j + i] = -(RI[i] * S[j] + RI[3 + i] * S[3 + j] + RI[6 + i] * S[6 + j]);
      Ha[3 * (3 + j) + i] = (i == j) ? 1.0 : 0.0;
    }
  skew3(dA, S);
  mat3_mul(RCtoG, S, T);
  for (int i = 0; i < 3; i++) // dpfg_dcalib[:, 0:3] = -R_CtoG skew(dA), [:, 3:6] = -R_CtoG
    for (int j = 0; j < 3; j++) {
      Hc[3 * j + i] = -T[3 * i + j];
      Hc[3 * (3 + j) + i] = -RCtoG[3 * i + j];
    }
  if (rep == 2) {
    for (int i = 0; i < 9; i++)
      M[i] = RCtoG[i];
  } else {
    if (rep == 3) {
      landmark_d_spherical(pA, D);
    } else { // lambda = (x/z, y/z, 1/z) (rep 4, and rep 5 before its bearing columns are projected out)
      const double rho = 1.0 / pA[2], al = pA[0] / pA[2], be = pA[1] / pA[2], ir = 1.0 / rho, ir2 = 1.0 / (rho * rho);
      const double d[9] = {ir, 0.0, -ir2 * al, 0.0, ir, -ir2 * be, 0.0, 0.0, -ir2};
      for (int i = 0; i < 9; i++)
        D[i] = d[i];
    }
    mat3_mul(RCtoG, D, M);
  }
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      L[3 * j + i] = M[3 * i + j];
}

} // namespace ovp

// ORACLE — TEST INFRASTRUCTURE ONLY.  CPU restatement (no Eigen) of the ov_plane hot path.
//
// Parity status: UNPINNED by the reference — rpng/ov_plane ships no tests, no golden vectors and cannot be
// compiled here (Eigen / Boost / OpenVINS ov_core are absent), see SURVEY.md §8(c).  Each function below cites
// the reference file:line it follows; the ov_core pieces (types, quat_ops, CamRadtan) are restated from the
// published OpenVINS algorithm (rpng/open_vins @ 74a63cf, pinned by /root/reference/ReadMe.md:39) and are
// additionally pinned by property tests (tests/test_oracle_*.py).
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may use this code.
// The product (ov_plane_b200/, include/) never includes, links or executes anything in oracle/.
//
// All arithmetic is IEEE double, column-major, single thread — like the reference's Eigen::MatrixXd path.
#pragma once
#include <algorithm>
#include <cassert>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <stdexcept>
#include <unordered_map>
#include <vector>

namespace orc {

// ---------------------------------------------------------------------------------------------------------------
// Minimal dense column-major matrix (stand-in for Eigen::MatrixXd)
// ---------------------------------------------------------------------------------------------------------------
struct Mat {
  int r = 0, c = 0;
  std::vector<double> a;
  Mat() {}
  Mat(int r_, int c_) : r(r_), c(c_), a((size_t)r_ * (size_t)c_, 0.0) {}
  static Mat Zero(int r, int c) { return Mat(r, c); }
  static Mat Identity(int n) {
    Mat m(n, n);
    for (int i = 0; i < n; i++)
      m(i, i) = 1.0;
    return m;
  }
  inline double &operator()(int i, int j) { return a[(size_t)j * r + i]; }
  inline double operator()(int i, int j) const { return a[(size_t)j * r + i]; }
  int rows() const { return r; }
  int cols() const { return c; }
  Mat block(int i0, int j0, int h, int w) const {
    Mat m(h, w);
    for (int j = 0; j < w; j++)
      for (int i = 0; i < h; i++)
        m(i, j) = (*this)(i0 + i, j0 + j);
    return m;
  }
  void setBlock(int i0, int j0, const Mat &m) {
    for (int j = 0; j < m.c; j++)
      for (int i = 0; i < m.r; i++)
        (*this)(i0 + i, j0 + j) = m(i, j);
  }
  void addBlock(int i0, int j0, const Mat &m) {
    for (int j = 0; j < m.c; j++)
      for (int i = 0; i < m.r; i++)
        (*this)(i0 + i, j0 + j) += m(i, j);
  }
  Mat T() const {
    Mat m(c, r);
    for (int j = 0; j < c; j++)
      for (int i = 0; i < r; i++)
        m(j, i) = (*this)(i, j);
    return m;
  }
  // Eigen conservativeResize semantics (keeps the top-left overlap, new entries zero)
  void conservativeResize(int nr, int nc) {
    Mat m(nr, nc);
    int hr = std::min(nr, r), hc = std::min(nc, c);
    for (int j = 0; j < hc; j++)
      for (int i = 0; i < hr; i++)
        m(i, j) = (*this)(i, j);
    *this = std::move(m);
  }
  double norm() const {
    double s = 0;
    for (double v : a)
      s += v * v;
    return std::sqrt(s);
  }
};

inline Mat operator*(const Mat &A, const Mat &B) {
  assert(A.c == B.r);
  Mat C(A.r, B.c);
  for (int j = 0; j < B.c; j++)
    for (int k = 0; k < A.c; k++) {
      double b = B(k, j);
      if (b == 0.0)
        continue;
      const double *ap = &A.a[(size_t)k * A.r];
      double *cp = &C.a[(size_t)j * C.r];
      for (int i = 0; i < A.r; i++)
        cp[i] += ap[i] * b;
    }
  return C;
}
inline Mat operator*(double s, const Mat &A) {
  Mat C = A;
  for (double &v : C.a)
    v *= s;
  return C;
}
inline Mat operator+(const Mat &A, const Mat &B) {
  assert(A.r == B.r && A.c == B.c);
  Mat C = A;
  for (size_t i = 0; i < C.a.size(); i++)
    C.a[i] += B.a[i];
  return C;
}
inline Mat operator-(const Mat &A, const Mat &B) {
  assert(A.r == B.r && A.c == B.c);
  Mat C = A;
  for (size_t i = 0; i < C.a.size(); i++)
    C.a[i] -= B.a[i];
  return C;
}
inline Mat vec3(double x, double y, double z) {
  Mat v(3, 1);
  v(0, 0) = x;
  v(1, 0) = y;
  v(2, 0) = z;
  return v;
}
inline double dot(const Mat &a, const Mat &b) {
  assert(a.a.size() == b.a.size());
  double s = 0;
  for (size_t i = 0; i < a.a.size(); i++)
    s += a.a[i] * b.a[i];
  return s;
}

// Cholesky (lower) of a symmetric matrix, reading the full matrix (Eigen LLT reads the lower triangle)
inline bool chol_lower(const Mat &S, Mat &L) {
  int n = S.r;
  L = Mat(n, n);
  for (int j = 0; j < n; j++) {
    double d = S(j, j);
    for (int k = 0; k < j; k++)
      d -= L(j, k) * L(j, k);
    if (!(d > 0.0))
      return false;
    double ljj = std::sqrt(d);
    L(j, j) = ljj;
    for (int i = j + 1; i < n; i++) {
      double s = S(i, j);
      for (int k = 0; k < j; k++)
        s -= L(i, k) * L(j, k);
      L(i, j) = s / ljj;
    }
  }
  return true;
}
// Solve L L^T X = B in place
inline void chol_solve_inplace(const Mat &L, Mat &B) {
  int n = L.r;
  for (int c = 0; c < B.c; c++) {
    for (int i = 0; i < n; i++) {
      double s = B(i, c);
      for (int k = 0; k < i; k++)
        s -= L(i, k) * B(k, c);
      B(i, c) = s / L(i, i);
    }
    for (int i = n - 1; i >= 0; i--) {
      double s = B(i, c);
      for (int k = i + 1; k < n; k++)
        s -= L(k, i) * B(k, c);
      B(i, c) = s / L(i, i);
    }
  }
}

// General small inverse by Gauss-Jordan with partial pivoting (stand-in for colPivHouseholderQr().inverse(),
// StateHelper.cpp:564; both are backward-stable for the 3x3 / 1x1 H_L blocks on this path)
inline Mat inverse_small(const Mat &A) {
  int n = A.r;
  assert(A.r == A.c);
  Mat M = A, I = Mat::Identity(n);
  for (int k = 0; k < n; k++) {
    int p = k;
    for (int i = k + 1; i < n; i++)
      if (std::fabs(M(i, k)) > std::fabs(M(p, k)))
        p = i;
    if (p != k)
      for (int j = 0; j < n; j++) {
        std::swap(M(k, j), M(p, j));
        std::swap(I(k, j), I(p, j));
      }
    double d = M(k, k);
    for (int j = 0; j < n; j++) {
      M(k, j) /= d;
      I(k, j) /= d;
    }
    for (int i = 0; i < n; i++)
      if (i != k) {
        double f = M(i, k);
        if (f == 0.0)
          continue;
        for (int j = 0; j < n; j++) {
          M(i, j) -= f * M(k, j);
          I(i, j) -= f * I(k, j);
        }
      }
  }
  return I;
}

// ---------------------------------------------------------------------------------------------------------------
// ov_core utils/quat_ops.h (JPL convention), restated.  Call sites: Propagator.cpp:384-404,476-566,
// UpdaterHelper.cpp:104,400,430.
// ---------------------------------------------------------------------------------------------------------------
inline Mat skew_x(const Mat &w) {
  Mat m(3, 3);
  m(0, 1) = -w(2, 0);
  m(0, 2) = w(1, 0);
  m(1, 0) = w(2, 0);
  m(1, 2) = -w(0, 0);
  m(2, 0) = -w(1, 0);
  m(2, 1) = w(0, 0);
  return m;
}
inline Mat quat_2_Rot(const Mat &q) {
  Mat v = q.block(0, 0, 3, 1);
  Mat qx = skew_x(v);
  double w = q(3, 0);
  Mat R = (2 * w * w - 1) * Mat::Identity(3) - (2 * w) * qx + 2.0 * (v * v.T());
  return R;
}
inline Mat quatnorm(Mat q) {
  if (q(3, 0) < 0)
    q = -1.0 * q;
  return (1.0 / q.norm()) * q;
}
inline Mat quat_multiply(const Mat &q, const Mat &p) {
  Mat Qm(4, 4);
  Mat v = q.block(0, 0, 3, 1);
  Qm.setBlock(0, 0, q(3, 0) * Mat::Identity(3) - skew_x(v));
  Qm.setBlock(0, 3, v);
  Qm.setBlock(3, 0, -1.0 * v.T());
  Qm(3, 3) = q(3, 0);
  Mat qt = Qm * p;
  if (qt(3, 0) < 0)
    qt = -1.0 * qt;
  return (1.0 / qt.norm()) * qt;
}
inline Mat rot_2_quat(const Mat &rot) {
  Mat q(4, 1);
  double T = rot(0, 0) + rot(1, 1) + rot(2, 2);
  if ((rot(0, 0) >= T) && (rot(0, 0) >= rot(1, 1)) && (rot(0, 0) >= rot(2, 2))) {
    q(0, 0) = std::sqrt((1 + (2 * rot(0, 0)) - T) / 4);
    q(1, 0) = (1 / (4 * q(0, 0))) * (rot(0, 1) + rot(1, 0));
    q(2, 0) = (1 / (4 * q(0, 0))) * (rot(0, 2) + rot(2, 0));
    q(3, 0) = (1 / (4 * q(0, 0))) * (rot(1, 2) - rot(2, 1));
  } else if ((rot(1, 1) >= T) && (rot(1, 1) >= rot(0, 0)) && (rot(1, 1) >= rot(2, 2))) {
    q(1, 0) = std::sqrt((1 + (2 * rot(1, 1)) - T) / 4);
    q(0, 0) = (1 / (4 * q(1, 0))) * (rot(0, 1) + rot(1, 0));
    q(2, 0) = (1 / (4 * q(1, 0))) * (rot(1, 2) + rot(2, 1));
    q(3, 0) = (1 / (4 * q(1, 0))) * (rot(2, 0) - rot(0, 2));
  } else if ((rot(2, 2) >= T) && (rot(2, 2) >= rot(0, 0)) && (rot(2, 2) >= rot(1, 1))) {
    q(2, 0) = std::sqrt((1 + (2 * rot(2, 2)) - T) / 4);
    q(0, 0) = (1 / (4 * q(2, 0))) * (rot(0, 2) + rot(2, 0));
    q(1, 0) = (1 / (4 * q(2, 0))) * (rot(1, 2) + rot(2, 1));
    q(3, 0) = (1 / (4 * q(2, 0))) * (rot(0, 1) - rot(1, 0));
  } else {
    q(3, 0) = std::sqrt((1 + T) / 4);
    q(0, 0) = (1 / (4 * q(3, 0))) * (rot(1, 2) - rot(2, 1));
    q(1, 0) = (1 / (4 * q(3, 0))) * (rot(2, 0) - rot(0, 2));
    q(2, 0) = (1 / (4 * q(3, 0))) * (rot(0, 1) - rot(1, 0));
  }
  if (q(3, 0) < 0)
    q = -1.0 * q;
  return (1.0 / q.norm()) * q;
}
inline Mat Omega(const Mat &w) {
  Mat m(4, 4);
  m.setBlock(0, 0, -1.0 * skew_x(w));
  m.setBlock(3, 0, -1.0 * w.T());
  m.setBlock(0, 3, w);
  return m;
}
inline Mat exp_so3(const Mat &w) {
  Mat wx = skew_x(w);
  double theta = w.norm();
  double A, B;
  if (theta < 1e-7) {
    A = 1;
    B = 0.5;
  } else {
    A = std::sin(theta) / theta;
    B = (1 - std::cos(theta)) / (theta * theta);
  }
  if (theta == 0)
    return Mat::Identity(3);
  return Mat::Identity(3) + A * wx + B * (wx * wx);
}
inline Mat Jl_so3(const Mat &w) {
  double theta = w.norm();
  if (theta < 1e-6)
    return Mat::Identity(3);
  Mat a = (1.0 / theta) * w;
  return (std::sin(theta) / theta) * Mat::Identity(3) + (1 - std::sin(theta) / theta) * (a * a.T()) +
         ((1 - std::cos(theta)) / theta) * skew_x(a);
}
inline Mat Jr_so3(const Mat &w) { return Jl_so3(-1.0 * w); }

// ---------------------------------------------------------------------------------------------------------------
// ov_type::{Type, JPLQuat, Vec, PoseJPL, IMU, Landmark} restated as one tagged struct.
// Call sites: StateHelper.cpp:54,192,340,365,381; UpdaterHelper.cpp:352-353,377-378; Propagator.cpp:369-387,448-453.
// ---------------------------------------------------------------------------------------------------------------
enum Kind { KIND_VEC = 0, KIND_POSE = 1, KIND_IMU = 2, KIND_LANDMARK = 3 };

struct Var {
  Kind kind = KIND_VEC;
  int sz = 0;            // error-state size
  int id = -1;           // location in the covariance (-1: not in the state)
  std::vector<double> value, fej;
  // Landmark extras
  size_t featid = 0;
  bool should_marg = false;
  int feat_representation = 0;        // Landmark::_feat_representation
  double anchor_clone_timestamp = -1; // Landmark::_anchor_clone_timestamp
  bool has_had_anchor_change = false;
  int handle = -1; // stable external identifier (tests use it to address variables)

  int size() const { return sz; }
  static std::shared_ptr<Var> makeVec(int n) {
    auto v = std::make_shared<Var>();
    v->kind = KIND_VEC;
    v->sz = n;
    v->value.assign(n, 0.0);
    v->fej.assign(n, 0.0);
    return v;
  }
  static std::shared_ptr<Var> makeLandmark(int n) {
    auto v = makeVec(n);
    v->kind = KIND_LANDMARK;
    return v;
  }
  static std::shared_ptr<Var> makePose() {
    auto v = std::make_shared<Var>();
    v->kind = KIND_POSE;
    v->sz = 6;
    v->value = {0, 0, 0, 1, 0, 0, 0};
    v->fej = v->value;
    return v;
  }
  static std::shared_ptr<Var> makeIMU() {
    auto v = std::make_shared<Var>();
    v->kind = KIND_IMU;
    v->sz = 15;
    v->value.assign(16, 0.0);
    v->value[3] = 1.0;
    v->fej = v->value;
    return v;
  }
  Mat quat(bool f = false) const {
    const auto &x = f ? fej : value;
    Mat q(4, 1);
    for (int i = 0; i < 4; i++)
      q(i, 0) = x[i];
    return q;
  }
  Mat Rot() const { return quat_2_Rot(quat(false)); }
  Mat Rot_fej() const { return quat_2_Rot(quat(true)); }
  Mat pos() const { return vec3(value[4], value[5], value[6]); }
  Mat pos_fej() const { return vec3(fej[4], fej[5], fej[6]); }
  Mat vel() const { return vec3(value[7], value[8], value[9]); }
  Mat vel_fej() const { return vec3(fej[7], fej[8], fej[9]); }
  Mat bias_g() const { return vec3(value[10], value[11], value[12]); }
  Mat bias_a() const { return vec3(value[13], value[14], value[15]); }
  Mat vecvalue(bool f = false) const {
    const auto &x = f ? fej : value;
    Mat v((int)x.size(), 1);
    for (size_t i = 0; i < x.size(); i++)
      v((int)i, 0) = x[i];
    return v;
  }

  // ov_type::*::update(dx): JPLQuat left-multiplicative, everything else additive
  void update(const double *dx) {
    if (kind == KIND_VEC || kind == KIND_LANDMARK) {
      for (int i = 0; i < sz; i++)
        value[i] += dx[i];
      return;
    }
    Mat dq(4, 1);
    dq(0, 0) = 0.5 * dx[0];
    dq(1, 0) = 0.5 * dx[1];
    dq(2, 0) = 0.5 * dx[2];
    dq(3, 0) = 1.0;
    dq = quatnorm(dq);
    Mat qn = quat_multiply(dq, quat(false));
    for (int i = 0; i < 4; i++)
      value[i] = qn(i, 0);
    for (int i = 0; i < 3; i++)
      value[4 + i] += dx[3 + i];
    if (kind == KIND_IMU)
      for (int i = 0; i < 9; i++)
        value[7 + i] += dx[6 + i];
  }
};
typedef std::shared_ptr<Var> VarP;

// ---------------------------------------------------------------------------------------------------------------
// ov_core::CamRadtan restated (distort_d / compute_distort_jacobian); call sites UpdaterHelper.cpp:365,389.
// cam = [fx fy cx cy k1 k2 p1 p2]
// ---------------------------------------------------------------------------------------------------------------
inline void radtan_distort_d(const double *cam, double x, double y, double &u, double &v) {
  double r = std::sqrt(x * x + y * y);
  double r_2 = r * r;
  double r_4 = r_2 * r_2;
  double x1 = x * (1 + cam[4] * r_2 + cam[5] * r_4) + 2 * cam[6] * x * y + cam[7] * (r_2 + 2 * x * x);
  double y1 = y * (1 + cam[4] * r_2 + cam[5] * r_4) + cam[6] * (r_2 + 2 * y * y) + 2 * cam[7] * x * y;
  u = cam[0] * x1 + cam[2];
  v = cam[1] * y1 + cam[3];
}
inline void radtan_distort_jacobian(const double *cam, double x, double y, Mat &H_dz_dzn, Mat &H_dz_dzeta) {
  double r = std::sqrt(x * x + y * y);
  double r_2 = r * r;
  double r_4 = r_2 * r_2;
  H_dz_dzn = Mat(2, 2);
  double x_2 = x * x, y_2 = y * y, x_y = x * y;
  H_dz_dzn(0, 0) = cam[0] * ((1 + cam[4] * r_2 + cam[5] * r_4) + (2 * cam[4] * x_2 + 4 * cam[5] * x_2 * (x_2 + y_2)) +
                             2 * cam[6] * y + (2 * cam[7] * x + 4 * cam[7] * x));
  H_dz_dzn(0, 1) = cam[0] * (2 * cam[4] * x_y + 4 * cam[5] * x_y * (x_2 + y_2) + 2 * cam[6] * x + 2 * cam[7] * y);
  H_dz_dzn(1, 0) = cam[1] * (2 * cam[4] * x_y + 4 * cam[5] * x_y * (x_2 + y_2) + 2 * cam[6] * x + 2 * cam[7] * y);
  H_dz_dzn(1, 1) = cam[1] * ((1 + cam[4] * r_2 + cam[5] * r_4) + (2 * cam[4] * y_2 + 4 * cam[5] * y_2 * (x_2 + y_2)) +
                             2 * cam[7] * x + (2 * cam[6] * y + 4 * cam[6] * y));
  double x1 = x * (1 + cam[4] * r_2 + cam[5] * r_4) + 2 * cam[6] * x_y + cam[7] * (r_2 + 2 * x_2);
  double y1 = y * (1 + cam[4] * r_2 + cam[5] * r_4) + cam[6] * (r_2 + 2 * y_2) + 2 * cam[7] * x_y;
  H_dz_dzeta = Mat(2, 8);
  H_dz_dzeta(0, 0) = x1;
  H_dz_dzeta(0, 2) = 1;
  H_dz_dzeta(0, 4) = cam[0] * x * r_2;
  H_dz_dzeta(0, 5) = cam[0] * x * r_4;
  H_dz_dzeta(0, 6) = 2 * cam[0] * x_y;
  H_dz_dzeta(0, 7) = cam[0] * (r_2 + 2 * x_2);
  H_dz_dzeta(1, 1) = y1;
  H_dz_dzeta(1, 3) = 1;
  H_dz_dzeta(1, 4) = cam[1] * y * r_2;
  H_dz_dzeta(1, 5) = cam[1] * y * r_4;
  H_dz_dzeta(1, 6) = cam[1] * (r_2 + 2 * y_2);
  H_dz_dzeta(1, 7) = 2 * cam[1] * x_y;
}

// ---------------------------------------------------------------------------------------------------------------
// Eigen::JacobiRotation::makeGivens (real) + applyOnTheLeft(0,1,G.adjoint()) restated
// (UpdaterHelper.cpp:528-534; formula from Eigen/src/Jacobi/Jacobi.h, see SURVEY.md §8(c))
// ---------------------------------------------------------------------------------------------------------------
struct Givens {
  double c, s;
  inline void make(double p, double q) {
    if (q == 0.0) {
      c = p < 0.0 ? -1.0 : 1.0;
      s = 0.0;
    } else if (p == 0.0) {
      c = 0.0;
      s = q < 0.0 ? 1.0 : -1.0;
    } else if (std::fabs(p) > std::fabs(q)) {
      double t = q / p;
      double u = std::sqrt(1.0 + t * t);
      if (p < 0.0)
        u = -u;
      c = 1.0 / u;
      s = -t * c;
    } else {
      double t = p / q;
      double u = std::sqrt(1.0 + t * t);
      if (q < 0.0)
        u = -u;
      s = -1.0 / u;
      c = -t * s;
    }
  }
  // rows (m-1, m) of M, columns [c0, c1): x' = c x - s y ; y' = s x + c y
  inline void apply(Mat &M, int m, int c0, int c1) const {
    for (int j = c0; j < c1; j++) {
      double x = M(m - 1, j), y = M(m, j);
      M(m - 1, j) = c * x - s * y;
      M(m, j) = s * x + c * y;
    }
  }
};

// ---------------------------------------------------------------------------------------------------------------
// State / StateOptions (state/State.h:53-134, State.cpp:33-102, StateOptions.h:41-153)
// ---------------------------------------------------------------------------------------------------------------
struct StateOptions {
  bool do_fej = true;
  bool imu_avg = false;
  bool use_rk4_integration = true;
  bool do_calib_camera_pose = false;
  bool do_calib_camera_intrinsics = false;
  bool do_calib_camera_timeoffset = false;
  int max_clone_size = 11;
  int max_slam_features = 25;
  int max_aruco_features = 1024;
  int num_cameras = 1;
  double sigma_constraint = 0.01;
  double const_init_multi = 1.0;
  double const_init_chi2 = 1.0;
  double sigma_plane_merge = 0.001;
  double plane_merge_chi2 = 1.0;
  double plane_merge_deg_max = 1.0;
};

struct State {
  StateOptions _options;
  double _timestamp = -1;
  VarP _imu;
  std::map<double, VarP> _clones_IMU;
  std::map<size_t, VarP> _features_SLAM; // reference uses unordered_map: iteration order implementation-defined
  VarP _calib_dt_CAMtoIMU;
  VarP _calib_IMUtoCAM; // mono (all shipped configs, SURVEY §7 hazard list)
  VarP _cam_intrinsics;
  std::map<size_t, VarP> _features_PLANE;
  std::map<size_t, size_t> _features_SLAM_to_PLANE;
  Mat _Cov;
  std::vector<VarP> _variables;
  std::vector<VarP> by_handle;

  VarP reg(VarP v) {
    v->handle = (int)by_handle.size();
    by_handle.push_back(v);
    return v;
  }

  // State.cpp:33-102
  explicit State(const StateOptions &opt) : _options(opt) {
    int current_id = 0;
    _imu = reg(Var::makeIMU());
    _imu->id = current_id;
    _variables.push_back(_imu);
    current_id += _imu->size();
    _calib_dt_CAMtoIMU = reg(Var::makeVec(1));
    if (_options.do_calib_camera_timeoffset) {
      _calib_dt_CAMtoIMU->id = current_id;
      _variables.push_back(_calib_dt_CAMtoIMU);
      current_id += 1;
    }
    _calib_IMUtoCAM = reg(Var::makePose());
    _cam_intrinsics = reg(Var::makeVec(8));
    if (_options.do_calib_camera_pose) {
      _calib_IMUtoCAM->id = current_id;
      _variables.push_back(_calib_IMUtoCAM);
      current_id += 6;
    }
    if (_options.do_calib_camera_intrinsics) {
      _cam_intrinsics->id = current_id;
      _variables.push_back(_cam_intrinsics);
      current_id += 8;
    }
    _Cov = std::pow(1e-3, 2) * Mat::Identity(current_id);
    if (_options.do_calib_camera_timeoffset)
      _Cov(_calib_dt_CAMtoIMU->id, _calib_dt_CAMtoIMU->id) = std::pow(0.01, 2);
    if (_options.do_calib_camera_pose) {
      int b = _calib_IMUtoCAM->id;
      for (int i = 0; i < 3; i++) {
        _Cov(b + i, b + i) = std::pow(0.005, 2);
        _Cov(b + 3 + i, b + 3 + i) = std::pow(0.01, 2);
      }
    }
    if (_options.do_calib_camera_intrinsics) {
      int b = _cam_intrinsics->id;
      for (int i = 0; i < 4; i++) {
        _Cov(b + i, b + i) = std::pow(1.0, 2);
        _Cov(b + 4 + i, b + 4 + i) = std::pow(0.005, 2);
      }
    }
  }
  double margtimestep() const {
    double t = INFINITY;
    for (auto &c : _clones_IMU)
      if (c.first < t)
        t = c.first;
    return t;
  }
  int max_covariance_size() const { return _Cov.rows(); }
};
typedef std::shared_ptr<State> StateP;

struct OracleExit : std::runtime_error {
  explicit OracleExit(const std::string &s) : std::runtime_error(s) {}
};
// reference prints + std::exit(EXIT_FAILURE); the oracle throws so the tests can observe it
[[noreturn]] inline void ref_exit(const char *what) { throw OracleExit(what); }

// TEST INSTRUMENTATION, NOT PART OF THE REFERENCE.  UpdaterPlane::measurement_compress_inplace keeps the top n rows of the Givens
// sweep over a stacked H_x that is exactly rank deficient on the plane paths (gauge directions, SURVEY.md §7); the n - rank kept
// rows whose H part is round-off still carry arbitrary, round-off defined unit projections of the stacked residual.  They do not
// move the posterior (zero Jacobian) but each adds its square to the plane chi2 the reference gates on, so that chi2 is not
// reproducible by the reference itself under a different FMA contraction (tools/oracle_sensitivity.py).  The probe lets a test
// split every gated chi2 into the well-defined part and that remainder: fn(rows, cols, H col-major, z) returns
// |projection of z onto the left null space of H|^2 (the test supplies an SVD).  With gate_without set the gate is evaluated on
// chi2 minus that remainder - the quantity the CUDA path computes; the default (fn == nullptr) is the unmodified reference.
struct GaugeProbe {
  double (*fn)(int rows, int cols, const double *H, const double *z) = nullptr;
  bool gate_without = false;
  std::vector<double> junk; // one entry per gated stacked system, in call order
  double probe(const struct Mat &H, const struct Mat &z);
};
inline GaugeProbe &gauge_probe() {
  static GaugeProbe g;
  return g;
}
inline double GaugeProbe::probe(const Mat &H, const Mat &z) {
  if (!fn)
    return 0.0;
  double j = fn(H.rows(), H.cols(), H.a.data(), z.a.data());
  junk.push_back(j);
  return gate_without ? j : 0.0;
}

// chi-squared 0.95 quantile: table injected by the test harness (scipy.stats.chi2.ppf; boost::math::quantile in
// the reference, UpdaterMSCKF.cpp:59-62).  Index = dof.
struct Chi2Table {
  std::vector<double> q;
  double at(int dof) const {
    if (dof < (int)q.size())
      return q[dof];
    // Wilson-Hilferty fallback only used beyond the injected table (never in the committed tests)
    double k = dof, z = 1.6448536269514722;
    double t = 1.0 - 2.0 / (9.0 * k) + z * std::sqrt(2.0 / (9.0 * k));
    return k * t * t * t;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// StateHelper (state/StateHelper.cpp)
// ---------------------------------------------------------------------------------------------------------------
struct StateHelper {

  // StateHelper.cpp:231-259
  static Mat get_marginal_covariance(StateP state, const std::vector<VarP> &small_variables) {
    int cov_size = 0;
    for (auto &v : small_variables)
      cov_size += v->size();
    Mat Small_cov(cov_size, cov_size);
    int i_index = 0;
    for (size_t i = 0; i < small_variables.size(); i++) {
      int k_index = 0;
      for (size_t k = 0; k < small_variables.size(); k++) {
        Small_cov.setBlock(i_index, k_index,
                           state->_Cov.block(small_variables[i]->id, small_variables[k]->id, small_variables[i]->size(),
                                             small_variables[k]->size()));
        k_index += small_variables[k]->size();
      }
      i_index += small_variables[i]->size();
    }
    return Small_cov;
  }

  // StateHelper.cpp:261-274
  static Mat get_full_covariance(StateP state) { return state->_Cov; }

  static void sym_from_upper(Mat &P) {
    for (int j = 0; j < P.c; j++)
      for (int i = j + 1; i < P.r; i++)
        P(i, j) = P(j, i);
  }

  // StateHelper.cpp:204-229
  static void set_initial_covariance(StateP state, const Mat &covariance, const std::vector<VarP> &order) {
    int i_index = 0;
    for (size_t i = 0; i < order.size(); i++) {
      int k_index = 0;
      for (size_t k = 0; k < order.size(); k++) {
        state->_Cov.setBlock(order[i]->id, order[k]->id, covariance.block(i_index, k_index, order[i]->size(), order[k]->size()));
        k_index += order[k]->size();
      }
      i_index += order[i]->size();
    }
    sym_from_upper(state->_Cov);
  }

  // StateHelper.cpp:41-119
  static void EKFPropagation(StateP state, const std::vector<VarP> &order_NEW, const std::vector<VarP> &order_OLD, const Mat &Phi,
                             const Mat &Q) {
    if (order_NEW.empty() || order_OLD.empty())
      ref_exit("EKFPropagation: empty variable arrays");
    int size_order_NEW = order_NEW.at(0)->size();
    for (size_t i = 0; i + 1 < order_NEW.size(); i++) {
      if (order_NEW.at(i)->id + order_NEW.at(i)->size() != order_NEW.at(i + 1)->id)
        ref_exit("EKFPropagation: non-contiguous state elements");
      size_order_NEW += order_NEW.at(i + 1)->size();
    }
    int size_order_OLD = order_OLD.at(0)->size();
    for (size_t i = 0; i + 1 < order_OLD.size(); i++)
      size_order_OLD += order_OLD.at(i + 1)->size();
    assert(size_order_NEW == Phi.rows());
    assert(size_order_OLD == Phi.cols());
    assert(size_order_NEW == Q.cols());
    assert(size_order_NEW == Q.rows());
    (void)size_order_OLD;
    int current_it = 0;
    std::vector<int> Phi_id;
    for (auto &var : order_OLD) {
      Phi_id.push_back(current_it);
      current_it += var->size();
    }
    int N = state->_Cov.rows();
    Mat Cov_PhiT(N, Phi.rows());
    for (size_t i = 0; i < order_OLD.size(); i++) {
      VarP var = order_OLD.at(i);
      Cov_PhiT = Cov_PhiT + state->_Cov.block(0, var->id, N, var->size()) * Phi.block(0, Phi_id[i], Phi.rows(), var->size()).T();
    }
    Mat Phi_Cov_PhiT = Q;
    sym_from_upper(Phi_Cov_PhiT);
    for (size_t i = 0; i < order_OLD.size(); i++) {
      VarP var = order_OLD.at(i);
      Phi_Cov_PhiT = Phi_Cov_PhiT + Phi.block(0, Phi_id[i], Phi.rows(), var->size()) * Cov_PhiT.block(var->id, 0, var->size(), Phi.rows());
    }
    int start_id = order_NEW.at(0)->id;
    state->_Cov.setBlock(start_id, 0, Cov_PhiT.T());
    state->_Cov.setBlock(0, start_id, Cov_PhiT);
    state->_Cov.setBlock(start_id, start_id, Phi_Cov_PhiT);
    for (int i = 0; i < N; i++)
      if (state->_Cov(i, i) < 0.0)
        ref_exit("EKFPropagation: negative diagonal");
  }

  // StateHelper.cpp:121-202
  static void EKFUpdate(StateP state, const std::vector<VarP> &H_order, const Mat &H, const Mat &res, const Mat &R) {
    assert(res.rows() == R.rows());
    assert(H.rows() == res.rows());
    int N = state->_Cov.rows();
    Mat M_a(N, res.rows());
    int current_it = 0;
    std::vector<int> H_id;
    for (auto &meas_var : H_order) {
      H_id.push_back(current_it);
      current_it += meas_var->size();
    }
    for (auto &var : state->_variables) {
      Mat M_i(var->size(), res.rows());
      for (size_t i = 0; i < H_order.size(); i++) {
        VarP meas_var = H_order[i];
        M_i = M_i + state->_Cov.block(var->id, meas_var->id, var->size(), meas_var->size()) *
                        H.block(0, H_id[i], H.rows(), meas_var->size()).T();
      }
      M_a.setBlock(var->id, 0, M_i);
    }
    Mat P_small = get_marginal_covariance(state, H_order);
    Mat S = H * P_small * H.T();
    // S.triangularView<Upper>() += R  then selfadjointView<Upper>
    for (int j = 0; j < S.c; j++)
      for (int i = 0; i <= j; i++)
        S(i, j) += R(i, j);
    sym_from_upper(S);
    Mat L;
    if (!chol_lower(S, L))
      ref_exit("EKFUpdate: S not positive definite");
    Mat Sinv = Mat::Identity(R.rows());
    chol_solve_inplace(L, Sinv);
    sym_from_upper(Sinv);
    Mat K = M_a * Sinv;
    Mat KMt = K * M_a.T();
    for (int j = 0; j < N; j++)
      for (int i = 0; i <= j; i++)
        state->_Cov(i, j) -= KMt(i, j);
    sym_from_upper(state->_Cov);
    for (int i = 0; i < N; i++)
      if (state->_Cov(i, i) < 0.0)
        ref_exit("EKFUpdate: negative diagonal");
    Mat dx = K * res;
    for (auto &v : state->_variables)
      v->update(&dx.a[v->id]);
    // (camera objects are refreshed from _cam_intrinsics here in the reference, :197-201: we read the Vec directly)
  }

  // StateHelper.cpp:276-344
  static void marginalize(StateP state, VarP marg) {
    if (std::find(state->_variables.begin(), state->_variables.end(), marg) == state->_variables.end())
      ref_exit("marginalize: variable not in the state");
    int marg_size = marg->size();
    int marg_id = marg->id;
    int N = state->_Cov.rows();
    int x2_size = N - marg_id - marg_size;
    Mat Cov_new(N - marg_size, N - marg_size);
    Cov_new.setBlock(0, 0, state->_Cov.block(0, 0, marg_id, marg_id));
    Cov_new.setBlock(0, marg_id, state->_Cov.block(0, marg_id + marg_size, marg_id, x2_size));
    Cov_new.setBlock(marg_id, 0, Cov_new.block(0, marg_id, marg_id, x2_size).T());
    Cov_new.setBlock(marg_id, marg_id, state->_Cov.block(marg_id + marg_size, marg_id + marg_size, x2_size, x2_size));
    state->_Cov = Cov_new;
    std::vector<VarP> remaining;
    for (auto &v : state->_variables) {
      if (v != marg) {
        if (v->id > marg_id)
          v->id -= marg_size;
        remaining.push_back(v);
      }
    }
    marg->id = -1;
    state->_variables = remaining;
  }

  // StateHelper.cpp:346-396, specialised to the only call site (clone of the IMU pose sub-variable, :598) and to
  // top-level variables
  static VarP clone(StateP state, VarP variable_to_clone, bool is_imu_pose) {
    int total_size = is_imu_pose ? 6 : variable_to_clone->size();
    int old_size = state->_Cov.rows();
    int new_loc = old_size;
    state->_Cov.conservativeResize(old_size + total_size, old_size + total_size);
    int old_loc = -1;
    for (auto &v : state->_variables)
      if (v == variable_to_clone)
        old_loc = v->id;
    if (old_loc < 0)
      ref_exit("clone: variable not in the state");
    state->_Cov.setBlock(new_loc, new_loc, state->_Cov.block(old_loc, old_loc, total_size, total_size));
    state->_Cov.setBlock(0, new_loc, state->_Cov.block(0, old_loc, old_size, total_size));
    state->_Cov.setBlock(new_loc, 0, state->_Cov.block(old_loc, 0, total_size, old_size));
    VarP nc;
    if (is_imu_pose) {
      nc = Var::makePose();
      for (int i = 0; i < 7; i++) {
        nc->value[i] = variable_to_clone->value[i];
        nc->fej[i] = variable_to_clone->fej[i];
      }
    } else {
      nc = std::make_shared<Var>(*variable_to_clone);
    }
    state->reg(nc);
    nc->id = new_loc;
    state->_variables.push_back(nc);
    return nc;
  }

  // StateHelper.cpp:588-625
  static VarP augment_clone(StateP state, const Mat &last_w) {
    if (state->_clones_IMU.find(state->_timestamp) != state->_clones_IMU.end())
      ref_exit("augment_clone: clone at the same time as an existing clone");
    VarP pose = clone(state, state->_imu, true);
    state->_clones_IMU[state->_timestamp] = pose;
    if (state->_options.do_calib_camera_timeoffset) {
      Mat dnc_dt(6, 1);
      dnc_dt.setBlock(0, 0, last_w);
      dnc_dt.setBlock(3, 0, state->_imu->vel());
      int N = state->_Cov.rows();
      int dt_id = state->_calib_dt_CAMtoIMU->id;
      Mat col = state->_Cov.block(0, dt_id, N, 1) * dnc_dt.T();
      state->_Cov.addBlock(0, pose->id, col);
      Mat row = dnc_dt * state->_Cov.block(dt_id, 0, 1, N);
      state->_Cov.addBlock(pose->id, 0, row);
    }
    return pose;
  }

  // StateHelper.cpp:627-636
  static void marginalize_old_clone(StateP state) {
    if ((int)state->_clones_IMU.size() > state->_options.max_clone_size) {
      double marginal_time = state->margtimestep();
      marginalize(state, state->_clones_IMU.at(marginal_time));
      state->_clones_IMU.erase(marginal_time);
    }
  }

  // StateHelper.cpp:638-652
  static void marginalize_slam(StateP state) {
    auto it0 = state->_features_SLAM.begin();
    while (it0 != state->_features_SLAM.end()) {
      if ((*it0).second->should_marg && (int)(*it0).first > 4 * state->_options.max_aruco_features) {
        marginalize(state, (*it0).second);
        state->_features_SLAM_to_PLANE.erase((*it0).first);
        it0 = state->_features_SLAM.erase(it0);
      } else {
        it0++;
      }
    }
  }

  static void check_isotropic(const Mat &R, const char *who) {
    assert(R.rows() == R.cols());
    assert(R.rows() > 0);
    for (int r = 0; r < R.rows(); r++)
      for (int c = 0; c < R.cols(); c++) {
        if (r == c && R(0, 0) != R(r, c))
          ref_exit(who);
        else if (r != c && R(r, c) != 0.0)
          ref_exit(who);
      }
  }

  // StateHelper.cpp:489-586
  static void initialize_invertible(StateP state, VarP new_variable, const std::vector<VarP> &H_order, const Mat &H_R, const Mat &H_L,
                                    const Mat &R, const Mat &res) {
    if (std::find(state->_variables.begin(), state->_variables.end(), new_variable) != state->_variables.end())
      ref_exit("initialize_invertible: variable already in the state");
    check_isotropic(R, "initialize_invertible: noise not isotropic");
    assert(res.rows() == R.rows());
    assert(H_L.rows() == res.rows());
    assert(H_L.rows() == H_R.rows());
    int N = state->_Cov.rows();
    Mat M_a(N, res.rows());
    int current_it = 0;
    std::vector<int> H_id;
    for (auto &meas_var : H_order) {
      H_id.push_back(current_it);
      current_it += meas_var->size();
    }
    for (auto &var : state->_variables) {
      Mat M_i(var->size(), res.rows());
      for (size_t i = 0; i < H_order.size(); i++) {
        VarP meas_var = H_order.at(i);
        M_i = M_i + state->_Cov.block(var->id, meas_var->id, var->size(), meas_var->size()) *
                        H_R.block(0, H_id[i], H_R.rows(), meas_var->size()).T();
      }
      M_a.setBlock(var->id, 0, M_i);
    }
    Mat P_small = get_marginal_covariance(state, H_order);
    Mat M = H_R * P_small * H_R.T();
    for (int j = 0; j < M.c; j++)
      for (int i = 0; i <= j; i++)
        M(i, j) += R(i, j);
    sym_from_upper(M);
    assert(H_L.rows() == H_L.cols());
    assert(H_L.rows() == new_variable->size());
    Mat H_Linv = inverse_small(H_L);
    Mat P_LL = H_Linv * M * H_Linv.T();
    int oldSize = N;
    int s = new_variable->size();
    state->_Cov.conservativeResize(oldSize + s, oldSize + s);
    Mat cross = -1.0 * (M_a * H_Linv.T());
    state->_Cov.setBlock(0, oldSize, cross);
    state->_Cov.setBlock(oldSize, 0, cross.T());
    state->_Cov.setBlock(oldSize, oldSize, P_LL);
    Mat dxn = H_Linv * res;
    new_variable->update(dxn.a.data());
    new_variable->id = oldSize;
    state->_variables.push_back(new_variable);
  }

  // StateHelper.cpp:398-487
  static bool initialize(StateP state, VarP new_variable, const std::vector<VarP> &H_order, Mat &H_R, Mat &H_L, Mat &R, Mat &res,
                         double chi_2_mult, const Chi2Table &chi2tab, bool do_update = true) {
    if (std::find(state->_variables.begin(), state->_variables.end(), new_variable) != state->_variables.end())
      ref_exit("initialize: variable already in the state");
    check_isotropic(R, "initialize: noise not isotropic");
    int new_var_size = new_variable->size();
    assert(new_var_size == H_L.cols());
    Givens G;
    for (int n = 0; n < H_L.cols(); ++n) {
      for (int m = H_L.rows() - 1; m > n; m--) {
        G.make(H_L(m - 1, n), H_L(m, n));
        G.apply(H_L, m, n, H_L.cols());
        G.apply(res, m, 0, 1);
        G.apply(H_R, m, 0, H_R.cols());
      }
    }
    Mat Hxinit = H_R.block(0, 0, new_var_size, H_R.cols());
    Mat H_finit = H_L.block(0, 0, new_var_size, new_var_size);
    Mat resinit = res.block(0, 0, new_var_size, 1);
    Mat Rinit = R.block(0, 0, new_var_size, new_var_size);
    Mat Hup = H_R.block(new_var_size, 0, H_R.rows() - new_var_size, H_R.cols());
    Mat resup = res.block(new_var_size, 0, res.rows() - new_var_size, 1);
    Mat Rup = R.block(new_var_size, new_var_size, R.rows() - new_var_size, R.rows() - new_var_size);
    Mat P_up = get_marginal_covariance(state, H_order);
    assert(Rup.rows() == Hup.rows());
    assert(Hup.cols() == P_up.cols());
    double chi2 = 0.0;
    if (Hup.rows() > 0) {
      Mat S = Hup * P_up * Hup.T() + Rup;
      Mat L;
      if (!chol_lower(S, L))
        ref_exit("initialize: S not positive definite");
      Mat y = resup;
      chol_solve_inplace(L, y);
      chi2 = dot(resup, y);
      chi2 -= gauge_probe().probe(Hup, resup); // instrumentation only (see GaugeProbe); default: subtracts 0
    }
    double chi2_check = chi2tab.at(res.rows()); // dof = full r, not r-s (:471-472)
    if (chi2 > chi_2_mult * chi2_check)
      return false;
    initialize_invertible(state, new_variable, H_order, Hxinit, H_finit, Rinit, resinit);
    if (Hup.rows() > 0 && do_update)
      EKFUpdate(state, H_order, Hup, resup, Rup);
    return true;
  }

  // StateHelper.cpp:654-758
  static void merge_planes_and_marginalize(StateP state, const std::map<size_t, size_t> &feat2plane,
                                           const std::map<size_t, std::set<size_t>> &plane2oldplane, const Chi2Table &chi2tab) {
    if (state->_features_PLANE.empty())
      return;
    auto it5 = state->_features_PLANE.begin();
    while (it5 != state->_features_PLANE.end()) {
      size_t planeid = (*it5).first;
      int planeid_new = -1;
      bool in_state = false;
      for (auto const &planeset : plane2oldplane) {
        if (planeset.second.find(planeid) != planeset.second.end()) {
          planeid_new = (int)planeset.first;
          in_state = (state->_features_PLANE.find(planeset.first) != state->_features_PLANE.end());
        }
      }
      if (planeid_new == -1 || (int)planeid == planeid_new) {
        it5++;
        continue;
      }
      if (!in_state) {
        state->_features_PLANE.insert({(size_t)planeid_new, state->_features_PLANE.at(planeid)});
        it5 = state->_features_PLANE.erase(it5);
      } else {
        auto plane_new = state->_features_PLANE.at(planeid_new);
        auto plane_old = state->_features_PLANE.at(planeid);
        Mat cp_new = plane_new->vecvalue();
        Mat cp_old = plane_old->vecvalue();
        Mat norm_new = (1.0 / cp_new.norm()) * cp_new;
        Mat norm_old = (1.0 / cp_old.norm()) * cp_old;
        double norm_dist = dot(norm_new, norm_old);
        double norm_angle = (180.0 / M_PI) * std::acos(norm_dist);
        double white_c = 1.0 / state->_options.sigma_plane_merge;
        Mat res = white_c * (Mat(3, 1) - (cp_new - cp_old));
        Mat H(3, 6);
        H.setBlock(0, 0, white_c * Mat::Identity(3));
        H.setBlock(0, 3, -white_c * Mat::Identity(3));
        std::vector<VarP> H_order = {plane_new, plane_old};
        Mat R = Mat::Identity(3);
        Mat P_marg = get_marginal_covariance(state, H_order);
        Mat S = H * P_marg * H.T() + R;
        Mat L;
        chol_lower(S, L);
        Mat y = res;
        chol_solve_inplace(L, y);
        double chi2 = dot(res, y);
        double chi2_check = state->_options.plane_merge_chi2 * chi2tab.at(3);
        if (chi2 < chi2_check && norm_angle < state->_options.plane_merge_deg_max)
          EKFUpdate(state, H_order, H, res, R);
        marginalize(state, plane_old);
        it5 = state->_features_PLANE.erase(it5);
      }
    }
    std::set<size_t> active_planes;
    for (auto const &featpair : feat2plane)
      active_planes.insert(featpair.second);
    it5 = state->_features_PLANE.begin();
    while (it5 != state->_features_PLANE.end()) {
      if (active_planes.find((*it5).first) == active_planes.end()) {
        marginalize(state, (*it5).second);
        it5 = state->_features_PLANE.erase(it5);
      } else {
        it5++;
      }
    }
  }
};

// ---------------------------------------------------------------------------------------------------------------
// UpdaterHelper (update/UpdaterHelper.cpp), GLOBAL_3D representation (the only one shipped configs use and the
// only one the plane constraint accepts, UpdaterHelper.cpp:455-456), mono camera.
// ---------------------------------------------------------------------------------------------------------------
struct Feature {
  size_t featid = 0;
  std::vector<double> timestamps; // clone timestamps (exact double keys, UpdaterHelper.cpp:233,351)
  std::vector<float> uvs;         // 2 floats per measurement (Eigen::VectorXf in the reference)
  Mat p_FinG = Mat(3, 1);
  Mat p_FinG_fej = Mat(3, 1);
  Mat p_FinG_original = Mat(3, 1); // value before the (out-of-scope) plane refinement, UpdaterMSCKF.cpp:160,663
  size_t planeid = 0;
  Mat cp_FinG = Mat(3, 1);
  Mat cp_FinG_fej = Mat(3, 1);
  bool to_delete = false;
  // ov_type::LandmarkRepresentation (0 GLOBAL_3D ... 5 ANCHORED_INVERSE_DEPTH_SINGLE) and, for the anchored forms, the anchor clone and the
  // feature in its camera frame (UpdaterHelper.h:61-99)
  int feat_representation = 0;
  double anchor_clone_timestamp = -1;
  Mat p_FinA = Mat(3, 1);
  Mat p_FinA_fej = Mat(3, 1);
};

struct UpdaterHelper {

  // UpdaterHelper.cpp:35-193: d p_FinG / d lambda for the six landmark representations (enum order of
  // ov_type::LandmarkRepresentation: GLOBAL_3D, GLOBAL_FULL_INVERSE_DEPTH, ANCHORED_3D, ANCHORED_FULL_INVERSE_DEPTH,
  // ANCHORED_MSCKF_INVERSE_DEPTH, ANCHORED_INVERSE_DEPTH_SINGLE) and, for the anchored ones, the Jacobians w.r.t. the anchor
  // clone (theta, p) and the camera extrinsics.  Plain-value interface: anchor pose / FEJ pose = [q_GtoI (JPL xyzw), p_IinG],
  // calib = [q_ItoC, p_IinC].  Returns whether anchor Jacobians were produced.
  static bool get_feature_jacobian_representation(int rep, bool do_fej, const Mat &p_FinG, const Mat &p_FinG_fej, const Mat &p_FinA_in,
                                                  const Mat &anchor, const Mat &anchor_fej, const Mat &calib, Mat &H_f, Mat &H_anc,
                                                  Mat &H_calib) {
    auto spherical = [](const Mat &p) { // :46-72 / :118-140: d p / d (theta, phi, rho) at the spherical coordinates of p
      double rho = 1.0 / p.norm();
      double phi = std::acos(rho * p(2, 0)), th = std::atan2(p(1, 0), p(0, 0));
      double st = std::sin(th), ct = std::cos(th), sp = std::sin(phi), cp = std::cos(phi);
      Mat J(3, 3);
      J(0, 0) = -(1.0 / rho) * st * sp;
      J(0, 1) = (1.0 / rho) * ct * cp;
      J(0, 2) = -(1.0 / (rho * rho)) * ct * sp;
      J(1, 0) = (1.0 / rho) * ct * sp;
      J(1, 1) = (1.0 / rho) * st * cp;
      J(1, 2) = -(1.0 / (rho * rho)) * st * sp;
      J(2, 0) = 0.0;
      J(2, 1) = -(1.0 / rho) * sp;
      J(2, 2) = -(1.0 / (rho * rho)) * cp;
      return J;
    };
    if (rep == 0) { // GLOBAL_3D (:39-43)
      H_f = Mat::Identity(3);
      return false;
    }
    if (rep == 1) { // GLOBAL_FULL_INVERSE_DEPTH (:46-72)
      H_f = spherical(do_fej ? p_FinG_fej : p_FinG);
      return false;
    }
    Mat R_ItoC = quat_2_Rot(calib.block(0, 0, 4, 1)), p_IinC = calib.block(4, 0, 3, 1);
    Mat R_GtoI = quat_2_Rot(anchor.block(0, 0, 4, 1)), p_IinG = anchor.block(4, 0, 3, 1);
    Mat p_FinA = p_FinA_in;
    if (do_fej) { // :88-96: best global point re-expressed in the FEJ anchor frame
      Mat best = R_GtoI.T() * R_ItoC.T() * (p_FinA - p_IinC) + p_IinG;
      R_GtoI = quat_2_Rot(anchor_fej.block(0, 0, 4, 1));
      p_IinG = anchor_fej.block(4, 0, 3, 1);
      p_FinA = (R_GtoI.T() * R_ItoC.T()).T() * (best - p_IinG) + p_IinC;
    }
    Mat R_CtoG = R_GtoI.T() * R_ItoC.T();
    H_anc = Mat(3, 6); // :100-102
    H_anc.setBlock(0, 0, (-1.0) * (R_GtoI.T() * skew_x(R_ItoC.T() * (p_FinA - p_IinC))));
    H_anc.setBlock(0, 3, Mat::Identity(3));
    H_calib = Mat(3, 6); // :109-115
    H_calib.setBlock(0, 0, (-1.0) * (R_CtoG * skew_x(p_FinA - p_IinC)));
    H_calib.setBlock(0, 3, (-1.0) * R_CtoG);
    if (rep == 2) { // ANCHORED_3D (:118-121)
      H_f = R_CtoG;
    } else if (rep == 3) { // ANCHORED_FULL_INVERSE_DEPTH (:124-150)
      H_f = R_CtoG * spherical(p_FinA);
    } else if (rep == 4) { // ANCHORED_MSCKF_INVERSE_DEPTH (:153-172)
      double alpha = p_FinA(0, 0) / p_FinA(2, 0), beta = p_FinA(1, 0) / p_FinA(2, 0), rho = 1.0 / p_FinA(2, 0);
      Mat J(3, 3);
      J(0, 0) = 1.0 / rho;
      J(0, 2) = -(1.0 / (rho * rho)) * alpha;
      J(1, 1) = 1.0 / rho;
      J(1, 2) = -(1.0 / (rho * rho)) * beta;
      J(2, 2) = -(1.0 / (rho * rho));
      H_f = R_CtoG * J;
    } else if (rep == 5) { // ANCHORED_INVERSE_DEPTH_SINGLE (:175-186)
      double rho = 1.0 / p_FinA(2, 0);
      Mat bearing = rho * p_FinA;
      H_f = R_CtoG * ((-(1.0 / (rho * rho))) * bearing);
    } else {
      ref_exit("get_feature_jacobian_representation: invalid representation");
    }
    return true;
  }


  // UpdaterHelper.cpp:195-513 (GLOBAL_3D: dpfg_dlambda = I, no anchor terms, :39-43)
  static void get_feature_jacobian_full(StateP state, const Feature &feature, double sigma_px, double sigma_c, Mat &H_f, Mat &H_x,
                                        Mat &res, std::vector<VarP> &x_order) {
    int total_meas = (int)feature.timestamps.size();
    x_order.clear();
    int total_hx = 0;
    std::unordered_map<Var *, int> map_hx;
    VarP calibration = state->_calib_IMUtoCAM;
    VarP distortion = state->_cam_intrinsics;
    if (total_meas > 0) { // the reference loops over cameras that have measurements (:209)
      if (state->_options.do_calib_camera_pose) {
        map_hx.insert({calibration.get(), total_hx});
        x_order.push_back(calibration);
        total_hx += calibration->size();
      }
      if (state->_options.do_calib_camera_intrinsics) {
        map_hx.insert({distortion.get(), total_hx});
        x_order.push_back(distortion);
        total_hx += distortion->size();
      }
      for (int m = 0; m < total_meas; m++) {
        VarP clone_Ci = state->_clones_IMU.at(feature.timestamps[m]);
        if (map_hx.find(clone_Ci.get()) == map_hx.end()) {
          map_hx.insert({clone_Ci.get(), total_hx});
          x_order.push_back(clone_Ci);
          total_hx += clone_Ci->size();
        }
      }
    }
    const bool relative = feature.feat_representation >= 2; // LandmarkRepresentation::is_relative_representation
    VarP clone_Ai;
    if (relative) { // :245-264: the anchor clone (and its extrinsics) take part even without a measurement from it
      clone_Ai = state->_clones_IMU.at(feature.anchor_clone_timestamp);
      if (map_hx.find(clone_Ai.get()) == map_hx.end()) {
        map_hx.insert({clone_Ai.get(), total_hx});
        x_order.push_back(clone_Ai);
        total_hx += clone_Ai->size();
      }
      if (state->_options.do_calib_camera_pose && map_hx.find(calibration.get()) == map_hx.end()) {
        map_hx.insert({calibration.get(), total_hx});
        x_order.push_back(calibration);
        total_hx += calibration->size();
      }
    }
    bool plane_in_state = (state->_features_PLANE.find(feature.planeid) != state->_features_PLANE.end());
    if (feature.planeid != 0 && plane_in_state) {
      VarP planecp = state->_features_PLANE.at(feature.planeid);
      if (map_hx.find(planecp.get()) == map_hx.end()) {
        map_hx.insert({planecp.get(), total_hx});
        x_order.push_back(planecp);
        total_hx += planecp->size();
      }
    }
    Mat p_FinG = feature.p_FinG;
    if (relative) // :281-293
      p_FinG = clone_Ai->Rot().T() * calibration->Rot().T() * (feature.p_FinA - calibration->pos()) + clone_Ai->pos();
    Mat p_FinG_fej = feature.p_FinG_fej;
    if (relative) // :297-301
      p_FinG_fej = p_FinG;
    // :318-323 derivative of p_FinG in the feature representation, computed once
    Mat dpfg_dlambda = Mat::Identity(3), dpfg_danchor, dpfg_dcalib;
    bool has_anchor_jac = false;
    if (feature.feat_representation != 0) {
      Mat anchor(7, 1), anchor_fej(7, 1), calib7(7, 1);
      for (int i = 0; i < 7; i++) {
        anchor(i, 0) = relative ? clone_Ai->value[i] : 0.0;
        anchor_fej(i, 0) = relative ? clone_Ai->fej[i] : 0.0;
        calib7(i, 0) = calibration->value[i];
      }
      has_anchor_jac = get_feature_jacobian_representation(feature.feat_representation, state->_options.do_fej, p_FinG, p_FinG_fej, feature.p_FinA,
                                                            anchor, anchor_fej, calib7, dpfg_dlambda, dpfg_danchor, dpfg_dcalib);
      if (feature.planeid != 0)
        ref_exit("the point-on-plane rows require GLOBAL_3D (assert, UpdaterHelper.cpp:455-456)");
    }

    int c = 0;
    int jacobsize = (feature.feat_representation != 5) ? 3 : 1;
    jacobsize += (feature.planeid != 0 && !plane_in_state) ? 3 : 0;
    int meassize = (feature.planeid != 0) ? (3 * total_meas) : (2 * total_meas);
    if (total_meas == 0 && feature.planeid != 0)
      meassize = 1;
    res = Mat(meassize, 1);
    H_f = Mat(meassize, jacobsize);
    H_x = Mat(meassize, total_hx);

    double white_px = 1.0 / sigma_px;
    Mat R_ItoC = calibration->Rot();
    Mat p_IinC = calibration->pos();
    const double *cam = distortion->value.data();
    for (int m = 0; m < total_meas; m++) {
      VarP clone_Ii = state->_clones_IMU.at(feature.timestamps[m]);
      Mat R_GtoIi = clone_Ii->Rot();
      Mat p_IiinG = clone_Ii->pos();
      Mat p_FinIi = R_GtoIi * (p_FinG - p_IiinG);
      Mat p_FinCi = R_ItoC * p_FinIi + p_IinC;
      double un = p_FinCi(0, 0) / p_FinCi(2, 0), vn = p_FinCi(1, 0) / p_FinCi(2, 0);
      double ud, vd;
      radtan_distort_d(cam, un, vn, ud, vd);
      double um = (double)feature.uvs[2 * m], vm = (double)feature.uvs[2 * m + 1];
      res(c, 0) = white_px * (um - ud);
      res(c + 1, 0) = white_px * (vm - vd);
      if (state->_options.do_fej) {
        R_GtoIi = clone_Ii->Rot_fej();
        p_IiinG = clone_Ii->pos_fej();
        p_FinIi = R_GtoIi * (p_FinG_fej - p_IiinG);
        p_FinCi = R_ItoC * p_FinIi + p_IinC;
        // uv_norm is NOT recomputed (:383)
      }
      Mat dz_dzn, dz_dzeta;
      radtan_distort_jacobian(cam, un, vn, dz_dzn, dz_dzeta);
      Mat dzn_dpfc(2, 3);
      double X = p_FinCi(0, 0), Y = p_FinCi(1, 0), Z = p_FinCi(2, 0);
      dzn_dpfc(0, 0) = 1 / Z;
      dzn_dpfc(0, 2) = -X / (Z * Z);
      dzn_dpfc(1, 1) = 1 / Z;
      dzn_dpfc(1, 2) = -Y / (Z * Z);
      Mat dpfc_dpfg = R_ItoC * R_GtoIi;
      Mat dpfc_dclone(3, 6);
      dpfc_dclone.setBlock(0, 0, R_ItoC * skew_x(p_FinIi));
      dpfc_dclone.setBlock(0, 3, -1.0 * dpfc_dpfg);
      Mat dz_dpfc = dz_dzn * dzn_dpfc;
      Mat dz_dpfg = dz_dpfc * dpfc_dpfg;
      H_f.setBlock(c, 0, (white_px * dz_dpfg) * dpfg_dlambda); // :411
      H_x.setBlock(c, map_hx[clone_Ii.get()], (white_px * dz_dpfc) * dpfc_dclone);
      if (has_anchor_jac) { // :418-420: we might be in the anchoring pose for this measurement, hence +=
        H_x.addBlock(c, map_hx[clone_Ai.get()], (white_px * dz_dpfg) * dpfg_danchor);
        if (state->_options.do_calib_camera_pose)
          H_x.addBlock(c, map_hx[calibration.get()], (white_px * dz_dpfg) * dpfg_dcalib);
      }
      if (state->_options.do_calib_camera_pose) {
        Mat dpfc_dcalib(3, 6);
        dpfc_dcalib.setBlock(0, 0, skew_x(p_FinCi - p_IinC));
        dpfc_dcalib.setBlock(0, 3, Mat::Identity(3));
        H_x.addBlock(c, map_hx[calibration.get()], (white_px * dz_dpfc) * dpfc_dcalib);
      }
      if (state->_options.do_calib_camera_intrinsics)
        H_x.setBlock(c, map_hx[distortion.get()], white_px * dz_dzeta);
      c += 2;
    }

    if (feature.planeid != 0) {
      auto add_constraint = [&]() {
        double white_c = 1.0 / sigma_c;
        Mat local_p_FinG = p_FinG;
        Mat cp_inG = feature.cp_FinG;
        double d_inG = cp_inG.norm();
        Mat n_inG = (1.0 / d_inG) * cp_inG;
        res(c, 0) = white_c * (0.0 - (dot(n_inG, local_p_FinG) - d_inG));
        if (state->_options.do_fej) {
          local_p_FinG = p_FinG_fej;
          cp_inG = feature.cp_FinG_fej;
          d_inG = cp_inG.norm();
          n_inG = (1.0 / d_inG) * cp_inG;
        }
        double ntp = dot(n_inG, local_p_FinG);
        Mat H_c_plane = (white_c * 1.0 / d_inG) * (local_p_FinG.T() - ntp * n_inG.T() - d_inG * n_inG.T());
        if (plane_in_state) {
          VarP planecp = state->_features_PLANE.at(feature.planeid);
          H_x.setBlock(c, map_hx[planecp.get()], H_c_plane);
        } else {
          H_f.setBlock(c, H_f.cols() - 3, H_c_plane);
        }
        H_f.setBlock(c, 0, white_c * n_inG.T());
        c += 1;
      };
      if (total_meas == 0) {
        add_constraint();
      } else {
        for (int m = 0; m < total_meas; m++)
          add_constraint();
      }
    }
  }

  // UpdaterHelper.cpp:515-546
  static void nullspace_project_inplace(Mat &H_f, Mat &H_x, Mat &res) {
    assert(H_f.rows() >= H_f.cols());
    Givens G;
    for (int n = 0; n < H_f.cols(); ++n) {
      for (int m = H_f.rows() - 1; m > n; m--) {
        G.make(H_f(m - 1, n), H_f(m, n));
        G.apply(H_f, m, n, H_f.cols());
        G.apply(H_x, m, 0, H_x.cols());
        G.apply(res, m, 0, 1);
      }
    }
    H_x = H_x.block(H_f.cols(), 0, H_x.rows() - H_f.cols(), H_x.cols());
    res = res.block(H_f.cols(), 0, res.rows() - H_f.cols(), res.cols());
  }

  // UpdaterHelper.cpp:548-579
  static void measurement_compress_inplace(Mat &H_x, Mat &res) {
    if (H_x.rows() <= H_x.cols())
      return;
    Givens G;
    for (int n = 0; n < H_x.cols(); n++) {
      for (int m = H_x.rows() - 1; m > n; m--) {
        G.make(H_x(m - 1, n), H_x(m, n));
        G.apply(H_x, m, n, H_x.cols());
        G.apply(res, m, 0, 1);
      }
    }
    int r = std::min(H_x.rows(), H_x.cols());
    H_x.conservativeResize(r, H_x.cols());
    res.conservativeResize(r, res.cols());
  }
};

// ---------------------------------------------------------------------------------------------------------------
// UpdaterPlane static Givens helpers (update/UpdaterPlane.cpp:483-552)
// ---------------------------------------------------------------------------------------------------------------
struct UpdaterPlane {
  static void nullspace_project_inplace(Mat &H_f, Mat &H_x, Mat &H_cp, Mat &res) {
    assert(H_f.rows() >= H_f.cols());
    Givens G;
    for (int n = 0; n < H_f.cols(); ++n) {
      for (int m = H_f.rows() - 1; m > n; m--) {
        G.make(H_f(m - 1, n), H_f(m, n));
        G.apply(H_f, m, n, H_f.cols());
        G.apply(H_x, m, 0, H_x.cols());
        G.apply(H_cp, m, 0, H_cp.cols());
        G.apply(res, m, 0, 1);
      }
    }
    H_x = H_x.block(H_f.cols(), 0, H_x.rows() - H_f.cols(), H_x.cols());
    H_cp = H_cp.block(H_f.cols(), 0, H_cp.rows() - H_f.cols(), H_cp.cols());
    res = res.block(H_f.cols(), 0, res.rows() - H_f.cols(), res.cols());
  }
  static void measurement_compress_inplace(Mat &H_x, Mat &H_cp, Mat &res) {
    if (H_x.rows() <= H_x.cols())
      return;
    Givens G;
    for (int n = 0; n < H_x.cols(); n++) {
      for (int m = H_x.rows() - 1; m > n; m--) {
        G.make(H_x(m - 1, n), H_x(m, n));
        G.apply(H_x, m, n, H_x.cols());
        G.apply(H_cp, m, 0, H_cp.cols());
        G.apply(res, m, 0, 1);
      }
    }
    int r = std::min(H_x.rows(), H_x.cols());
    H_x.conservativeResize(r, H_x.cols());
    H_cp.conservativeResize(r, H_cp.cols());
    res.conservativeResize(r, res.cols());
  }
};

// ---------------------------------------------------------------------------------------------------------------
// UpdaterMSCKF::update from "plane linearisation points known" onward (update/UpdaterMSCKF.cpp:407-828).
// Triangulation / RANSAC / Ceres refinement (:142-404) are upstream of the path: their outputs arrive as inputs
// (Feature::p_FinG, p_FinG_original, plane_estimates_cp_inG).
// ---------------------------------------------------------------------------------------------------------------
struct MsckfTimers {
  double plane_updates = 0, feat_system = 0, compression = 0, update = 0;
};
struct MsckfResult {
  std::vector<size_t> used_plane_featids;          // features consumed by a successful plane update
  std::vector<std::pair<size_t, int>> plane_status; // (planeid, 1 pass / 0 chi2 fail)
  std::vector<std::pair<size_t, int>> feat_status;  // point path: (featid, 1 accept / 0 chi2 reject)
  std::vector<int> Hx_order_handles;                // Hx_order_big of the final point update (variable handles)
  std::vector<std::vector<int>> plane_Hx_order_handles;
  std::vector<double> plane_chi2;
  std::vector<double> feat_chi2;
  int point_rows = 0, point_cols = 0;
  MsckfTimers t;
};

struct UpdaterMSCKF {
  double sigma_pix = 1.0;
  double chi2_multipler = 1.0;
  Chi2Table chi2tab;
  bool time_stages = false;

  static double now() {
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
  }

  // feature_vec: MSCKF features in the caller's order (VioManager.cpp:608-623); feat2plane as the tracker/sim
  // produced it; plane_estimates_cp_inG: std::map ⇒ ascending plane id (UpdaterMSCKF.cpp:198,413)
  MsckfResult update(StateP state, std::vector<Feature> &feature_vec, const std::map<size_t, size_t> &feat2plane,
                     const std::map<size_t, Mat> &plane_estimates_cp_inG) {
    MsckfResult out;
    if (feature_vec.empty())
      return out;
    double t0 = now();
    // plane_feats in feature_vec order (:207-217); SLAM-feature members (:236-254) are not part of this restatement
    std::map<size_t, std::vector<Feature *>> plane_feats;
    for (auto &feat : feature_vec) {
      auto it = feat2plane.find(feat.featid);
      if (it == feat2plane.end())
        continue;
      plane_feats[it->second].push_back(&feat);
    }

    std::set<size_t> features_used_already;
    for (auto const &planepair : plane_estimates_cp_inG) {
      size_t planeid = planepair.first;
      if (plane_feats.find(planeid) == plane_feats.end())
        continue;
      bool is_slam_plane = (state->_features_PLANE.find(planeid) != state->_features_PLANE.end());
      std::vector<Feature *> features = plane_feats.at(planeid);
      assert(planeid != 0);
      assert(is_slam_plane || features.size() > 3);
      size_t max_meas_size = 0;
      for (auto *f : features) {
        max_meas_size += 3 * f->timestamps.size();
        if (f->timestamps.empty())
          max_meas_size += 1;
      }
      size_t max_hx_size = state->max_covariance_size();
      Mat res_big((int)max_meas_size, 1);
      Mat Hx_big((int)max_meas_size, (int)max_hx_size);
      Mat Hcp_big((int)max_meas_size, 3);
      std::unordered_map<Var *, size_t> Hx_mapping;
      std::vector<VarP> Hx_order_big;
      size_t ct_jacob = 0, ct_meas = 0;
      for (auto *feature : features) {
        Feature feat = *feature;
        feat.planeid = planeid;
        if (is_slam_plane) {
          feat.cp_FinG = state->_features_PLANE.at(planeid)->vecvalue(false);
          feat.cp_FinG_fej = state->_features_PLANE.at(planeid)->vecvalue(true);
        } else {
          feat.cp_FinG = plane_estimates_cp_inG.at(planeid);
          feat.cp_FinG_fej = plane_estimates_cp_inG.at(planeid);
        }
        feat.p_FinG_fej = feat.p_FinG; // MSCKF feature (:499-500)
        Mat H_f_tmp, H_x_tmp, res;
        std::vector<VarP> Hx_order_tmp;
        UpdaterHelper::get_feature_jacobian_full(state, feat, sigma_pix, state->_options.sigma_constraint, H_f_tmp, H_x_tmp, res,
                                                 Hx_order_tmp);
        Mat H_cp, H_f, H_x;
        std::vector<VarP> Hx_order;
        if (is_slam_plane) {
          int planeindex = state->_features_PLANE.at(planeid)->id;
          int planesize = 3;
          H_x = Mat(H_x_tmp.rows(), H_x_tmp.cols() - planesize);
          int ct_hx = 0, ct_hx_new = 0;
          for (auto &var : Hx_order_tmp) {
            if (var->id == planeindex) {
              H_cp = H_x_tmp.block(0, ct_hx, H_x_tmp.rows(), var->size());
            } else {
              Hx_order.push_back(var);
              H_x.setBlock(0, ct_hx_new, H_x_tmp.block(0, ct_hx, H_x_tmp.rows(), var->size()));
              ct_hx_new += var->size();
            }
            ct_hx += var->size();
          }
          H_f = H_f_tmp;
        } else {
          H_cp = H_f_tmp.block(0, H_f_tmp.cols() - 3, H_f_tmp.rows(), 3);
          H_f = H_f_tmp.block(0, 0, H_f_tmp.rows(), 3);
          H_x = H_x_tmp;
          Hx_order = Hx_order_tmp;
        }
        UpdaterPlane::nullspace_project_inplace(H_f, H_x, H_cp, res);
        size_t ct_hx = 0;
        for (auto &var : Hx_order) {
          if (Hx_mapping.find(var.get()) == Hx_mapping.end()) {
            Hx_mapping.insert({var.get(), ct_jacob});
            Hx_order_big.push_back(var);
            ct_jacob += var->size();
          }
          Hx_big.setBlock((int)ct_meas, (int)Hx_mapping[var.get()], H_x.block(0, (int)ct_hx, H_x.rows(), var->size()));
          ct_hx += var->size();
        }
        Hcp_big.setBlock((int)ct_meas, 0, H_cp);
        res_big.setBlock((int)ct_meas, 0, res);
        ct_meas += res.rows();
      }
      assert(ct_meas > 0);
      res_big.conservativeResize((int)ct_meas, 1);
      Hx_big.conservativeResize((int)ct_meas, (int)ct_jacob);
      Hcp_big.conservativeResize((int)ct_meas, 3);
      UpdaterPlane::measurement_compress_inplace(Hx_big, Hcp_big, res_big);
      if (is_slam_plane) {
        Mat H_xcp = Hx_big;
        H_xcp.conservativeResize(Hx_big.rows(), Hx_big.cols() + Hcp_big.cols());
        H_xcp.setBlock(0, Hx_big.cols(), Hcp_big);
        Hx_order_big.push_back(state->_features_PLANE.at(planeid));
        Hx_big = H_xcp;
      } else {
        assert(ct_meas > 3);
        UpdaterHelper::nullspace_project_inplace(Hcp_big, Hx_big, res_big);
      }
      Mat P_marg = StateHelper::get_marginal_covariance(state, Hx_order_big);
      Mat S = Hx_big * P_marg * Hx_big.T();
      for (int i = 0; i < S.rows(); i++)
        S(i, i) += 1.0;
      Mat L;
      if (!chol_lower(S, L))
        ref_exit("UpdaterMSCKF: plane S not positive definite");
      Mat y = res_big;
      chol_solve_inplace(L, y);
      double chi2 = dot(res_big, y);
      double chi2_check = chi2tab.at(res_big.rows());
      std::vector<int> handles;
      for (auto &v : Hx_order_big)
        handles.push_back(v->handle);
      out.plane_Hx_order_handles.push_back(handles);
      out.plane_chi2.push_back(chi2);
      const double chi2_gate = chi2 - gauge_probe().probe(Hx_big, res_big); // instrumentation only (see GaugeProbe); default: chi2
      if (chi2_gate > chi2_multipler * chi2_check) {
        out.plane_status.push_back({planeid, 0});
        continue;
      }
      out.plane_status.push_back({planeid, 1});
      for (auto *feature : features) {
        feature->to_delete = true;
        features_used_already.insert(feature->featid);
        out.used_plane_featids.push_back(feature->featid);
      }
      Mat R_big = Mat::Identity(res_big.rows());
      StateHelper::EKFUpdate(state, Hx_order_big, Hx_big, res_big, R_big);
    }
    double t1 = now();
    out.t.plane_updates = t1 - t0;

    // Remaining point features (:656-668)
    std::vector<Feature *> fv;
    for (auto &feature : feature_vec) {
      if (features_used_already.find(feature.featid) != features_used_already.end())
        continue;
      feature.p_FinG = feature.p_FinG_original;
      fv.push_back(&feature);
    }
    if (fv.empty())
      return out;
    size_t max_meas_size = 0;
    for (auto *f : fv)
      max_meas_size += 3 * f->timestamps.size();
    size_t max_hx_size = state->max_covariance_size();
    for (auto &landmark : state->_features_SLAM)
      max_hx_size -= landmark.second->size();
    Mat res_big((int)max_meas_size, 1);
    Mat Hx_big((int)max_meas_size, (int)max_hx_size);
    std::unordered_map<Var *, size_t> Hx_mapping;
    std::vector<VarP> Hx_order_big;
    size_t ct_jacob = 0, ct_meas = 0;
    for (auto *f : fv) {
      Feature feat = *f;
      feat.planeid = 0;
      feat.p_FinG_fej = feat.p_FinG; // :721-722
      Mat H_f, H_x, res;
      std::vector<VarP> Hx_order;
      UpdaterHelper::get_feature_jacobian_full(state, feat, sigma_pix, state->_options.sigma_constraint, H_f, H_x, res, Hx_order);
      UpdaterHelper::nullspace_project_inplace(H_f, H_x, res);
      Mat P_marg = StateHelper::get_marginal_covariance(state, Hx_order);
      Mat S = H_x * P_marg * H_x.T();
      for (int i = 0; i < S.rows(); i++)
        S(i, i) += 1.0;
      Mat L;
      if (!chol_lower(S, L))
        ref_exit("UpdaterMSCKF: feature S not positive definite");
      Mat y = res;
      chol_solve_inplace(L, y);
      double chi2 = dot(res, y);
      double chi2_check = chi2tab.at(res.rows());
      out.feat_chi2.push_back(chi2);
      if (chi2 > chi2_multipler * chi2_check) {
        f->to_delete = true;
        out.feat_status.push_back({f->featid, 0});
        continue;
      }
      out.feat_status.push_back({f->featid, 1});
      size_t ct_hx = 0;
      for (auto &var : Hx_order) {
        if (Hx_mapping.find(var.get()) == Hx_mapping.end()) {
          Hx_mapping.insert({var.get(), ct_jacob});
          Hx_order_big.push_back(var);
          ct_jacob += var->size();
        }
        Hx_big.setBlock((int)ct_meas, (int)Hx_mapping[var.get()], H_x.block(0, (int)ct_hx, H_x.rows(), var->size()));
        ct_hx += var->size();
      }
      res_big.setBlock((int)ct_meas, 0, res);
      ct_meas += res.rows();
      f->to_delete = true;
    }
    double t2 = now();
    out.t.feat_system = t2 - t1;
    if (ct_meas < 1)
      return out;
    res_big.conservativeResize((int)ct_meas, 1);
    Hx_big.conservativeResize((int)ct_meas, (int)ct_jacob);
    out.point_rows = (int)ct_meas;
    out.point_cols = (int)ct_jacob;
    UpdaterHelper::measurement_compress_inplace(Hx_big, res_big);
    double t3 = now();
    out.t.compression = t3 - t2;
    if (Hx_big.rows() < 1)
      return out;
    for (auto &v : Hx_order_big)
      out.Hx_order_handles.push_back(v->handle);
    Mat R_big = Mat::Identity(res_big.rows());
    StateHelper::EKFUpdate(state, Hx_order_big, Hx_big, res_big, R_big);
    out.t.update = now() - t3;
    return out;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// UpdaterPlane::init_vio_plane from "plane linearisation points known" onward (update/UpdaterPlane.cpp:297-481); the
// RANSAC fit / Ceres refinement before it (:61-293) are upstream of the path, their outputs arrive as inputs.
// ---------------------------------------------------------------------------------------------------------------
struct PlaneInitResult {
  std::vector<std::pair<size_t, int>> plane_status; // (planeid, 1 initialised / 0 rejected)
  std::vector<int> new_handles;
};
struct UpdaterPlaneInit {
  double sigma_pix = 1.0;
  Chi2Table chi2tab;
  PlaneInitResult init_vio_plane(StateP state, std::vector<Feature> &feature_vec, const std::map<size_t, size_t> &feat2plane,
                                 const std::map<size_t, Mat> &plane_estimates_cp_inG) {
    PlaneInitResult out;
    std::map<size_t, std::vector<Feature *>> plane_feats;
    for (auto &feat : feature_vec) {
      auto it = feat2plane.find(feat.featid);
      if (it != feat2plane.end())
        plane_feats[it->second].push_back(&feat);
    }
    for (auto const &planepair : plane_estimates_cp_inG) {
      size_t planeid = planepair.first;
      Mat cp_inG = planepair.second;
      if (plane_feats.find(planeid) == plane_feats.end())
        continue;
      if (state->_features_PLANE.find(planeid) != state->_features_PLANE.end())
        continue; // only planes that are not in the state are initialised (:304)
      std::vector<Feature *> features = plane_feats.at(planeid);
      if (features.size() < 3)
        continue; // assert(features.size() >= 3), :303
      size_t max_meas_size = 0;
      for (auto *f : features)
        max_meas_size += 3 * f->timestamps.size();
      size_t max_hx_size = state->max_covariance_size();
      Mat res_big((int)max_meas_size, 1), Hx_big((int)max_meas_size, (int)max_hx_size), Hcp_big((int)max_meas_size, 3);
      std::unordered_map<Var *, size_t> Hx_mapping;
      std::vector<VarP> Hx_order_big;
      size_t ct_jacob = 0, ct_meas = 0;
      for (auto *feature : features) {
        Feature feat = *feature;
        feat.planeid = planeid;
        feat.cp_FinG = cp_inG;
        feat.cp_FinG_fej = cp_inG;
        feat.p_FinG_fej = feat.p_FinG;
        Mat H_f, H_x, res;
        std::vector<VarP> Hx_order;
        double sigma_c = state->_options.const_init_multi * state->_options.sigma_constraint; // :384
        UpdaterHelper::get_feature_jacobian_full(state, feat, sigma_pix, sigma_c, H_f, H_x, res, Hx_order);
        assert(H_f.cols() == 6);
        Mat H_cp = H_f.block(0, 3, H_f.rows(), 3);
        H_f = H_f.block(0, 0, H_f.rows(), 3);
        UpdaterPlane::nullspace_project_inplace(H_f, H_x, H_cp, res);
        size_t ct_hx = 0;
        for (auto &var : Hx_order) {
          if (Hx_mapping.find(var.get()) == Hx_mapping.end()) {
            Hx_mapping.insert({var.get(), ct_jacob});
            Hx_order_big.push_back(var);
            ct_jacob += var->size();
          }
          Hx_big.setBlock((int)ct_meas, (int)Hx_mapping[var.get()], H_x.block(0, (int)ct_hx, H_x.rows(), var->size()));
          ct_hx += var->size();
        }
        Hcp_big.setBlock((int)ct_meas, 0, H_cp);
        res_big.setBlock((int)ct_meas, 0, res);
        ct_meas += res.rows();
      }
      res_big.conservativeResize((int)ct_meas, 1);
      Hx_big.conservativeResize((int)ct_meas, (int)ct_jacob);
      Hcp_big.conservativeResize((int)ct_meas, 3);
      UpdaterPlane::measurement_compress_inplace(Hx_big, Hcp_big, res_big);
      Mat R_big = Mat::Identity(res_big.rows());
      VarP plane = Var::makeVec(3);
      for (int i = 0; i < 3; i++) {
        plane->value[i] = cp_inG(i, 0);
        plane->fej[i] = cp_inG(i, 0);
      }
      if (StateHelper::initialize(state, plane, Hx_order_big, Hx_big, Hcp_big, R_big, res_big, state->_options.const_init_chi2, chi2tab)) {
        state->reg(plane);
        state->_features_PLANE.insert({planeid, plane});
        out.plane_status.push_back({planeid, 1});
        out.new_handles.push_back(plane->handle);
      } else {
        out.plane_status.push_back({planeid, 0});
        out.new_handles.push_back(-1);
      }
    }
    return out;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// UpdaterSLAM (update/UpdaterSLAM.cpp): update (:376-682) from "measurements cleaned" on, delayed_init (:205-364) from
// "triangulated (and plane-refined)" on.  GLOBAL_3D landmarks, no ArUco.
// ---------------------------------------------------------------------------------------------------------------
struct SlamOptions {
  double sigma_pix = 1.0, chi2_multipler = 1.0;
  bool use_plane_constraint_slamu = true, use_plane_constraint_slamd = true;
};
// ---------------------------------------------------------------------------------------------------------------
// ov_type::Landmark::get_xyz / set_from_xyz (ov_core @74a63cf, not in the tree: restated) and UpdaterSLAM::change_anchors /
// perform_anchor_change (update/UpdaterSLAM.cpp:684-850).  Landmark forms 0..4 (the single-depth form needs the initial bearing).
// ---------------------------------------------------------------------------------------------------------------
struct LandmarkOps {
  static Mat get_xyz(const Var &lm, bool isfej) {
    const std::vector<double> &v = isfej ? lm.fej : lm.value;
    const int rep = lm.feat_representation;
    if (rep == 0 || rep == 2)
      return vec3(v[0], v[1], v[2]);
    if (rep == 4)
      return vec3(v[0] / v[2], v[1] / v[2], 1.0 / v[2]);
    if (rep == 1 || rep == 3)
      return (1.0 / v[2]) * vec3(std::cos(v[0]) * std::sin(v[1]), std::sin(v[0]) * std::sin(v[1]), std::cos(v[1]));
    ref_exit("Landmark::get_xyz: representation not carried");
    return Mat(3, 1);
  }
  static void set_from_xyz(Var &lm, const Mat &p, bool isfej) {
    std::vector<double> &v = isfej ? lm.fej : lm.value;
    const int rep = lm.feat_representation;
    if (rep == 0 || rep == 2) {
      v[0] = p(0, 0), v[1] = p(1, 0), v[2] = p(2, 0);
    } else if (rep == 4) {
      v[0] = p(0, 0) / p(2, 0), v[1] = p(1, 0) / p(2, 0), v[2] = 1.0 / p(2, 0);
    } else if (rep == 1 || rep == 3) {
      double g_rho = 1.0 / p.norm();
      v[0] = std::atan2(p(1, 0), p(0, 0));
      v[1] = std::acos(g_rho * p(2, 0));
      v[2] = g_rho;
    } else {
      ref_exit("Landmark::set_from_xyz: representation not carried");
    }
  }
  // UpdaterSLAM::perform_anchor_change (:706-850), mono camera (anchor_cam_id = 0)
  static void perform_anchor_change(StateP state, VarP landmark, double new_anchor_timestamp) {
    const int rep = landmark->feat_representation;
    if (rep < 2)
      ref_exit("perform_anchor_change: not an anchored representation (assert, :710)");
    VarP calibv = state->_calib_IMUtoCAM;
    VarP cl_old = state->_clones_IMU.at(landmark->anchor_clone_timestamp), cl_new = state->_clones_IMU.at(new_anchor_timestamp);
    auto pose7 = [](const VarP &v, bool fej) {
      Mat m(7, 1);
      for (int i = 0; i < 7; i++)
        m(i, 0) = fej ? v->fej[i] : v->value[i];
      return m;
    };
    Mat p_FinA = get_xyz(*landmark, false), p_FinA_fej = get_xyz(*landmark, true);
    Mat H_f_old, Ha_old, Hc_old, H_f_new, Ha_new, Hc_new, zero3(3, 1);
    UpdaterHelper::get_feature_jacobian_representation(rep, state->_options.do_fej, zero3, zero3, p_FinA, pose7(cl_old, false), pose7(cl_old, true),
                                                       pose7(calibv, false), H_f_old, Ha_old, Hc_old);
    // :739-777 the landmark in the new anchor camera, best and first estimates (the extrinsics have no first estimate)
    auto reanchor = [&](bool fej, const Mat &p_in) {
      Mat R_GtoOLD = calibv->Rot() * (fej ? cl_old->Rot_fej() : cl_old->Rot());
      Mat p_OLDinG = (fej ? cl_old->pos_fej() : cl_old->pos()) - R_GtoOLD.T() * calibv->pos();
      Mat R_GtoNEW = calibv->Rot() * (fej ? cl_new->Rot_fej() : cl_new->Rot());
      Mat p_NEWinG = (fej ? cl_new->pos_fej() : cl_new->pos()) - R_GtoNEW.T() * calibv->pos();
      Mat R_OLDtoNEW = R_GtoNEW * R_GtoOLD.T();
      Mat p_OLDinNEW = R_GtoNEW * (p_OLDinG - p_NEWinG);
      return R_OLDtoNEW * p_in + p_OLDinNEW;
    };
    Mat p_FinA_new = reanchor(false, p_FinA), p_FinA_new_fej = reanchor(true, p_FinA_fej);
    UpdaterHelper::get_feature_jacobian_representation(rep, state->_options.do_fej, zero3, zero3, p_FinA_new, pose7(cl_new, false), pose7(cl_new, true),
                                                       pose7(calibv, false), H_f_new, Ha_new, Hc_new);
    std::vector<VarP> x_order_old = {cl_old}, x_order_new = {cl_new};
    std::vector<Mat> H_x_old = {Ha_old}, H_x_new = {Ha_new};
    if (state->_options.do_calib_camera_pose) {
      x_order_old.push_back(calibv);
      H_x_old.push_back(Hc_old);
      x_order_new.push_back(calibv);
      H_x_new.push_back(Hc_new);
    }
    std::vector<VarP> phi_order_NEW = {landmark}, phi_order_OLD;
    int current_it = 0;
    std::map<Var *, int> Phi_id_map;
    for (auto &var : x_order_old)
      if (Phi_id_map.find(var.get()) == Phi_id_map.end()) {
        Phi_id_map.insert({var.get(), current_it});
        phi_order_OLD.push_back(var);
        current_it += var->size();
      }
    for (auto &var : x_order_new)
      if (Phi_id_map.find(var.get()) == Phi_id_map.end()) {
        Phi_id_map.insert({var.get(), current_it});
        phi_order_OLD.push_back(var);
        current_it += var->size();
      }
    Phi_id_map.insert({landmark.get(), current_it});
    phi_order_OLD.push_back(landmark);
    current_it += landmark->size();
    Mat Phi(3, current_it), Q(3, 3);
    Mat H_f_new_inv = inverse_small(H_f_new);
    for (size_t i = 0; i < H_x_old.size(); i++)
      Phi.addBlock(0, Phi_id_map.at(x_order_old[i].get()), H_f_new_inv * H_x_old[i]);
    Phi.setBlock(0, Phi_id_map.at(landmark.get()), H_f_new_inv * H_f_old);
    for (size_t i = 0; i < H_x_new.size(); i++)
      Phi.addBlock(0, Phi_id_map.at(x_order_new[i].get()), (-1.0) * (H_f_new_inv * H_x_new[i]));
    StateHelper::EKFPropagation(state, phi_order_NEW, phi_order_OLD, Phi, Q);
    landmark->anchor_clone_timestamp = new_anchor_timestamp;
    set_from_xyz(*landmark, p_FinA_new, false);
    set_from_xyz(*landmark, p_FinA_new_fej, true);
    landmark->has_had_anchor_change = true;
  }
  // UpdaterSLAM::change_anchors (:684-704)
  static int change_anchors(StateP state) {
    if ((int)state->_clones_IMU.size() <= state->_options.max_clone_size)
      return 0;
    int n = 0;
    double marg_timestep = state->margtimestep();
    for (auto &f : state->_features_SLAM) {
      if (f.second->feat_representation < 2)
        continue;
      if (f.second->anchor_clone_timestamp == marg_timestep) {
        perform_anchor_change(state, f.second, state->_timestamp);
        n++;
      }
    }
    return n;
  }
};

struct UpdaterSLAM {
  SlamOptions opt;
  Chi2Table chi2tab;

  // returns per feature: 1 accepted (with its plane constraint if any), 3 accepted after dropping the plane constraint, 0 rejected
  std::vector<int> update(StateP state, std::vector<Feature> &feature_vec, const std::map<size_t, size_t> &feat2plane,
                          std::vector<double> *chi2_out = nullptr) {
    std::vector<int> status(feature_vec.size(), 0);
    if (chi2_out)
      chi2_out->assign(feature_vec.size(), NAN);
    if (feature_vec.empty())
      return status;
    size_t max_meas_size = 0;
    for (auto &f : feature_vec)
      max_meas_size += 3 * f.timestamps.size();
    size_t max_hx_size = state->max_covariance_size();
    Mat res_big((int)max_meas_size, 1), Hx_big((int)max_meas_size, (int)max_hx_size);
    std::unordered_map<Var *, size_t> Hx_mapping;
    std::vector<VarP> Hx_order_big;
    size_t ct_jacob = 0, ct_meas = 0;
    for (size_t fi = 0; fi < feature_vec.size(); fi++) {
      Feature feat = feature_vec[fi];
      VarP landmark = state->_features_SLAM.at(feat.featid);
      feat.planeid = 0;
      auto itp = feat2plane.find(feat.featid);
      if (opt.use_plane_constraint_slamu && itp != feat2plane.end() && state->_features_PLANE.count(itp->second)) {
        auto its = state->_features_SLAM_to_PLANE.find(feat.featid);
        if (its == state->_features_SLAM_to_PLANE.end() || its->second != 0) {
          feat.planeid = itp->second;
          feat.cp_FinG = state->_features_PLANE.at(itp->second)->vecvalue(false);
          feat.cp_FinG_fej = state->_features_PLANE.at(itp->second)->vecvalue(true);
        }
      }
      feat.p_FinG = landmark->vecvalue(false);
      feat.p_FinG_fej = landmark->vecvalue(true);
      Mat H_f, H_x, res;
      std::vector<VarP> Hx_order;
      auto build = [&](Mat &H_xf, std::vector<VarP> &Hxf_order, double &chi2) {
        UpdaterHelper::get_feature_jacobian_full(state, feat, opt.sigma_pix, state->_options.sigma_constraint, H_f, H_x, res, Hx_order);
        H_xf = H_x;
        H_xf.conservativeResize(H_x.rows(), H_x.cols() + H_f.cols());
        H_xf.setBlock(0, H_x.cols(), H_f);
        Hxf_order = Hx_order;
        Hxf_order.push_back(landmark);
        Mat P_marg = StateHelper::get_marginal_covariance(state, Hxf_order);
        Mat S = H_xf * P_marg * H_xf.T();
        for (int i = 0; i < S.rows(); i++)
          S(i, i) += 1.0;
        Mat L;
        if (!chol_lower(S, L))
          ref_exit("UpdaterSLAM: S not positive definite");
        Mat y = res;
        chol_solve_inplace(L, y);
        chi2 = dot(res, y);
      };
      Mat H_xf;
      std::vector<VarP> Hxf_order;
      double chi2;
      build(H_xf, Hxf_order, chi2);
      double chi2_check = chi2tab.at(res.rows());
      int st = 1;
      if (feat.planeid != 0 && chi2 > opt.chi2_multipler * chi2_check) {
        feat.planeid = 0; // fallback without the plane (:547-609)
        state->_features_SLAM_to_PLANE[feat.featid] = 0;
        build(H_xf, Hxf_order, chi2);
        chi2_check = chi2tab.at(res.rows());
        st = 3;
        if (chi2 > opt.chi2_multipler * chi2_check) {
          if ((int)feat.featid >= state->_options.max_aruco_features) // ArUco tags are not flagged (:600-605)
            landmark->should_marg = true;
          status[fi] = 0;
          if (chi2_out)
            (*chi2_out)[fi] = chi2;
          continue;
        }
      } else if (chi2 > opt.chi2_multipler * chi2_check) {
        if ((int)feat.featid >= state->_options.max_aruco_features) // ArUco tags are not flagged (:613-618)
          landmark->should_marg = true;
        status[fi] = 0;
        if (chi2_out)
          (*chi2_out)[fi] = chi2;
        continue;
      }
      if (chi2_out)
        (*chi2_out)[fi] = chi2;
      if (feat.planeid != 0)
        state->_features_SLAM_to_PLANE[feat.featid] = feat.planeid;
      status[fi] = st;
      size_t ct_hx = 0;
      for (auto &var : Hxf_order) {
        if (Hx_mapping.find(var.get()) == Hx_mapping.end()) {
          Hx_mapping.insert({var.get(), ct_jacob});
          Hx_order_big.push_back(var);
          ct_jacob += var->size();
        }
        Hx_big.setBlock((int)ct_meas, (int)Hx_mapping[var.get()], H_xf.block(0, (int)ct_hx, H_xf.rows(), var->size()));
        ct_hx += var->size();
      }
      res_big.setBlock((int)ct_meas, 0, res);
      ct_meas += res.rows();
    }
    if (ct_meas < 1)
      return status;
    res_big.conservativeResize((int)ct_meas, 1);
    Hx_big.conservativeResize((int)ct_meas, (int)ct_jacob);
    Mat R_big = Mat::Identity((int)ct_meas);
    StateHelper::EKFUpdate(state, Hx_order_big, Hx_big, res_big, R_big); // no compression (:672-673)
    return status;
  }

  // returns per feature: 1 initialised (with plane constraint if any), 3 initialised after dropping the plane, 0 failed
  std::vector<int> delayed_init(StateP state, std::vector<Feature> &feature_vec, const std::map<size_t, size_t> &feat2plane,
                                std::vector<int> *handles_out = nullptr) {
    std::vector<int> status(feature_vec.size(), 0);
    if (handles_out)
      handles_out->assign(feature_vec.size(), -1);
    for (size_t fi = 0; fi < feature_vec.size(); fi++) {
      Feature feat = feature_vec[fi];
      feat.planeid = 0;
      auto itp = feat2plane.find(feat.featid);
      if (opt.use_plane_constraint_slamd && itp != feat2plane.end() && state->_features_PLANE.count(itp->second)) {
        auto its = state->_features_SLAM_to_PLANE.find(feat.featid);
        if (its == state->_features_SLAM_to_PLANE.end() || its->second != 0) {
          feat.planeid = itp->second;
          feat.cp_FinG = state->_features_PLANE.at(itp->second)->vecvalue(false);
          feat.cp_FinG_fej = state->_features_PLANE.at(itp->second)->vecvalue(true);
        }
      }
      feat.p_FinG_fej = feat.p_FinG;
      auto attempt = [&]() -> bool {
        Mat H_f, H_x, res;
        std::vector<VarP> Hx_order;
        UpdaterHelper::get_feature_jacobian_full(state, feat, opt.sigma_pix, state->_options.sigma_constraint, H_f, H_x, res, Hx_order);
        VarP landmark = Var::makeLandmark(3);
        landmark->featid = feat.featid;
        for (int i = 0; i < 3; i++) {
          landmark->value[i] = feat.p_FinG(i, 0);
          landmark->fej[i] = feat.p_FinG_fej(i, 0);
        }
        Mat R = Mat::Identity(res.rows());
        if (StateHelper::initialize(state, landmark, Hx_order, H_x, H_f, R, res, opt.chi2_multipler, chi2tab)) {
          state->reg(landmark);
          state->_features_SLAM.insert({feat.featid, landmark});
          if (handles_out)
            (*handles_out)[fi] = landmark->handle;
          return true;
        }
        return false;
      };
      if (attempt()) {
        status[fi] = 1;
        if (feat.planeid != 0)
          state->_features_SLAM_to_PLANE[feat.featid] = feat.planeid;
      } else if (feat.planeid != 0) {
        feat.planeid = 0; // fallback (:310-359): no plane, position before the plane refinement
        state->_features_SLAM_to_PLANE[feat.featid] = 0;
        feat.p_FinG = feat.p_FinG_original;
        feat.p_FinG_fej = feat.p_FinG_original;
        if (attempt())
          status[fi] = 3;
      }
    }
    return status;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// Propagator (state/Propagator.cpp)
// ---------------------------------------------------------------------------------------------------------------
struct ImuData {
  double timestamp;
  Mat wm = Mat(3, 1), am = Mat(3, 1);
};
struct NoiseManager { // utils/NoiseManager.h:41-63
  double sigma_w = 1.6968e-04, sigma_wb = 1.9393e-05, sigma_a = 2.0000e-3, sigma_ab = 3.0000e-03;
  double sigma_w_2() const { return sigma_w * sigma_w; }
  double sigma_wb_2() const { return sigma_wb * sigma_wb; }
  double sigma_a_2() const { return sigma_a * sigma_a; }
  double sigma_ab_2() const { return sigma_ab * sigma_ab; }
};

struct Propagator {
  NoiseManager _noises;
  Mat _gravity = vec3(0, 0, 9.81);
  std::vector<ImuData> imu_data;
  double last_prop_time_offset = 0.0;
  bool have_last_prop_time_offset = false;

  // Propagator.h:146-156
  static ImuData interpolate_data(const ImuData &imu_1, const ImuData &imu_2, double timestamp) {
    double lambda = (timestamp - imu_1.timestamp) / (imu_2.timestamp - imu_1.timestamp);
    ImuData data;
    data.timestamp = timestamp;
    data.am = (1 - lambda) * imu_1.am + lambda * imu_2.am;
    data.wm = (1 - lambda) * imu_1.wm + lambda * imu_2.wm;
    return data;
  }

  // Propagator.cpp:226-341
  static std::vector<ImuData> select_imu_readings(const std::vector<ImuData> &imu_data, double time0, double time1) {
    std::vector<ImuData> prop_data;
    if (imu_data.empty())
      return prop_data;
    for (size_t i = 0; i + 1 < imu_data.size(); i++) {
      if (imu_data.at(i + 1).timestamp > time0 && imu_data.at(i).timestamp < time0) {
        prop_data.push_back(interpolate_data(imu_data.at(i), imu_data.at(i + 1), time0));
        continue;
      }
      if (imu_data.at(i).timestamp >= time0 && imu_data.at(i + 1).timestamp <= time1) {
        prop_data.push_back(imu_data.at(i));
        continue;
      }
      if (imu_data.at(i + 1).timestamp > time1) {
        if (imu_data.at(i).timestamp > time1 && i == 0) {
          break;
        } else if (imu_data.at(i).timestamp > time1) {
          prop_data.push_back(interpolate_data(imu_data.at(i - 1), imu_data.at(i), time1));
        } else {
          prop_data.push_back(imu_data.at(i));
        }
        if (prop_data.at(prop_data.size() - 1).timestamp != time1)
          prop_data.push_back(interpolate_data(imu_data.at(i), imu_data.at(i + 1), time1));
        break;
      }
    }
    if (prop_data.empty())
      return prop_data;
    for (size_t i = 0; i + 1 < prop_data.size(); i++) {
      if (std::abs(prop_data.at(i + 1).timestamp - prop_data.at(i).timestamp) < 1e-12) {
        prop_data.erase(prop_data.begin() + i);
        i--;
      }
    }
    return prop_data;
  }

  // Propagator.cpp:456-488
  void predict_mean_discrete(StateP state, double dt, const Mat &w_hat1, const Mat &a_hat1, const Mat &w_hat2, const Mat &a_hat2,
                             Mat &new_q, Mat &new_v, Mat &new_p) {
    Mat w_hat = w_hat1, a_hat = a_hat1;
    if (state->_options.imu_avg) {
      w_hat = .5 * (w_hat1 + w_hat2);
      a_hat = .5 * (a_hat1 + a_hat2);
    }
    double w_norm = w_hat.norm();
    Mat I4 = Mat::Identity(4);
    Mat R_Gtoi = state->_imu->Rot();
    Mat bigO;
    if (w_norm > 1e-20)
      bigO = std::cos(0.5 * w_norm * dt) * I4 + (1 / w_norm * std::sin(0.5 * w_norm * dt)) * Omega(w_hat);
    else
      bigO = I4 + (0.5 * dt) * Omega(w_hat);
    new_q = quatnorm(bigO * state->_imu->quat());
    new_v = state->_imu->vel() + dt * (R_Gtoi.T() * a_hat) - dt * _gravity;
    new_p = state->_imu->pos() + dt * state->_imu->vel() + (0.5 * dt * dt) * (R_Gtoi.T() * a_hat) - (0.5 * dt * dt) * _gravity;
  }

  // Propagator.cpp:490-569
  void predict_mean_rk4(StateP state, double dt, const Mat &w_hat1, const Mat &a_hat1, const Mat &w_hat2, const Mat &a_hat2, Mat &new_q,
                        Mat &new_v, Mat &new_p) {
    Mat w_hat = w_hat1, a_hat = a_hat1;
    Mat w_alpha = (1.0 / dt) * (w_hat2 - w_hat1);
    Mat a_jerk = (1.0 / dt) * (a_hat2 - a_hat1);
    Mat q_0 = state->_imu->quat();
    Mat p_0 = state->_imu->pos();
    Mat v_0 = state->_imu->vel();
    Mat dq_0(4, 1);
    dq_0(3, 0) = 1;
    Mat q0_dot = 0.5 * (Omega(w_hat) * dq_0);
    Mat p0_dot = v_0;
    Mat R_Gto0 = quat_2_Rot(quat_multiply(dq_0, q_0));
    Mat v0_dot = R_Gto0.T() * a_hat - _gravity;
    Mat k1_q = dt * q0_dot, k1_p = dt * p0_dot, k1_v = dt * v0_dot;
    w_hat = w_hat + (0.5 * dt) * w_alpha;
    a_hat = a_hat + (0.5 * dt) * a_jerk;
    Mat dq_1 = quatnorm(dq_0 + 0.5 * k1_q);
    Mat v_1 = v_0 + 0.5 * k1_v;
    Mat q1_dot = 0.5 * (Omega(w_hat) * dq_1);
    Mat p1_dot = v_1;
    Mat R_Gto1 = quat_2_Rot(quat_multiply(dq_1, q_0));
    Mat v1_dot = R_Gto1.T() * a_hat - _gravity;
    Mat k2_q = dt * q1_dot, k2_p = dt * p1_dot, k2_v = dt * v1_dot;
    Mat dq_2 = quatnorm(dq_0 + 0.5 * k2_q);
    Mat v_2 = v_0 + 0.5 * k2_v;
    Mat q2_dot = 0.5 * (Omega(w_hat) * dq_2);
    Mat p2_dot = v_2;
    Mat R_Gto2 = quat_2_Rot(quat_multiply(dq_2, q_0));
    Mat v2_dot = R_Gto2.T() * a_hat - _gravity;
    Mat k3_q = dt * q2_dot, k3_p = dt * p2_dot, k3_v = dt * v2_dot;
    w_hat = w_hat + (0.5 * dt) * w_alpha;
    a_hat = a_hat + (0.5 * dt) * a_jerk;
    Mat dq_3 = quatnorm(dq_0 + k3_q);
    Mat v_3 = v_0 + k3_v;
    Mat q3_dot = 0.5 * (Omega(w_hat) * dq_3);
    Mat p3_dot = v_3;
    Mat R_Gto3 = quat_2_Rot(quat_multiply(dq_3, q_0));
    Mat v3_dot = R_Gto3.T() * a_hat - _gravity;
    Mat k4_q = dt * q3_dot, k4_p = dt * p3_dot, k4_v = dt * v3_dot;
    Mat dq = quatnorm(dq_0 + (1.0 / 6.0) * k1_q + (1.0 / 3.0) * k2_q + (1.0 / 3.0) * k3_q + (1.0 / 6.0) * k4_q);
    new_q = quat_multiply(dq, q_0);
    new_p = p_0 + (1.0 / 6.0) * k1_p + (1.0 / 3.0) * k2_p + (1.0 / 3.0) * k3_p + (1.0 / 6.0) * k4_p;
    new_v = v_0 + (1.0 / 6.0) * k1_v + (1.0 / 3.0) * k2_v + (1.0 / 3.0) * k3_v + (1.0 / 6.0) * k4_v;
  }

  // Propagator.cpp:343-454.  IMU sub-variable ids: th 0, p 3, v 6, bg 9, ba 12 (:369-373)
  void predict_and_compute(StateP state, const ImuData &data_minus, const ImuData &data_plus, Mat &F, Mat &Qd) {
    F = Mat(15, 15);
    Qd = Mat(15, 15);
    double dt = data_plus.timestamp - data_minus.timestamp;
    Mat w_hat = data_minus.wm - state->_imu->bias_g();
    Mat a_hat = data_minus.am - state->_imu->bias_a();
    Mat w_hat2 = data_plus.wm - state->_imu->bias_g();
    Mat a_hat2 = data_plus.am - state->_imu->bias_a();
    Mat new_q, new_v, new_p;
    if (state->_options.use_rk4_integration)
      predict_mean_rk4(state, dt, w_hat, a_hat, w_hat2, a_hat2, new_q, new_v, new_p);
    else
      predict_mean_discrete(state, dt, w_hat, a_hat, w_hat2, a_hat2, new_q, new_v, new_p);
    const int th_id = 0, p_id = 3, v_id = 6, bg_id = 9, ba_id = 12;
    Mat G(15, 12);
    Mat I3 = Mat::Identity(3);
    if (state->_options.do_fej) {
      Mat Rfej = state->_imu->Rot_fej();
      Mat dR = quat_2_Rot(new_q) * Rfej.T();
      Mat v_fej = state->_imu->vel_fej();
      Mat p_fej = state->_imu->pos_fej();
      Mat JrT = Jr_so3((-dt) * w_hat);
      F.setBlock(th_id, th_id, dR);
      F.setBlock(th_id, bg_id, (-dt) * (dR * JrT));
      F.setBlock(bg_id, bg_id, I3);
      F.setBlock(v_id, th_id, -1.0 * (skew_x(new_v - v_fej + dt * _gravity) * Rfej.T()));
      F.setBlock(v_id, v_id, I3);
      F.setBlock(v_id, ba_id, (-dt) * Rfej.T());
      F.setBlock(ba_id, ba_id, I3);
      F.setBlock(p_id, th_id, -1.0 * (skew_x(new_p - p_fej - dt * v_fej + (0.5 * dt * dt) * _gravity) * Rfej.T()));
      F.setBlock(p_id, v_id, dt * I3);
      F.setBlock(p_id, ba_id, (-0.5 * dt * dt) * Rfej.T());
      F.setBlock(p_id, p_id, I3);
      G.setBlock(th_id, 0, (-dt) * (dR * JrT));
      G.setBlock(v_id, 3, (-dt) * Rfej.T());
      G.setBlock(p_id, 3, (-0.5 * dt * dt) * Rfej.T());
      G.setBlock(bg_id, 6, I3);
      G.setBlock(ba_id, 9, I3);
    } else {
      Mat R_Gtoi = state->_imu->Rot();
      Mat E = exp_so3((-dt) * w_hat);
      Mat JrT = Jr_so3((-dt) * w_hat);
      F.setBlock(th_id, th_id, E);
      F.setBlock(th_id, bg_id, (-dt) * (E * JrT));
      F.setBlock(bg_id, bg_id, I3);
      F.setBlock(v_id, th_id, -1.0 * (R_Gtoi.T() * skew_x(dt * a_hat)));
      F.setBlock(v_id, v_id, I3);
      F.setBlock(v_id, ba_id, (-dt) * R_Gtoi.T());
      F.setBlock(ba_id, ba_id, I3);
      F.setBlock(p_id, th_id, -0.5 * (R_Gtoi.T() * skew_x((dt * dt) * a_hat)));
      F.setBlock(p_id, v_id, dt * I3);
      F.setBlock(p_id, ba_id, (-0.5 * dt * dt) * R_Gtoi.T());
      F.setBlock(p_id, p_id, I3);
      G.setBlock(th_id, 0, (-dt) * (E * JrT));
      G.setBlock(v_id, 3, (-dt) * R_Gtoi.T());
      G.setBlock(p_id, 3, (-0.5 * dt * dt) * R_Gtoi.T());
      G.setBlock(bg_id, 6, I3);
      G.setBlock(ba_id, 9, I3);
    }
    Mat Qc(12, 12);
    for (int i = 0; i < 3; i++) {
      Qc(i, i) = _noises.sigma_w_2() / dt;
      Qc(3 + i, 3 + i) = _noises.sigma_a_2() / dt;
      Qc(6 + i, 6 + i) = _noises.sigma_wb_2() * dt;
      Qc(9 + i, 9 + i) = _noises.sigma_ab_2() * dt;
    }
    Qd = G * Qc * G.T();
    Qd = 0.5 * (Qd + Qd.T());
    for (int i = 0; i < 4; i++)
      state->_imu->value[i] = new_q(i, 0);
    for (int i = 0; i < 3; i++) {
      state->_imu->value[4 + i] = new_p(i, 0);
      state->_imu->value[7 + i] = new_v(i, 0);
    }
    state->_imu->fej = state->_imu->value;
  }

  // Propagator.cpp:37-126; returns Phi_summed / Qd_summed for stage-level parity tests
  // Propagator.cpp:128-224: IMU-rate prediction of (q, p, v_local, w) and of the 12x12 pose/velocity covariance on a COPY of the IMU
  // marginal; the state is not touched.  Zero-order quaternion, constant-acceleration discrete model with averaged measurements.
  bool fast_state_propagate(StateP state, double timestamp, Mat &state_plus, Mat &covariance) {
    Mat est = state->_imu->vecvalue();                                        // 16 x 1 (:133)
    Mat cov = StateHelper::get_marginal_covariance(state, {state->_imu});    // 15 x 15 (:134)
    const double t_off = state->_calib_dt_CAMtoIMU->value[0];
    std::vector<ImuData> prop = select_imu_readings(imu_data, state->_timestamp + t_off, timestamp + t_off);
    if (prop.size() < 2)
      return false; // (:147-148)
    const Mat bg = est.block(10, 0, 3, 1), ba = est.block(13, 0, 3, 1);
    for (size_t i = 0; i + 1 < prop.size(); i++) {
      const double dt = prop[i + 1].timestamp - prop[i].timestamp;
      const Mat w_hat = 0.5 * (prop[i + 1].wm + prop[i].wm) - bg, a_hat = 0.5 * (prop[i + 1].am + prop[i].am) - ba; // (:160-161)
      const Mat R = quat_2_Rot(est.block(0, 0, 4, 1)), RT = R.T();
      const Mat v = est.block(7, 0, 3, 1), pp = est.block(4, 0, 3, 1);
      const Mat E = exp_so3((-dt) * w_hat), EJ = (-dt) * (E * Jr_so3((-dt) * w_hat));
      Mat F(15, 15), G(15, 12);
      F.setBlock(0, 0, E);                                   // (:169-181)
      F.setBlock(0, 9, EJ);
      F.setBlock(9, 9, Mat::Identity(3));
      F.setBlock(6, 0, (-1.0) * (RT * skew_x(dt * a_hat)));
      F.setBlock(6, 6, Mat::Identity(3));
      F.setBlock(6, 12, (-dt) * RT);
      F.setBlock(12, 12, Mat::Identity(3));
      F.setBlock(3, 0, (-0.5) * (RT * skew_x((dt * dt) * a_hat)));
      F.setBlock(3, 6, dt * Mat::Identity(3));
      F.setBlock(3, 12, (-0.5 * dt * dt) * RT);
      F.setBlock(3, 3, Mat::Identity(3));
      G.setBlock(0, 0, EJ);                                  // (:182-187)
      G.setBlock(6, 3, (-dt) * RT);
      G.setBlock(3, 3, (-0.5 * dt * dt) * RT);
      G.setBlock(9, 6, Mat::Identity(3));
      G.setBlock(12, 9, Mat::Identity(3));
      Mat Qc(12, 12);                                        // (:192-196)
      for (int k = 0; k < 3; k++) {
        Qc(k, k) = _noises.sigma_w_2() / dt;
        Qc(3 + k, 3 + k) = _noises.sigma_a_2() / dt;
        Qc(6 + k, 6 + k) = _noises.sigma_wb_2() * dt;
        Qc(9 + k, 9 + k) = _noises.sigma_ab_2() * dt;
      }
      Mat Qd = G * Qc * G.T();
      Qd = 0.5 * (Qd + Qd.T());
      cov = F * cov * F.T() + Qd;                            // (:199)
      est.setBlock(0, 0, rot_2_quat(E * R));                 // (:202-204)
      est.setBlock(4, 0, pp + dt * v + (0.5 * dt * dt) * (RT * a_hat) - (0.5 * dt * dt) * _gravity);
      est.setBlock(7, 0, v + dt * (RT * a_hat) - dt * _gravity);
    }
    const Mat q = est.block(0, 0, 4, 1);
    state_plus = Mat(13, 1);                                 // (:208-215)
    state_plus.setBlock(0, 0, q);
    state_plus.setBlock(4, 0, est.block(4, 0, 3, 1));
    state_plus.setBlock(7, 0, quat_2_Rot(q) * est.block(7, 0, 3, 1));
    const size_t n = prop.size();
    state_plus.setBlock(10, 0, 0.5 * (prop[n - 1].wm + prop[n - 2].wm) - bg);
    Mat Phi = Mat::Identity(15);                             // (:220-226)
    Phi.setBlock(6, 6, quat_2_Rot(q));
    cov = Phi * cov * Phi.T();
    covariance = Mat(12, 12);
    covariance.setBlock(0, 0, cov.block(0, 0, 9, 9));
    const double dtl = prop[n - 1].timestamp - prop[n - 2].timestamp;
    for (int k = 0; k < 3; k++)
      covariance(9 + k, 9 + k) = _noises.sigma_w_2() / dtl;
    return true;
  }

  void propagate_and_clone(StateP state, double timestamp, Mat *Phi_out = nullptr, Mat *Qd_out = nullptr) {
    if (state->_timestamp == timestamp)
      ref_exit("propagate_and_clone: same timestep");
    if (state->_timestamp > timestamp)
      ref_exit("propagate_and_clone: backwards in time");
    if (!have_last_prop_time_offset) {
      last_prop_time_offset = state->_calib_dt_CAMtoIMU->value[0];
      have_last_prop_time_offset = true;
    }
    double t_off_new = state->_calib_dt_CAMtoIMU->value[0];
    double time0 = state->_timestamp + last_prop_time_offset;
    double time1 = timestamp + t_off_new;
    std::vector<ImuData> prop_data = select_imu_readings(imu_data, time0, time1);
    Mat Phi_summed = Mat::Identity(15);
    Mat Qd_summed(15, 15);
    if (prop_data.size() > 1) {
      for (size_t i = 0; i + 1 < prop_data.size(); i++) {
        Mat F, Qdi;
        predict_and_compute(state, prop_data.at(i), prop_data.at(i + 1), F, Qdi);
        Phi_summed = F * Phi_summed;
        Qd_summed = F * Qd_summed * F.T() + Qdi;
        Qd_summed = 0.5 * (Qd_summed + Qd_summed.T());
      }
    }
    Mat last_w(3, 1);
    if (prop_data.size() > 1)
      last_w = prop_data.at(prop_data.size() - 2).wm - state->_imu->bias_g();
    else if (!prop_data.empty())
      last_w = prop_data.at(prop_data.size() - 1).wm - state->_imu->bias_g();
    std::vector<VarP> Phi_order = {state->_imu};
    StateHelper::EKFPropagation(state, Phi_order, Phi_order, Phi_summed, Qd_summed);
    state->_timestamp = timestamp;
    last_prop_time_offset = t_off_new;
    StateHelper::augment_clone(state, last_w);
    if (Phi_out)
      *Phi_out = Phi_summed;
    if (Qd_out)
      *Qd_out = Qd_summed;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// UpdaterZeroVelocity::try_update (update/UpdaterZeroVelocity.cpp:68-318) with the flags the reference hard-codes
// (:113-116: integrated_accel_constraint = false, model_time_varying_bias = true, override_with_disparity_check = true,
// explicitly_enforce_zero_motion = false).  FeatureHelper::compute_disparity (ov_core, front end) is upstream: its outputs
// arrive as inputs.  H_order is {q, bg, ba} of the IMU (:119-121); the oracle's Var has no sub-variables, so H is laid out
// over the whole IMU variable (15 columns, zeros for p and v) - the zero columns add exact zeros to every product of
// EKFUpdate.  The bias propagation EKFPropagation({bg, ba}, {bg, ba}, I, Q_bias) (:253-259) with Phi = I changes exactly
// the six diagonal entries P_ii += Q_ii (StateHelper.cpp:85-105: C = P[:, new] I, D = Q + I C[new rows]).
// ---------------------------------------------------------------------------------------------------------------
struct UpdaterZeroVelocity {
  NoiseManager _noises;
  Mat _gravity = vec3(0, 0, 9.81);
  double _zupt_max_velocity = 1.0, _zupt_noise_multiplier = 1.0, _zupt_max_disparity = 1.0, chi2_multipler = 1.0;
  std::vector<ImuData> imu_data;
  double last_prop_time_offset = 0.0;
  bool have_last_prop_time_offset = false;
  double last_zupt_state_timestamp = 0.0;
  double last_chi2 = 0.0;

  bool try_update(StateP state, double timestamp, double average_disparity, int num_features, const Chi2Table &chi2tab) {
    if (imu_data.empty()) {
      last_zupt_state_timestamp = 0.0;
      return false;
    }
    if (state->_timestamp == timestamp) {
      last_zupt_state_timestamp = 0.0;
      return false;
    }
    const double dtv = state->_calib_dt_CAMtoIMU->value[0];
    if (!have_last_prop_time_offset) {
      last_prop_time_offset = dtv;
      have_last_prop_time_offset = true;
    }
    double t_off_new = dtv;
    double time0 = state->_timestamp + last_prop_time_offset;
    double time1 = timestamp + t_off_new;
    std::vector<ImuData> imu_recent = Propagator::select_imu_readings(imu_data, time0, time1);
    last_prop_time_offset = t_off_new;
    if (imu_recent.size() < 2) {
      last_zupt_state_timestamp = 0.0;
      return false;
    }
    VarP imu = state->_imu;
    int h_size = 15;
    int m_size = 6 * ((int)imu_recent.size() - 1);
    Mat H(m_size, h_size), res(m_size, 1);
    Mat R = Mat::Identity(m_size);
    double dt_summed = 0;
    for (size_t i = 0; i + 1 < imu_recent.size(); i++) {
      double dt = imu_recent.at(i + 1).timestamp - imu_recent.at(i).timestamp;
      Mat a_hat = imu_recent.at(i).am - imu->bias_a();
      Mat r_w = -1.0 * (imu_recent.at(i).wm - imu->bias_g());
      Mat r_a = -1.0 * (a_hat - imu->Rot() * _gravity);
      for (int j = 0; j < 3; j++) {
        res((int)(6 * i) + j, 0) = r_w(j, 0);
        res((int)(6 * i) + 3 + j, 0) = r_a(j, 0);
      }
      Mat R_GtoI_jacob = state->_options.do_fej ? imu->Rot_fej() : imu->Rot();
      Mat sk = -1.0 * skew_x(R_GtoI_jacob * _gravity);
      for (int j = 0; j < 3; j++) {
        H((int)(6 * i) + j, 9 + j) = -1.0; // d w / d bg   (:164; bg = IMU columns 9..11)
        for (int l = 0; l < 3; l++)
          H((int)(6 * i) + 3 + j, l) = sk(j, l); // d a / d theta (:166)
        H((int)(6 * i) + 3 + j, 12 + j) = -1.0;  // d a / d ba    (:167; ba = IMU columns 12..14)
      }
      for (int j = 0; j < 3; j++) {
        R((int)(6 * i) + j, (int)(6 * i) + j) *= _noises.sigma_w * _noises.sigma_w / dt;
        R((int)(6 * i) + 3 + j, (int)(6 * i) + 3 + j) *= _noises.sigma_a * _noises.sigma_a / dt;
      }
      dt_summed += dt;
    }
    R = _zupt_noise_multiplier * R;
    double Qb[6];
    for (int j = 0; j < 3; j++) {
      Qb[j] = dt_summed * _noises.sigma_wb; // the reference multiplies by sigma_wb / sigma_ab here, NOT by their squares (:186-187):
      Qb[3 + j] = dt_summed * _noises.sigma_ab; // a property of the reference that parity has to reproduce
    }
    std::vector<VarP> Hx_order = {imu};
    Mat P_marg = StateHelper::get_marginal_covariance(state, Hx_order);
    for (int j = 0; j < 6; j++)
      P_marg(9 + j, 9 + j) += Qb[j];
    Mat S = H * P_marg * H.T() + R;
    Mat L;
    if (!chol_lower(S, L))
      ref_exit("UpdaterZeroVelocity: S not positive definite");
    Mat y = res;
    chol_solve_inplace(L, y);
    double chi2 = dot(res, y);
    last_chi2 = chi2;
    double chi2_check = chi2tab.at(res.rows());
    bool disparity_passed = (average_disparity < _zupt_max_disparity && num_features > 20); // :219
    if (!disparity_passed && (chi2 > chi2_multipler * chi2_check || imu->vel().norm() > _zupt_max_velocity)) {
      last_zupt_state_timestamp = 0.0;
      return false;
    }
    // accepted: propagate the biases (Phi = I, see the header comment), then update with the IMU measurements
    const int ib = imu->id + 9;
    for (int j = 0; j < 6; j++) {
      state->_Cov(ib + j, ib + j) += Qb[j];
      if (state->_Cov(ib + j, ib + j) < 0.0)
        ref_exit("EKFPropagation: negative diagonal");
    }
    StateHelper::EKFUpdate(state, Hx_order, H, res, R);
    state->_timestamp = timestamp;
    last_zupt_state_timestamp = timestamp;
    return true;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// ov_core::FeatureInitializer::single_triangulation + single_gaussnewton (OpenVINS @74a63cf, NOT under /root/reference:
// restated from the published algorithm; call sites UpdaterMSCKF.cpp:142-194, UpdaterSLAM.cpp:118-160).  Dense Mat arithmetic,
// inverse by cofactors, extreme singular values by cyclic Jacobi - deliberately different numerics from the CUDA path's
// closed forms (parity unpinned by the reference: this checks the restatement against itself in two formulations).
// ---------------------------------------------------------------------------------------------------------------
struct FeatureInitializerOptions {
  int max_runs = 5;
  double init_lamda = 1e-3, max_lamda = 1e10, min_dx = 1e-6, min_dcost = 1e-6, lam_mult = 10, min_dist = 0.10, max_dist = 60, max_baseline = 40,
         max_cond_number = 10000;
};
struct FeatureInitializer {
  FeatureInitializerOptions _options;
  struct ClonePose {
    Mat R, p;
  };
  static void sym_eig_minmax(Mat A, double &emin, double &emax) { // cyclic Jacobi on a symmetric 3x3
    for (int sweep = 0; sweep < 30; sweep++)
      for (int p = 0; p < 3; p++)
        for (int q = p + 1; q < 3; q++) {
          if (std::abs(A(p, q)) < 1e-300)
            continue;
          double th = 0.5 * std::atan2(2 * A(p, q), A(q, q) - A(p, p));
          double c = std::cos(th), s = std::sin(th);
          Mat J = Mat::Identity(3);
          J(p, p) = c;
          J(q, q) = c;
          J(p, q) = s;
          J(q, p) = -s;
          A = J.T() * A * J;
        }
    emin = std::min(A(0, 0), std::min(A(1, 1), A(2, 2)));
    emax = std::max(A(0, 0), std::max(A(1, 1), A(2, 2)));
  }
  double compute_error(const std::vector<ClonePose> &cams, const std::vector<float> &uvn, double alpha, double beta, double rho) const {
    double err = 0;
    const Mat &R_GtoA = cams.back().R;
    const Mat &p_AinG = cams.back().p;
    for (size_t m = 0; m < cams.size(); m++) {
      Mat R_AtoCi = cams[m].R * R_GtoA.T();
      Mat p_CiinA = R_GtoA * (cams[m].p - p_AinG);
      Mat p_AinCi = -1.0 * (R_AtoCi * p_CiinA);
      double hi1 = R_AtoCi(0, 0) * alpha + R_AtoCi(0, 1) * beta + R_AtoCi(0, 2) + rho * p_AinCi(0, 0);
      double hi2 = R_AtoCi(1, 0) * alpha + R_AtoCi(1, 1) * beta + R_AtoCi(1, 2) + rho * p_AinCi(1, 0);
      double hi3 = R_AtoCi(2, 0) * alpha + R_AtoCi(2, 1) * beta + R_AtoCi(2, 2) + rho * p_AinCi(2, 0);
      float z0 = (float)(hi1 / hi3), z1 = (float)(hi2 / hi3);
      float r0 = uvn[2 * m] - z0, r1 = uvn[2 * m + 1] - z1;
      float n = std::sqrt(r0 * r0 + r1 * r1);
      err += std::pow(n, 2);
    }
    return err;
  }
  bool triangulate_and_refine(const std::vector<ClonePose> &cams, const std::vector<float> &uvn, Mat &p_FinG) const {
    const Mat &R_GtoA = cams.back().R;
    const Mat &p_AinG = cams.back().p;
    Mat A(3, 3), b(3, 1);
    for (size_t m = 0; m < cams.size(); m++) {
      Mat R_AtoCi = cams[m].R * R_GtoA.T();
      Mat p_CiinA = R_GtoA * (cams[m].p - p_AinG);
      Mat b_i = R_AtoCi.T() * vec3(uvn[2 * m], uvn[2 * m + 1], 1.0);
      b_i = (1.0 / b_i.norm()) * b_i;
      Mat Bperp = skew_x(b_i);
      Mat Ai = Bperp.T() * Bperp;
      A = A + Ai;
      b = b + Ai * p_CiinA;
    }
    Mat p_f = inverse_small(A) * b;
    double emin, emax;
    sym_eig_minmax(A, emin, emax);
    double condA = emax / emin;
    if (std::abs(condA) > _options.max_cond_number || p_f(2, 0) < _options.min_dist || p_f(2, 0) > _options.max_dist || std::isnan(p_f.norm()))
      return false;
    double rho = 1 / p_f(2, 0), alpha = p_f(0, 0) / p_f(2, 0), beta = p_f(1, 0) / p_f(2, 0);
    double lam = _options.init_lamda, eps = 10000;
    int runs = 0;
    bool recompute = true;
    double cost_old = compute_error(cams, uvn, alpha, beta, rho);
    Mat Hess(3, 3), grad(3, 1);
    while (runs < _options.max_runs && lam < _options.max_lamda && eps > _options.min_dx) {
      if (recompute) {
        Hess = Mat(3, 3);
        grad = Mat(3, 1);
        for (size_t m = 0; m < cams.size(); m++) {
          Mat R_AtoCi = cams[m].R * R_GtoA.T();
          Mat p_CiinA = R_GtoA * (cams[m].p - p_AinG);
          Mat p_AinCi = -1.0 * (R_AtoCi * p_CiinA);
          double hi1 = R_AtoCi(0, 0) * alpha + R_AtoCi(0, 1) * beta + R_AtoCi(0, 2) + rho * p_AinCi(0, 0);
          double hi2 = R_AtoCi(1, 0) * alpha + R_AtoCi(1, 1) * beta + R_AtoCi(1, 2) + rho * p_AinCi(1, 0);
          double hi3 = R_AtoCi(2, 0) * alpha + R_AtoCi(2, 1) * beta + R_AtoCi(2, 2) + rho * p_AinCi(2, 0);
          Mat H(2, 3);
          H(0, 0) = (R_AtoCi(0, 0) * hi3 - hi1 * R_AtoCi(2, 0)) / (std::pow(hi3, 2));
          H(0, 1) = (R_AtoCi(0, 1) * hi3 - hi1 * R_AtoCi(2, 1)) / (std::pow(hi3, 2));
          H(0, 2) = (p_AinCi(0, 0) * hi3 - hi1 * p_AinCi(2, 0)) / (std::pow(hi3, 2));
          H(1, 0) = (R_AtoCi(1, 0) * hi3 - hi2 * R_AtoCi(2, 0)) / (std::pow(hi3, 2));
          H(1, 1) = (R_AtoCi(1, 1) * hi3 - hi2 * R_AtoCi(2, 1)) / (std::pow(hi3, 2));
          H(1, 2) = (p_AinCi(1, 0) * hi3 - hi2 * p_AinCi(2, 0)) / (std::pow(hi3, 2));
          float z0 = (float)(hi1 / hi3), z1 = (float)(hi2 / hi3);
          Mat res(2, 1);
          res(0, 0) = (double)(uvn[2 * m] - z0);
          res(1, 0) = (double)(uvn[2 * m + 1] - z1);
          grad = grad + H.T() * res;
          Hess = Hess + H.T() * H;
        }
      }
      Mat Hess_l = Hess;
      for (int r = 0; r < 3; r++)
        Hess_l(r, r) *= (1.0 + lam);
      Mat dx = inverse_small(Hess_l) * grad;
      double cost = compute_error(cams, uvn, alpha + dx(0, 0), beta + dx(1, 0), rho + dx(2, 0));
      if (cost <= cost_old && (cost_old - cost) / cost_old < _options.min_dcost) {
        alpha += dx(0, 0);
        beta += dx(1, 0);
        rho += dx(2, 0);
        eps = 0;
        break;
      }
      if (cost <= cost_old) {
        recompute = true;
        cost_old = cost;
        alpha += dx(0, 0);
        beta += dx(1, 0);
        rho += dx(2, 0);
        runs++;
        lam = lam / _options.lam_mult;
        eps = dx.norm();
      } else {
        recompute = false;
        lam = lam * _options.lam_mult;
        continue;
      }
    }
    Mat p_FinA = vec3(alpha / rho, beta / rho, 1 / rho);
    // tangent plane of the bearing: the two directions orthogonal to p_FinA (ov_core takes them from a Householder QR of p_FinA)
    Mat n = (1.0 / p_FinA.norm()) * p_FinA;
    Mat t1 = (std::abs(n(0, 0)) < 0.9) ? vec3(1, 0, 0) : vec3(0, 1, 0);
    t1 = t1 - dot(t1, n) * n;
    t1 = (1.0 / t1.norm()) * t1;
    Mat t2 = skew_x(n) * t1;
    double base_line_max = 0.0;
    for (size_t m = 0; m < cams.size(); m++) {
      Mat p_CiinA = R_GtoA * (cams[m].p - p_AinG);
      double base_line = std::sqrt(std::pow(dot(t1, p_CiinA), 2) + std::pow(dot(t2, p_CiinA), 2));
      if (base_line > base_line_max)
        base_line_max = base_line;
    }
    if (p_FinA(2, 0) < _options.min_dist || p_FinA(2, 0) > _options.max_dist || (p_FinA.norm() / base_line_max) > _options.max_baseline ||
        std::isnan(p_FinA.norm()))
      return false;
    p_FinG = R_GtoA.T() * p_FinA + p_AinG;
    return true;
  }
};

} // namespace orc

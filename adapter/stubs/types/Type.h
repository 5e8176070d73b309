// MINIMAL STAND-IN for OpenVINS ov_core types/{Type,Vec,JPLQuat,PoseJPL,IMU,Landmark}.h (syntax check of adapter/*.cpp only).
#pragma once
#include <Eigen/Dense>
#include <memory>
namespace ov_type {
class Type {
public:
  explicit Type(int size) : _size(size) {}
  virtual ~Type() {}
  virtual void set_local_id(int new_id) { _id = new_id; }
  int id() { return _id; }
  int size() { return _size; }
  virtual const Eigen::MatrixXd &value() const { return _value; }
  virtual const Eigen::MatrixXd &fej() const { return _fej; }
  virtual void set_value(const Eigen::MatrixXd &new_value) { _value = new_value; }
  virtual void set_fej(const Eigen::MatrixXd &new_value) { _fej = new_value; }

protected:
  Eigen::MatrixXd _value, _fej;
  int _id = -1, _size = -1;
};
class Vec : public Type {
public:
  explicit Vec(int dim) : Type(dim) {}
};
class JPLQuat : public Type {
public:
  JPLQuat() : Type(3) {}
};
class PoseJPL : public Type {
public:
  PoseJPL() : Type(6) {}
};
class IMU : public Type {
public:
  IMU() : Type(15) {}
  std::shared_ptr<PoseJPL> pose() { return _pose; }

private:
  std::shared_ptr<PoseJPL> _pose;
};
class LandmarkRepresentation { // types/LandmarkRepresentation.h
public:
  enum Representation {
    GLOBAL_3D,
    GLOBAL_FULL_INVERSE_DEPTH,
    ANCHORED_3D,
    ANCHORED_FULL_INVERSE_DEPTH,
    ANCHORED_MSCKF_INVERSE_DEPTH,
    ANCHORED_INVERSE_DEPTH_SINGLE,
    UNKNOWN
  };
  static bool is_relative_representation(Representation feat_representation) {
    return feat_representation == ANCHORED_3D || feat_representation == ANCHORED_FULL_INVERSE_DEPTH ||
           feat_representation == ANCHORED_MSCKF_INVERSE_DEPTH || feat_representation == ANCHORED_INVERSE_DEPTH_SINGLE;
  }
};
class Landmark : public Vec {
public:
  explicit Landmark(int dim) : Vec(dim) {}
  size_t _featid = 0;
  int _unique_camera_id = -1;
  int _anchor_cam_id = -1;
  double _anchor_clone_timestamp = -1;
  bool should_marg = false;
  LandmarkRepresentation::Representation _feat_representation = LandmarkRepresentation::UNKNOWN;
  Eigen::Vector3d uv_norm_zero;     // ANCHORED_INVERSE_DEPTH_SINGLE: the bearing rho p_FinA it was set from
  Eigen::Vector3d uv_norm_zero_fej; // and its first-estimate copy
};
} // namespace ov_type

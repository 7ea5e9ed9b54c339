// imu_process_facade.hpp — flb::ImuProcessGpu, a stand-in for ImuProcess (src/IMU_Processing.hpp) with the same setters
// and call shape, running on a front end (flb_frontend, see scan_frontend_facade.hpp):
//
//   flb::ImuProcessGpu p_imu;                    // next to `shared_ptr<ImuProcess> p_imu` (laserMapping.cpp)
//   p_imu.set_extrinsic(Lidar_T_wrt_IMU, Lidar_R_wrt_IMU);   p_imu.set_gyr_cov(...); ... (laserMapping.cpp:2142-2146)
//   p_imu.attach(fe.handle(), filter_size_surf_min);         // once, after the setters
//   ... per scan, after the raw scan is on the front end (flb_frontend_preprocess / flb_frontend_upload):
//   p_imu.Process(Measures, kf, feats_undistort);            // laserMapping.cpp:2256
//
// Process runs IMU_init on the host and, once initialised, the forward propagation, the undistortion and the voxel
// filter on the device in one call (flb_imu_process): kf's state and covariance become the prior, and feats_down_body
// is left on the device as the session's current scan.  The undistorted cloud stays on the device as well;
// pcl_un_ is not written (flb_frontend_download_undistorted reads it); scan_ready() replaces the reference's
// `feats_undistort->empty()` test.  Only member names of the reference types are used: meas.imu (a sequence of
// pointers with header.stamp.toSec(), linear_acceleration, angular_velocity), meas.lidar_beg_time / lidar_end_time,
// kf.get_x / change_x / get_P / change_P, and the state_ikfom members (pack_state26 / unpack_state26).
#pragma once
#include <cstdio>
#include <vector>

#include "../fastlio_b200.h"
#include "lio_gpu_frontend.hpp"

namespace flb {

class ImuProcessGpu {
 public:
  ImuProcessGpu() { flb_imu_default_config(&cfg_); }
  ~ImuProcessGpu() { if (imu_) flb_imu_destroy(imu_); }
  ImuProcessGpu(const ImuProcessGpu&) = delete;
  ImuProcessGpu& operator=(const ImuProcessGpu&) = delete;

  // set_extrinsic(MD(4,4)) / (V3D) / (V3D, M3D) (:108-132)
  template <class M4>
  void set_extrinsic(const M4& T) {
    for (int i = 0; i < 3; ++i) {
      cfg_.Lidar_T_wrt_IMU[i] = T(i, 3);
      for (int j = 0; j < 3; ++j) cfg_.Lidar_R_wrt_IMU[3 * i + j] = T(i, j);
    }
  }
  template <class V3>
  void set_extrinsic_T(const V3& t) {
    for (int i = 0; i < 3; ++i) {
      cfg_.Lidar_T_wrt_IMU[i] = t[i];
      for (int j = 0; j < 3; ++j) cfg_.Lidar_R_wrt_IMU[3 * i + j] = i == j ? 1.0 : 0.0;
    }
  }
  template <class V3, class M3>
  void set_extrinsic(const V3& t, const M3& R) {
    for (int i = 0; i < 3; ++i) {
      cfg_.Lidar_T_wrt_IMU[i] = t[i];
      for (int j = 0; j < 3; ++j) cfg_.Lidar_R_wrt_IMU[3 * i + j] = R(i, j);
    }
  }
  template <class V3> void set_gyr_cov(const V3& v) { for (int i = 0; i < 3; ++i) cfg_.cov_gyr_scale[i] = v[i]; }
  template <class V3> void set_acc_cov(const V3& v) { for (int i = 0; i < 3; ++i) cfg_.cov_acc_scale[i] = v[i]; }
  template <class V3> void set_gyr_bias_cov(const V3& v) { for (int i = 0; i < 3; ++i) cfg_.cov_bias_gyr[i] = v[i]; }
  template <class V3> void set_acc_bias_cov(const V3& v) { for (int i = 0; i < 3; ++i) cfg_.cov_bias_acc[i] = v[i]; }

  // The propagation runs on `fe` (the setters above must come first); leaf > 0 also runs the voxel filter
  // (downSizeFilterSurf, laserMapping.cpp:2322-2323).  Destroy this object before the front end.
  bool attach(flb_frontend* fe, float leaf) {
    leaf_ = leaf;
    if (imu_) { flb_imu_destroy(imu_); imu_ = nullptr; }
    if (flb_imu_create(fe, &cfg_, &imu_)) { std::fprintf(stderr, "[fastlio_b200] %s\n", flb_last_error()); imu_ = nullptr; return false; }
    return true;
  }

  void Reset() { if (imu_) flb_imu_reset(imu_); }

  template <class Meas, class KF, class Cloud>
  void Process(const Meas& meas, KF& kf, Cloud& /*pcl_un_*/) {
    last_ = flb_imu_result{};
    if (!imu_) { std::fprintf(stderr, "[fastlio_b200] ImuProcessGpu::Process before attach\n"); return; }
    imu7_.clear();
    for (const auto& m : meas.imu) {
      const double r[7] = {m->header.stamp.toSec(), m->linear_acceleration.x, m->linear_acceleration.y, m->linear_acceleration.z,
                           m->angular_velocity.x, m->angular_velocity.y, m->angular_velocity.z};
      imu7_.insert(imu7_.end(), r, r + 7);
    }
    auto x = kf.get_x();
    auto P = kf.get_P();
    double st[FLB_STATE_DIM];
    double Pm[FLB_STATE_DOF * FLB_STATE_DOF];
    pack_state26(x, st);
    for (int i = 0; i < FLB_STATE_DOF; ++i)
      for (int j = 0; j < FLB_STATE_DOF; ++j) Pm[i * FLB_STATE_DOF + j] = P(i, j);
    if (flb_imu_process(imu_, imu7_.empty() ? nullptr : imu7_.data(), (int)(imu7_.size() / 7), meas.lidar_beg_time, meas.lidar_end_time,
                        st, Pm, leaf_, &last_)) {
      std::fprintf(stderr, "[fastlio_b200] ImuProcessGpu::Process: %s\n", flb_last_error());
      last_ = flb_imu_result{};
      return;
    }
    if (last_.status == FLB_IMU_EMPTY) return;
    unpack_state26(st, x);
    for (int i = 0; i < FLB_STATE_DOF; ++i)
      for (int j = 0; j < FLB_STATE_DOF; ++j) P(i, j) = Pm[i * FLB_STATE_DOF + j];
    kf.change_x(x);
    kf.change_P(P);
  }

  bool scan_ready() const { return last_.status == FLB_IMU_PROPAGATED; }   // feats_undistort is not empty
  int feats_down_size() const { return last_.n_down; }
  const flb_imu_result& last_result() const { return last_; }
  // IMUpose of the last propagation (Pose6D records of 22 doubles)
  int imu_poses(std::vector<double>& out22) {
    int n = 0;
    if (flb_imu_download_poses(imu_, nullptr, 0, &n)) return -1;
    out22.assign((size_t)n * FLB_IMU_POSE_DOUBLES, 0.0);
    if (flb_imu_download_poses(imu_, out22.data(), n, &n)) return -1;
    return n;
  }
  flb_imu* handle() { return imu_; }

 private:
  flb_imu_config cfg_{};
  flb_imu* imu_ = nullptr;
  float leaf_ = 0.f;
  flb_imu_result last_{};
  std::vector<double> imu7_;
};

}  // namespace flb

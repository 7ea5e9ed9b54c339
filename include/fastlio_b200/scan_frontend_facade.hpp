// scan_frontend_facade.hpp — drop-in C++ shapes for the two steps immediately before the per-scan update, so that the raw
// scan stays on the GPU from the driver callback to the posterior (SURVEY.md §8f ranks 1, 2 and 4):
//
//   * flb::ScanFrontEnd::undistort(...)  replaces the per-point backward pass of ImuProcess::UndistortPcl
//     (src/IMU_Processing.hpp:243 sort, :334-386); the forward propagation (:260-329, kf_state.predict per IMU sample)
//     stays where it is and hands over its IMUpose vector and imu_state;
//   * flb::VoxelGridGpu<PointT>          keeps the pcl::VoxelGrid call shape used at src/laserMapping.cpp:2135 and
//     :2322-2323:   downSizeFilterSurf.setLeafSize(l, l, l);  .setInputCloud(feats_undistort);  .filter(*feats_down_body);
//     its result is ALSO the session's current scan, so LioGpu::begin_scan (the upload) is no longer needed;
//   * flb::ScanFrontEnd::to_world(...)   replaces the RGBpointBodyToWorld loops of publish_frame_world
//     (src/laserMapping.cpp:1502-1540);
//   * flb::ScanFrontEnd::set_camera / upload_image / colorize replace paramSetting, imageCallback and the loops of
//     publish_frame_world_color (src/laserMapping.cpp:250-392); to_imu(...) replaces the loop of publish_frame_body
//     (:1543-1558);
//   * flb::ScanFrontEnd::preprocess(...) replaces Preprocess::process (src/preprocess.cpp, feature extraction off) for a
//     sensor_msgs::PointCloud2 (Velodyne, Ouster) or livox_ros_driver::CustomMsg: the driver message is uploaded once
//     and its preprocessed cloud stays on the device as the current scan, which undistort(poses, imu_state) then uses.
//
//   flb::ScanFrontEnd fe;  fe.attach(gpu.handle(), 300000);        // next to `flb::LioGpu gpu;`
//   // in ImuProcess::UndistortPcl, instead of lines 334-386:
//   fe.undistort(*meas.lidar, IMUpose, imu_state, pcl_out);        // pcl_out = time-sorted, compensated cloud
//   // in main(), instead of lines 2322-2323:
//   flb::VoxelGridGpu<PointType> downSizeFilterSurf(&fe);  ...  downSizeFilterSurf.filter(*feats_down_body);
//
// Only member names of the reference types are needed (Pose6D: offset_time, acc, gyr, vel, pos, rot —
// msg/Pose6D.msg; pcl::PointCloud: points; PointType: x,y,z,intensity,curvature; PointCloud2: fields[].name/.offset,
// point_step, width, height, data; CustomMsg: point_num, points[] with offset_time, x,y,z, reflectivity, tag, line;
// cv::Mat: rows, cols, step[0], data; livox_ros::Point: x,y,z, intensity, b,g,r,a), so the header compiles without
// ROS/PCL/OpenCV.
#pragma once
#include <cstddef>
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

#include "../fastlio_b200.h"
#include "lio_gpu_frontend.hpp"

namespace flb {

class ScanFrontEnd {
 public:
  ~ScanFrontEnd() { if (fe_) flb_frontend_destroy(fe_); }
  bool attach(flb_session* ses, int max_raw_points) {
    if (flb_frontend_create(ses, max_raw_points, &fe_)) { std::fprintf(stderr, "[fastlio_b200] %s\n", flb_last_error()); fe_ = nullptr; return false; }
    cap_ = max_raw_points;
    return true;
  }
  flb_frontend* handle() { return fe_; }

  // meas.lidar -> device (IMU_Processing.hpp:242 "pcl_out = *(meas.lidar)")
  template <class Cloud>
  bool upload(const Cloud& cloud) {
    typedef typename std::remove_reference<decltype(cloud.points[0])>::type P;
    const int n = (int)cloud.points.size();
    const P* p0 = n ? &cloud.points[0] : nullptr;
    const int off_i = n ? (int)((const char*)&p0->intensity - (const char*)p0) : -1;
    const int off_c = n ? (int)((const char*)&p0->curvature - (const char*)p0) : -1;
    return ok(flb_frontend_upload(fe_, p0, n, (int)sizeof(P), off_i, off_c), "upload");
  }

  // The backward pass of UndistortPcl.  poses = IMUpose (vector<Pose6D>), imu_state = kf_state.get_x() after the last
  // predict.  When `out` is given it receives the time-sorted compensated cloud (x,y,z,intensity,curvature), i.e. pcl_out.
  template <class Cloud, class PoseVec, class State>
  bool undistort(const Cloud& lidar, const PoseVec& poses, const State& imu_state, Cloud* out = nullptr) {
    if (!upload(lidar) || !undistort(poses, imu_state)) return false;
    return !out || download_undistorted(*out);
  }

  // The backward pass of UndistortPcl on the scan the front end already holds (the output of preprocess()).
  template <class PoseVec, class State>
  bool undistort(const PoseVec& poses, const State& imu_state) {
    std::vector<double> pz(poses.size() * FLB_IMU_POSE_DOUBLES);
    for (size_t k = 0; k < poses.size(); ++k) {
      double* o = &pz[k * FLB_IMU_POSE_DOUBLES];
      o[0] = poses[k].offset_time;
      for (int i = 0; i < 3; ++i) { o[1 + i] = poses[k].acc[i]; o[4 + i] = poses[k].gyr[i]; o[7 + i] = poses[k].vel[i]; o[10 + i] = poses[k].pos[i]; }
      for (int i = 0; i < 9; ++i) o[13 + i] = poses[k].rot[i];
    }
    double st[FLB_STATE_DIM];
    pack_state26(imu_state, st);
    return ok(flb_frontend_undistort(fe_, pz.data(), (int)poses.size(), st), "undistort");
  }

  // The front end's current raw scan (time-sorted and compensated after undistort), x,y,z,intensity,curvature: pcl_out.
  template <class Cloud>
  bool download_undistorted(Cloud& out) {
    int n = 0;
    if (!ok(flb_frontend_download_undistorted(fe_, nullptr, nullptr, nullptr, 0, &n), "download")) return false;
    xyzi_.resize((size_t)n * 4 + 4);
    curv_.resize(n + 1);
    int m = 0;
    if (!ok(flb_frontend_download_undistorted(fe_, xyzi_.data(), curv_.data(), nullptr, n, &m), "download")) return false;
    out.points.resize(m);
    for (int i = 0; i < m; ++i) fill(out.points[i], &xyzi_[4 * (size_t)i], curv_[i]);
    return true;
  }

  // Preprocess::process(const sensor_msgs::PointCloud2::ConstPtr&, ...) for VELO16 / OUST64 (cfg.lidar_type 2 / 3):
  // field offsets are found by name in msg.fields as pcl::fromROSMsg does (x, y, z, intensity, ring, and `time` for
  // Velodyne / `t` for Ouster; a missing field reads as 0).  Returns pl_surf.size() (or -1); *last_curvature =
  // pl_surf.points.back().curvature, the two values sync_packages needs (laserMapping.cpp:1374-1405).
  template <class PointCloud2>
  auto preprocess(const PointCloud2& msg, const flb_preprocess_config& cfg, float* last_curvature = nullptr)
      -> decltype((void)msg.point_step, (void)msg.fields, int()) {
    flb_raw_layout L;
    L.stride = (int)msg.point_step;
    L.off_x = L.off_y = L.off_z = L.off_intensity = L.off_time = L.off_ring = L.off_tag = L.off_line = -1;
    const char* time_name = cfg.lidar_type == 3 ? "t" : "time";
    for (const auto& f : msg.fields) {
      const char* nm = f.name.c_str();
      const int off = (int)f.offset;
      if (!std::strcmp(nm, "x")) L.off_x = off;
      else if (!std::strcmp(nm, "y")) L.off_y = off;
      else if (!std::strcmp(nm, "z")) L.off_z = off;
      else if (!std::strcmp(nm, "intensity")) L.off_intensity = off;
      else if (!std::strcmp(nm, time_name)) L.off_time = off;
      else if (!std::strcmp(nm, "ring")) L.off_ring = off;
    }
    const int n = (int)((size_t)msg.width * msg.height);
    return run_preprocess(cfg, L, n ? (const void*)msg.data.data() : nullptr, n, last_curvature);
  }

  // Preprocess::process(const livox_ros_driver::CustomMsg::ConstPtr&, ...) for LIVOX (cfg.lidar_type 1).
  template <class CustomMsg>
  auto preprocess(const CustomMsg& msg, const flb_preprocess_config& cfg, float* last_curvature = nullptr)
      -> decltype((void)msg.point_num, (void)msg.points, int()) {
    typedef typename std::remove_reference<decltype(msg.points[0])>::type P;
    const int n = (int)std::min<size_t>((size_t)msg.point_num, msg.points.size());
    flb_raw_layout L;
    L.stride = (int)sizeof(P);
    const P probe = P();
    const char* b = (const char*)&probe;
    L.off_x = (int)((const char*)&probe.x - b);
    L.off_y = (int)((const char*)&probe.y - b);
    L.off_z = (int)((const char*)&probe.z - b);
    L.off_intensity = (int)((const char*)&probe.reflectivity - b);
    L.off_time = (int)((const char*)&probe.offset_time - b);
    L.off_ring = -1;
    L.off_tag = (int)((const char*)&probe.tag - b);
    L.off_line = (int)((const char*)&probe.line - b);
    return run_preprocess(cfg, L, n ? (const void*)&msg.points[0] : nullptr, n, last_curvature);
  }

  // downSizeFilterSurf.filter(*feats_down_body): leaves feats_down_body as the session's current scan; returns
  // feats_down_size (or -1).  `out` (optional) receives the centroids on the host as well.
  template <class Cloud>
  int voxel_filter(float leaf, Cloud* out) {
    int n = 0;
    if (!ok(flb_frontend_voxel_filter(fe_, leaf, &n), "voxel_filter")) return -1;
    if (out) {
      xyzi_.resize((size_t)n * 4 + 4);
      curv_.resize(n + 1);
      int m = 0;
      if (!ok(flb_frontend_download_down(fe_, xyzi_.data(), curv_.data(), n, &m), "download")) return -1;
      out->points.resize(n);
      for (int i = 0; i < n; ++i) fill(out->points[i], &xyzi_[4 * (size_t)i], curv_[i]);
    }
    return n;
  }

  // publish_frame_world (laserMapping.cpp:1506-1514, :1529-1536): dense = feats_undistort, else feats_down_body
  template <class State, class Cloud>
  bool to_world(const State& state_point, bool dense, Cloud& laserCloudWorld, int capacity) {
    double st[FLB_STATE_DIM];
    pack_state26(state_point, st);
    xyzi_.resize((size_t)capacity * 4 + 4);
    int n = 0;
    if (!ok(flb_frontend_points_to_world(fe_, dense ? 1 : 0, st, xyzi_.data(), capacity, &n), "to_world")) return false;
    if (n > capacity) n = capacity;
    laserCloudWorld.points.resize(n);
    for (int i = 0; i < n; ++i) fill(laserCloudWorld.points[i], &xyzi_[4 * (size_t)i], 0.f);
    return true;
  }

  // paramSetting (laserMapping.cpp:279-289): cam_ex = 16, cam_in = 12 row-major values (vector<double>, :2045-2046);
  // width x height bounds the image (the reference's Wmax x Hmax).  Zero-fills the device image.
  template <class VecEx, class VecIn>
  bool set_camera(const VecEx& cam_ex, const VecIn& cam_in, int width = 1280, int height = 720) {
    if (cam_ex.size() < 16 || cam_in.size() < 12) { std::fprintf(stderr, "[fastlio_b200] set_camera: cam_ex needs 16 and cam_in 12 values\n"); return false; }
    double ex[16], in[12];
    for (int k = 0; k < 16; ++k) ex[k] = cam_ex[k];
    for (int k = 0; k < 12; ++k) in[k] = cam_in[k];
    return ok(flb_frontend_camera_config(fe_, ex, in, width, height), "set_camera");
  }

  // imageCallback (:250-276): img = cv_bridge::toCvShare(msg, "bgr8")->image (members rows, cols, step[0], data)
  template <class Mat>
  bool upload_image(const Mat& img) {
    return ok(flb_frontend_camera_image(fe_, (const unsigned char*)img.data, (int)img.rows, (int)img.cols, (int)img.step[0]),
              "upload_image");
  }

  // The two loops of publish_frame_world_color (:323-381): colorCloud (pcl::PointCloud<livox_ros::Point>) receives the kept
  // points of feats_undistort (dense_pub_en) or feats_down_body in the world frame, x, y, z, intensity, b, g, r, a set by
  // member name and every other field zero.
  template <class State, class Cloud>
  bool colorize(const State& state_point, bool dense_pub_en, Cloud& colorCloud) {
    double st[FLB_STATE_DIM];
    pack_state26(state_point, st);
    xyzi_.resize((size_t)cap_ * 4 + 4);
    bgra_.resize((size_t)cap_ + 1);
    int n = 0;
    if (!ok(flb_frontend_points_colorize(fe_, dense_pub_en ? 1 : 0, st, xyzi_.data(), bgra_.data(), cap_, &n), "colorize")) return false;
    if (n > cap_) n = cap_;
    colorCloud.points.resize(n);
    for (int i = 0; i < n; ++i) {
      auto& p = colorCloud.points[i];
      typedef typename std::remove_reference<decltype(p)>::type P;
      p = P();
      const float* v = &xyzi_[4 * (size_t)i];
      const unsigned c = bgra_[i];
      p.x = v[0]; p.y = v[1]; p.z = v[2]; p.intensity = v[3];
      p.b = (unsigned char)(c & 0xFFu); p.g = (unsigned char)((c >> 8) & 0xFFu); p.r = (unsigned char)((c >> 16) & 0xFFu);
      p.a = (unsigned char)(c >> 24);
    }
    return true;
  }

  // publish_frame_body (:1543-1558): feats_undistort in the IMU frame (RGBpointBodyLidarToIMU), curvature 0
  template <class State, class Cloud>
  bool to_imu(const State& state_point, Cloud& laserCloudIMUBody) {
    double st[FLB_STATE_DIM];
    pack_state26(state_point, st);
    xyzi_.resize((size_t)cap_ * 4 + 4);
    int n = 0;
    if (!ok(flb_frontend_points_to_imu(fe_, st, xyzi_.data(), cap_, &n), "to_imu")) return false;
    if (n > cap_) n = cap_;
    laserCloudIMUBody.points.resize(n);
    for (int i = 0; i < n; ++i) fill(laserCloudIMUBody.points[i], &xyzi_[4 * (size_t)i], 0.f);
    return true;
  }

 private:
  int run_preprocess(const flb_preprocess_config& cfg, flb_raw_layout L, const void* rec, int n, float* last_curvature) {
    if (n == 0) L = flb_raw_layout{12, 0, 4, 8, -1, -1, -1, -1, -1};   // nothing to decode; the call still resets the scan
    int m = 0;
    float last = 0.f;
    if (!ok(flb_frontend_preprocess(fe_, &cfg, &L, rec, n, &m, &last), "preprocess")) return -1;
    if (last_curvature) *last_curvature = last;
    return m;
  }
  template <class P>
  static void fill(P& p, const float* v, float curvature) {
    p = P();
    p.x = v[0]; p.y = v[1]; p.z = v[2]; p.intensity = v[3]; p.curvature = curvature;
  }
  static bool ok(int rc, const char* what) {
    if (rc) std::fprintf(stderr, "[fastlio_b200] %s: %s\n", what, flb_last_error());
    return rc == 0;
  }
  flb_frontend* fe_ = nullptr;
  int cap_ = 0;   // max_raw_points: no cloud of the front end is larger
  std::vector<float> xyzi_, curv_;
  std::vector<unsigned> bgra_;
};

// pcl::VoxelGrid<PointT> call shape on top of a ScanFrontEnd.  setInputCloud() is accepted for source compatibility: the
// cloud that is filtered is the one the front end already holds on the device (the output of undistort(), or of an
// explicit ScanFrontEnd::upload() when the caller has no IMU step).
template <class PointT>
class VoxelGridGpu {
 public:
  explicit VoxelGridGpu(ScanFrontEnd* fe = nullptr) : fe_(fe) {}
  void attach(ScanFrontEnd* fe) { fe_ = fe; }
  void setLeafSize(float lx, float ly, float lz) {
    if (lx != ly || lx != lz) std::fprintf(stderr, "[fastlio_b200] VoxelGridGpu: anisotropic leaves are not supported (the reference never uses them)\n");
    leaf_ = lx;
  }
  template <class CloudPtr>
  void setInputCloud(const CloudPtr&) {}
  template <class Cloud>
  void filter(Cloud& output) {
    const int n = fe_ ? fe_->voxel_filter(leaf_, &output) : -1;
    if (n < 0) output.points.clear();
  }

 private:
  ScanFrontEnd* fe_;
  float leaf_ = 0.5f;
};

}  // namespace flb

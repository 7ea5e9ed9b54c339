// Compiles flb::ScanFrontEnd::preprocess against PointCloud2 / CustomMsg look-alikes (member names of
// sensor_msgs::PointCloud2 and livox_ros_driver::CustomMsg) and, when a GPU is present, runs driver message ->
// preprocess -> undistort(current scan) -> VoxelGrid -> h_share_model.
// Built by tests/test_oracle_preprocess.py with:
//   g++ -Ioracle/shim -Iinclude tests/cpp/preprocess_facade_smoke.cpp -Lbetter_fastlio2_b200 -lfastlio_b200
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include <fastlio_b200/ikd_tree_facade.hpp>
#include <fastlio_b200/lio_gpu_frontend.hpp>
#include <fastlio_b200/scan_frontend_facade.hpp>

typedef pcl::PointXYZINormal PointType;
typedef std::vector<PointType, Eigen::aligned_allocator<PointType>> PointVector;
struct PointCloudXYZI { PointVector points; };

struct Vec3 { double v[3]; double operator[](int i) const { return v[i]; } };
struct Quat { double c[4]; const double* coeffs() const { return c; } };
struct state_ikfom { Vec3 pos; Quat rot; Quat offset_R_L_I; Vec3 offset_T_L_I, vel, bg, ba, grav; };
struct MatX { std::vector<double> a; int r = 0, c = 0; void resize(int R, int C) { r = R; c = C; a.assign((size_t)R * C, 0.0); } double* data() { return a.data(); } int rows() const { return r; } };
struct VecX { std::vector<double> a; void resize(int n) { a.assign(n, 0.0); } double* data() { return a.data(); } };
struct dyn_share_datastruct { bool valid = true, converge = true; MatX h_x; VecX h; };
struct Pose6D { double offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9]; };

// sensor_msgs::PointField / PointCloud2 and livox_ros_driver::CustomPoint / CustomMsg look-alikes
struct PointField { std::string name; uint32_t offset; uint8_t datatype; uint32_t count; };
struct PointCloud2 { uint32_t height = 1, width = 0; std::vector<PointField> fields; bool is_bigendian = false; uint32_t point_step = 0, row_step = 0; std::vector<uint8_t> data; bool is_dense = true; };
struct CustomPoint { uint32_t offset_time; float x, y, z; uint8_t reflectivity, tag, line; };
struct CustomMsg { uint64_t timebase = 0; uint32_t point_num = 0; uint8_t lidar_id = 0; std::vector<CustomPoint> points; };

KD_TREE<PointType> ikdtree;
flb::LioGpu gpu;

int main() {
  // packed Velodyne cloud without per-point time: x y z intensity f32, ring u16 (point_step 18)
  PointCloud2 velo;
  velo.fields = {{"x", 0, 7, 1}, {"y", 4, 7, 1}, {"z", 8, 7, 1}, {"intensity", 12, 7, 1}, {"ring", 16, 4, 1}};
  velo.point_step = 18;
  const int rings = 16, cols = 900;
  std::mt19937 rng(3);
  std::uniform_real_distribution<float> U(-1.f, 1.f);
  PointVector map;
  for (int c = 0; c < cols; ++c)
    for (int r = 0; r < rings; ++r) {
      const float az = (float)(0.5 - c * 0.4) * 3.14159265f / 180.f, el = (-15.f + 2.f * r) * 3.14159265f / 180.f;
      // a square room of half-width 8 m, floor at -1.5 m
      const float dx = std::cos(el) * std::cos(az), dy = std::cos(el) * std::sin(az), dz = std::sin(el);
      float t = 8.f / std::fmax(std::fabs(dx), std::fabs(dy));
      if (dz < 0.f) t = std::fmin(t, -1.5f / dz);
      float rec[4] = {dx * t, dy * t, dz * t, (float)((c + r) % 200)};
      const uint16_t ring = (uint16_t)r;
      const size_t o = velo.data.size();
      velo.data.resize(o + 18);
      std::memcpy(&velo.data[o], rec, 16);
      std::memcpy(&velo.data[o + 16], &ring, 2);
      PointType p{};
      p.x = rec[0] + 0.01f * U(rng); p.y = rec[1] + 0.01f * U(rng); p.z = rec[2] + 0.01f * U(rng);
      map.push_back(p);
    }
  velo.width = rings * cols;
  CustomMsg livox;
  for (int i = 0; i < 2000; ++i) livox.points.push_back(CustomPoint{(uint32_t)(i * 50000), 5.f + U(rng), U(rng), U(rng), (uint8_t)(i % 256), (uint8_t)(i % 7 == 0 ? 0x20 : 0x00), (uint8_t)(i % 4)});
  livox.point_num = (uint32_t)livox.points.size();

  if (flb_device_count() <= 0) { std::printf("NO_GPU compile-only ok\n"); return 0; }
  ikdtree.set_capacity(1 << 20, 1 << 16);
  ikdtree.set_downsample_param(0.2f);
  ikdtree.Build(map);
  if (!gpu.attach(ikdtree.handle(), false, 3, 0.2)) return 2;
  flb::ScanFrontEnd fe;
  if (!fe.attach(gpu.handle(), 1 << 17)) return 3;

  flb_preprocess_config cfg{2, rings, 10, 1, 0, 1.0};   // VELO16, 16 rings, 10 Hz, every point, SEC, blind 1 m
  float last = -1.f;
  const int n = fe.preprocess(velo, cfg, &last);
  // every ring's first record is dropped; 900 columns x 0.4 deg = 360 deg: the last column sits just short of a wrap
  if (n != rings * (cols - 1)) { std::printf("velodyne size %d\n", n); return 4; }
  if (!(last > 90.f && last < 100.f)) { std::printf("velodyne last curvature %f\n", last); return 5; }
  state_ikfom s{};
  s.rot.c[3] = 1.0; s.offset_R_L_I.c[3] = 1.0; s.grav.v[2] = -9.809;
  std::vector<Pose6D> IMUpose(3);
  for (int k = 0; k < 3; ++k) {   // at rest: the compensation is the identity, only the time sort remains
    Pose6D q{};
    q.offset_time = 0.05 * k;
    q.rot[0] = q.rot[4] = q.rot[8] = 1.0;
    IMUpose[k] = q;
  }
  PointCloudXYZI und, down;
  if (!fe.undistort(IMUpose, s) || !fe.download_undistorted(und) || (int)und.points.size() != n) return 6;
  for (int i = 1; i < n; ++i)
    if (und.points[i].curvature < und.points[i - 1].curvature) return 7;
  if (und.points.back().curvature != last) return 8;   // the latest point of this sweep is its last record
  flb::VoxelGridGpu<PointType> ds(&fe);
  ds.setLeafSize(0.5f, 0.5f, 0.5f);
  ds.filter(down);
  if (down.points.size() < 100) return 9;
  dyn_share_datastruct d;
  gpu.h_share_model(s, d);
  if (!d.valid || gpu.effct_feat_num < 100) return 10;

  cfg = flb_preprocess_config{1, 4, 10, 1, 1, 0.5};   // LIVOX, 4 lines
  const int nl = fe.preprocess(livox, cfg, &last);
  int expect = 0;
  for (int i = 1; i < 2000; ++i) expect += (i % 7 != 0);
  if (nl != expect || last != (float)(1999 * 50000) / 1e6f) { std::printf("livox %d/%d %f\n", nl, expect, last); return 11; }
  CustomMsg empty;
  if (fe.preprocess(empty, cfg, &last) != 0 || last != 0.f) return 12;
  cfg = flb_preprocess_config{2, 4, 10, 1, 0, 1.0};    // 16 rings into n_scans 4: an error, not undefined behaviour
  if (fe.preprocess(velo, cfg, &last) != -1) return 13;
  std::printf("PREPROCESS_FACADE_OK velodyne=%d livox=%d down=%d M=%d\n", n, nl, (int)down.points.size(), gpu.effct_feat_num);
  return 0;
}

// Compiles flb::ImuProcessGpu against look-alikes of the reference types (MeasureGroup with sensor_msgs::Imu pointers,
// esekfom::esekf's get_x / change_x / get_P / change_P, state_ikfom with MTK::S2's `vec`) and, when a GPU is present,
// runs twelve scans: one of IMU_init (20 samples pass MAX_INI_COUNT), then eleven propagations that undistort and
// filter a raw scan on the device.
// Built by tests/test_gpu_imu.py (build_facade_smoke) with g++ -Ioracle/shim -Iinclude ... -lfastlio_b200.
#include <cmath>
#include <cstdio>
#include <deque>
#include <memory>
#include <vector>

#include <fastlio_b200/ikd_tree_facade.hpp>
#include <fastlio_b200/imu_process_facade.hpp>
#include <fastlio_b200/lio_gpu_frontend.hpp>
#include <fastlio_b200/scan_frontend_facade.hpp>

typedef pcl::PointXYZINormal PointType;
typedef std::vector<PointType, Eigen::aligned_allocator<PointType>> PointVector;
struct PointCloudXYZI { PointVector points; };

struct Time { double s; double toSec() const { return s; } };
struct Header { Time stamp; };
struct Vector3 { double x, y, z; };
struct Imu { Header header; Vector3 linear_acceleration, angular_velocity; };
typedef std::shared_ptr<const Imu> ImuConstPtr;
struct MeasureGroup { double lidar_beg_time = 0, lidar_end_time = 0; std::deque<ImuConstPtr> imu; };

struct Vec3 { double v[3] = {0, 0, 0}; double& operator[](int i) { return v[i]; } double operator[](int i) const { return v[i]; } };
struct Quat { double c[4] = {0, 0, 0, 1}; double* coeffs() { return c; } const double* coeffs() const { return c; } };
struct S2 { Vec3 vec; double operator[](int i) const { return vec[i]; } };
struct state_ikfom { Vec3 pos; Quat rot; Quat offset_R_L_I; Vec3 offset_T_L_I, vel, bg, ba; S2 grav; };
struct Mat23 { double a[23 * 23] = {0}; double& operator()(int i, int j) { return a[j * 23 + i]; } };   // column-major, as Eigen
struct Esekf {
  state_ikfom x;
  Mat23 P;
  state_ikfom get_x() const { return x; }
  Mat23 get_P() const { return P; }
  void change_x(const state_ikfom& s) { x = s; }
  void change_P(const Mat23& p) { P = p; }
};
struct Mat3 { double m[9]; double operator()(int i, int j) const { return m[3 * i + j]; } };

KD_TREE<PointType> ikdtree;
flb::LioGpu gpu;

int main() {
  flb::ScanFrontEnd fe;        // declared first: the IMU processor is destroyed before its front end
  flb::ImuProcessGpu p_imu;
  Vec3 T;
  T[0] = 0.04; T[1] = -0.02; T[2] = 0.03;
  const Mat3 R{{1, 0, 0, 0, 1, 0, 0, 0, 1}};
  Vec3 cg, ca, bg, ba;
  for (int i = 0; i < 3; ++i) { cg[i] = 0.1; ca[i] = 0.1; bg[i] = 1e-4; ba[i] = 1e-4; }
  p_imu.set_extrinsic(T, R);
  p_imu.set_gyr_cov(cg);
  p_imu.set_acc_cov(ca);
  p_imu.set_gyr_bias_cov(bg);
  p_imu.set_acc_bias_cov(ba);
  if (flb_device_count() <= 0) { std::printf("NO_GPU compile-only ok\n"); return 0; }

  // a square room of half-width 8 m with a floor, scanned by 16 rings
  PointVector map;
  PointCloudXYZI raw;
  for (int c = 0; c < 900; ++c)
    for (int r = 0; r < 16; ++r) {
      const double az = (0.5 - c * 0.4) * M_PI / 180.0, el = (-15.0 + 2.0 * r) * M_PI / 180.0;
      const double dx = std::cos(el) * std::cos(az), dy = std::cos(el) * std::sin(az), dz = std::sin(el);
      double t = 8.0 / std::fmax(std::fabs(dx), std::fabs(dy));
      if (dz < 0.0) t = std::fmin(t, -1.5 / dz);
      PointType p{};
      p.x = (float)(dx * t); p.y = (float)(dy * t); p.z = (float)(dz * t);
      p.intensity = (float)r;
      p.curvature = (float)(c * 100.0 / 900.0);   // ms inside the sweep
      map.push_back(p);
      raw.points.push_back(p);
    }
  ikdtree.set_capacity(1 << 20, 1 << 16);
  ikdtree.set_downsample_param(0.2f);
  ikdtree.Build(map);
  if (!gpu.attach(ikdtree.handle(), false, 3, 0.2)) return 2;
  if (!fe.attach(gpu.handle(), 1 << 16)) return 3;
  if (!p_imu.attach(fe.handle(), 0.5f)) return 4;

  Esekf kf;
  for (int i = 0; i < 23; ++i) kf.P(i, i) = 1.0;
  kf.x.grav.vec[2] = -9.809;
  int propagated = 0;
  for (int k = 0; k < 12; ++k) {
    MeasureGroup meas;
    meas.lidar_beg_time = 0.1 * k;
    meas.lidar_end_time = 0.1 * k + 0.1;
    for (int s = 0; s < 20; ++s) {
      auto m = std::make_shared<Imu>();
      m->header.stamp.s = 0.1 * k + 0.005 * s;
      m->linear_acceleration = Vector3{0.01, -0.02, 9.81};
      m->angular_velocity = Vector3{0.001, 0.0, 0.02};
      meas.imu.push_back(m);
    }
    if (!fe.upload(raw)) return 5;
    PointCloudXYZI undistorted;
    p_imu.Process(meas, kf, undistorted);
    const flb_imu_result& r = p_imu.last_result();
    if (k == 0 && r.status != FLB_IMU_INIT) { std::printf("expected initialisation, status %d\n", r.status); return 6; }
    if (!p_imu.scan_ready()) continue;
    ++propagated;
    if (r.n_poses != 21 && r.n_poses != 20) { std::printf("n_poses %d\n", r.n_poses); return 7; }
    if (p_imu.feats_down_size() <= 100) return 8;
    std::vector<double> poses;
    if (p_imu.imu_poses(poses) != r.n_poses) return 9;
    if (!(std::fabs(kf.x.grav[2] + 9.809) < 1e-3) || !(kf.x.rot.c[3] > 0.99)) return 10;
    if (!(kf.P(12, 12) > 1.0)) return 11;   // the velocity covariance grew
  }
  if (propagated != 11) { std::printf("propagated %d scans\n", propagated); return 12; }
  std::printf("IMU_FACADE_OK\n");
  return 0;
}

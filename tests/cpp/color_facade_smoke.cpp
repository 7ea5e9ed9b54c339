// Compiles flb::ScanFrontEnd::set_camera / upload_image / colorize / to_imu against cv::Mat- and livox_ros::Point-shaped
// look-alikes as src/laserMapping.cpp would use them in paramSetting, imageCallback, publish_frame_world_color and
// publish_frame_body and, when a GPU is present, colours a cloud in front of a forward-looking camera.  Without a GPU the
// facade cannot be attached: its calls report the error on stderr and return false, and the program prints NO_GPU.
// Built by tests/test_color_cpu.py with:
//   g++ -Ioracle/shim -Iinclude tests/cpp/color_facade_smoke.cpp -Lbetter_fastlio2_b200 -lfastlio_b200
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#include <fastlio_b200/ikd_tree_facade.hpp>
#include <fastlio_b200/lio_gpu_frontend.hpp>
#include <fastlio_b200/scan_frontend_facade.hpp>

typedef pcl::PointXYZINormal PointType;
typedef std::vector<PointType, Eigen::aligned_allocator<PointType>> PointVector;
struct PointCloudXYZI { PointVector points; };

namespace cv {   // the members of cv::Mat the facade reads
struct MatStep { size_t s[2]; size_t operator[](int i) const { return s[i]; } };
struct Mat { int rows, cols; MatStep step; unsigned char* data; };
}  // namespace cv
namespace livox_ros {   // preprocess.h:77-87: PCL_ADD_POINT4D, intensity, tag, line, reflectivity, offset_time, PCL_ADD_RGB
struct Point {
  float x, y, z, pad;
  float intensity;
  uint8_t tag, line, reflectivity;
  uint32_t offset_time;
  union { struct { uint8_t b, g, r, a; }; float rgb; uint32_t rgba; };
};
}  // namespace livox_ros
struct ColorCloud { std::vector<livox_ros::Point> points; };

struct Vec3 { double v[3]; double operator[](int i) const { return v[i]; } };
struct Quat { double c[4]; const double* coeffs() const { return c; } };
struct state_ikfom { Vec3 pos; Quat rot; Quat offset_R_L_I; Vec3 offset_T_L_I, vel, bg, ba, grav; };

KD_TREE<PointType> ikdtree;
flb::LioGpu gpu;

int main() {
  const int W = 1280, H = 720;
  // paramSetting's inputs: lidar x forward -> camera z, fx = fy = 900, principal point at the image centre
  std::vector<double> cam_ex = {0, -1, 0, 0, 0, 0, -1, 0, 1, 0, 0, 0, 0, 0, 0, 1};
  std::vector<double> cam_in = {900, 0, W / 2.0, 0, 0, 900, H / 2.0, 0, 0, 0, 1, 0};
  // a bgr8 frame with padded rows: b = u % 256, g = v % 256, r = 7
  const int step = 3 * W + 64;
  std::vector<unsigned char> pixels((size_t)step * H, 0);
  for (int v = 0; v < H; ++v)
    for (int u = 0; u < W; ++u) {
      unsigned char* p = &pixels[(size_t)v * step + 3 * u];
      p[0] = (unsigned char)(u % 256); p[1] = (unsigned char)(v % 256); p[2] = 7;
    }
  cv::Mat image{H, W, {{(size_t)step, 3}}, pixels.data()};

  flb::ScanFrontEnd fe;
  if (flb_device_count() <= 0) {
    const bool any = fe.set_camera(cam_ex, cam_in) || fe.upload_image(image);
    std::printf("NO_GPU compile-only ok\n");
    return any ? 1 : 0;
  }
  std::mt19937 rng(3);
  std::uniform_real_distribution<float> X(-5.f, 30.f), Y(-20.f, 20.f), Z(-5.f, 5.f);
  PointVector map;
  for (int i = 0; i < 20000; ++i) { PointType p{}; p.x = X(rng); p.y = Y(rng); p.z = Z(rng); map.push_back(p); }
  ikdtree.set_capacity(1 << 20, 1 << 16);
  ikdtree.set_downsample_param(0.2f);
  ikdtree.Build(map);
  if (!gpu.attach(ikdtree.handle(), false, 3, 0.2)) return 2;
  if (!fe.attach(gpu.handle(), 1 << 16)) return 3;
  PointCloudXYZI lidar;
  for (int i = 0; i < 30000; ++i) {
    PointType p{};
    p.x = X(rng); p.y = Y(rng); p.z = Z(rng); p.intensity = (float)(i % 97);
    lidar.points.push_back(p);
  }
  if (!fe.upload(lidar)) return 4;
  if (!fe.set_camera(cam_ex, cam_in) || !fe.upload_image(image)) return 5;
  state_ikfom s{};
  s.rot.c[3] = 1.0; s.offset_R_L_I.c[3] = 1.0;
  ColorCloud colorCloud;
  if (!fe.colorize(s, true, colorCloud)) return 6;
  // the same selection and colours computed here (identity state: world = lidar frame)
  size_t k = 0;
  for (const PointType& p : lidar.points) {
    const double c0 = -900.0 * p.y + (W / 2.0) * p.x, c1 = -900.0 * p.z + (H / 2.0) * p.x, c2 = p.x;
    const double u = c0 / c2, v = c1 / c2;
    if (!(p.x > 0 && u > -1.0 && u < W && v > -1.0 && v < H)) continue;
    if (k >= colorCloud.points.size()) return 7;
    const livox_ros::Point& q = colorCloud.points[k++];
    if (q.x != p.x || q.y != p.y || q.z != p.z || q.intensity != p.intensity) return 8;
    if (q.b != (int)u % 256 || q.g != (int)v % 256 || q.r != 7 || q.a != 255 || q.tag || q.line || q.reflectivity || q.offset_time) return 9;
  }
  if (k != colorCloud.points.size() || k < 1000) return 10;
  PointCloudXYZI body;
  if (!fe.to_imu(s, body) || body.points.size() != lidar.points.size()) return 11;
  for (size_t i = 0; i < body.points.size(); ++i)
    if (body.points[i].x != lidar.points[i].x || body.points[i].intensity != lidar.points[i].intensity) return 12;
  std::printf("COLOR_FACADE_OK kept=%zu of %zu\n", k, lidar.points.size());
  return 0;
}

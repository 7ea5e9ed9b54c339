// Compiles flb::KeyFrameStore::icp with flb::IcpParams / flb::IcpResult against PointType / PointTypePose / Affine3f /
// Matrix4f look-alikes as src/laserMapping.cpp would use them in performLoopClosure (:946-987) and, when a GPU is present,
// registers a key frame onto a shifted copy of itself.  Without a GPU the store cannot be attached: the facade reports it
// on stderr and the program exits with 2.  Built by tests/test_icp_cpu.py with:
//   g++ -Ioracle/shim -Iinclude tests/cpp/icp_facade_smoke.cpp -Lbetter_fastlio2_b200 -lfastlio_b200
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include <fastlio_b200/ikd_tree_facade.hpp>
#include <fastlio_b200/keyframe_store_facade.hpp>

typedef pcl::PointXYZINormal PointType;
typedef std::vector<PointType, Eigen::aligned_allocator<PointType>> PointVector;
struct PointCloudXYZI { PointVector points; };
struct PointTypePose { float x, y, z, intensity, roll, pitch, yaw; double time; };   // PointXYZIRPYT, common_lib.h
struct Affine3f {   // the member Eigen::Affine3f offers: operator()(row, col)
  float m[3][4];
  float operator()(int r, int c) const { return m[r][c]; }
};
struct Matrix4f {   // the member Eigen::Matrix4f offers: operator()(row, col)
  float m[4][4];
  float& operator()(int r, int c) { return m[r][c]; }
};

KD_TREE<PointType> ikdtree;

int main() {
  std::mt19937 rng(11);
  std::uniform_real_distribution<float> U(-20.f, 20.f), H(0.f, 6.f);
  std::normal_distribution<float> N(0.f, 0.01f);
  PointCloudXYZI scene, shifted;
  for (int i = 0; i < 30000; ++i) {   // a ground, two walls and a pole
    PointType p{};
    const int k = i % 4;
    if (k == 0) { p.x = U(rng); p.y = U(rng); p.z = N(rng); }
    else if (k == 1) { p.x = U(rng); p.y = 12.f + N(rng); p.z = H(rng); }
    else if (k == 2) { p.x = -9.f + N(rng); p.y = U(rng); p.z = H(rng); }
    else { const float a = 0.001f * i; p.x = 4.f + std::cos(a); p.y = -3.f + std::sin(a); p.z = H(rng); }
    p.intensity = (float)(i % 100);
    scene.points.push_back(p);
    PointType q = p;   // the same scene seen from 0.3 m further along x and 0.2 m along y
    q.x -= 0.3f; q.y -= 0.2f;
    shifted.points.push_back(q);
  }
  std::vector<Affine3f> eye(1);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) eye[0].m[r][c] = (r == c) ? 1.f : 0.f;
  PointTypePose com{};   // the Scan Context yaw: 0 here

  // performLoopClosure's settings (:947-952)
  flb::IcpParams icp;
  icp.setMaxCorrespondenceDistance(200);
  icp.setMaximumIterations(100);
  icp.setTransformationEpsilon(1e-6);
  icp.setEuclideanFitnessEpsilon(1e-6);
  icp.setRANSACIterations(0);
  flb::IcpResult reg;

  flb::KeyFrameStore keyframes;
  if (flb_device_count() <= 0) {
    std::printf("NO_GPU: the store needs a device\n");
    return keyframes.attach(ikdtree.handle(), 1 << 17, 8) ? 1 : 2;
  }
  ikdtree.set_capacity(1 << 20, 1 << 16);
  ikdtree.set_downsample_param(0.2f);
  if (!keyframes.attach(ikdtree.handle(), 1 << 17, 8)) return 3;
  if (keyframes.push_back(scene) != 0 || keyframes.push_back(shifted) != 1) return 4;
  std::vector<int> cur = {1}, pre = {0};
  if (!keyframes.icp(cur, eye, com, pre, eye, icp, reg)) return 5;
  Matrix4f correctionLidarFrame;
  reg.getFinalTransformation(correctionLidarFrame);
  const double dx = correctionLidarFrame(0, 3) - 0.3, dy = correctionLidarFrame(1, 3) - 0.2;
  if (!reg.hasConverged() || !(reg.getFitnessScore() < 0.3) || std::fabs(dx) > 0.02 || std::fabs(dy) > 0.02) return 6;
  // errors are reported, not thrown
  std::vector<int> bad = {0, 9};
  if (keyframes.icp(bad, std::vector<Affine3f>(2, eye[0]), com, pre, eye, icp, reg)) return 7;
  icp.setRANSACIterations(10);
  if (keyframes.icp(cur, eye, com, pre, eye, icp, reg)) return 8;
  std::printf("ICP_FACADE_OK t=(%.4f, %.4f, %.4f) fitness=%.6f\n", correctionLidarFrame(0, 3), correctionLidarFrame(1, 3),
              correctionLidarFrame(2, 3), reg.getFitnessScore());
  return 0;
}

// Compiles flb::KeyFrameStore::icp_batch with flb::IcpPairSel / flb::IcpParams / flb::IcpResult against PointType /
// PointTypePose / Matrix4f look-alikes as the multi-session mapper (Incremental_mapping.cpp addSCloops / addRSloops) would
// use them and, when a GPU is present, registers two pairs: a key frame onto a shifted copy of itself, with zero poses
// (the local-frame Scan Context pairs) and with the copy's own pose (the central-frame radius-search pairs).  Without a
// GPU the store cannot be attached: the facade reports it on stderr and the program exits with 2.  Built by
// tests/test_icp_batch_cpu.py with:
//   g++ -Ioracle/shim -Iinclude tests/cpp/icp_batch_facade_smoke.cpp -Lbetter_fastlio2_b200 -lfastlio_b200
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
struct Matrix4f {   // the member Eigen::Matrix4f offers: operator()(row, col)
  float m[4][4];
  float& operator()(int r, int c) { return m[r][c]; }
};

KD_TREE<PointType> ikdtree;

int main() {
  std::mt19937 rng(12);
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
  PointTypePose zero{}, back{};   // back: the copy's pose, which puts it onto the scene
  back.x = 0.3f; back.y = 0.2f;

  // doICPVirtualRelative / doICPGlobalRelative's settings (Incremental_mapping.cpp:484-488, :546-550)
  flb::IcpParams icp;
  icp.setMaxCorrespondenceDistance(30);
  icp.setMaximumIterations(10);
  icp.setTransformationEpsilon(1e-6);
  icp.setEuclideanFitnessEpsilon(1e-6);
  icp.setRANSACIterations(0);

  flb::KeyFrameStore keyframes;
  if (flb_device_count() <= 0) {
    std::printf("NO_GPU: the store needs a device\n");
    return keyframes.attach(ikdtree.handle(), 1 << 17, 8) ? 1 : 2;
  }
  ikdtree.set_capacity(1 << 20, 1 << 16);
  ikdtree.set_downsample_param(0.2f);
  if (!keyframes.attach(ikdtree.handle(), 1 << 17, 8)) return 3;
  if (keyframes.push_back(scene) != 0 || keyframes.push_back(shifted) != 1) return 4;
  std::vector<flb::IcpPairSel> pairs(2);
  pairs[0].addSrc(1, zero);   // SC pair: both in their local frames
  pairs[0].addTgt(0, zero);
  pairs[1].addSrc(1, back);   // RS pair: both in the central frame
  pairs[1].addTgt(0, zero);
  std::vector<flb::IcpResult> regs;
  flb_icp_batch_stats st{};
  if (!keyframes.icp_batch(pairs, 0.2f, icp, regs, &st) || regs.size() != 2 || st.rounds != 1) return 5;
  Matrix4f T0, T1;
  regs[0].getFinalTransformation(T0);
  regs[1].getFinalTransformation(T1);
  if (!regs[0].hasConverged() || !(regs[0].getFitnessScore() < 0.3) || std::fabs(T0(0, 3) - 0.3f) > 0.05 || std::fabs(T0(1, 3) - 0.2f) > 0.05)
    return 6;
  if (!regs[1].hasConverged() || std::fabs(T1(0, 3)) > 0.02 || std::fabs(T1(1, 3)) > 0.02) return 7;
  // errors are reported, not thrown
  flb::IcpPairSel bad = pairs[0];
  bad.addSrc(9, zero);
  if (keyframes.icp_batch({bad}, 0.2f, icp, regs)) return 8;
  icp.setRANSACIterations(10);
  if (keyframes.icp_batch(pairs, 0.2f, icp, regs)) return 9;
  std::printf("ICP_BATCH_FACADE_OK t0=(%.4f, %.4f) t1=(%.4f, %.4f) syncs=%d+%d\n", T0(0, 3), T0(1, 3), T1(0, 3), T1(1, 3), st.setup_syncs,
              st.iteration_syncs);
  return 0;
}

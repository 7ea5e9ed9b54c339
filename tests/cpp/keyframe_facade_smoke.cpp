// Compiles flb::KeyFrameStore against PointType / PointTypePose / Affine3f look-alikes exactly as src/laserMapping.cpp
// would use it and, when a GPU is present, runs front end -> key frame -> sub-map rebuild -> global / loop maps -> saver.
// Built by tests/test_keyframes_cpu.py with:
//   g++ -Ioracle/shim -Iinclude tests/cpp/keyframe_facade_smoke.cpp -Lbetter_fastlio2_b200 -lfastlio_b200
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include <fastlio_b200/ikd_tree_facade.hpp>
#include <fastlio_b200/keyframe_store_facade.hpp>
#include <fastlio_b200/lio_gpu_frontend.hpp>
#include <fastlio_b200/scan_frontend_facade.hpp>

typedef pcl::PointXYZINormal PointType;
typedef std::vector<PointType, Eigen::aligned_allocator<PointType>> PointVector;
struct PointCloudXYZI { PointVector points; };
struct PointTypePose { float x, y, z, intensity, roll, pitch, yaw; double time; };   // PointXYZIRPYT, common_lib.h
struct PoseCloud { std::vector<PointTypePose> points; };
struct Affine3f {   // the member Eigen::Affine3f offers: operator()(row, col)
  float m[3][4];
  float operator()(int r, int c) const { return m[r][c]; }
};

KD_TREE<PointType> ikdtree;
flb::LioGpu gpu;

int main() {
  std::mt19937 rng(5);
  std::uniform_real_distribution<float> U(-20.f, 20.f);
  PointCloudXYZI scan;
  for (int i = 0; i < 5000; ++i) {
    PointType p{};
    p.x = U(rng); p.y = U(rng); p.z = 0.1f * U(rng); p.intensity = (float)(i % 100); p.curvature = 0.02f * i;
    scan.points.push_back(p);
  }
  PoseCloud cloudKeyPoses6D;
  cloudKeyPoses6D.points.push_back(PointTypePose{0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.0});
  cloudKeyPoses6D.points.push_back(PointTypePose{2.f, 1.f, 0.f, 1.f, 0.01f, -0.02f, 0.3f, 0.1});
  std::vector<Affine3f> finalTrans(2);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) { finalTrans[0].m[r][c] = (r == c) ? 1.f : 0.f; finalTrans[1].m[r][c] = (r == c) ? 1.f : (c == 3 ? 0.5f : 0.f); }

  if (flb_device_count() <= 0) { std::printf("NO_GPU compile-only ok\n"); return 0; }
  ikdtree.set_capacity(1 << 20, 1 << 16);
  ikdtree.set_downsample_param(0.2f);
  ikdtree.Build(scan.points);
  if (!gpu.attach(ikdtree.handle(), false, 3, 0.2)) return 2;
  flb::ScanFrontEnd fe;
  if (!fe.attach(gpu.handle(), 1 << 14)) return 3;
  flb::KeyFrameStore keyframes;
  if (!keyframes.attach(ikdtree.handle(), 1 << 16, 8)) return 4;

  // saveKeyFramesAndFactor: the front end's scan (no IMU step here: upload order) and a host cloud
  if (!fe.upload(scan) || keyframes.push_back(fe) != 0) return 5;
  if (keyframes.push_back(scan) != 1 || keyframes.size() != 2 || keyframes.points(1) != 5000) return 6;
  PointCloudXYZI saved;
  if (!keyframes.at(0, saved) || saved.points.size() != scan.points.size()) return 7;
  for (size_t i = 0; i < scan.points.size(); ++i)
    if (saved.points[i].x != scan.points[i].x || saved.points[i].intensity != scan.points[i].intensity ||
        saved.points[i].curvature != scan.points[i].curvature)
      return 8;
  // recontructIKdTree
  std::vector<int> ids = {0, 1};
  PointVector featsFromMap;
  if (!keyframes.reconstruct(ikdtree, ids, cloudKeyPoses6D, 0.4f, featsFromMap)) return 9;
  if (featsFromMap.empty() || ikdtree.validnum() != (int)featsFromMap.size() || ikdtree.Root_Node == nullptr) return 10;
  // publishGlobalMap / saveMapService (dense and filtered)
  PointCloudXYZI dense, filtered, nearKeyframes;
  if (!keyframes.assemble(ids, cloudKeyPoses6D, 0.f, dense) || dense.points.size() != 10000) return 11;
  if (!keyframes.assemble(ids, cloudKeyPoses6D, 0.7f, filtered) || filtered.points.empty() || filtered.points.size() >= 10000) return 12;
  // loopFindNearKeyframes: the key frame itself is copied (curvature kept), the neighbour transformed (curvature 0)
  if (!keyframes.assemble(ids, finalTrans, 0.f, nearKeyframes) || nearKeyframes.points.size() != 10000) return 13;
  if (nearKeyframes.points[7].curvature != scan.points[7].curvature || nearKeyframes.points[5007].curvature != 0.f) return 14;
  if (nearKeyframes.points[5007].x != scan.points[7].x + 0.5f) return 15;
  // the map-side scratch a whole-map assembly leaves behind is reported and given back
  if (keyframes.scratch_bytes() <= 0 || !keyframes.release_scratch() || keyframes.scratch_bytes() != 0) return 17;
  // errors are reported, not thrown
  std::vector<int> bad = {0, 9};
  if (keyframes.assemble(bad, cloudKeyPoses6D, 0.f, dense) || keyframes.at(9, saved)) return 16;
  std::printf("KEYFRAME_FACADE_OK keyframes=%d featsFromMap=%d dense=%d filtered=%d\n", keyframes.size(), (int)featsFromMap.size(),
              (int)dense.points.size(), (int)filtered.points.size());
  return 0;
}

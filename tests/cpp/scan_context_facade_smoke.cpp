// Compiles flb::KeyFrameStore::scan_context / scan_contexts against PointType / PointTypePose / Affine3f / MatrixXd
// look-alikes as src/laserMapping.cpp would use them and, when a GPU is present, runs one loop attempt (two descriptors,
// the gate, the clouds only after it passes) and the key-frame saver.  Built by tests/test_scan_context_cpu.py with:
//   g++ -Ioracle/shim -Iinclude tests/cpp/scan_context_facade_smoke.cpp -Lbetter_fastlio2_b200 -lfastlio_b200
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
struct PoseCloud { std::vector<PointTypePose> points; };
struct Affine3f {   // the member Eigen::Affine3f offers: operator()(row, col)
  float m[3][4];
  float operator()(int r, int c) const { return m[r][c]; }
};
struct MatrixXd {   // the members Eigen::MatrixXd offers: resize(rows, cols), operator()(row, col), rows(), cols()
  std::vector<double> v;
  int r = 0, c = 0;
  void resize(int rows, int cols) { r = rows; c = cols; v.assign((size_t)rows * cols, -1.0); }
  double& operator()(int i, int j) { return v[(size_t)i * c + j]; }
  double operator()(int i, int j) const { return v[(size_t)i * c + j]; }
  int rows() const { return r; }
  int cols() const { return c; }
};

// SCManager::distanceBtnScanContext without the sector-key pre-alignment: the smallest column-wise cosine distance over
// every circular shift (enough for a smoke run of the gate)
static double sc_distance(const MatrixXd& a, const MatrixXd& b) {
  double best = 1e9;
  for (int s = 0; s < a.cols(); ++s) {
    double sum = 0;
    int cnt = 0;
    for (int j = 0; j < a.cols(); ++j) {
      double dot = 0, na = 0, nb = 0;
      for (int i = 0; i < a.rows(); ++i) {
        const double x = a(i, j), y = b(i, (j + s) % b.cols());
        dot += x * y; na += x * x; nb += y * y;
      }
      if (na == 0 || nb == 0) continue;
      sum += dot / (std::sqrt(na) * std::sqrt(nb));
      ++cnt;
    }
    if (cnt > 0 && 1.0 - sum / cnt < best) best = 1.0 - sum / cnt;
  }
  return best;
}

KD_TREE<PointType> ikdtree;

int main() {
  std::mt19937 rng(5);
  std::uniform_real_distribution<float> U(-40.f, 40.f), H(-1.f, 3.f);
  PointCloudXYZI scan;
  for (int i = 0; i < 20000; ++i) {
    PointType p{};
    p.x = U(rng); p.y = U(rng); p.z = H(rng); p.intensity = (float)(i % 100);
    scan.points.push_back(p);
  }
  PoseCloud cloudKeyPoses6D;
  for (int k = 0; k < 3; ++k) cloudKeyPoses6D.points.push_back(PointTypePose{0.5f * k, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.1 * k});
  std::vector<Affine3f> finalTrans(2);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) { finalTrans[0].m[r][c] = (r == c) ? 1.f : 0.f; finalTrans[1].m[r][c] = (r == c) ? 1.f : (c == 3 ? 0.25f : 0.f); }
  const double LIDAR_HEIGHT = 1.5;   // scLoop.LIDAR_HEIGHT

  if (flb_device_count() <= 0) { std::printf("NO_GPU compile-only ok\n"); return 0; }
  ikdtree.set_capacity(1 << 20, 1 << 16);
  ikdtree.set_downsample_param(0.2f);
  flb::KeyFrameStore keyframes;
  if (!keyframes.attach(ikdtree.handle(), 1 << 17, 8)) return 2;
  for (int k = 0; k < 3; ++k)
    if (keyframes.push_back(scan) != k) return 3;

  // performLoopClosure: current key frame 1 with its neighbour 2, candidate 0 with its neighbour 1
  std::vector<int> cur = {1, 2}, prev = {0, 1};
  MatrixXd cureKeyframeSC, prevKeyframeSC;
  if (!keyframes.scan_context(cur, finalTrans, LIDAR_HEIGHT, cureKeyframeSC)) return 4;
  if (!keyframes.scan_context(prev, finalTrans, LIDAR_HEIGHT, prevKeyframeSC)) return 5;
  if (cureKeyframeSC.rows() != FLB_SC_RINGS || cureKeyframeSC.cols() != FLB_SC_SECTORS) return 6;
  int filled = 0;
  for (int i = 0; i < FLB_SC_RINGS; ++i)
    for (int j = 0; j < FLB_SC_SECTORS; ++j) filled += cureKeyframeSC(i, j) != 0;
  if (filled < 200) return 7;
  const double dist = sc_distance(cureKeyframeSC, prevKeyframeSC);
  if (!(dist <= 0.3)) return 8;   // SC_DIST_THRES: the same scene, so the gate passes and ICP gets its clouds
  PointCloudXYZI cureKeyframeCloud;
  if (!keyframes.assemble(cur, finalTrans, 0.f, cureKeyframeCloud) || cureKeyframeCloud.points.size() != 40000) return 9;
  // the same descriptor from poses
  MatrixXd byPose;
  if (!keyframes.scan_context(std::vector<int>{2}, cloudKeyPoses6D, LIDAR_HEIGHT, byPose)) return 10;

  // the saver: one call over all key frames; descs[i] goes to scLoop.saveScancontextAndKeys
  std::vector<MatrixXd> descs;
  std::vector<int> all = {0, 1, 2};
  if (!keyframes.scan_contexts(all, LIDAR_HEIGHT, descs) || descs.size() != 3) return 11;
  MatrixXd single;
  std::vector<Affine3f> eye(1, finalTrans[0]);
  if (!keyframes.scan_context(std::vector<int>{1}, eye, LIDAR_HEIGHT, single)) return 12;
  if (single.v != descs[1].v || descs[0].v != descs[2].v) return 13;   // stored records as they are: all the same scan

  // errors are reported, not thrown
  std::vector<int> bad = {0, 9};
  if (keyframes.scan_context(bad, cloudKeyPoses6D, LIDAR_HEIGHT, single) || keyframes.scan_contexts(bad, LIDAR_HEIGHT, descs)) return 14;
  if (keyframes.scan_context(cur, finalTrans, NAN, single)) return 15;
  std::printf("SCAN_CONTEXT_FACADE_OK filled=%d dist=%.4f\n", filled, dist);
  return 0;
}

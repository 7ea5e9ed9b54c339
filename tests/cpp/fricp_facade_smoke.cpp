// Compiles flb::KeyFrameStore::fricp with flb::FricpParams against PointType / PointTypePose / Eigen::MatrixXd look-alikes
// as src/online_relocalization.cpp's pose_estimator::run would use them (pose_estimator.cpp:184-198): the prior session's
// key frames pushed back once, then one call per scan.  Syntax-checked by tests/test_fricp_cpu.py with:
//   g++ -fsyntax-only -Ioracle/shim -Iinclude tests/cpp/fricp_facade_smoke.cpp
#include <vector>

#include <fastlio_b200/ikd_tree_facade.hpp>
#include <fastlio_b200/keyframe_store_facade.hpp>

typedef pcl::PointXYZINormal PointType;
typedef std::vector<PointType, Eigen::aligned_allocator<PointType>> PointVector;
struct PointCloudXYZI { PointVector points; };
struct PointTypePose { float x, y, z, intensity, roll, pitch, yaw; double time; };   // PointXYZIRPYT, common_lib.h
struct Poses6D { std::vector<PointTypePose> points; };                              // *cloudKeyPoses6D
struct MatrixXd {   // the members of Eigen::MatrixXd the node uses: operator()(row, col)
  double m[4][4];
  double& operator()(int r, int c) { return m[r][c]; }
};

int relocalise(flb::KeyFrameStore& keyframes, const std::vector<PointCloudXYZI>& all_cloud, const Poses6D& poses6D,
               const PointCloudXYZI& cur, const PointTypePose& initPose, const PointTypePose& pose_ext, int regMode) {
  for (const PointCloudXYZI& c : all_cloud) keyframes.push_back(c);
  const std::vector<int> near{0, 1, 2};   // searchNum key frames around the pose
  flb::FricpParams fr(regMode);
  MatrixXd T;
  flb_fricp_result info;
  if (!keyframes.fricp(cur, initPose, near, pose_ext, poses6D, fr, T, &info)) return 1;
  return info.status == FLB_FRICP_OK && T(3, 3) == 1.0 ? 0 : 1;
}

int main() { return 0; }

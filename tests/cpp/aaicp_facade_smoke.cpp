// Compiles flb::KeyFrameStore::aaicp with flb::AaicpParams against PointType / PointTypePose / Eigen::MatrixXd look-alikes
// as pose_estimator::run would dispatch regMode 1 (AA-ICP) to it: the prior session's key frames pushed back once, then
// one call per scan, regMode 7 going to sicp and the other point-to-point modes to fricp.  Syntax-checked by
// tests/test_aaicp_cpu.py with:
//   g++ -fsyntax-only -Ioracle/shim -Iinclude tests/cpp/aaicp_facade_smoke.cpp
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
  MatrixXd T;
  if (regMode == 1) {   // case AA_ICP
    flb::AaicpParams ap;
    flb_aaicp_result info;
    if (!keyframes.aaicp(cur, initPose, near, pose_ext, poses6D, ap, T, &info)) return 1;
    return info.status == FLB_FRICP_OK && info.history >= 2 && T(3, 3) == 1.0 ? 0 : 1;
  }
  if (regMode == 7) {   // case SparseICP
    flb::SicpParams sp;
    flb_sicp_result info;
    if (!keyframes.sicp(cur, initPose, near, pose_ext, poses6D, sp, T, &info)) return 1;
    return info.status == FLB_FRICP_OK && T(3, 3) == 1.0 ? 0 : 1;
  }
  flb::FricpParams fr(regMode);
  flb_fricp_result info;
  if (!keyframes.fricp(cur, initPose, near, pose_ext, poses6D, fr, T, &info)) return 1;
  return info.status == FLB_FRICP_OK && T(3, 3) == 1.0 ? 0 : 1;
}

int main() { return 0; }

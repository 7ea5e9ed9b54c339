// keyframe_store_facade.hpp — surfCloudKeyFrames (src/laserMapping.cpp:756-758) kept on the GPU, with the reader shapes
// laserMapping.cpp uses, so that no key-frame cloud has to live in host RAM:
//
//   flb::KeyFrameStore keyframes;  keyframes.attach(ikdtree.handle(), 40000000LL, 4000);   // next to `flb::LioGpu gpu;`
//   // saveKeyFramesAndFactor, instead of :756-758 (copyPointCloud(*feats_undistort) + push_back):
//   keyframes.push_back(fe);                                             // fe: the flb::ScanFrontEnd of the scan
//   // recontructIKdTree, instead of :636-664 (transform + VoxelGrid + ikdtree.reconstruct + featsFromMap):
//   keyframes.reconstruct(ikdtree, ids, *cloudKeyPoses6D, leaf, featsFromMap->points);
//   // publishGlobalMap (:1858-1869) and saveMapService (:1763-1798): poses per key frame, leaf 0 = dense
//   keyframes.assemble(ids, *cloudKeyPoses6D, globalMapVisualizationLeafSize, *globalMapKeyFramesDS);
//   // loopFindNearKeyframes (:856-883): one affine per key frame, the identity for keyNear == key
//   keyframes.assemble(ids, finalTrans, 0.f, *nearKeyframes);
//   // the per-key-frame saver at shutdown (:2501-2505):
//   keyframes.at(i, *save_cloud);
//   // the Scan Context gate of performLoopClosure (:932-940), before any cloud is assembled: same ids and affines
//   keyframes.scan_context(ids, finalTrans, scLoop.LIDAR_HEIGHT, cureKeyframeSC);
//   // every key frame's descriptor for the saver (:2504-2505), then scLoop.saveScancontextAndKeys(descs[i])
//   keyframes.scan_contexts(all_ids, scLoop.LIDAR_HEIGHT, descs);
//   // the ICP of performLoopClosure (:946-974) once the gate passed: the same selections, com = the SC yaw pose
//   flb::IcpParams icp;  icp.setMaxCorrespondenceDistance(200); ...;  flb::IcpResult reg;
//   keyframes.icp(curIds, curT, com, preIds, preT, icp, reg);  reg.hasConverged(), reg.getFitnessScore(), ...
//   // the multi-session mapper's inter-session loops (Incremental_mapping.cpp addSCloops :651-696, addRSloops :787-837):
//   // both sessions' key frames in one store, one IcpPairSel per loop pair, every pair of the loop list in one call
//   flb::IcpPairSel sel;  sel.addSrc(id, pose);  sel.addTgt(id, pose);  ...;  std::vector<flb::IcpResult> regs;
//   keyframes.icp_batch(pairs, 0.2f, icp, regs);  regs[p].hasConverged(), regs[p].getFitnessScore(), ...
//   // the relocaliser (pose_estimator.cpp:184-198, :566-596), the prior session's key frames pushed back once:
//   flb::FricpParams fr(regMode);  Eigen::MatrixXd T(4, 4);
//   keyframes.fricp(*cloudBuffer[idx], initPose, nearIds, pose_ext, *poses6D, fr, T);
//   // regMode 7 (Sparse ICP, registeration.h:143-146) on the same clouds
//   flb::SicpParams sp;  keyframes.sicp(*cloudBuffer[idx], initPose, nearIds, pose_ext, *poses6D, sp, T);
//   // regMode 1 (AA-ICP, registeration.h:86-91) on the same clouds
//   flb::AaicpParams ap;  keyframes.aaicp(*cloudBuffer[idx], initPose, nearIds, pose_ext, *poses6D, ap, T);
//
// Poses6D is anything with points[k].{x, y, z, roll, pitch, yaw} (pcl::PointCloud<PointTypePose>); an affine is
// anything with operator()(row, col) (Eigen::Affine3f).  Clouds come back with x, y, z, intensity and curvature set
// and the other PointType fields zero.  Nothing here takes a lock: calls are serialised with every other call on the map
// from all threads — the loop-closure thread and the main loop hold one common mutex around their calls (INTEGRATION.md
// §3 "Key-frame clouds on the GPU", §5).  Errors are reported on stderr and returned as false / -1.
#pragma once
#include <cstdio>
#include <type_traits>
#include <vector>

#include "../fastlio_b200.h"
#include "ikd_tree_facade.hpp"
#include "scan_frontend_facade.hpp"

namespace flb {

// The five setters of pcl::IterativeClosestPoint that performLoopClosure calls (:947-952), with its values as defaults.
struct IcpParams {
  flb_icp_config cfg{200.0, 100, 1e-6, 1e-6};
  int ransac_iterations = 0;
  void setMaxCorrespondenceDistance(double d) { cfg.max_correspondence_distance = d; }
  void setMaximumIterations(int n) { cfg.max_iterations = n; }
  void setTransformationEpsilon(double e) { cfg.transformation_epsilon = e; }
  void setEuclideanFitnessEpsilon(double e) { cfg.euclidean_fitness_epsilon = e; }
  void setRANSACIterations(int n) { ransac_iterations = n; }   // only 0, the reference's value, is accepted
};

// The three getters the node reads after icp.align(..) (:966-987).
struct IcpResult {
  flb_icp_result r{};
  bool hasConverged() const { return r.converged != 0; }
  double getFitnessScore() const { return r.fitness_score; }
  // into anything with operator()(row, col) of a 4x4, i.e. Eigen::Matrix4f (correctionLidarFrame.matrix())
  template <class M>
  void getFinalTransformation(M& T) const {
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j) T(i, j) = r.final_transformation[4 * i + j];
  }
};

// One pair of flb_keyframes_icp_batch: the source and the target selections, each key frame with its own pose (anything
// with x, y, z, roll, pitch, yaw: PointTypePose; a zero pose for the local-frame Scan Context pairs).
struct IcpPairSel {
  std::vector<int> srcIds, tgtIds;
  std::vector<float> srcPoses6, tgtPoses6;   // 6 per id
  template <class Pose> void addSrc(int id, const Pose& p) { add(srcIds, srcPoses6, id, p); }
  template <class Pose> void addTgt(int id, const Pose& p) { add(tgtIds, tgtPoses6, id, p); }

 private:
  template <class Pose>
  static void add(std::vector<int>& ids, std::vector<float>& p6, int id, const Pose& p) {
    ids.push_back(id);
    p6.insert(p6.end(), {p.x, p.y, p.z, p.roll, p.pitch, p.yaw});
  }
};

// Registeration(regMode) of the relocaliser (registeration.h:24-33) with ICP::Parameters' values (ICP.h:518-566); the
// mode numbers are the reference's: 0 ICP, 2 Fast ICP, 3 Robust ICP, 4 Fast and Robust ICP (config/online_relo.yaml).
struct FricpParams {
  flb_fricp_config cfg{};
  explicit FricpParams(int regMode = FLB_FRICP_FAST_ROBUST) {
    flb_fricp_default_config(&cfg);
    cfg.mode = regMode;
  }
};

// Registeration's SICP::Parameters for regMode 7 (registeration.h:67-69: ICP.h's defaults with p = 0.4).
struct SicpParams {
  flb_sicp_config cfg{};
  SicpParams() { flb_sicp_default_config(&cfg); }
};

// Registeration's ICP::Parameters as regMode 1 (AAICP::point_to_point_aaicp) reads them: max_icp, stop and
// error_overflow_threshold_ (ICP.h:518-566).
struct AaicpParams {
  flb_aaicp_config cfg{};
  AaicpParams() { flb_aaicp_default_config(&cfg); }
};

class KeyFrameStore {
 public:
  KeyFrameStore() = default;
  KeyFrameStore(const KeyFrameStore&) = delete;
  KeyFrameStore& operator=(const KeyFrameStore&) = delete;
  ~KeyFrameStore() { if (kf_) flb_keyframes_destroy(kf_); }

  // capacity: points over all key frames (20 device bytes each) and number of key frames
  bool attach(flb_map* map, long long max_points, int max_keyframes) {
    if (flb_keyframes_create(map, max_points, max_keyframes, &kf_)) { kf_ = nullptr; return ok(1, "attach"); }
    map_ = map;
    return true;
  }
  flb_keyframes* handle() { return kf_; }

  int size() const {   // surfCloudKeyFrames.size()
    int n = 0;
    return kf_ && !flb_keyframes_info(kf_, &n, nullptr, nullptr, nullptr) ? n : 0;
  }
  int points(int k) const { return kf_ ? flb_keyframes_size(kf_, k) : -1; }
  // device bytes of the readers' scratch the map keeps, and a way to free it (e.g. at the end of saveMapService)
  long long scratch_bytes() const {
    long long b = 0;
    return kf_ && !flb_keyframes_info(kf_, nullptr, nullptr, nullptr, &b) ? b : 0;
  }
  bool release_scratch() { return map_ && ok(flb_map_release_keyframe_scratch(map_), "release_scratch"); }

  // surfCloudKeyFrames.push_back(copy of feats_undistort): the front end's current scan, device to device.  Returns the
  // key frame's id, or -1.
  int push_back(ScanFrontEnd& fe) {
    int id = -1;
    return ok(flb_keyframes_append_frontend(kf_, fe.handle(), &id), "push_back") ? id : -1;
  }
  // the same from a host cloud (restoring a saved session)
  template <class Cloud>
  int push_back(const Cloud& cloud) {
    typedef typename std::remove_reference<decltype(cloud.points[0])>::type P;
    const int n = (int)cloud.points.size();
    const P* p0 = n ? &cloud.points[0] : nullptr;
    const int off_i = n ? (int)((const char*)&p0->intensity - (const char*)p0) : -1;
    const int off_c = n ? (int)((const char*)&p0->curvature - (const char*)p0) : -1;
    int id = -1;
    return ok(flb_keyframes_append(kf_, p0, n, (int)sizeof(P), off_i, off_c, &id), "push_back") ? id : -1;
  }

  // recontructIKdTree (laserMapping.cpp:636-664): subMap += transformPointCloud(key frame ids[j], poses.points[ids[j]]),
  // VoxelGrid(leaf), tree.reconstruct, featsFromMap = the filtered sub-map.
  template <class PointT, class Poses6D, class PointVec>
  bool reconstruct(KD_TREE<PointT>& tree, const std::vector<int>& ids, const Poses6D& poses, float leaf, PointVec& featsFromMap) {
    const std::vector<float> p6 = poses6(ids, poses);
    const int cap = selection_size(ids);
    if (cap < 0) return false;
    xyzi_.resize((size_t)cap * 4 + 4);
    int n = 0;
    const bool good = ok(flb_map_reconstruct_from_keyframes(tree.handle(), kf_, ids.data(), (int)ids.size(), p6.data(), leaf, xyzi_.data(),
                                                            cap, &n), "reconstruct");
    tree.refresh_root();
    if (!good) return false;
    featsFromMap.resize(n);
    for (int i = 0; i < n; ++i) fill(featsFromMap[i], &xyzi_[4 * (size_t)i], 0.f);
    return true;
  }

  // *out = sum over j of transformPointCloud(key frame ids[j], poses.points[ids[j]]), VoxelGrid(leaf) when leaf > 0
  template <class Poses6D, class Cloud>
  bool assemble(const std::vector<int>& ids, const Poses6D& poses, float leaf, Cloud& out) {
    const std::vector<float> p6 = poses6(ids, poses);
    return run_assemble(ids, FLB_KF_POSE6, p6, leaf, out);
  }
  // the same with one affine per selected key frame (T[j] for ids[j]); the identity copies the stored records
  template <class Affine, class Alloc, class Cloud>
  bool assemble(const std::vector<int>& ids, const std::vector<Affine, Alloc>& T, float leaf, Cloud& out) {
    if (T.size() != ids.size()) return ok(1, "assemble: one affine per key frame");
    return run_assemble(ids, FLB_KF_AFFINE, affines12(T), leaf, out);
  }

  // scLoop.makeScancontext(*nearKeyframes) for the loop sub-map that assemble(ids, T, 0.f, ..) would return
  // (performLoopClosure :932-933), computed on the device without assembling or downloading the cloud.  Mat is anything
  // with resize(rows, cols) and operator()(row, col), i.e. Eigen::MatrixXd: 20 rings x 60 sectors.
  template <class Affine, class Alloc, class Mat>
  bool scan_context(const std::vector<int>& ids, const std::vector<Affine, Alloc>& T, double lidar_height, Mat& desc) {
    if (T.size() != ids.size()) return ok(1, "scan_context: one affine per key frame");
    return run_scan_context(ids, FLB_KF_AFFINE, affines12(T), lidar_height, desc);
  }
  // the same with the key frames' poses (poses.points[ids[j]])
  template <class Poses6D, class Mat>
  bool scan_context(const std::vector<int>& ids, const Poses6D& poses, double lidar_height, Mat& desc) {
    return run_scan_context(ids, FLB_KF_POSE6, poses6(ids, poses), lidar_height, desc);
  }
  // makeScancontext(*surfCloudKeyFrames[ids[j]]) for every j (the key-frame saver, :2501-2505): descs[j], 20 x 60 each
  template <class Mat, class Alloc>
  bool scan_contexts(const std::vector<int>& ids, double lidar_height, std::vector<Mat, Alloc>& descs) {
    sc_.resize(ids.size() * kScBins + 1);
    if (!ok(flb_keyframes_scan_contexts(kf_, ids.data(), (int)ids.size(), lidar_height, sc_.data()), "scan_contexts")) return false;
    descs.resize(ids.size());
    for (size_t j = 0; j < ids.size(); ++j) to_mat(&sc_[j * kScBins], descs[j]);
    return true;
  }

  // performLoopClosure's ICP (:946-974) on the device: the loop sub-map of (curIds, curT) moved by the pose `com`
  // (transformPointCloud(cureKeyframeCloud, &com), :954-962) registered onto the loop sub-map of (preIds, preT), with the
  // same ids and affines as the Scan Context gate.  No cloud is assembled on the host or downloaded.  com is anything
  // with x, y, z, roll, pitch, yaw (PointTypePose).
  template <class Affine, class Alloc, class Pose>
  bool icp(const std::vector<int>& curIds, const std::vector<Affine, Alloc>& curT, const Pose& com, const std::vector<int>& preIds,
           const std::vector<Affine, Alloc>& preT, const IcpParams& params, IcpResult& result) {
    result = IcpResult();
    if (curT.size() != curIds.size() || preT.size() != preIds.size()) return ok(1, "icp: one affine per key frame");
    if (params.ransac_iterations != 0) {
      std::fprintf(stderr, "[fastlio_b200] KeyFrameStore::icp: RANSAC rejection is not offered (setRANSACIterations(0))\n");
      return false;
    }
    const float pre[6] = {com.x, com.y, com.z, com.roll, com.pitch, com.yaw};
    const std::vector<float> a = affines12(curT), b = affines12(preT);
    return ok(flb_keyframes_icp(kf_, curIds.data(), (int)curIds.size(), FLB_KF_AFFINE, a.data(), pre, preIds.data(), (int)preIds.size(),
                                FLB_KF_AFFINE, b.data(), &params.cfg, &result.r, nullptr, nullptr),
              "icp");
  }

  // IncreMapping's inter-session registrations (doICPVirtualRelative :462-522, doICPGlobalRelative :525-583) of every
  // pair in one call: each selection assembled with its poses and VoxelGrid(leaf)-filtered (leaf 0: dense), each pair
  // registered as icp() registers it with no pre-pose.  results[p] is pair p's registration; stats may be null.
  bool icp_batch(const std::vector<IcpPairSel>& pairs, float leaf, const IcpParams& params, std::vector<IcpResult>& results,
                 flb_icp_batch_stats* stats = nullptr) {
    results.assign(pairs.size(), IcpResult());
    if (params.ransac_iterations != 0) {
      std::fprintf(stderr, "[fastlio_b200] KeyFrameStore::icp_batch: RANSAC rejection is not offered (setRANSACIterations(0))\n");
      return false;
    }
    std::vector<int> so(1, 0), to(1, 0), si, ti;
    std::vector<float> sp, tp;
    for (const IcpPairSel& q : pairs) {
      if (q.srcPoses6.size() != 6 * q.srcIds.size() || q.tgtPoses6.size() != 6 * q.tgtIds.size())
        return ok(1, "icp_batch: one pose per key frame");
      si.insert(si.end(), q.srcIds.begin(), q.srcIds.end());
      ti.insert(ti.end(), q.tgtIds.begin(), q.tgtIds.end());
      sp.insert(sp.end(), q.srcPoses6.begin(), q.srcPoses6.end());
      tp.insert(tp.end(), q.tgtPoses6.begin(), q.tgtPoses6.end());
      so.push_back((int)si.size());
      to.push_back((int)ti.size());
    }
    std::vector<flb_icp_result> r(pairs.size() + 1);
    if (!ok(flb_keyframes_icp_batch(kf_, (int)pairs.size(), so.data(), si.data(), sp.data(), to.data(), ti.data(), tp.data(), leaf,
                                    &params.cfg, r.data(), stats),
            "icp_batch"))
      return false;
    for (size_t p = 0; p < pairs.size(); ++p) results[p].r = r[p];
    return true;
  }

  // pose_estimator::run's registration (pose_estimator.cpp:184-198) with the prior session's key frames in the store:
  // curCloud moved by initPose, onto the key frames ids each moved by pose_ext and then by poses6D.points[ids[j]], with
  // Registeration(params.cfg.mode).run.  T receives res_trans (anything with operator()(row, col) of a 4x4, i.e. the
  // Eigen::MatrixXd the node reads at :197-198, sized by the caller).  Pose is anything with x, y, z, roll, pitch, yaw
  // (PointTypePose); info (optional) receives the whole result.
  template <class Cloud, class Pose, class Poses6D, class Mat>
  bool fricp(const Cloud& curCloud, const Pose& initPose, const std::vector<int>& ids, const Pose& pose_ext, const Poses6D& poses6D,
             const FricpParams& params, Mat& T, flb_fricp_result* info = nullptr) {
    return run_reloc(flb_keyframes_fricp, "fricp", curCloud, initPose, ids, pose_ext, poses6D, params.cfg, T, info);
  }

  // The same registration with regMode 7 (Sparse ICP, registeration.h:143-146): the clouds of fricp(), the result into T.
  template <class Cloud, class Pose, class Poses6D, class Mat>
  bool sicp(const Cloud& curCloud, const Pose& initPose, const std::vector<int>& ids, const Pose& pose_ext, const Poses6D& poses6D,
            const SicpParams& params, Mat& T, flb_sicp_result* info = nullptr) {
    return run_reloc(flb_keyframes_sicp, "sicp", curCloud, initPose, ids, pose_ext, poses6D, params.cfg, T, info);
  }

  // The same registration with regMode 1 (AA-ICP, registeration.h:86-91): the clouds of fricp(), the result into T.
  template <class Cloud, class Pose, class Poses6D, class Mat>
  bool aaicp(const Cloud& curCloud, const Pose& initPose, const std::vector<int>& ids, const Pose& pose_ext, const Poses6D& poses6D,
             const AaicpParams& params, Mat& T, flb_aaicp_result* info = nullptr) {
    return run_reloc(flb_keyframes_aaicp, "aaicp", curCloud, initPose, ids, pose_ext, poses6D, params.cfg, T, info);
  }

  // pcl::copyPointCloud(*surfCloudKeyFrames[k], out)
  template <class Cloud>
  bool at(int k, Cloud& out) {
    const int cap = points(k);
    if (cap < 0) return ok(1, "at");
    xyzi_.resize((size_t)cap * 4 + 4);
    curv_.resize((size_t)cap + 1);
    int n = 0;
    if (!ok(flb_keyframes_download(kf_, k, xyzi_.data(), curv_.data(), cap, &n), "at")) return false;
    out.points.resize(n);
    for (int i = 0; i < n; ++i) fill(out.points[i], &xyzi_[4 * (size_t)i], curv_[i]);
    return true;
  }

 private:
  template <class Poses6D>
  static std::vector<float> poses6(const std::vector<int>& ids, const Poses6D& poses) {
    std::vector<float> p(ids.size() * 6 + 6, 0.f);
    for (size_t j = 0; j < ids.size(); ++j) {
      if (ids[j] < 0 || (size_t)ids[j] >= poses.points.size()) continue;   // the store rejects the id
      const auto& q = poses.points[ids[j]];
      float* o = &p[j * 6];
      o[0] = q.x; o[1] = q.y; o[2] = q.z; o[3] = q.roll; o[4] = q.pitch; o[5] = q.yaw;
    }
    return p;
  }
  template <class Affine, class Alloc>
  static std::vector<float> affines12(const std::vector<Affine, Alloc>& T) {
    std::vector<float> t(T.size() * 12 + 12, 0.f);
    for (size_t j = 0; j < T.size(); ++j)
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 4; ++c) t[j * 12 + r * 4 + c] = T[j](r, c);
    return t;
  }
  // fricp / sicp / aaicp through their C entry point fn: curCloud's records uploaded as they are, res_trans into T
  template <class Cfg, class R, class Cloud, class Pose, class Poses6D, class Mat>
  bool run_reloc(int (*fn)(flb_keyframes*, const void*, int, int, int, const float*, const int*, int, const float*, const float*,
                           const Cfg*, R*, int*, double*, double*, int),
                 const char* what, const Cloud& curCloud, const Pose& initPose, const std::vector<int>& ids, const Pose& pose_ext,
                 const Poses6D& poses6D, const Cfg& cfg, Mat& T, R* info) {
    typedef typename std::remove_reference<decltype(curCloud.points[0])>::type P;
    const int n = (int)curCloud.points.size();
    const P* p0 = n ? &curCloud.points[0] : nullptr;
    const int off_i = n ? (int)((const char*)&p0->intensity - (const char*)p0) : -1;
    const float init6[6] = {initPose.x, initPose.y, initPose.z, initPose.roll, initPose.pitch, initPose.yaw};
    const float ext6[6] = {pose_ext.x, pose_ext.y, pose_ext.z, pose_ext.roll, pose_ext.pitch, pose_ext.yaw};
    const std::vector<float> p6 = poses6(ids, poses6D);
    R r{};
    if (!ok(fn(kf_, p0, n, (int)sizeof(P), off_i, init6, ids.data(), (int)ids.size(), ext6, p6.data(), &cfg, &r, nullptr, nullptr,
               nullptr, 0),
            what))
      return false;
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j) T(i, j) = r.res_trans[4 * i + j];
    if (info) *info = r;
    return true;
  }
  template <class Mat>
  bool run_scan_context(const std::vector<int>& ids, int kind, const std::vector<float>& t, double lidar_height, Mat& desc) {
    sc_.resize(kScBins);
    if (!ok(flb_keyframes_scan_context(kf_, ids.data(), (int)ids.size(), kind, t.data(), lidar_height, sc_.data()), "scan_context"))
      return false;
    to_mat(sc_.data(), desc);
    return true;
  }
  template <class Mat>
  static void to_mat(const double* d, Mat& m) {   // row-major (ring, sector)
    m.resize(FLB_SC_RINGS, FLB_SC_SECTORS);
    for (int r = 0; r < FLB_SC_RINGS; ++r)
      for (int c = 0; c < FLB_SC_SECTORS; ++c) m(r, c) = d[r * FLB_SC_SECTORS + c];
  }
  int selection_size(const std::vector<int>& ids) const {
    long long t = 0;
    for (int k : ids) {
      const int c = points(k);
      if (c < 0) { ok(1, "selection"); return -1; }
      t += c;
    }
    if (t > 0x7fffffffLL) { std::fprintf(stderr, "[fastlio_b200] selection of %lld points is too large\n", t); return -1; }
    return (int)t;
  }
  template <class Cloud>
  bool run_assemble(const std::vector<int>& ids, int kind, const std::vector<float>& t, float leaf, Cloud& out) {
    const int cap = selection_size(ids);
    if (cap < 0) return false;
    xyzi_.resize((size_t)cap * 4 + 4);
    curv_.resize((size_t)cap + 1);
    int n = 0;
    if (!ok(flb_keyframes_assemble(kf_, ids.data(), (int)ids.size(), kind, t.data(), leaf, xyzi_.data(), curv_.data(), cap, &n), "assemble"))
      return false;
    out.points.resize(n);
    for (int i = 0; i < n; ++i) fill(out.points[i], &xyzi_[4 * (size_t)i], curv_[i]);
    return true;
  }
  template <class P>
  static void fill(P& p, const float* v, float curvature) {
    p = P();
    p.x = v[0]; p.y = v[1]; p.z = v[2]; p.intensity = v[3]; p.curvature = curvature;
  }
  static bool ok(int rc, const char* what) {
    if (rc) std::fprintf(stderr, "[fastlio_b200] KeyFrameStore::%s: %s\n", what, flb_last_error());
    return rc == 0;
  }

  flb_keyframes* kf_ = nullptr;
  flb_map* map_ = nullptr;
  static const int kScBins = FLB_SC_RINGS * FLB_SC_SECTORS;
  std::vector<float> xyzi_, curv_;
  std::vector<double> sc_;
};

}  // namespace flb

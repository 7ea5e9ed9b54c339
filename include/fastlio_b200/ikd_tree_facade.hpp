// ikd_tree_facade.hpp — drop-in replacement for the reference's `#include <ikd-Tree/ikd_Tree.h>`:
// the same global names (BoxPointType, delete_point_storage_set, KD_TREE<PointType>) and the public members that
// src/laserMapping.cpp touches (SURVEY.md §8b: Root_Node, PCL_Storage, set_downsample_param, Build, validnum, size,
// Nearest_Search, Add_Points, Delete_Point_Boxes, reconstruct, flatten, acquire_removed_points), implemented on the
// device hashed-voxel map behind the C ABI of fastlio_b200.h.  Reference API: include/ikd-Tree/ikd_Tree.h:225-249.
//
// Differences that are part of the contract (see DESIGN.md §"Deviations"):
//   * only x,y,z of a point are stored in the map; neighbours come back with the other PointType fields zeroed
//     (the hot path reads x,y,z only: laserMapping.cpp:1459-1481, common_lib.h:514-516);
//   * size() == validnum() (no lazily deleted nodes); Add_Point_Boxes (un-delete) is not supported (never called by
//     the reference node); the rebuild thread / balance criteria do not exist (setters are accepted and ignored).
//   * errors never throw: they are reported on stderr and through last_error(); searches then return no neighbours.
#pragma once
#include <pcl/point_types.h>  // same include as ikd_Tree.h:11 (point structs + Eigen::aligned_allocator)
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../fastlio_b200.h"

struct BoxPointType {  // ikd_Tree.h:32-35
  float vertex_min[3];
  float vertex_max[3];
};
enum delete_point_storage_set { NOT_RECORD, DELETE_POINTS_REC, MULTI_THREAD_REC };  // ikd_Tree.h:39

template <typename PointType>
class KD_TREE {
 public:
  using PointVector = std::vector<PointType, Eigen::aligned_allocator<PointType>>;
  using Ptr = std::shared_ptr<KD_TREE<PointType>>;
  struct KD_TREE_NODE {};  // opaque: callers only compare Root_Node with nullptr / pass it back to flatten()

  explicit KD_TREE(float delete_param = 0.5f, float balance_param = 0.6f, float box_length = 0.2f)
      : downsample_size_(box_length) { (void)delete_param; (void)balance_param; }
  ~KD_TREE() { if (map_) flb_map_destroy(map_); }
  KD_TREE(const KD_TREE&) = delete;
  KD_TREE& operator=(const KD_TREE&) = delete;

  // capacity knobs (no reference counterpart; call before the first Build/Add)
  void set_capacity(int max_points, int max_blocks = 0, int device = 0) { max_points_ = max_points; max_blocks_ = max_blocks; device_ = device; }

  void Set_delete_criterion_param(float) {}
  void Set_balance_criterion_param(float) {}
  void set_downsample_param(float box_length) {
    downsample_size_ = box_length;
    if (map_ && flb_map_set_downsample_param(map_, box_length)) report("set_downsample_param");
  }
  void InitializeKDTree(float, float, float box_length = 0.2f) { set_downsample_param(box_length); }

  int size() { return map_ ? flb_map_size(map_) : 0; }
  int validnum() { return map_ ? flb_map_validnum(map_) : 0; }
  void root_alpha(float& alpha_bal, float& alpha_del) { alpha_bal = 0.5f; alpha_del = 0.f; }

  void Build(PointVector point_cloud) {
    if (!ensure()) return;
    if (flb_map_build_pt(map_, xyz(point_cloud), (int)point_cloud.size(), (int)sizeof(PointType), off_intensity())) report("Build");
    sync_root();
  }
  void reconstruct(PointVector point_cloud) {
    if (!ensure()) return;
    if (flb_map_reconstruct_pt(map_, xyz(point_cloud), (int)point_cloud.size(), (int)sizeof(PointType), off_intensity())) report("reconstruct");
    sync_root();
  }

  void Nearest_Search(PointType point, int k_nearest, PointVector& Nearest_Points, std::vector<float>& Point_Distance,
                      double max_dist = INFINITY) {
    PointVector().swap(Nearest_Points);
    std::vector<float>().swap(Point_Distance);
    if (!map_ || k_nearest < 1) return;
    std::vector<float> oxyz((size_t)k_nearest * 4), od2(k_nearest);
    int cnt = 0;
    const float md = std::isfinite(max_dist) ? (float)max_dist : 0.f;
    if (flb_map_nearest_search_xyzi(map_, &point.x, 1, (int)sizeof(PointType), k_nearest, md, oxyz.data(), od2.data(), &cnt)) {
      report("Nearest_Search");
      return;
    }
    fill(Nearest_Points, oxyz.data(), cnt);
    Point_Distance.assign(od2.begin(), od2.begin() + cnt);
  }
  // Batched form (what the GPU wants): nq queries at once. Outputs are [nq][k] row-major; counts[nq].
  int Nearest_Search_Batch(const PointVector& queries, int k_nearest, std::vector<float>& out_xyz, std::vector<float>& out_d2,
                           std::vector<int>& counts, double max_dist = INFINITY) {
    const int nq = (int)queries.size();
    out_xyz.assign((size_t)nq * k_nearest * 3, NAN);
    out_d2.assign((size_t)nq * k_nearest, INFINITY);
    counts.assign(nq, 0);
    if (!map_ || nq == 0) return 0;
    const float md = std::isfinite(max_dist) ? (float)max_dist : 0.f;
    if (flb_map_nearest_search(map_, xyz(queries), nq, (int)sizeof(PointType), k_nearest, md, out_xyz.data(), out_d2.data(), counts.data())) {
      report("Nearest_Search_Batch");
      return 1;
    }
    return 0;
  }
  void Box_Search(const BoxPointType& Box_of_Point, PointVector& Storage) {
    Storage.clear();
    if (!map_) return;
    const float b[6] = {Box_of_Point.vertex_min[0], Box_of_Point.vertex_min[1], Box_of_Point.vertex_min[2],
                        Box_of_Point.vertex_max[0], Box_of_Point.vertex_max[1], Box_of_Point.vertex_max[2]};
    int n = 0;
    if (flb_map_box_search_xyzi(map_, b, nullptr, 0, &n)) { report("Box_Search"); return; }
    std::vector<float> o((size_t)std::max(n, 1) * 4);
    if (flb_map_box_search_xyzi(map_, b, o.data(), n, &n)) { report("Box_Search"); return; }
    fill(Storage, o.data(), n);
  }
  void Radius_Search(PointType point, const float radius, PointVector& Storage) {
    Storage.clear();
    if (!map_) return;
    int n = 0;
    if (flb_map_radius_search_xyzi(map_, &point.x, radius, nullptr, 0, &n)) { report("Radius_Search"); return; }
    std::vector<float> o((size_t)std::max(n, 1) * 4);
    if (flb_map_radius_search_xyzi(map_, &point.x, radius, o.data(), n, &n)) { report("Radius_Search"); return; }
    fill(Storage, o.data(), n);
  }

  int Add_Points(PointVector& PointToAdd, bool downsample_on) {
    if (PointToAdd.empty()) return 0;
    if (!ensure()) return 0;
    int added = 0;
    if (flb_map_add_points_pt(map_, xyz(PointToAdd), (int)PointToAdd.size(), (int)sizeof(PointType), off_intensity(), downsample_on ? 1 : 0, &added)) report("Add_Points");
    sync_root();
    return added;
  }
  void Add_Point_Boxes(std::vector<BoxPointType>&) { std::fprintf(stderr, "[fastlio_b200] Add_Point_Boxes is not supported (unused by the reference node)\n"); }
  void Delete_Points(PointVector& PointToDel) {
    if (!map_ || PointToDel.empty()) return;
    int nd = 0;
    if (flb_map_delete_points(map_, xyz(PointToDel), (int)PointToDel.size(), (int)sizeof(PointType), &nd)) report("Delete_Points");
  }
  int Delete_Point_Boxes(std::vector<BoxPointType>& BoxPoints) {
    if (!map_ || BoxPoints.empty()) return 0;
    static_assert(sizeof(BoxPointType) == 6 * sizeof(float), "BoxPointType must be 6 packed floats");
    int nd = 0;
    if (flb_map_delete_boxes(map_, BoxPoints[0].vertex_min, (int)BoxPoints.size(), &nd)) report("Delete_Point_Boxes");
    return nd;
  }
  void flatten(KD_TREE_NODE* root, PointVector& Storage, delete_point_storage_set) {
    if (!root || !map_) return;
    int n = 0;
    if (flb_map_flatten_xyzi(map_, nullptr, 0, &n)) { report("flatten"); return; }
    std::vector<float> o((size_t)std::max(n, 1) * 4);
    if (flb_map_flatten_xyzi(map_, o.data(), n, &n)) { report("flatten"); return; }
    const size_t base = Storage.size();
    Storage.resize(base + n);
    for (int i = 0; i < n; ++i) set(Storage[base + i], &o[4 * (size_t)i]);
  }
  void acquire_removed_points(PointVector& removed_points) { (void)removed_points; }  // dead in the reference (laserMapping.cpp:1124-1130)
  BoxPointType tree_range() {
    BoxPointType b{};
    float r[6] = {0, 0, 0, 0, 0, 0};
    if (map_ && flb_map_range(map_, r)) report("tree_range");
    for (int i = 0; i < 3; ++i) { b.vertex_min[i] = r[i]; b.vertex_max[i] = r[3 + i]; }
    return b;
  }

  flb_map* handle() { ensure(); return map_; }  // for flb_session_create
  // Root_Node after the map was rebuilt through another C-ABI call on handle() (flb::KeyFrameStore::reconstruct)
  void refresh_root() { sync_root(); }
  const std::string& last_error() const { return err_; }

  PointVector PCL_Storage;           // ikd_Tree.h:247
  KD_TREE_NODE* Root_Node = nullptr; // ikd_Tree.h:248
  int max_queue_size = 0;

 private:
  bool ensure() {
    if (map_) return true;
    flb_map_config c;
    c.voxel_size = downsample_size_;
    c.max_points = max_points_;
    c.max_blocks = max_blocks_;
    c.device = device_;
    if (flb_map_create(&c, &map_)) { map_ = nullptr; report("KD_TREE (flb_map_create)"); return false; }
    return true;
  }
  void sync_root() { Root_Node = (map_ && flb_map_has_root(map_)) ? &dummy_ : nullptr; }
  void report(const char* where) {
    err_ = std::string(where) + ": " + flb_last_error();
    std::fprintf(stderr, "[fastlio_b200] %s\n", err_.c_str());
  }
  static const float* xyz(const PointVector& v) { return v.empty() ? nullptr : &v[0].x; }
  // the map keeps x, y, z, intensity of every point (what FAST-LIO's map points carry: normals and curvature are zero,
  // laserMapping.cpp:1101-1110); records handed back have those four fields set and the rest zeroed
  static int off_intensity() { return (int)offsetof(PointType, intensity); }
  static void set(PointType& p, const float* c) { std::memset(&p, 0, sizeof(PointType)); p.x = c[0]; p.y = c[1]; p.z = c[2]; p.intensity = c[3]; }
  static void fill(PointVector& out, const float* c, int n) {
    out.resize(n);
    for (int i = 0; i < n; ++i) set(out[i], c + 4 * (size_t)i);
  }

  flb_map* map_ = nullptr;
  float downsample_size_ = 0.2f;
  int max_points_ = 0, max_blocks_ = 0, device_ = 0;
  KD_TREE_NODE dummy_;
  std::string err_;
};

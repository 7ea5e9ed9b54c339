// frontend_host.cuh — C-ABI entry points of the rows either side of the per-scan path (SURVEY.md §8f ranks 1-4).
// Included at the end of fastlio_b200.cu (uses its flb_map / flb_session definitions and error helpers).
#pragma once
#include "frontend_kernels.cuh"
#include <cub/device/device_radix_sort.cuh>

// ------------------------------------------------------------------------------------------------ voxel-grid workspace
struct VgWork {
  int cap = 0;   // points the arrays and the CUB scratch are sized for
  DevBuf<unsigned> keys_a, keys_b;
  DevBuf<int> vals_a, vals_b, flags, pos;
  DevBuf<unsigned char> tmp;   // CUB temporary storage
  DevBuf<unsigned> d_mm;       // 8 words, see k_vg_init
  PinnedBuf<unsigned> h_mm;    // pinned mirror
};
static int vg_ensure(VgWork& w, int n) {
  if (n <= w.cap) return 0;
  w.cap = 0;   // (until every array has grown)
  const int cap = std::max(n, 1 << 12);
  size_t t1 = 0, t2 = 0;
  CU(cub::DeviceRadixSort::SortPairs(nullptr, t1, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, cap));
  CU(cub::DeviceScan::ExclusiveSum(nullptr, t2, (const int*)nullptr, (int*)nullptr, cap));
  const size_t words = sizeof(unsigned) * (size_t)cap;
  if (grow(w.keys_a, words, 0) || grow(w.keys_b, words, 0) || grow(w.vals_a, words, 0) || grow(w.vals_b, words, 0) ||
      grow(w.flags, words, 0) || grow(w.pos, words, 0) || grow(w.tmp, std::max(t1, t2) + 256, 0) ||
      grow(w.d_mm, sizeof(unsigned) * 8, 0) || grow(w.h_mm, sizeof(unsigned) * 8, 0))
    return 1;
  w.cap = cap;
  return 0;
}
static size_t vg_device_bytes(const VgWork& w) {
  return w.keys_a.cap + w.keys_b.cap + w.vals_a.cap + w.vals_b.cap + w.flags.cap + w.pos.cap + w.tmp.cap + w.d_mm.cap;
}

// pcl::VoxelGrid::applyFilter on n device points (x,y,z,intensity [+curvature]) -> out (capacity out_cap points), all on
// `st`.  The output count and PCL's overflow flag are copied to w.h_mm[7] / w.h_mm[6]; valid after the stream drained.
static int vg_enqueue(flb_map* m, VgWork& w, const float4* pts, const float* curv, int n, float leaf, float4* out, float* out_curv,
                      int out_cap, cudaStream_t st) {
  if (vg_ensure(w, n)) return 1;
  unsigned* mm = w.d_mm.p;
  const float inv = 1.0f / leaf;   // inverse_leaf_size_
  const int g = grid_for(std::max(n, 1), 256, m->sm_count * 8);
  k_vg_init<<<1, 32, 0, st>>>(mm);
  m->launches++;
  if (n > 0) {
    k_vg_minmax<<<g, 256, 0, st>>>(pts, n, mm);
    k_vg_keys<<<g, 256, 0, st>>>(pts, n, inv, mm, w.keys_a.p, w.vals_a.p);
    size_t tb = w.tmp.cap;
    CU(cub::DeviceRadixSort::SortPairs(w.tmp.p, tb, (const unsigned*)w.keys_a.p, w.keys_b.p, (const int*)w.vals_a.p, w.vals_b.p, n, 0, 32, st));
    k_vg_heads<<<g, 256, 0, st>>>(w.keys_b.p, n, w.flags.p);
    tb = w.tmp.cap;
    CU(cub::DeviceScan::ExclusiveSum(w.tmp.p, tb, (const int*)w.flags.p, w.pos.p, n, st));
    k_vg_centroid<<<g, 256, 0, st>>>(pts, curv, w.keys_b.p, w.vals_b.p, w.flags.p, w.pos.p, n, out, out_curv, out_cap, mm);
    m->launches += 4 + 6;   // + the radix-sort (histogram, 4 onesweep passes) and scan kernels of CUB
  }
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(w.h_mm.p, mm, sizeof(unsigned) * 8, cudaMemcpyDeviceToHost, st));
  return 0;
}

// ------------------------------------------------------------------------------------------------ front end object
struct PpWork;                          // preprocess scratch (preprocess_host.cuh)
static void pp_release(PpWork* w);
struct ColorCam;                        // camera state of the colour publisher (color_host.cuh)
static void cam_release(ColorCam* c);
struct flb_frontend {
  flb_session* ses = nullptr;
  int cap = 0;
  int n_raw = 0;            // points of the current raw scan (meas.lidar)
  int n_down = -1;          // points of feats_down_body after the last voxel filter (-1: none yet)
  bool sorted = false;      // pts_t holds feats_undistort (time order); else `pts` (upload order) is current
  DevBuf<unsigned char> raw;   // staging of host records
  float4 *pts = nullptr, *pts_t = nullptr;
  float *curv = nullptr, *curv_t = nullptr, *down_curv = nullptr;
  int* perm = nullptr;      // time-sorted position -> upload index
  float4* world = nullptr;  // publish scratch
  double *d_poses = nullptr, *h_poses = nullptr;
  cudaEvent_t ev_poses = nullptr;
  VgWork vg;
  PpWork* pp = nullptr;
  ColorCam* cam = nullptr;  // null until flb_frontend_camera_config
  bool holds_ref = false;
};

extern "C" int flb_frontend_create(flb_session* s, int max_raw_points, flb_frontend** out) {
  if (!s || !out) return set_err("flb_frontend_create: null argument");
  if (max_raw_points <= 0) return set_err("max_raw_points must be > 0");
  CU(cudaSetDevice(s->map->cfg.device));
  flb_frontend* f = new (std::nothrow) flb_frontend();
  if (!f) return set_err("out of host memory");
  f->ses = s;
  f->cap = max_raw_points;
  const size_t N = (size_t)max_raw_points;
  cudaError_t e = cudaSuccess;
  auto A = [&](void** p, size_t b) { if (e == cudaSuccess) e = cudaMalloc(p, b); };
  A((void**)&f->pts, sizeof(float4) * N);
  A((void**)&f->pts_t, sizeof(float4) * N);
  A((void**)&f->world, sizeof(float4) * N);
  A((void**)&f->curv, sizeof(float) * N);
  A((void**)&f->curv_t, sizeof(float) * N);
  A((void**)&f->down_curv, sizeof(float) * N);
  A((void**)&f->perm, sizeof(int) * N);
  A((void**)&f->d_poses, sizeof(double) * IMU_POSE_DOUBLES * MAX_IMU_POSES);
  if (e == cudaSuccess) e = cudaMallocHost((void**)&f->h_poses, sizeof(double) * IMU_POSE_DOUBLES * MAX_IMU_POSES);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&f->ev_poses, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    cudaGetLastError();
    flb_frontend_destroy(f);
    return set_err("flb_frontend_create: %s", cudaGetErrorString(e));
  }
  if (vg_ensure(f->vg, max_raw_points)) { flb_frontend_destroy(f); return 1; }
  s->map->refs++;   // keeps the map (and its stream) alive
  f->holds_ref = true;
  *out = f;
  return 0;
}

extern "C" void flb_frontend_destroy(flb_frontend* f) {
  if (!f) return;
  flb_map* m = f->ses ? f->ses->map : nullptr;
  if (m) { Q(cudaSetDevice(m->cfg.device)); Q(cudaStreamSynchronize(m->stream)); }
  void* ptrs[] = {f->pts, f->pts_t, f->world, f->curv, f->curv_t, f->down_curv, f->perm, f->d_poses};
  for (void* p : ptrs) if (p) Q(cudaFree(p));
  if (f->h_poses) Q(cudaFreeHost(f->h_poses));
  if (f->ev_poses) Q(cudaEventDestroy(f->ev_poses));
  const bool counted = f->holds_ref;
  pp_release(f->pp);
  cam_release(f->cam);
  delete f;
  if (m && counted) map_release(m);
}

static inline const float4* fe_cloud(const flb_frontend* f) { return f->sorted ? f->pts_t : f->pts; }
static inline const float* fe_curv(const flb_frontend* f) { return f->sorted ? f->curv_t : f->curv; }

extern "C" int flb_frontend_upload(flb_frontend* f, const void* pts, int n, int stride, int off_intensity, int off_curvature) {
  if (!f) return set_err("null front end");
  if (n < 0 || n > f->cap) return set_err("raw scan of %d points exceeds max_raw_points=%d", n, f->cap);
  if (n > 0 && (!pts || stride < 12)) return set_err("bad raw scan buffer");
  if ((off_intensity >= 0 && off_intensity + 4 > stride) || (off_curvature >= 0 && off_curvature + 4 > stride))
    return set_err("field offset outside the point stride");
  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  f->n_raw = n;
  f->sorted = false;
  f->n_down = -1;
  if (n == 0) return 0;
  // the staging is sized once for the capacity (scans vary in size); with the curvature always written, every stride packs
  return upload_records(m, m->stream, f->raw, (size_t)f->cap * (size_t)stride, pts, n, stride, off_intensity, off_curvature, f->pts, f->curv);
}

// time sort + backward compensation of the current raw scan (n_raw > 0) with the poses in f->d_poses, on the map stream.
// end26 / np_dev null: end pose `e` and n_poses from the host; else both are read on the device and n_poses is the
// capacity the launch reserves (see k_undistort).
static int fe_undistort_enqueue(flb_frontend* f, int n_poses, const UndistortEnd& e, const double* end26, const int* np_dev) {
  flb_map* m = f->ses->map;
  cudaStream_t st = m->stream;
  const int n = f->n_raw;
  const int g = grid_for(n, 256, m->sm_count * 8);
  // sort(pcl_out.points.begin(), pcl_out.points.end(), time_list)  (IMU_Processing.hpp:243) — stable here
  VgWork& v = f->vg;
  k_time_keys<<<g, 256, 0, st>>>(f->curv, v.keys_a.p, v.vals_a.p, n);
  size_t tb = v.tmp.cap;
  CU(cub::DeviceRadixSort::SortPairs(v.tmp.p, tb, (const unsigned*)v.keys_a.p, v.keys_b.p, (const int*)v.vals_a.p, f->perm, n, 0, 32, st));
  k_undistort<<<g, 256, sizeof(double) * IMU_POSE_DOUBLES * (size_t)n_poses, st>>>(f->pts, f->curv, f->perm, n, f->d_poses, n_poses, e,
                                                                                  f->pts_t, f->curv_t, end26, np_dev);
  m->launches += 2 + 5;
  CU(cudaGetLastError());
  f->sorted = true;
  return 0;
}

extern "C" int flb_frontend_undistort(flb_frontend* f, const double* imu_poses22, int n_poses, const double* state26_end) {
  if (!f) return set_err("null front end");
  if (!imu_poses22 || !state26_end) return set_err("flb_frontend_undistort: null argument");
  if (n_poses < 1 || n_poses > MAX_IMU_POSES) return set_err("n_poses must be in [1, %d]", MAX_IMU_POSES);
  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  const int n = f->n_raw;
  if (n == 0) { f->sorted = true; return 0; }
  cudaStream_t st = m->stream;
  // pinned staging (a pageable cudaMemcpyAsync measured ~7 ms per call here); the event guards its reuse
  CU(cudaEventSynchronize(f->ev_poses));
  memcpy(f->h_poses, imu_poses22, sizeof(double) * IMU_POSE_DOUBLES * (size_t)n_poses);
  CU(cudaMemcpyAsync(f->d_poses, f->h_poses, sizeof(double) * IMU_POSE_DOUBLES * (size_t)n_poses, cudaMemcpyHostToDevice, st));
  CU(cudaEventRecord(f->ev_poses, st));
  UndistortEnd e;
  for (int k = 0; k < 4; ++k) { e.rot[k] = state26_end[3 + k]; e.offR[k] = state26_end[7 + k]; }
  for (int k = 0; k < 3; ++k) { e.pos[k] = state26_end[k]; e.offT[k] = state26_end[11 + k]; }
  return fe_undistort_enqueue(f, n_poses, e, nullptr, nullptr);
}

extern "C" int flb_frontend_voxel_filter(flb_frontend* f, float leaf, int* n_out) {
  if (!f) return set_err("null front end");
  if (!(leaf > 0.f)) return set_err("leaf size must be > 0");
  flb_session* s = f->ses;
  flb_map* m = s->map;
  CU(cudaSetDevice(m->cfg.device));
  if (s->pending_n >= 0) return set_err("flb_frontend_voxel_filter: a prefetched scan is pending on this session");
  const int n = f->n_raw;
  // the centroids are written straight into the session's feats_down_body buffer
  if (vg_enqueue(m, f->vg, fe_cloud(f), fe_curv(f), n, leaf, s->body, f->down_curv, s->cap, m->stream)) return 1;
  CU(cudaStreamSynchronize(m->stream));
  int nd = (int)f->vg.h_mm.p[7];
  if (f->vg.h_mm.p[6]) {
    // PCL: "Leaf size is too small for the input dataset. Integer indices would overflow." -> output = input
    if (n > s->cap) return set_err("voxel filter overflow guard: unfiltered scan of %d points exceeds max_scan_points=%d", n, s->cap);
    CU(cudaMemcpyAsync(s->body, fe_cloud(f), sizeof(float4) * (size_t)n, cudaMemcpyDeviceToDevice, m->stream));
    CU(cudaMemcpyAsync(f->down_curv, fe_curv(f), sizeof(float) * (size_t)n, cudaMemcpyDeviceToDevice, m->stream));
    nd = n;
  }
  if (nd > s->cap) return set_err("filtered scan of %d points exceeds max_scan_points=%d", nd, s->cap);
  f->n_down = nd;
  if (n_out) *n_out = nd;
  return scan_reset(s, nd);
}

// upload + undistort + voxel filter in one call (one synchronisation): meas.lidar -> feats_down_body on the device
extern "C" int flb_frontend_process(flb_frontend* f, const void* pts, int n, int stride, int off_intensity, int off_curvature,
                                    const double* imu_poses22, int n_poses, const double* state26_end, float leaf, int* n_out) {
  if (flb_frontend_upload(f, pts, n, stride, off_intensity, off_curvature)) return 1;
  if (imu_poses22 && n_poses > 0 && flb_frontend_undistort(f, imu_poses22, n_poses, state26_end)) return 1;
  return flb_frontend_voxel_filter(f, leaf, n_out);
}

static int fe_download(flb_map* m, const float4* src, const float* src_curv, int n, float* out_xyzi, float* out_curv, int cap) {
  const int c = std::min(n, cap);
  if (c > 0 && out_xyzi) CU(cudaMemcpyAsync(out_xyzi, src, sizeof(float4) * (size_t)c, cudaMemcpyDeviceToHost, m->stream));
  if (c > 0 && out_curv && src_curv) CU(cudaMemcpyAsync(out_curv, src_curv, sizeof(float) * (size_t)c, cudaMemcpyDeviceToHost, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  return 0;
}

extern "C" int flb_frontend_download_undistorted(flb_frontend* f, float* out_xyzi, float* out_curv, int* out_perm, int cap, int* n) {
  if (!f) return set_err("null front end");
  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  if (n) *n = f->n_raw;
  const int c = std::min(f->n_raw, cap);
  if (c > 0 && out_perm) {
    if (f->sorted) CU(cudaMemcpyAsync(out_perm, f->perm, sizeof(int) * (size_t)c, cudaMemcpyDeviceToHost, m->stream));
    else for (int i = 0; i < c; ++i) out_perm[i] = i;
  }
  return fe_download(m, fe_cloud(f), fe_curv(f), f->n_raw, out_xyzi, out_curv, cap);
}

extern "C" int flb_frontend_download_down(flb_frontend* f, float* out_xyzi, float* out_curv, int cap, int* n) {
  if (!f) return set_err("null front end");
  if (f->n_down < 0) return set_err("flb_frontend_download_down: no filtered scan yet");
  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  if (n) *n = f->n_down;
  return fe_download(m, f->ses->body, f->down_curv, f->n_down, out_xyzi, out_curv, cap);
}

extern "C" int flb_frontend_points_to_world(flb_frontend* f, int which, const double* state26, float* out_xyzi, int cap, int* n) {
  if (!f) return set_err("null front end");
  if (!state26) return set_err("null state");
  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  const float4* src;
  int cnt;
  if (which == 0) {   // feats_down_body (dense_pub_en == false)
    src = f->ses->body;
    cnt = f->ses->n;
  } else if (which == 1) {   // feats_undistort (dense_pub_en == true, map_save_en)
    src = fe_cloud(f);
    cnt = f->n_raw;
  } else {
    return set_err("which must be 0 (feats_down_body) or 1 (feats_undistort)");
  }
  if (n) *n = cnt;
  if (cnt > f->cap) return set_err("cloud of %d points exceeds the front end capacity %d", cnt, f->cap);
  if (cnt > 0) {
    k_transform<<<grid_for(cnt, 256, m->sm_count * 8), 256, 0, m->stream>>>(pose_from(state26), src, f->world, cnt);
    m->launches++;
    CU(cudaGetLastError());
  }
  return fe_download(m, f->world, nullptr, cnt, out_xyzi, nullptr, cap);
}

// ------------------------------------------------------------------------------------------------ stand-alone filters
extern "C" int flb_voxel_grid_filter(flb_map* m, const void* pts, int n, int stride, int off_intensity, float leaf, float* out_xyzi,
                                     int cap, int* n_out) {
  if (!m) return set_err("null map");
  if (n_out) *n_out = 0;
  if (n < 0) return set_err("negative point count");
  if (!(leaf > 0.f)) return set_err("leaf size must be > 0");
  if (n == 0) return 0;
  if (!pts || stride < 12) return set_err("bad point buffer");
  if (off_intensity >= 0 && off_intensity + 4 > stride) return set_err("field offset outside the point stride");
  CU(cudaSetDevice(m->cfg.device));
  VgWork w;                     // per-call workspace and staging, freed on return
  DevBuf<unsigned char> raw;
  float4 *in = nullptr, *out = nullptr;
  int rc = 0;
  auto body = [&]() -> int {
    CU(cudaMalloc((void**)&in, sizeof(float4) * (size_t)n));
    CU(cudaMalloc((void**)&out, sizeof(float4) * (size_t)n));
    if (upload_records(m, m->stream, raw, 0, pts, n, stride, off_intensity, -1, in, nullptr)) return 1;
    if (vg_enqueue(m, w, in, nullptr, n, leaf, out, nullptr, n, m->stream)) return 1;
    CU(cudaStreamSynchronize(m->stream));
    const bool ovf = w.h_mm.p[6] != 0;
    const int nd = ovf ? n : (int)w.h_mm.p[7];
    if (n_out) *n_out = nd;
    const int c = std::min(nd, cap);
    if (c > 0 && out_xyzi) CU(cudaMemcpy(out_xyzi, ovf ? in : out, sizeof(float4) * (size_t)c, cudaMemcpyDeviceToHost));
    return 0;
  };
  rc = body();
  if (in) Q(cudaFree(in));
  if (out) Q(cudaFree(out));
  return rc;
}

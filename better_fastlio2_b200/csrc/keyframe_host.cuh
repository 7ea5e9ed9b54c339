// keyframe_host.cuh — the device key-frame store (flb_keyframes) and the readers of the key-frame clouds
// (surfCloudKeyFrames, laserMapping.cpp:756-758): the sub-map rebuild (recontructIKdTree :612-669), the loop sub-maps
// (loopFindNearKeyframes :856-883), the published global map (publishGlobalMap :1840-1872) and the saved maps
// (saveMapService :1763-1798, the per-key-frame saver :2501-2530).  Every reader assembles its selection with one
// k_kf_assemble launch.  Included at the end of fastlio_b200.cu after frontend_host.cuh (uses VgWork, flb_frontend).
#pragma once
#include "icp_batch_kernels.cuh"
#include "icp_kernels.cuh"
#include "keyframe_kernels.cuh"
#include "scan_context_kernels.cuh"

// ------------------------------------------------------------------------------------------------ map-side scratch
// Kept with the map and only ever grown, like kf_raw / kf_in / kf_out: the readers run every kd_step key frames or on a
// service call with selections of similar size, and cudaMalloc / cudaFree of a few hundred MB cost more than the kernels.
// Each path allocates only the buffers it uses; flb_keyframes_info reports the total and
// flb_map_release_keyframe_scratch frees it (e.g. after saving a map of the whole run).
// The grid index of flb_keyframes_icp and flb_keyframes_fricp (icp_host.cuh) and the reductions' scratch.  Both calls
// run on the map's stream and synchronise before returning, so they share it.
struct IcpIndex {
  DevBuf<float4> sorted;                       // sorted finite target (w = original index)
  DevBuf<unsigned> keys_a, keys_b;             // radix-sort keys
  DevBuf<int> vals_a, vals_b, order, open;     // radix-sort values (vals_b: the sorted original indices); source visiting
                                               // order; open queries of the fine rings
  DevBuf<int> cs;                              // CSR cell offsets (n_cells + 1)
  DevBuf<IcpBox> box;                          // coarse-cell point boxes
  DevBuf<unsigned char> tmp;                   // CUB temporary storage
  DevBuf<double> partials;                     // reduction block partials
  DevBuf<unsigned> misc;                       // bounds keys (6), finite count, open count, reduction counter
  PinnedBuf<unsigned> h_misc;
};

// flb_keyframes_icp's own scratch (icp_host.cuh)
struct IcpWork {
  DevBuf<float4> src_raw, src, x, tgt;         // assembled source, pre-transformed source, input_transformed, target
  DevBuf<int> corr;                            // nearest target per source
  DevBuf<float> corr_d2;
  DevBuf<double> sums;                         // the pairs record (8) and the cross products (9)
  PinnedBuf<double> h_sums;
};

// flb_keyframes_icp_batch's own scratch (icp_batch_host.cuh): one round's pairs packed back to back
struct IcpBatchWork {
  DevBuf<float4> raw;                          // dense assembly of one selection before its voxel grid
  DevBuf<float4> src, tgt, x, sorted;          // sources, targets, moved sources, sorted finite targets (w = index)
  DevBuf<int> order, corr, cs;                 // sources' visiting order, nearest target per source, CSR cell offsets
  DevBuf<float> corr_d2;
  DevBuf<int2> open;                           // open queries of the fine rings (source index, item)
  DevBuf<IcpBox> box;                          // coarse-cell point boxes
  DevBuf<IcpBatchItem> items;                  // the active pairs of a pass
  PinnedBuf<IcpBatchItem> h_items;             //   and their staging
  DevBuf<double> partials, sums;               // reduction block partials; the pairs' sum records (ICPB_REC each)
  PinnedBuf<double> h_sums;
  DevBuf<unsigned> counters;                   // one reduction counter per pair, then the open count
};

// flb_keyframes_fricp's own scratch (fricp_host.cuh)
struct FricpWork {
  DevBuf<unsigned char> raw;                   // staged source records
  DevBuf<float4> src_raw, src, tgt_a, tgt, tgtf;   // uploaded / pre-transformed source, the two target stages, float target
  DevBuf<double4> x, tn, sorted_d;             // normalised source, normalised target, sorted finite target (w = index)
  DevBuf<int> pos, corr;                       // sorted position of the nearest target; its original index
  DevBuf<double> d2, med, sort_a, sort_b;      // 1-NN d²; 7-NN medians; sort input / output of a median
  DevBuf<double> sums;                         // reduction records
  PinnedBuf<double> h_sums;
};

// flb_keyframes_sicp's own scratch (sicp_host.cuh); its clouds, matches and index are flb_keyframes_fricp's
struct SicpWork {
  DevBuf<double4> q, z, c, xo2;                // per source point: match, shrunk residual, multiplier, X of the last ICP
                                               // iteration
  DevBuf<double> sched;                        // μ, Ba, ha per outer iteration
  PinnedBuf<double> h_sched;
  DevBuf<double> part, rec;                    // the ADMM kernel's block partials and its per-iteration record
  PinnedBuf<double> h_rec;
};

struct KfWork {
  VgWork vg;                                   // voxel grid of the sub-map / saved map
  DevBuf<float> cin, cout;                     // curvature of an assembly and of its filtered output
  DevBuf<KfSeg> d_seg;                         // segment table of k_kf_assemble
  PinnedBuf<KfSeg> h_seg;                      //   and its staging
  cudaEvent_t ev_seg = nullptr;                // the last copy out of h_seg
  DevBuf<ScChunk> d_chunk;                     // chunk table of k_sc_bins
  PinnedBuf<ScChunk> h_chunk;                  //   and its staging
  DevBuf<unsigned> d_sc_keys;                  // Scan Context keys, SC_BINS per descriptor
  PinnedBuf<unsigned> h_sc_keys;               //   and their staging
  IcpIndex index;                              // the registrations' target index and reductions
  IcpWork icp;                                 // flb_keyframes_icp's sub-maps and matches
  IcpBatchWork icpb;                           // flb_keyframes_icp_batch's packed rounds
  FricpWork fricp;                             // flb_keyframes_fricp's clouds, matches and medians
  SicpWork sicp;                               // flb_keyframes_sicp's ADMM state
};

static void kfw_release(KfWork* w) {
  if (!w) return;
  if (w->ev_seg) Q(cudaEventDestroy(w->ev_seg));
  delete w;
}

// growth policy of the key-frame buffers that follow the selection size: a quarter of headroom
template <typename T>
static int kf_grow(DevBuf<T>& b, size_t need) { return grow(b, need, need + need / 4); }

// The map's KfWork, created on first use.
static int kf_work(flb_map* m) {
  if (m->kfw) return 0;
  cudaEvent_t ev = nullptr;
  CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  m->kfw = new (std::nothrow) KfWork();
  if (!m->kfw) { Q(cudaEventDestroy(ev)); return set_err("out of host memory"); }
  m->kfw->ev_seg = ev;
  return 0;
}

// Scratch for an assembly of n points: kf_in (the assembled cloud) and, when asked for, its curvature; with a filter
// also kf_out (the filtered cloud), its curvature and the voxel-grid workspace.  A failure leaves the map's contents
// untouched.
static int kf_scratch(flb_map* m, int n, bool curv, bool filter) {
  if (kf_work(m)) return 1;
  KfWork& w = *m->kfw;
  const size_t pts = sizeof(float4) * (size_t)n, cur = sizeof(float) * (size_t)n;
  if (kf_grow(m->kf_in, pts)) return 1;
  if (curv && kf_grow(w.cin, cur)) return 1;
  if (!filter) return 0;
  if (kf_grow(m->kf_out, pts)) return 1;
  if (curv && kf_grow(w.cout, cur)) return 1;
  return vg_ensure(w.vg, n);
}

static long long kf_scratch_bytes(const flb_map* m) {
  size_t b = m->kf_raw.cap + m->kf_in.cap + m->kf_out.cap;   // device bytes (the pinned staging is not counted)
  if (const KfWork* w = m->kfw) {
    const IcpIndex& x = w->index;
    const IcpWork& i = w->icp;
    const FricpWork& f = w->fricp;
    b += w->cin.cap + w->cout.cap + w->d_seg.cap + w->d_chunk.cap + w->d_sc_keys.cap + vg_device_bytes(w->vg);
    b += x.sorted.cap + x.keys_a.cap + x.keys_b.cap + x.vals_a.cap + x.vals_b.cap + x.order.cap + x.open.cap + x.cs.cap + x.box.cap +
         x.tmp.cap + x.partials.cap + x.misc.cap;
    b += i.src_raw.cap + i.src.cap + i.x.cap + i.tgt.cap + i.corr.cap + i.corr_d2.cap + i.sums.cap;
    const IcpBatchWork& bw = w->icpb;
    b += bw.raw.cap + bw.src.cap + bw.tgt.cap + bw.x.cap + bw.sorted.cap + bw.order.cap + bw.corr.cap + bw.cs.cap + bw.corr_d2.cap +
         bw.open.cap + bw.box.cap + bw.items.cap + bw.partials.cap + bw.sums.cap + bw.counters.cap;
    b += f.raw.cap + f.src_raw.cap + f.src.cap + f.tgt_a.cap + f.tgt.cap + f.tgtf.cap + f.x.cap + f.tn.cap + f.sorted_d.cap + f.pos.cap +
         f.corr.cap + f.d2.cap + f.med.cap + f.sort_a.cap + f.sort_b.cap + f.sums.cap;
    const SicpWork& s = w->sicp;
    b += s.q.cap + s.z.cap + s.c.cap + s.xo2.cap + s.sched.cap + s.part.cap + s.rec.cap;
  }
  return (long long)b;
}

extern "C" int flb_map_release_keyframe_scratch(flb_map* m) {
  if (!m) return set_err("null map");
  CU(cudaSetDevice(m->cfg.device));
  CU(cudaStreamSynchronize(m->stream));
  m->kf_raw.release();
  m->kf_in.release();
  m->kf_out.release();
  kfw_release(m->kfw);
  m->kfw = nullptr;
  return 0;
}

// pcl::getTransformation(x, y, z, roll, pitch, yaw) (PCL 1.10 common/impl/eigen.hpp), float, as transformPointCloud
// uses it (common_lib.h:720-721)
static Affine12 affine_from_rpy(const float* p6) {
  Affine12 a;
  const float x = p6[0], y = p6[1], z = p6[2], roll = p6[3], pitch = p6[4], yaw = p6[5];
  const float A = std::cos(yaw), B = std::sin(yaw), C = std::cos(pitch), D = std::sin(pitch);
  const float E = std::cos(roll), F = std::sin(roll), DE = D * E, DF = D * F;
  a.t[0] = A * C; a.t[1] = A * DF - B * E; a.t[2] = B * F + A * DE; a.t[3] = x;
  a.t[4] = B * C; a.t[5] = A * E + B * DF; a.t[6] = B * DE - A * F; a.t[7] = y;
  a.t[8] = -D;    a.t[9] = C * F;          a.t[10] = C * E;         a.t[11] = z;
  return a;
}

static KfSeg kf_seg(const float* t12, bool copy, long long src_off, int dst_off, int count) {
  KfSeg s{};
  for (int i = 0; i < 12; ++i) s.t[i] = t12[i];
  s.src_off = src_off;
  s.dst_off = dst_off;
  s.count = count;
  s.copy = copy ? 1 : 0;
  return s;
}

// The segment table into w.d_seg (through the pinned staging), on the map stream.
static int kf_upload_segs(flb_map* m, const std::vector<KfSeg>& segs) {
  KfWork& w = *m->kfw;
  const int ns = (int)segs.size();
  CU(cudaEventSynchronize(w.ev_seg));   // the previous table copy has left the pinned staging
  const size_t bytes = sizeof(KfSeg) * (size_t)ns, floor = sizeof(KfSeg) * 256;
  if (grow(w.d_seg, bytes, floor) || grow(w.h_seg, bytes, floor)) return 1;
  memcpy(w.h_seg.p, segs.data(), bytes);
  CU(cudaMemcpyAsync(w.d_seg.p, w.h_seg.p, bytes, cudaMemcpyHostToDevice, m->stream));
  CU(cudaEventRecord(w.ev_seg, m->stream));
  return 0;
}

// One launch: out[dst_off + j] = segment transform of src[src_off + j] for every (non-empty) segment, in table order.
static int kf_assemble_enqueue(flb_map* m, const std::vector<KfSeg>& segs, const float4* src, const float* src_curv, int n, float4* out,
                               float* out_curv) {
  if (n == 0) return 0;
  if (kf_upload_segs(m, segs)) return 1;
  k_kf_assemble<<<grid_for(n, 256, m->sm_count * 8), 256, 0, m->stream>>>(m->kfw->d_seg.p, (int)segs.size(), src, src_curv, n, out,
                                                                          out_curv);
  m->launches++;
  CU(cudaGetLastError());
  return 0;
}

// The tail of recontructIKdTree on the n assembled points in kf_in: downSizeFilterGlobalMapKeyFrames.filter
// (laserMapping.cpp:640-643), ikdtree.reconstruct (:656), featsFromMap->points = subMapKeyFramesDS->points (:664).
static int kf_rebuild_tail(flb_map* m, int n, float leaf, float* out_xyzi, int cap, int* n_points) {
  VgWork& w = m->kfw->vg;
  if (vg_enqueue(m, w, m->kf_in.p, nullptr, n, leaf, m->kf_out.p, nullptr, n, m->stream)) return 1;
  CU(cudaStreamSynchronize(m->stream));
  const bool ovf = w.h_mm.p[6] != 0;
  const int nd = ovf ? n : (int)w.h_mm.p[7];
  const float4* ds = ovf ? m->kf_in.p : m->kf_out.p;
  if (n_points) *n_points = nd;
  if (map_reset_storage(m)) return 1;
  if (nd > 0 && insert_device(m, ds, nullptr, nd, 0)) return 1;
  if (fetch_counters(m)) return 1;
  const int c = std::min(nd, cap);
  if (c > 0 && out_xyzi) CU(cudaMemcpy(out_xyzi, ds, sizeof(float4) * (size_t)c, cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int flb_map_reconstruct_keyframes(flb_map* m, const void* const* clouds, const int* sizes, int n_kf, int stride,
                                             int off_intensity, const float* poses6, float leaf, float* out_xyzi, int cap,
                                             int* n_points) {
  if (!m) return set_err("null map");
  if (n_points) *n_points = 0;
  if (n_kf < 0 || (n_kf > 0 && (!clouds || !sizes || !poses6))) return set_err("flb_map_reconstruct_keyframes: bad arguments");
  if (!(leaf > 0.f)) return set_err("leaf size must be > 0");
  if (stride < 12) return set_err("stride_bytes must be >= 12");
  if (off_intensity >= 0 && off_intensity + 4 > stride) return set_err("field offset outside the point stride");
  long long total = 0;
  for (int k = 0; k < n_kf; ++k) {
    if (sizes[k] < 0 || (sizes[k] > 0 && !clouds[k])) return set_err("key frame %d: bad cloud", k);
    total += sizes[k];
  }
  if (total > INT_MAX) return set_err("sub-map of %lld points is too large", total);
  CU(cudaSetDevice(m->cfg.device));
  const int n = (int)total;
  if (n == 0) return map_reset_storage(m);   // reconstruct with an empty cloud: everything deleted
  if (kf_scratch(m, n, false, true)) return 1;
  if (kf_grow(m->kf_raw, (size_t)n * stride)) return 1;
  // all clouds share the stride: staged back to back, packed by one launch, then transformed by one assembly
  std::vector<KfSeg> segs;
  segs.reserve(n_kf);
  long long off = 0;
  for (int k = 0; k < n_kf; ++k) {
    const int c = sizes[k];
    if (c == 0) continue;
    CU(cudaMemcpyAsync(m->kf_raw.p + (size_t)off * stride, clouds[k], (size_t)c * stride, cudaMemcpyHostToDevice, m->stream));
    segs.push_back(kf_seg(affine_from_rpy(poses6 + 6 * k).t, false, off, (int)off, c));
    off += c;
  }
  if (pack_records(m, m->stream, m->kf_raw.p, n, stride, off_intensity, -1, m->kf_out.p, nullptr)) return 1;
  // *subMapKeyFrames += *transformPointCloud(surfCloudKeyFrames[k], &cloudKeyPoses6D->points[k])  (laserMapping.cpp:636)
  if (kf_assemble_enqueue(m, segs, m->kf_out.p, nullptr, n, m->kf_in.p, nullptr)) return 1;
  return kf_rebuild_tail(m, n, leaf, out_xyzi, cap, n_points);
}

// ------------------------------------------------------------------------------------------------ key-frame store
struct flb_keyframes {
  flb_map* map = nullptr;
  long long cap_pts = 0;
  int cap_kf = 0;
  float4* xyzi = nullptr;            // x, y, z, intensity of every stored point (key frames back to back)
  float* curv = nullptr;             // curvature (the point's time offset in ms)
  std::vector<long long> off;        // first point of key frame k
  std::vector<int> cnt;              // its size
  long long n_pts = 0;
  DevBuf<unsigned char> raw;         // staging of host records (flb_keyframes_append)
  bool holds_ref = false;
};

extern "C" int flb_keyframes_create(flb_map* m, long long max_points, int max_keyframes, flb_keyframes** out) {
  if (!m || !out) return set_err("flb_keyframes_create: null argument");
  *out = nullptr;
  if (max_points <= 0 || max_keyframes <= 0) return set_err("flb_keyframes_create: max_points and max_keyframes must be > 0");
  CU(cudaSetDevice(m->cfg.device));
  flb_keyframes* k = new (std::nothrow) flb_keyframes();
  if (!k) return set_err("out of host memory");
  k->map = m;
  k->cap_pts = max_points;
  k->cap_kf = max_keyframes;
  try {   // reserved up front: an append never reallocates the table
    k->off.reserve((size_t)max_keyframes);
    k->cnt.reserve((size_t)max_keyframes);
  } catch (...) {
    delete k;
    return set_err("flb_keyframes_create: out of host memory for %d key frames", max_keyframes);
  }
  cudaError_t e = cudaMalloc((void**)&k->xyzi, sizeof(float4) * (size_t)max_points);
  if (e == cudaSuccess) e = cudaMalloc((void**)&k->curv, sizeof(float) * (size_t)max_points);
  if (e != cudaSuccess) {
    cudaGetLastError();
    flb_keyframes_destroy(k);
    return set_err("flb_keyframes_create: %lld points: %s", max_points, cudaGetErrorString(e));
  }
  m->refs++;   // keeps the map (and its stream) alive
  k->holds_ref = true;
  *out = k;
  return 0;
}

extern "C" void flb_keyframes_destroy(flb_keyframes* k) {
  if (!k) return;
  flb_map* m = k->map;
  Q(cudaSetDevice(m->cfg.device));
  Q(cudaStreamSynchronize(m->stream));
  void* ptrs[] = {k->xyzi, k->curv};
  for (void* p : ptrs) if (p) Q(cudaFree(p));
  const bool counted = k->holds_ref;
  delete k;
  if (counted) map_release(m);
}

static int kf_room(const flb_keyframes* k, long long n) {
  if ((int)k->cnt.size() >= k->cap_kf) return set_err("key-frame store full: %d key frames (max_keyframes)", k->cap_kf);
  if (k->n_pts + n > k->cap_pts)
    return set_err("key frame of %lld points does not fit: %lld of max_points=%lld in use", n, k->n_pts, k->cap_pts);
  return 0;
}

static void kf_commit(flb_keyframes* k, int n, int* index) {
  if (index) *index = (int)k->cnt.size();
  k->off.push_back(k->n_pts);
  k->cnt.push_back(n);
  k->n_pts += n;
}

extern "C" int flb_keyframes_append_frontend(flb_keyframes* k, flb_frontend* f, int* index) {
  if (!k || !f) return set_err("flb_keyframes_append_frontend: null argument");
  flb_map* m = k->map;
  if (f->ses->map != m) return set_err("flb_keyframes_append_frontend: the front end works on another map");
  const int n = f->n_raw;
  if (kf_room(k, n)) return 1;
  CU(cudaSetDevice(m->cfg.device));
  // pcl::copyPointCloud(*feats_undistort, *thisSurfKeyFrame)  (laserMapping.cpp:757): device to device, stream ordered
  if (n > 0) {
    CU(cudaMemcpyAsync(k->xyzi + k->n_pts, fe_cloud(f), sizeof(float4) * (size_t)n, cudaMemcpyDeviceToDevice, m->stream));
    CU(cudaMemcpyAsync(k->curv + k->n_pts, fe_curv(f), sizeof(float) * (size_t)n, cudaMemcpyDeviceToDevice, m->stream));
  }
  kf_commit(k, n, index);
  return 0;
}

extern "C" int flb_keyframes_append(flb_keyframes* k, const void* pts, int n, int stride, int off_intensity, int off_curvature, int* index) {
  if (!k) return set_err("null key-frame store");
  if (n < 0) return set_err("negative point count");
  if (n > 0 && (!pts || stride < 12)) return set_err("bad point buffer");
  if ((off_intensity >= 0 && off_intensity + 4 > stride) || (off_curvature >= 0 && off_curvature + 4 > stride))
    return set_err("field offset outside the point stride");
  if (kf_room(k, n)) return 1;
  flb_map* m = k->map;
  CU(cudaSetDevice(m->cfg.device));
  if (n > 0) {
    const size_t bytes = (size_t)n * stride;   // staging with a quarter of headroom, as kf_grow
    if (upload_records(m, m->stream, k->raw, bytes + bytes / 4, pts, n, stride, off_intensity, off_curvature, k->xyzi + k->n_pts,
                       k->curv + k->n_pts))
      return 1;
  }
  kf_commit(k, n, index);
  return 0;
}

extern "C" int flb_keyframes_download(flb_keyframes* k, int id, float* out_xyzi, float* out_curvature, int cap, int* n) {
  if (!k) return set_err("null key-frame store");
  if (id < 0 || id >= (int)k->cnt.size()) return set_err("key frame %d out of range [0, %d)", id, (int)k->cnt.size());
  if (n) *n = k->cnt[id];
  flb_map* m = k->map;
  CU(cudaSetDevice(m->cfg.device));
  return fe_download(m, k->xyzi + k->off[id], k->curv + k->off[id], k->cnt[id], out_xyzi, out_curvature, cap);
}

extern "C" int flb_keyframes_info(const flb_keyframes* k, int* n_keyframes, long long* n_points, long long* device_bytes,
                                  long long* map_scratch_bytes) {
  if (!k) return set_err("null key-frame store");
  if (n_keyframes) *n_keyframes = (int)k->cnt.size();
  if (n_points) *n_points = k->n_pts;
  if (device_bytes) *device_bytes = (long long)((sizeof(float4) + sizeof(float)) * (size_t)k->cap_pts + k->raw.cap);
  if (map_scratch_bytes) *map_scratch_bytes = kf_scratch_bytes(k->map);
  return 0;
}

extern "C" int flb_keyframes_size(const flb_keyframes* k, int id) {
  if (!k) return -set_err("null key-frame store");
  if (id < 0 || id >= (int)k->cnt.size()) return -set_err("key frame %d out of range [0, %d)", id, (int)k->cnt.size());
  return k->cnt[id];
}

// every id of a selection checked (before any device work)
static int kf_check_ids(const flb_keyframes* k, const int* ids, int n_ids, const char* who) {
  for (int j = 0; j < n_ids; ++j)
    if (ids[j] < 0 || ids[j] >= (int)k->cnt.size())
      return set_err("%s: key frame id %d (entry %d) out of range [0, %d)", who, ids[j], j, (int)k->cnt.size());
  return 0;
}

// the selection's size, with every id checked (before any device work)
static int kf_selection(const flb_keyframes* k, const int* ids, int n_ids, const char* who, int* total) {
  if (kf_check_ids(k, ids, n_ids, who)) return 1;
  long long t = 0;
  for (int j = 0; j < n_ids; ++j) t += k->cnt[ids[j]];
  if (t > INT_MAX) return set_err("%s: selection of %lld points is too large", who, t);
  *total = (int)t;
  return 0;
}

extern "C" int flb_map_reconstruct_from_keyframes(flb_map* m, const flb_keyframes* k, const int* ids, int n_ids, const float* poses6,
                                                  float leaf, float* out_xyzi, int cap, int* n_points) {
  if (!m || !k) return set_err("flb_map_reconstruct_from_keyframes: null map or store");
  if (n_points) *n_points = 0;
  if (k->map != m) return set_err("flb_map_reconstruct_from_keyframes: the store belongs to another map");
  if (n_ids < 0 || (n_ids > 0 && (!ids || !poses6))) return set_err("flb_map_reconstruct_from_keyframes: bad arguments");
  if (!(leaf > 0.f)) return set_err("leaf size must be > 0");
  int n = 0;
  if (kf_selection(k, ids, n_ids, "flb_map_reconstruct_from_keyframes", &n)) return 1;
  CU(cudaSetDevice(m->cfg.device));
  if (n == 0) return map_reset_storage(m);
  if (kf_scratch(m, n, false, true)) return 1;
  std::vector<KfSeg> segs;
  segs.reserve(n_ids);
  int dst = 0;
  for (int j = 0; j < n_ids; ++j) {
    const int c = k->cnt[ids[j]];
    if (c == 0) continue;
    segs.push_back(kf_seg(affine_from_rpy(poses6 + 6 * j).t, false, k->off[ids[j]], dst, c));
    dst += c;
  }
  if (kf_assemble_enqueue(m, segs, k->xyzi, nullptr, n, m->kf_in.p, nullptr)) return 1;
  return kf_rebuild_tail(m, n, leaf, out_xyzi, cap, n_points);
}

static bool is_identity(const float* t) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c)
      if (t[r * 4 + c] != (r == c ? 1.f : 0.f)) return false;
  return true;
}

// The segment table of a selection: ids[j] with transforms[j] (FLB_KF_POSE6 / FLB_KF_AFFINE, the identity affine
// copies), back to back from output point 0, empty key frames dropped.
static void kf_selection_segs(const flb_keyframes* k, const int* ids, int n_ids, int transform_kind, const float* transforms,
                              std::vector<KfSeg>& segs) {
  segs.clear();
  segs.reserve(n_ids);
  int dst = 0;
  for (int j = 0; j < n_ids; ++j) {
    const int c = k->cnt[ids[j]];
    if (c == 0) continue;
    if (transform_kind == FLB_KF_POSE6) {
      segs.push_back(kf_seg(affine_from_rpy(transforms + 6 * j).t, false, k->off[ids[j]], dst, c));
    } else {
      const float* t = transforms + 12 * j;
      segs.push_back(kf_seg(t, is_identity(t), k->off[ids[j]], dst, c));
    }
    dst += c;
  }
}

extern "C" int flb_keyframes_assemble(flb_keyframes* k, const int* ids, int n_ids, int transform_kind, const float* transforms, float leaf,
                                      float* out_xyzi, float* out_curvature, int cap, int* n_out) {
  if (!k) return set_err("null key-frame store");
  if (n_out) *n_out = 0;
  if (transform_kind != FLB_KF_POSE6 && transform_kind != FLB_KF_AFFINE)
    return set_err("transform_kind must be FLB_KF_POSE6 (%d) or FLB_KF_AFFINE (%d)", FLB_KF_POSE6, FLB_KF_AFFINE);
  if (n_ids < 0 || (n_ids > 0 && (!ids || !transforms))) return set_err("flb_keyframes_assemble: bad arguments");
  if (!(leaf >= 0.f)) return set_err("leaf size must be >= 0 (0: no filter)");
  int n = 0;
  if (kf_selection(k, ids, n_ids, "flb_keyframes_assemble", &n)) return 1;
  if (n == 0) return 0;
  flb_map* m = k->map;
  CU(cudaSetDevice(m->cfg.device));
  if (kf_scratch(m, n, true, leaf > 0.f)) return 1;
  KfWork& w = *m->kfw;
  std::vector<KfSeg> segs;
  kf_selection_segs(k, ids, n_ids, transform_kind, transforms, segs);
  if (kf_assemble_enqueue(m, segs, k->xyzi, k->curv, n, m->kf_in.p, w.cin.p)) return 1;
  if (leaf == 0.f) {   // the dense concatenation (GlobalMap.pcd, the loop sub-maps)
    if (n_out) *n_out = n;
    return fe_download(m, m->kf_in.p, w.cin.p, n, out_xyzi, out_curvature, cap);
  }
  // downSizeFilterSurf / downSizeFilterGlobalMapKeyFrames .filter (laserMapping.cpp:1780-1789, :1866-1869)
  if (vg_enqueue(m, w.vg, m->kf_in.p, w.cin.p, n, leaf, m->kf_out.p, w.cout.p, n, m->stream)) return 1;
  CU(cudaStreamSynchronize(m->stream));
  const bool ovf = w.vg.h_mm.p[6] != 0;   // PCL's int32 overflow guard: the input comes back unchanged
  const int nd = ovf ? n : (int)w.vg.h_mm.p[7];
  if (n_out) *n_out = nd;
  return fe_download(m, ovf ? m->kf_in.p : m->kf_out.p, ovf ? w.cin.p : w.cout.p, nd, out_xyzi, out_curvature, cap);
}

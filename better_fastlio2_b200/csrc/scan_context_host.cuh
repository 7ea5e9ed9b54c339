// scan_context_host.cuh — Scan Context descriptors (SCManager::makeScancontext, include/sc-relo/Scancontext.cpp:195-251)
// of key-frame selections in the device store, for the loop gate of performLoopClosure (laserMapping.cpp:932-940) and
// the key-frame saver at shutdown (:2501-2505).  One k_sc_bins launch per call over the selection's segment table, the
// same table k_kf_assemble reads; one synchronisation; the store is not modified.  Included after keyframe_host.cuh.
#pragma once
#include <cmath>

#include "scan_context_kernels.cuh"

// Grow-only Scan Context scratch in the map's KfWork: n_chunks chunk-table rows and n_desc descriptors of keys, each
// on the device and in pinned staging.
static int sc_scratch(flb_map* m, int n_chunks, int n_desc) {
  if (kf_work(m)) return 1;
  KfWork& w = *m->kfw;
  const size_t chunks = sizeof(ScChunk) * (size_t)n_chunks, chunk_floor = sizeof(ScChunk) * 1024;
  const size_t keys = sizeof(unsigned) * SC_BINS * (size_t)n_desc;
  if (grow(w.d_chunk, chunks, chunk_floor) || grow(w.h_chunk, chunks, chunk_floor)) return 1;
  return grow(w.d_sc_keys, keys, 0) || grow(w.h_sc_keys, keys, 0);
}

// The float a key stands for, as a double; key 0 (no point beat -1000) is the reference's NO_POINT reset to 0.
static double sc_value(unsigned key) {
  if (key == 0u) return 0.0;
  const unsigned b = (key & 0x80000000u) ? (key & 0x7fffffffu) : ~key;
  float v;
  memcpy(&v, &b, sizeof(v));
  return (double)v;
}

// makeScancontext of every segment group: segment s feeds descriptor seg_desc[s]; n_desc descriptors of SC_RINGS x
// SC_SECTORS doubles, row-major (ring, sector), written to out.  Key frames are split into chunks of SC_CHUNK points.
static int sc_run(flb_keyframes* k, const std::vector<KfSeg>& segs, const std::vector<int>& seg_desc, int n_desc,
                  double lidar_height, double* out) {
  flb_map* m = k->map;
  CU(cudaSetDevice(m->cfg.device));
  std::vector<ScChunk> chunks;
  for (int s = 0; s < (int)segs.size(); ++s)
    for (int b = 0; b < segs[s].count; b += SC_CHUNK)
      chunks.push_back(ScChunk{s, segs[s].dst_off + b, std::min(SC_CHUNK, segs[s].count - b), seg_desc[s]});
  const int nc = (int)chunks.size();
  if (sc_scratch(m, nc, n_desc)) return 1;
  KfWork& w = *m->kfw;
  const size_t key_bytes = sizeof(unsigned) * SC_BINS * (size_t)n_desc;
  CU(cudaMemsetAsync(w.d_sc_keys.p, 0, key_bytes, m->stream));
  if (nc > 0) {
    if (kf_upload_segs(m, segs)) return 1;
    memcpy(w.h_chunk.p, chunks.data(), sizeof(ScChunk) * (size_t)nc);   // free: every call ends in a synchronisation
    CU(cudaMemcpyAsync(w.d_chunk.p, w.h_chunk.p, sizeof(ScChunk) * (size_t)nc, cudaMemcpyHostToDevice, m->stream));
    k_sc_bins<<<std::min(nc, m->sm_count * 8), 256, 0, m->stream>>>(w.d_seg.p, w.d_chunk.p, nc, k->xyzi, lidar_height, w.d_sc_keys.p);
    m->launches++;
    CU(cudaGetLastError());
  }
  CU(cudaMemcpyAsync(w.h_sc_keys.p, w.d_sc_keys.p, key_bytes, cudaMemcpyDeviceToHost, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  for (size_t b = 0; b < (size_t)SC_BINS * n_desc; ++b) out[b] = sc_value(w.h_sc_keys.p[b]);
  return 0;
}

extern "C" int flb_keyframes_scan_context(flb_keyframes* k, const int* ids, int n_ids, int transform_kind, const float* transforms,
                                          double lidar_height, double* out_desc) {
  const char* who = "flb_keyframes_scan_context";
  if (n_ids < 0) return set_err("%s: negative n_ids", who);
  if (!out_desc) return set_err("%s: null out_desc", who);
  if (n_ids > 0 && (!ids || !transforms)) return set_err("%s: null ids or transforms", who);
  if (transform_kind != FLB_KF_POSE6 && transform_kind != FLB_KF_AFFINE)
    return set_err("%s: transform_kind must be FLB_KF_POSE6 (%d) or FLB_KF_AFFINE (%d)", who, FLB_KF_POSE6, FLB_KF_AFFINE);
  if (!std::isfinite(lidar_height)) return set_err("%s: lidar_height must be finite", who);
  if (!k) return set_err("%s: null key-frame store", who);
  int n = 0;
  if (kf_selection(k, ids, n_ids, who, &n)) return 1;
  if (n == 0) {   // makeScancontext of an empty cloud: every bin NO_POINT, reset to 0
    for (int b = 0; b < SC_BINS; ++b) out_desc[b] = 0.0;
    return 0;
  }
  std::vector<KfSeg> segs;
  kf_selection_segs(k, ids, n_ids, transform_kind, transforms, segs);
  return sc_run(k, segs, std::vector<int>(segs.size(), 0), 1, lidar_height, out_desc);
}

extern "C" int flb_keyframes_scan_contexts(flb_keyframes* k, const int* ids, int n_ids, double lidar_height, double* out_descs) {
  const char* who = "flb_keyframes_scan_contexts";
  if (n_ids < 0) return set_err("%s: negative n_ids", who);
  if (n_ids > 0 && (!ids || !out_descs)) return set_err("%s: null ids or out_descs", who);
  if (!std::isfinite(lidar_height)) return set_err("%s: lidar_height must be finite", who);
  if (!k) return set_err("%s: null key-frame store", who);
  if (kf_check_ids(k, ids, n_ids, who)) return 1;
  if (n_ids == 0) return 0;
  // key frame ids[j] as stored (copyPointCloud(*surfCloudKeyFrames[i], *save_cloud), :2504), into descriptor j; each
  // segment counts from 0, so a whole run may hold more than INT_MAX points
  static const float eye[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  std::vector<KfSeg> segs;
  std::vector<int> seg_desc;
  for (int j = 0; j < n_ids; ++j) {
    const int c = k->cnt[ids[j]];
    if (c == 0) continue;
    segs.push_back(kf_seg(eye, true, k->off[ids[j]], 0, c));
    seg_desc.push_back(j);
  }
  return sc_run(k, segs, seg_desc, n_ids, lidar_height, out_descs);
}

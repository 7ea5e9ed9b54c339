// preprocess_host.cuh — C-ABI entry point of Preprocess::process on the device (flb_frontend_preprocess).
// Included at the end of fastlio_b200.cu after frontend_host.cuh (uses flb_frontend and its voxel-grid workspace).
#pragma once
#include "preprocess_kernels.cuh"

// scratch of the preprocess call that the front end does not already own (allocated on first use, grown only)
struct PpWork {
  int cap = 0;          // points
  int ring_cap = 0;     // rings
  double* yaw = nullptr;
  int* ring_first = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
  PpOut* d_out = nullptr;
  PpOut* h_out = nullptr;   // pinned
};
static void pp_release(PpWork* w) {
  if (!w) return;
  void* ptrs[] = {w->yaw, w->ring_first, w->tmp, w->d_out};
  for (void* p : ptrs) if (p) Q(cudaFree(p));
  if (w->h_out) Q(cudaFreeHost(w->h_out));
  delete w;
}
static int pp_ensure(PpWork& w, int cap, int rings) {
  if (!w.d_out) {
    CU(cudaMalloc((void**)&w.d_out, sizeof(PpOut)));
    CU(cudaMallocHost((void**)&w.h_out, sizeof(PpOut)));
  }
  if (cap > w.cap) {
    if (w.yaw) Q(cudaFree(w.yaw));
    if (w.tmp) Q(cudaFree(w.tmp));
    w.yaw = nullptr; w.tmp = nullptr; w.cap = 0;
    size_t t1 = 0, t2 = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, t1, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr,
                                       cap, 0, 16));
    CU(cub::DeviceScan::InclusiveScan(nullptr, t2, (const unsigned*)nullptr, (unsigned*)nullptr, PpMapCompose(), cap));
    w.tmp_bytes = std::max(t1, t2) + 256;
    CU(cudaMalloc((void**)&w.yaw, sizeof(double) * (size_t)cap));
    CU(cudaMalloc(&w.tmp, w.tmp_bytes));
    w.cap = cap;
  }
  if (rings > w.ring_cap) {
    if (w.ring_first) Q(cudaFree(w.ring_first));
    w.ring_first = nullptr; w.ring_cap = 0;
    CU(cudaMalloc((void**)&w.ring_first, sizeof(int) * (size_t)rings));
    w.ring_cap = rings;
  }
  return 0;
}

static int pp_check_field(const char* name, int off, int size, int stride, bool required) {
  if (off < 0) return required ? set_err("flb_frontend_preprocess: field %s is required", name) : 0;
  if (off + size > stride) return set_err("flb_frontend_preprocess: field %s (offset %d, %d bytes) outside the %d-byte record", name, off, size, stride);
  return 0;
}

extern "C" int flb_frontend_preprocess(flb_frontend* f, const flb_preprocess_config* cfg, const flb_raw_layout* lay, const void* records,
                                       int n, int* n_out, float* last_curvature) {
  // the handle is checked after the arguments, so that every argument check is reachable without a device
  if (!cfg || !lay) return set_err("flb_frontend_preprocess: null config or layout");
  const int type = cfg->lidar_type;
  if (type != PP_LIVOX && type != PP_VELO16 && type != PP_OUST64)
    return set_err("flb_frontend_preprocess: lidar_type %d is not 1 (LIVOX), 2 (VELO16) or 3 (OUST64)", type);
  if (cfg->point_filter_num < 1) return set_err("flb_frontend_preprocess: point_filter_num must be >= 1");
  if (cfg->n_scans < 1) return set_err("flb_frontend_preprocess: n_scans must be >= 1");
  if (n < 0) return set_err("flb_frontend_preprocess: negative number of records");
  if (n > 0 && !records) return set_err("flb_frontend_preprocess: null records");
  const int s = lay->stride;
  if (s < 1) return set_err("flb_frontend_preprocess: stride must be >= 1");
  if (pp_check_field("x", lay->off_x, 4, s, true) || pp_check_field("y", lay->off_y, 4, s, true) ||
      pp_check_field("z", lay->off_z, 4, s, true) || pp_check_field("time", lay->off_time, 4, s, false) ||
      pp_check_field("intensity", lay->off_intensity, type == PP_LIVOX ? 1 : 4, s, false))
    return 1;
  if (type == PP_VELO16 && pp_check_field("ring", lay->off_ring, 2, s, false)) return 1;
  if (type == PP_LIVOX && (pp_check_field("tag", lay->off_tag, 1, s, false) || pp_check_field("line", lay->off_line, 1, s, false)))
    return 1;
  if (!f) return set_err("null front end");
  if (n > f->cap) return set_err("raw scan of %d records exceeds max_raw_points=%d", n, f->cap);

  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  f->n_raw = 0;
  f->sorted = false;
  f->n_down = -1;
  if (n_out) *n_out = 0;
  if (last_curvature) *last_curvature = 0.f;
  if (n == 0) return 0;

  PpParams p;
  p.n = n; p.stride = s; p.pfn = cfg->point_filter_num; p.n_scans = cfg->n_scans;
  p.off_x = lay->off_x; p.off_y = lay->off_y; p.off_z = lay->off_z; p.off_i = lay->off_intensity; p.off_t = lay->off_time;
  p.off_ring = lay->off_ring; p.off_tag = lay->off_tag; p.off_line = lay->off_line;
  switch (cfg->time_unit) {   // Preprocess::process (preprocess.cpp:65-82)
    case 0: p.tscale = 1.e3f; break;
    case 2: p.tscale = 1.e-3f; break;
    case 3: p.tscale = 1.e-6f; break;
    default: p.tscale = 1.f; break;
  }
  p.blind2 = cfg->blind * cfg->blind;
  p.omega_l = 0.361 * cfg->scan_rate;
  p.wrap = 360.0 / p.omega_l;
  // given_offset_time = (last record's time > 0), read on the host: it picks the launch sequence (:322-340)
  bool synth = false;
  if (type == PP_VELO16) {
    float t_last = 0.f;
    if (lay->off_time >= 0) memcpy(&t_last, (const unsigned char*)records + (size_t)(n - 1) * s + lay->off_time, sizeof(float));
    synth = !(t_last > 0.f);
  }
  const int rings = std::min(cfg->n_scans, 65536);   // ring is a u16
  if (!f->pp) {
    f->pp = new (std::nothrow) PpWork();
    if (!f->pp) return set_err("out of host memory");
  }
  PpWork& w = *f->pp;
  if (pp_ensure(w, f->cap, rings)) return 1;
  if (fe_stage_raw(f, m, records, n, s)) return 1;   // the one H2D copy

  cudaStream_t st = m->stream;
  const int g = grid_for(n, 256, m->sm_count * 8);
  VgWork& v = f->vg;   // its arrays hold max_raw_points entries; free between front-end calls
  int* keep = v.flags;
  int* pos = v.pos;
  CU(cudaMemsetAsync(w.d_out, 0, sizeof(PpOut), st));
  if (type == PP_OUST64) {
    k_pp_ouster<<<g, 256, 0, st>>>(f->raw, p, f->pts_t, f->curv_t, keep);
    m->launches++;
  } else if (type == PP_VELO16) {
    if (synth) CU(cudaMemsetAsync(w.ring_first, 0x7F, sizeof(int) * (size_t)rings, st));   // 0x7F7F7F7F > any index
    k_pp_velo<<<g, 256, 0, st>>>(f->raw, p, synth ? 1 : 0, f->pts_t, f->curv_t, keep, v.keys_a, v.vals_a, w.yaw, w.ring_first, w.d_out);
    m->launches++;
    if (synth) {
      int end_bit = 1;
      while (end_bit < 17 && (1 << end_bit) <= rings) ++end_bit;   // keys are min(ring, n_scans) <= rings
      size_t tb = w.tmp_bytes;
      CU(cub::DeviceRadixSort::SortPairs(w.tmp, tb, (const unsigned*)v.keys_a, v.keys_b, (const int*)v.vals_a, v.vals_b, n, 0, end_bit, st));
      k_pp_velo_maps<<<g, 256, 0, st>>>(v.keys_b, v.vals_b, w.yaw, w.ring_first, p, v.keys_a);
      tb = w.tmp_bytes;
      CU(cub::DeviceScan::InclusiveScan(w.tmp, tb, (const unsigned*)v.keys_a, (unsigned*)v.vals_a, PpMapCompose(), n, st));
      k_pp_velo_apply<<<g, 256, 0, st>>>(v.keys_b, v.vals_b, w.yaw, w.ring_first, (const unsigned*)v.vals_a, p, f->curv_t, keep);
      m->launches += 3 + 4 + 2;   // + CUB's radix sort and scan kernels
    }
  } else {
    k_pp_livox<<<g, 256, 0, st>>>(f->raw, p, f->pts_t, f->curv_t, v.vals_a);
    size_t tb = v.tmp_bytes;
    CU(cub::DeviceScan::ExclusiveSum(v.tmp, tb, (const int*)v.vals_a, v.vals_b, n, st));
    k_pp_livox_keep<<<g, 256, 0, st>>>(f->pts_t, v.vals_a, v.vals_b, p, keep);
    m->launches += 2 + 2;
  }
  size_t tb = v.tmp_bytes;
  CU(cub::DeviceScan::ExclusiveSum(v.tmp, tb, (const int*)keep, pos, n, st));
  k_pp_scatter<<<g, 256, 0, st>>>(f->pts_t, f->curv_t, keep, pos, n, f->pts, f->curv, w.d_out);
  m->launches += 1 + 2;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(w.h_out, w.d_out, sizeof(PpOut), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const PpOut r = *w.h_out;
  if (r.bad_ring)
    return set_err("flb_frontend_preprocess: ring %d >= n_scans=%d (scan_line does not match the sensor)", r.bad_ring - 1, cfg->n_scans);
  f->n_raw = r.count;
  if (n_out) *n_out = r.count;
  if (last_curvature) *last_curvature = r.last_curv;
  return 0;
}

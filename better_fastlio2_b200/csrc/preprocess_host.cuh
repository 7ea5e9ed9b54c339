// preprocess_host.cuh — C-ABI entry point of Preprocess::process on the device (flb_frontend_preprocess).
// Included at the end of fastlio_b200.cu after frontend_host.cuh (uses flb_frontend and its voxel-grid workspace).
#pragma once
#include "preprocess_kernels.cuh"

// scratch of the preprocess call that the front end does not already own (allocated on first use, grown only)
struct PpWork {
  int cap = 0;                 // points yaw and the CUB scratch are sized for
  DevBuf<double> yaw;
  DevBuf<int> ring_first;
  DevBuf<unsigned char> tmp;   // CUB temporary storage
  DevBuf<PpOut> d_out;
  PinnedBuf<PpOut> h_out;
};
static void pp_release(PpWork* w) { delete w; }
static int pp_ensure(PpWork& w, int cap, int rings) {
  if (grow(w.d_out, sizeof(PpOut), 0) || grow(w.h_out, sizeof(PpOut), 0)) return 1;
  if (cap > w.cap) {
    w.cap = 0;   // (until both have grown)
    size_t t1 = 0, t2 = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, t1, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr,
                                       cap, 0, 16));
    CU(cub::DeviceScan::InclusiveScan(nullptr, t2, (const unsigned*)nullptr, (unsigned*)nullptr, PpMapCompose(), cap));
    if (grow(w.yaw, sizeof(double) * (size_t)cap, 0) || grow(w.tmp, std::max(t1, t2) + 256, 0)) return 1;
    w.cap = cap;
  }
  return grow(w.ring_first, sizeof(int) * (size_t)rings, 0);
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
  // the one H2D copy, into the front end's staging (sized once for its capacity)
  if (grow(f->raw, (size_t)n * s, (size_t)f->cap * s)) return 1;
  CU(cudaMemcpyAsync(f->raw.p, records, (size_t)n * s, cudaMemcpyHostToDevice, m->stream));

  cudaStream_t st = m->stream;
  const int g = grid_for(n, 256, m->sm_count * 8);
  VgWork& v = f->vg;   // its arrays hold max_raw_points entries; free between front-end calls
  int* keep = v.flags.p;
  int* pos = v.pos.p;
  CU(cudaMemsetAsync(w.d_out.p, 0, sizeof(PpOut), st));
  if (type == PP_OUST64) {
    k_pp_ouster<<<g, 256, 0, st>>>(f->raw.p, p, f->pts_t, f->curv_t, keep);
    m->launches++;
  } else if (type == PP_VELO16) {
    if (synth) CU(cudaMemsetAsync(w.ring_first.p, 0x7F, sizeof(int) * (size_t)rings, st));   // 0x7F7F7F7F > any index
    k_pp_velo<<<g, 256, 0, st>>>(f->raw.p, p, synth ? 1 : 0, f->pts_t, f->curv_t, keep, v.keys_a.p, v.vals_a.p, w.yaw.p, w.ring_first.p, w.d_out.p);
    m->launches++;
    if (synth) {
      int end_bit = 1;
      while (end_bit < 17 && (1 << end_bit) <= rings) ++end_bit;   // keys are min(ring, n_scans) <= rings
      size_t tb = w.tmp.cap;
      CU(cub::DeviceRadixSort::SortPairs(w.tmp.p, tb, (const unsigned*)v.keys_a.p, v.keys_b.p, (const int*)v.vals_a.p, v.vals_b.p, n, 0, end_bit, st));
      k_pp_velo_maps<<<g, 256, 0, st>>>(v.keys_b.p, v.vals_b.p, w.yaw.p, w.ring_first.p, p, v.keys_a.p);
      tb = w.tmp.cap;
      CU(cub::DeviceScan::InclusiveScan(w.tmp.p, tb, (const unsigned*)v.keys_a.p, (unsigned*)v.vals_a.p, PpMapCompose(), n, st));
      k_pp_velo_apply<<<g, 256, 0, st>>>(v.keys_b.p, v.vals_b.p, w.yaw.p, w.ring_first.p, (const unsigned*)v.vals_a.p, p, f->curv_t, keep);
      m->launches += 3 + 4 + 2;   // + CUB's radix sort and scan kernels
    }
  } else {
    k_pp_livox<<<g, 256, 0, st>>>(f->raw.p, p, f->pts_t, f->curv_t, v.vals_a.p);
    size_t tb = v.tmp.cap;
    CU(cub::DeviceScan::ExclusiveSum(v.tmp.p, tb, (const int*)v.vals_a.p, v.vals_b.p, n, st));
    k_pp_livox_keep<<<g, 256, 0, st>>>(f->pts_t, v.vals_a.p, v.vals_b.p, p, keep);
    m->launches += 2 + 2;
  }
  size_t tb = v.tmp.cap;
  CU(cub::DeviceScan::ExclusiveSum(v.tmp.p, tb, (const int*)keep, pos, n, st));
  k_pp_scatter<<<g, 256, 0, st>>>(f->pts_t, f->curv_t, keep, pos, n, f->pts, f->curv, w.d_out.p);
  m->launches += 1 + 2;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(w.h_out.p, w.d_out.p, sizeof(PpOut), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const PpOut r = *w.h_out.p;
  if (r.bad_ring)
    return set_err("flb_frontend_preprocess: ring %d >= n_scans=%d (scan_line does not match the sensor)", r.bad_ring - 1, cfg->n_scans);
  f->n_raw = r.count;
  if (n_out) *n_out = r.count;
  if (last_curvature) *last_curvature = r.last_curv;
  return 0;
}

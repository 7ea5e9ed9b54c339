// color_host.cuh — C-ABI entry points of the camera-coloured and IMU-frame scan publishers (color_kernels.cuh).
// Included at the end of fastlio_b200.cu after frontend_host.cuh (uses flb_frontend, fe_cloud, fe_download).
#pragma once
#include "color_kernels.cuh"
#include <cmath>

// Camera state of a front end (paramSetting, the global image_color), created by flb_frontend_camera_config.
struct ColorCam {
  CamProj proj{};
  DevBuf<unsigned char> img;   // H × W × 3 bytes, bgr8, row pitch 3·W
  // pinned mirror of the colour pass's output: k_color_emit writes the records and the count straight into it, so a call
  // needs one synchronisation (the count is known only on the device)
  PinnedBuf<float4> h_xyzi;
  PinnedBuf<unsigned> h_bgra;
  PinnedBuf<int> h_count;
};
static void cam_release(ColorCam* c) { delete c; }

extern "C" int flb_frontend_camera_config(flb_frontend* f, const double* cam_ex, const double* cam_in, int width, int height) {
  if (!cam_ex || !cam_in) return set_err("flb_frontend_camera_config: null argument");
  if (width <= 0 || height <= 0) return set_err("flb_frontend_camera_config: image size %d x %d must be positive", width, height);
  if ((size_t)width * (size_t)height * 3 > (size_t)INT_MAX) return set_err("flb_frontend_camera_config: image of %d x %d is too large", width, height);
  for (int k = 0; k < 16; ++k)
    if (!std::isfinite(cam_ex[k])) return set_err("flb_frontend_camera_config: cam_ex[%d] is not finite", k);
  for (int k = 0; k < 12; ++k)
    if (!std::isfinite(cam_in[k])) return set_err("flb_frontend_camera_config: cam_in[%d] is not finite", k);
  if (!f) return set_err("null front end");
  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  if (!f->cam) {
    f->cam = new (std::nothrow) ColorCam();
    if (!f->cam) return set_err("out of host memory");
  }
  ColorCam& c = *f->cam;
  // internalMatProject * externalMat: each element a sum over k = 0..3 in index order, no FMA
  for (int r = 0; r < 3; ++r)
    for (int j = 0; j < 4; ++j) {
      double s = cam_in[4 * r + 0] * cam_ex[0 + j];
      for (int k = 1; k < 4; ++k) s = s + cam_in[4 * r + k] * cam_ex[4 * k + j];
      c.proj.M[4 * r + j] = s;
    }
  const size_t bytes = (size_t)width * (size_t)height * 3;
  const size_t recs = (size_t)f->cap;
  if (grow(c.img, bytes, 0) || grow(c.h_xyzi, sizeof(float4) * recs, 0) || grow(c.h_bgra, sizeof(unsigned) * recs, 0) ||
      grow(c.h_count, sizeof(int), 0))
    return 1;
  c.proj.W = width;
  c.proj.H = height;
  // no image yet: all zero, as the reference's zero-initialised global image_color
  CU(cudaMemsetAsync(c.img.p, 0, bytes, m->stream));
  return 0;
}

extern "C" int flb_frontend_camera_image(flb_frontend* f, const unsigned char* bgr8, int rows, int cols, int step_bytes) {
  if (!bgr8) return set_err("flb_frontend_camera_image: null image");
  if (rows <= 0 || cols <= 0) return set_err("flb_frontend_camera_image: image size %d x %d must be positive", cols, rows);
  if ((long long)step_bytes < 3LL * cols) return set_err("flb_frontend_camera_image: row step %d is below 3 * cols = %lld", step_bytes, 3LL * cols);
  if (!f) return set_err("null front end");
  if (!f->cam) return set_err("flb_frontend_camera_image: camera not configured (flb_frontend_camera_config)");
  const CamProj& p = f->cam->proj;
  if (rows < p.H || cols < p.W)
    return set_err("flb_frontend_camera_image: image of %d x %d is smaller than the configured %d x %d", cols, rows, p.W, p.H);
  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  // imageCallback: the top-left H × W window
  CU(cudaMemcpy2DAsync(f->cam->img.p, (size_t)p.W * 3, bgr8, (size_t)step_bytes, (size_t)p.W * 3, (size_t)p.H, cudaMemcpyHostToDevice,
                       m->stream));
  return 0;
}

extern "C" int flb_frontend_points_colorize(flb_frontend* f, int which, const double* state26, float* out_xyzi, unsigned* out_bgra,
                                            int cap, int* n) {
  if (which != 0 && which != 1) return set_err("which must be 0 (feats_down_body) or 1 (feats_undistort)");
  if (!state26 || !n) return set_err("flb_frontend_points_colorize: null argument");
  if (cap < 0) return set_err("flb_frontend_points_colorize: negative capacity");
  if (cap > 0 && (!out_xyzi || !out_bgra)) return set_err("flb_frontend_points_colorize: null output buffer");
  if (!f) return set_err("null front end");
  if (!f->cam) return set_err("flb_frontend_points_colorize: camera not configured (flb_frontend_camera_config)");
  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  const float4* src = which == 0 ? f->ses->body : fe_cloud(f);
  const int cnt = which == 0 ? f->ses->n : f->n_raw;
  *n = 0;
  if (cnt > f->cap) return set_err("cloud of %d points exceeds the front end capacity %d", cnt, f->cap);
  if (cnt == 0) return 0;
  ColorCam& c = *f->cam;
  VgWork& w = f->vg;   // scratch: pixel index, keep flag, output slot (the voxel filter's, free between its calls)
  if (vg_ensure(w, cnt)) return 1;
  float4* d_xyzi = nullptr;
  unsigned* d_bgra = nullptr;
  int* d_count = nullptr;
  CU(cudaHostGetDevicePointer((void**)&d_xyzi, c.h_xyzi.p, 0));
  CU(cudaHostGetDevicePointer((void**)&d_bgra, c.h_bgra.p, 0));
  CU(cudaHostGetDevicePointer((void**)&d_count, c.h_count.p, 0));
  cudaStream_t st = m->stream;
  const int g = grid_for(cnt, 256, m->sm_count * 8);
  k_color_mark<<<g, 256, 0, st>>>(c.proj, src, cnt, w.vals_a.p, w.flags.p);
  size_t tb = w.tmp.cap;
  CU(cub::DeviceScan::ExclusiveSum(w.tmp.p, tb, (const int*)w.flags.p, w.pos.p, cnt, st));
  k_color_emit<<<g, 256, 0, st>>>(pose_from(state26), src, cnt, w.vals_a.p, w.pos.p, c.img.p, d_xyzi, d_bgra, d_count);
  m->launches += 2 + 1;
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(st));
  const int kept = *c.h_count.p;
  const int k = std::min(kept, cap);
  if (k > 0) {
    memcpy(out_xyzi, c.h_xyzi.p, sizeof(float4) * (size_t)k);
    memcpy(out_bgra, c.h_bgra.p, sizeof(unsigned) * (size_t)k);
  }
  *n = kept;
  return 0;
}

extern "C" int flb_frontend_points_to_imu(flb_frontend* f, const double* state26, float* out_xyzi, int cap, int* n) {
  if (!state26) return set_err("null state");
  if (!f) return set_err("null front end");
  flb_map* m = f->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  const int cnt = f->n_raw;   // feats_undistort (publish_frame_body)
  if (n) *n = cnt;
  if (cnt > 0) {
    k_to_imu<<<grid_for(cnt, 256, m->sm_count * 8), 256, 0, m->stream>>>(pose_from(state26), fe_cloud(f), f->world, cnt);
    m->launches++;
    CU(cudaGetLastError());
  }
  return fe_download(m, f->world, nullptr, cnt, out_xyzi, nullptr, cap);
}

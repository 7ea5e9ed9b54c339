// color_kernels.cuh — the two scan publishers of the main loop that still walk the cloud on the host, as sm_90a kernels:
//   publish_frame_world_color   src/laserMapping.cpp:310-392 (image: imageCallback :250-276, matrices: paramSetting :279-289)
//   publish_frame_body          src/laserMapping.cpp:1543-1558 (RGBpointBodyLidarToIMU :1113-1122)
// The colour pass is order-preserving stream compaction: k_color_mark projects every point and flags the kept ones, a
// cub::DeviceScan gives each kept point its output slot (as vg_enqueue), k_color_emit gathers the pixel and writes the
// world-frame record.  DESIGN.md §9 states the contract.  The TU is compiled with -fmad=false; the double arithmetic is
// written with explicit round-to-nearest intrinsics as well, so no contraction can change a pixel.
#pragma once
#include "frontend_kernels.cuh"

namespace flb {

// M = internalMatProject · externalMat, row-major 3×4 (computed on the host in double, sums in index order)
struct CamProj { double M[12]; int W, H; };

// c = M·(p, 1) with the sums in index order; u = c0/c2, v = c1/c2.  A pixel is kept iff trunc(u) ∈ [0, W) and trunc(v)
// ∈ [0, H), i.e. −1 < u < W and −1 < v < H (NaN and ±inf fail both), and the lidar-frame x > 0.  Returns the pixel
// index v·W + u, or −1.
__device__ __forceinline__ int color_pixel(const CamProj& c, float4 p) {
  if (!(p.x > 0.f)) return -1;
  const double x = p.x, y = p.y, z = p.z;
  double r[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double* m = c.M + 4 * k;
    r[k] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dmul_rn(m[1], y)), __dmul_rn(m[2], z)), m[3]);
  }
  const double u = __ddiv_rn(r[0], r[2]), v = __ddiv_rn(r[1], r[2]);
  if (!(u > -1.0 && u < (double)c.W && v > -1.0 && v < (double)c.H)) return -1;
  return (int)v * c.W + (int)u;
}

__global__ void k_color_mark(CamProj c, const float4* __restrict__ pts, int n, int* __restrict__ pix, int* __restrict__ flags) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int q = color_pixel(c, pts[i]);
    pix[i] = q;
    flags[i] = q >= 0 ? 1 : 0;
  }
}

// Kept point i goes to slot pos[i] (exclusive scan of the flags): x, y, z in the world frame (body_to_world, the same
// arithmetic as flb_frontend_points_to_world), intensity carried, colour as PCL_ADD_RGB's bytes b, g, r, a = 255.  The
// thread of the last point writes the count.
__global__ void k_color_emit(PoseDev s, const float4* __restrict__ pts, int n, const int* __restrict__ pix,
                             const int* __restrict__ pos, const unsigned char* __restrict__ img, float4* __restrict__ out_xyzi,
                             unsigned* __restrict__ out_bgra, int* __restrict__ count) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int q = pix[i];
    if (q >= 0) {
      const int o = pos[i];
      const unsigned char* b = img + 3 * (size_t)q;
      out_xyzi[o] = body_to_world(s, pts[i]);
      out_bgra[o] = (unsigned)b[0] | ((unsigned)b[1] << 8) | ((unsigned)b[2] << 16) | (255u << 24);
    }
    if (i == n - 1) *count = pos[i] + (q >= 0 ? 1 : 0);
  }
}

// RGBpointBodyLidarToIMU: offR·p + offT in double (the first half of body_to_world), rounded to float, intensity carried
__global__ void k_to_imu(PoseDev s, const float4* __restrict__ body, float4* __restrict__ out, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 pb = body[i];
    double ax, ay, az;
    qrot_d(s.offR, (double)pb.x, (double)pb.y, (double)pb.z, ax, ay, az);
    out[i] = make_float4((float)__dadd_rn(ax, s.offT[0]), (float)__dadd_rn(ay, s.offT[1]), (float)__dadd_rn(az, s.offT[2]), pb.w);
  }
}

}  // namespace flb

// frontend_kernels.cuh — the rows either side of the per-scan path (SURVEY.md §8f), as sm_90a kernels:
//   rank 2  UndistortPcl backward pass          src/IMU_Processing.hpp:241-243 (time sort), :334-386 (compensation)
//   rank 1  pcl::VoxelGrid centroid filter      src/laserMapping.cpp:2322-2323 (leaf :2135); PCL 1.10 voxel_grid.hpp
//   rank 3  transformPointCloud (key frames)    include/common_lib.h:711-734, used by recontructIKdTree laserMapping.cpp:636
//           (the kernel is k_kf_assemble in keyframe_kernels.cuh)
//   rank 4  pointBodyToWorld / RGBpointBodyToWorld for publishing   src/laserMapping.cpp:1077-1110, :1502-1540
// All of it is per-point streaming work (HBM bound, a few dozen bytes per point); sorting is cub::DeviceRadixSort.
// The TU is compiled with -fmad=false: the reference is built without FMA contraction (CMakeLists.txt:9, no -march).
#pragma once
#include "knn_kernels.cuh"

namespace flb {

// monotone float -> uint map (radix-sortable; -0.0 < +0.0 as for the total order, NaN sorts last for positive NaN)
__device__ __forceinline__ unsigned f2ordu(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordu2f(unsigned o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o);
}

// strided host-layout points (e.g. 48-byte pcl::PointXYZINormal: x@0 y@4 z@8 intensity@32 curvature@36) -> float4
// (x,y,z,intensity) + curvature; a negative offset means "field absent" (0).
__global__ void k_pack_xyzic(const unsigned char* __restrict__ src, int stride, int off_i, int off_c, float4* __restrict__ dst,
                             float* __restrict__ curv, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned char* b = src + (size_t)i * stride;
    const float* p = reinterpret_cast<const float*>(b);
    const float in = off_i >= 0 ? *reinterpret_cast<const float*>(b + off_i) : 0.f;
    dst[i] = make_float4(p[0], p[1], p[2], in);
    if (curv) curv[i] = off_c >= 0 ? *reinterpret_cast<const float*>(b + off_c) : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------ undistortion
constexpr int IMU_POSE_DOUBLES = 22;   // Pose6D: offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9] (msg/Pose6D.msg)
constexpr int MAX_IMU_POSES = 256;     // 22*8*256 = 44 KB staged in shared memory (typical scans: 20-100 IMU samples)

struct UndistortEnd {   // imu_state after the forward propagation (IMU_Processing.hpp:329)
  double rot[4], offR[4], pos[3], offT[3];
};

__global__ void k_time_keys(const float* __restrict__ curv, unsigned* __restrict__ keys, int* __restrict__ vals, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    keys[i] = f2ordu(curv[i]);
    vals[i] = i;
  }
}

__device__ __forceinline__ void exp_so3_d(const double* w, double dt, double* R) {   // Exp(ang_vel, dt), math_tools.h:39-61
  const double n = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  R[0] = 1.0; R[1] = 0.0; R[2] = 0.0; R[3] = 0.0; R[4] = 1.0; R[5] = 0.0; R[6] = 0.0; R[7] = 0.0; R[8] = 1.0;
  if (!(n > 0.0000001)) return;
  const double a0 = w[0] / n, a1 = w[1] / n, a2 = w[2] / n;
  const double K[9] = {0.0, -a2, a1, a2, 0.0, -a0, -a1, a0, 0.0};
  const double r = n * dt;
  double s, c;
  sincos(r, &s, &c);
  const double c1 = 1.0 - c;
  double cK[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) cK[i] = c1 * K[i];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double kk = cK[i * 3 + 0] * K[j] + cK[i * 3 + 1] * K[3 + j] + cK[i * 3 + 2] * K[6 + j];
      R[i * 3 + j] = (R[i * 3 + j] + s * K[i * 3 + j]) + kk;
    }
}

// one compensation with segment (head, tail) (IMU_Processing.hpp:353-378)
__device__ __forceinline__ void undistort_point(float& px, float& py, float& pz, double t, const double* head, const double* tail,
                                                const UndistortEnd& e) {
  const double dt = t - head[0];
  double E[9], Ri[9];
  exp_so3_d(tail + 4, dt, E);
  const double* Rm = head + 13;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Ri[i * 3 + j] = Rm[i * 3] * E[j] + Rm[i * 3 + 1] * E[3 + j] + Rm[i * 3 + 2] * E[6 + j];
  double T[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) T[k] = ((head[10 + k] + head[7 + k] * dt) + ((0.5 * tail[1 + k]) * dt) * dt) - e.pos[k];
  double ax, ay, az;
  qrot_d(e.offR, (double)px, (double)py, (double)pz, ax, ay, az);
  ax += e.offT[0]; ay += e.offT[1]; az += e.offT[2];
  double bx = (Ri[0] * ax + Ri[1] * ay + Ri[2] * az) + T[0];
  double by = (Ri[3] * ax + Ri[4] * ay + Ri[5] * az) + T[1];
  double bz = (Ri[6] * ax + Ri[7] * ay + Ri[8] * az) + T[2];
  const double rc[4] = {-e.rot[0], -e.rot[1], -e.rot[2], e.rot[3]};
  const double oc[4] = {-e.offR[0], -e.offR[1], -e.offR[2], e.offR[3]};
  double cx, cy, cz, dx, dy, dz;
  qrot_d(rc, bx, by, bz, cx, cy, cz);
  cx -= e.offT[0]; cy -= e.offT[1]; cz -= e.offT[2];
  qrot_d(oc, cx, cy, cz, dx, dy, dz);
  px = (float)dx; py = (float)dy; pz = (float)dz;
}

// Thread j handles the j-th point in time order (perm from the stable radix sort by curvature).  A point belongs to
// the LAST segment whose head time it exceeds (what the reference's backward double sweep computes for time-sorted
// points); points not later than IMUpose[0] stay untouched.  Quirk kept: the first sorted point is compensated again by
// every earlier segment whose head time it exceeds (the `break` at begin() leaves the iterator on it, :382-383).
// end26 / np_dev (both null, or both set): the end pose and the pose count come from the device (the state26 and
// n_poses of the IMU propagation's record) instead of `e` / `np`; np is then the capacity the shared memory holds.
__global__ void k_undistort(const float4* __restrict__ pts, const float* __restrict__ curv, const int* __restrict__ perm, int n,
                            const double* __restrict__ poses, int np, UndistortEnd e, float4* __restrict__ out,
                            float* __restrict__ out_curv, const double* __restrict__ end26 = nullptr,
                            const int* __restrict__ np_dev = nullptr) {
  extern __shared__ double sp[];
  if (end26) {
    np = *np_dev;
    for (int k = 0; k < 4; ++k) { e.rot[k] = end26[3 + k]; e.offR[k] = end26[7 + k]; }
    for (int k = 0; k < 3; ++k) { e.pos[k] = end26[k]; e.offT[k] = end26[11 + k]; }
  }
  for (int k = threadIdx.x; k < np * IMU_POSE_DOUBLES; k += blockDim.x) sp[k] = poses[k];
  __syncthreads();
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const int i = perm[j];
    float4 p = pts[i];
    const float cf = curv[i];
    const double t = (double)cf / double(1000);
    int h = np - 2;
    while (h >= 0 && !(t > sp[h * IMU_POSE_DOUBLES])) --h;
    if (h >= 0) {
      undistort_point(p.x, p.y, p.z, t, sp + h * IMU_POSE_DOUBLES, sp + (h + 1) * IMU_POSE_DOUBLES, e);
      if (j == 0) {
        for (int g = h - 1; g >= 0; --g)
          if (t > sp[g * IMU_POSE_DOUBLES])
            undistort_point(p.x, p.y, p.z, t, sp + g * IMU_POSE_DOUBLES, sp + (g + 1) * IMU_POSE_DOUBLES, e);
      }
    }
    out[j] = p;
    out_curv[j] = cf;
  }
}

// ------------------------------------------------------------------------------------------------ voxel grid
// d_mm[0..2] = ordered-uint min x,y,z ; d_mm[3..5] = ordered-uint max ; d_mm[6] = overflow flag ; d_mm[7] = #outputs
__global__ void k_vg_init(unsigned* mm) {
  if (threadIdx.x < 3) mm[threadIdx.x] = 0xFFFFFFFFu;
  else if (threadIdx.x < 8) mm[threadIdx.x] = 0u;
}
__global__ void k_vg_minmax(const float4* __restrict__ pts, int n, unsigned* __restrict__ mm) {   // getMinMax3D
  unsigned lo[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, hi[3] = {0u, 0u, 0u};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = pts[i];
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) continue;
    const unsigned ox = f2ordu(p.x), oy = f2ordu(p.y), oz = f2ordu(p.z);
    lo[0] = min(lo[0], ox); lo[1] = min(lo[1], oy); lo[2] = min(lo[2], oz);
    hi[0] = max(hi[0], ox); hi[1] = max(hi[1], oy); hi[2] = max(hi[2], oz);
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    lo[k] = __reduce_min_sync(FULL, lo[k]);
    hi[k] = __reduce_max_sync(FULL, hi[k]);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      atomicMin(&mm[k], lo[k]);
      atomicMax(&mm[3 + k], hi[k]);
    }
  }
}

struct VgGrid { int min_b[3]; int mul[3]; bool overflow; };
// min_b_, div_b_, divb_mul_ and the overflow guard of applyFilter, recomputed per thread from the 6 extrema (cheap)
__device__ __forceinline__ VgGrid vg_grid(const unsigned* mm, float inv) {
  VgGrid g;
  float mn[3], mx[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) { mn[k] = ordu2f(mm[k]); mx[k] = ordu2f(mm[3 + k]); }
  const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1;
  const long long dy = (long long)((mx[1] - mn[1]) * inv) + 1;
  const long long dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  g.overflow = (dx * dy * dz) > (long long)INT_MAX;
  int div[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    g.min_b[k] = (int)floorf(mn[k] * inv);
    div[k] = (int)floorf(mx[k] * inv) - g.min_b[k] + 1;
  }
  g.mul[0] = 1; g.mul[1] = div[0]; g.mul[2] = div[0] * div[1];
  return g;
}

__global__ void k_vg_keys(const float4* __restrict__ pts, int n, float inv, unsigned* __restrict__ mm, unsigned* __restrict__ keys,
                          int* __restrict__ vals) {
  const VgGrid g = vg_grid(mm, inv);
  if (blockIdx.x == 0 && threadIdx.x == 0) mm[6] = g.overflow ? 1u : 0u;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = pts[i];
    unsigned key = 0xFFFFFFFFu;   // non-finite points are dropped (PCL does so for non-dense clouds)
    if (!g.overflow && isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      const int i0 = (int)(floorf(p.x * inv) - (float)g.min_b[0]);
      const int i1 = (int)(floorf(p.y * inv) - (float)g.min_b[1]);
      const int i2 = (int)(floorf(p.z * inv) - (float)g.min_b[2]);
      key = (unsigned)(i0 * g.mul[0] + i1 * g.mul[1] + i2 * g.mul[2]);
    }
    keys[i] = key;
    vals[i] = i;
  }
}

__global__ void k_vg_heads(const unsigned* __restrict__ keys, int n, int* __restrict__ flags) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned k = keys[i];
    flags[i] = (k != 0xFFFFFFFFu && (i == 0 || keys[i - 1] != k)) ? 1 : 0;
  }
}

// The thread of each leaf's first sorted point sums the leaf sequentially in sorted order (stable sort => ascending
// input index, a fixed order) exactly as CentroidPoint does: float sums, then division by the count as a float.
__global__ void k_vg_centroid(const float4* __restrict__ pts, const float* __restrict__ curv, const unsigned* __restrict__ keys,
                              const int* __restrict__ vals, const int* __restrict__ flags, const int* __restrict__ pos, int n,
                              float4* __restrict__ out, float* __restrict__ out_curv, int out_cap, unsigned* __restrict__ mm) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!flags[i]) continue;
    const unsigned k = keys[i];
    float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f, sc = 0.f;
    int j = i;
    for (; j < n && keys[j] == k; ++j) {
      const int src = vals[j];
      const float4 p = pts[src];
      sx += p.x; sy += p.y; sz += p.z; si += p.w;
      if (curv) sc += curv[src];
    }
    const float cnt = (float)(j - i);
    const int o = pos[i];
    if (o < out_cap) {
      out[o] = make_float4(sx / cnt, sy / cnt, sz / cnt, si / cnt);
      if (out_curv) out_curv[o] = sc / cnt;
    }
    if (j == n || keys[j] == 0xFFFFFFFFu) mm[7] = (unsigned)(o + 1);   // the last leaf publishes the output count
  }
}

// ------------------------------------------------------------------------------------------------ transforms
// transformPointCloud (common_lib.h:711-734): float affine "t00*x + t01*y + t02*z + t03", intensity copied; applied to
// key-frame clouds by k_kf_assemble (keyframe_kernels.cuh)
struct Affine12 { float t[12]; };

}  // namespace flb

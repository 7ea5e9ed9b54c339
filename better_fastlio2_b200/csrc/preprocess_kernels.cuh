// preprocess_kernels.cuh — Preprocess::process with feature extraction off (src/preprocess.cpp), as sm_90a kernels:
//   LIVOX  CustomMsg     livox_handler, feature-off branch        preprocess.cpp:178-204
//   VELO16 PointCloud2   velodyne_handler                         preprocess.cpp:302-340, :417-473
//   OUST64 PointCloud2   oust64_handler, feature-off branch       preprocess.cpp:271-297
// Driver records are decoded in place from the uploaded message (any stride, unaligned fields allowed), the kept points
// are compacted in input order into the front end's raw-scan buffers.  The TU is compiled with -fmad=false; the float
// expressions below are additionally spelled with _rn intrinsics where the reference's evaluation order matters.
#pragma once
#include "frontend_kernels.cuh"

namespace flb {

enum { PP_LIVOX = 1, PP_VELO16 = 2, PP_OUST64 = 3 };

struct PpParams {
  int n, stride, pfn, n_scans;
  int off_x, off_y, off_z, off_i, off_t, off_ring, off_tag, off_line;
  float tscale;     // time_unit_scale
  double blind2;    // blind * blind
  double omega_l;   // 0.361 * SCAN_RATE
  double wrap;      // 360.0 / omega_l
};

struct PpOut {      // the one read-back of a preprocess call
  int count;        // pl_surf.size()
  float last_curv;  // pl_surf.points.back().curvature
  int bad_ring;     // 1 + the largest ring >= n_scans seen (0: none)
  int pad;
};

// field loads from a record: little endian, alignment checked at run time (packed PointCloud2 layouts put a float at
// byte 18), a negative offset reads as 0 like pcl::fromROSMsg does for a field it cannot match
__device__ __forceinline__ unsigned pp_u32(const unsigned char* b, int off) {
  if (off < 0) return 0u;
  const unsigned char* p = b + off;
  if (((size_t)p & 3) == 0) return *reinterpret_cast<const unsigned*>(p);
  return (unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16) | ((unsigned)p[3] << 24);
}
__device__ __forceinline__ float pp_f32(const unsigned char* b, int off) { return __uint_as_float(pp_u32(b, off)); }
__device__ __forceinline__ unsigned pp_u16(const unsigned char* b, int off) {
  if (off < 0) return 0u;
  const unsigned char* p = b + off;
  return (unsigned)p[0] | ((unsigned)p[1] << 8);
}
__device__ __forceinline__ unsigned pp_u8(const unsigned char* b, int off) { return off < 0 ? 0u : (unsigned)b[off]; }

// x*x + y*y + z*z in float, left to right, no contraction
__device__ __forceinline__ float pp_r2(float x, float y, float z) {
  return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
}

// ------------------------------------------------------------------------------------------------ Ouster (:276-296)
__global__ void k_pp_ouster(const unsigned char* __restrict__ raw, PpParams p, float4* __restrict__ pts, float* __restrict__ curv,
                            int* __restrict__ keep) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    const unsigned char* b = raw + (size_t)i * p.stride;
    const float x = pp_f32(b, p.off_x), y = pp_f32(b, p.off_y), z = pp_f32(b, p.off_z);
    pts[i] = make_float4(x, y, z, pp_f32(b, p.off_i));
    curv[i] = __fmul_rn(__uint2float_rn(pp_u32(b, p.off_t)), p.tscale);
    // `if (range < blind*blind) continue;` with range a double from a float sum: NaN and r == blind are kept
    keep[i] = (i % p.pfn == 0) && !((double)pp_r2(x, y, z) < p.blind2);
  }
}

// ------------------------------------------------------------------------------------------------ Velodyne (:419-472)
// Decode.  With given_offset_time the curvature is time * time_unit_scale; otherwise the ring key (stable-sorted next),
// the yaw in degrees and the first input index of every ring are produced for the time synthesis.
__global__ void k_pp_velo(const unsigned char* __restrict__ raw, PpParams p, int synth, float4* __restrict__ pts,
                          float* __restrict__ curv, int* __restrict__ keep, unsigned* __restrict__ ring_key,
                          int* __restrict__ idx, double* __restrict__ yaw, int* __restrict__ ring_first, PpOut* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    const unsigned char* b = raw + (size_t)i * p.stride;
    const float x = pp_f32(b, p.off_x), y = pp_f32(b, p.off_y), z = pp_f32(b, p.off_z);
    pts[i] = make_float4(x, y, z, pp_f32(b, p.off_i));
    curv[i] = __fmul_rn(pp_f32(b, p.off_t), p.tscale);
    keep[i] = (i % p.pfn == 0) && ((double)pp_r2(x, y, z) > p.blind2);
    if (synth) {
      const int ring = (int)pp_u16(b, p.off_ring);
      if (ring >= p.n_scans) atomicMax(&out->bad_ring, ring + 1);
      else atomicMin(&ring_first[ring], i);
      ring_key[i] = (unsigned)min(ring, p.n_scans);
      idx[i] = i;
      yaw[i] = __dmul_rn(atan2((double)y, (double)x), 57.2957);
    }
  }
}

// (yaw <= yaw_fp ? yaw_fp - yaw : yaw_fp - yaw + 360.0) / omega_l, stored to float (:450-457)
__device__ __forceinline__ float pp_base(double yfp, double yw, double omega_l) {
  const double d = (yw <= yfp) ? __dsub_rn(yfp, yw) : __dadd_rn(__dsub_rn(yfp, yw), 360.0);
  return __double2float_rn(__ddiv_rn(d, omega_l));
}
// curvature += 360.0/omega_l: float + double in double, rounded to float (:459)
__device__ __forceinline__ float pp_wrapped(float base, double wrap) { return __double2float_rn(__dadd_rn((double)base, wrap)); }

// The ring-sequential recurrence `if (curvature < time_last) curvature += P; time_last = curvature;` as a scan: the
// value before point k is its predecessor's base or base + P (0 after the ring's first point), so point k is a map
// {0,1} -> {0,1} on "the predecessor wrapped".  Code: bit0 = f(0), bit1 = f(1), bit2 = first point of a ring (a
// segment head; its map is the constant 0 since the first point's curvature is 0).
struct PpMapCompose {   // a then b (segmented): associative
  __device__ __forceinline__ unsigned operator()(unsigned a, unsigned b) const {
    if (b & 4u) return b;
    const unsigned r0 = (b >> (a & 1u)) & 1u, r1 = (b >> ((a >> 1) & 1u)) & 1u;
    return r0 | (r1 << 1) | (a & 4u);
  }
};

// k = position in ring order (stable sort: input order inside a ring)
__global__ void k_pp_velo_maps(const unsigned* __restrict__ key, const int* __restrict__ idx, const double* __restrict__ yaw,
                               const int* __restrict__ ring_first, PpParams p, unsigned* __restrict__ maps) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < p.n; k += gridDim.x * blockDim.x) {
    const unsigned r = key[k];
    const bool head = (k == 0 || key[k - 1] != r);
    unsigned code = 4u;
    if (!head && (int)r < p.n_scans) {
      const double yfp = yaw[ring_first[r]];
      const float bj = pp_base(yfp, yaw[idx[k]], p.omega_l);
      float tl0 = 0.f, tl1 = 0.f;   // the predecessor is the ring's first point: time_last = 0
      if (!(k == 1 || key[k - 2] != r)) {
        tl0 = pp_base(yfp, yaw[idx[k - 1]], p.omega_l);
        tl1 = pp_wrapped(tl0, p.wrap);
      }
      code = (bj < tl0 ? 1u : 0u) | (bj < tl1 ? 2u : 0u);   // NaN compares false, as in the reference
    }
    maps[k] = code;
  }
}

// after the inclusive segmented scan: bit0 of scanned[k] = "point k wrapped"; ring heads are dropped (the `continue`)
__global__ void k_pp_velo_apply(const unsigned* __restrict__ key, const int* __restrict__ idx, const double* __restrict__ yaw,
                                const int* __restrict__ ring_first, const unsigned* __restrict__ scanned, PpParams p,
                                float* __restrict__ curv, int* __restrict__ keep) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < p.n; k += gridDim.x * blockDim.x) {
    const unsigned r = key[k];
    if ((int)r >= p.n_scans) continue;   // the call fails on such a ring
    const int i = idx[k];
    if (k == 0 || key[k - 1] != r) {
      keep[i] = 0;
      curv[i] = 0.f;
      continue;
    }
    const float b = pp_base(yaw[ring_first[r]], yaw[i], p.omega_l);
    curv[i] = (scanned[k] & 1u) ? pp_wrapped(b, p.wrap) : b;
  }
}

// ------------------------------------------------------------------------------------------------ Livox (:181-203)
__global__ void k_pp_livox(const unsigned char* __restrict__ raw, PpParams p, float4* __restrict__ pts, float* __restrict__ curv,
                           int* __restrict__ valid) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    const unsigned char* b = raw + (size_t)i * p.stride;
    pts[i] = make_float4(pp_f32(b, p.off_x), pp_f32(b, p.off_y), pp_f32(b, p.off_z), (float)pp_u8(b, p.off_i));
    curv[i] = __fdiv_rn(__uint2float_rn(pp_u32(b, p.off_t)), 1000000.f);   // offset_time / float(1000000)
    const unsigned tag = pp_u8(b, p.off_tag) & 0x30u;
    valid[i] = (i >= 1 && (int)pp_u8(b, p.off_line) < p.n_scans && (tag == 0x10u || tag == 0x00u)) ? 1 : 0;
  }
}

// excl[i] = valid records before i, so valid_num at i is excl[i] + valid[i] and at i-1 it is excl[i].  A record is
// filled when valid_num % point_filter_num == 0; pl_full[i-1] is the previous record if that one was filled, else the
// zero point pl_full.resize() left there.
__global__ void k_pp_livox_keep(const float4* __restrict__ pts, const int* __restrict__ valid, const int* __restrict__ excl,
                                PpParams p, int* __restrict__ keep) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    const unsigned pf = (unsigned)p.pfn;
    const unsigned vn = (unsigned)excl[i] + (unsigned)valid[i];
    int k = 0;
    if (valid[i] && vn % pf == 0u) {
      const bool prev_filled = i >= 2 && valid[i - 1] && ((unsigned)excl[i] % pf == 0u);
      const float4 c = pts[i];
      const float4 q = prev_filled ? pts[i - 1] : make_float4(0.f, 0.f, 0.f, 0.f);
      const double ax = fabsf(__fsub_rn(c.x, q.x)), ay = fabsf(__fsub_rn(c.y, q.y)), az = fabsf(__fsub_rn(c.z, q.z));
      // `a || b || c && d`: the blind cut only applies when x and y both repeat (:197)
      k = (ax > 1e-7 || ay > 1e-7 || (az > 1e-7 && (double)pp_r2(c.x, c.y, c.z) > p.blind2)) ? 1 : 0;
    }
    keep[i] = k;
  }
}

// ------------------------------------------------------------------------------------------------ compaction
// pos = exclusive scan of keep; kept points land in input order in the raw-scan buffers (pl_surf.push_back order)
__global__ void k_pp_scatter(const float4* __restrict__ pts, const float* __restrict__ curv, const int* __restrict__ keep,
                             const int* __restrict__ pos, int n, float4* __restrict__ out, float* __restrict__ out_curv,
                             PpOut* __restrict__ res) {
  const int total = pos[n - 1] + keep[n - 1];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    res->count = total;
    if (total == 0) res->last_curv = 0.f;
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!keep[i]) continue;
    const int o = pos[i];
    out[o] = pts[i];
    out_curv[o] = curv[i];
    if (o == total - 1) res->last_curv = curv[i];
  }
}

}  // namespace flb

// scan_context_kernels.cuh — the Scan Context descriptor (SCManager::makeScancontext, include/sc-relo/Scancontext.cpp
// :195-251) of key-frame selections, fused into the key-frame store's gather: each point is read once (16 B), transformed
// by its segment exactly as k_kf_assemble writes it (kf_point), binned and max-reduced.  Nothing is materialised.
//   loop gate   makeScancontext(*cureKeyframeCloud / *prevKeyframeCloud)   laserMapping.cpp:932-933
//   saver       makeAndSaveScancontextAndKeys(*save_cloud)                 laserMapping.cpp:2504-2505
// The TU is compiled with -fmad=false: every float / double operation below rounds as the reference's host code does.
#pragma once
#include "keyframe_kernels.cuh"

namespace flb {

constexpr int SC_RINGS = 20, SC_SECTORS = 60, SC_BINS = SC_RINGS * SC_SECTORS;   // PC_NUM_RING, PC_NUM_SECTOR
constexpr double SC_MAX_RADIUS = 80.0;                                           // PC_MAX_RADIUS
constexpr int SC_CHUNK = 4096;                                                   // points per chunk (one CTA pass)

// Points [begin, begin + count) of segment seg (indices as kf_point takes them) go into descriptor desc.
struct ScChunk {
  int seg, begin, count, desc;
};

// xy2theta (Scancontext.cpp:23-36) with the reference's types: float quotient, double atan and degrees, float result.
// The branches are taken literally (& of two tests; -0.0 >= 0), so x = -0, y > 0 gives -90 and x = ±0, y = 0 gives NaN.
__device__ __forceinline__ float sc_theta(float x, float y) {
  const double r2d = 180 / M_PI;
  if ((x >= 0) & (y >= 0)) return (float)(r2d * atan((double)(y / x)));
  if ((x < 0) & (y >= 0)) return (float)(180 - (r2d * atan((double)(y / (-x)))));
  if ((x < 0) & (y < 0)) return (float)(180 + (r2d * atan((double)(y / x))));
  return (float)(360 - (r2d * atan((double)((-y) / x))));
}

// Order-preserving key of a float: larger float, larger unsigned.  0 is below every key of a value > -1000, so it marks
// an untouched bin.
__device__ __forceinline__ unsigned sc_key(float v) {
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// The bin (ring * 60 + sector, 0-based) a point updates, or -1 when it updates none: out of range (> 80 m, compared in
// double; a NaN range is kept) or a height that cannot beat the bin's initial -1000 (<= -1000 or NaN).  A NaN reaches
// int() as 0 here and as INT_MIN on x86; both clamp to index 1.  *v = pt.z = (float)(z + LIDAR_HEIGHT), the sum in double.
__device__ __forceinline__ int sc_bin(float4 p, double lidar_height, float* v) {
  const float z = (float)((double)p.z + lidar_height) + 0.f;   // + 0: a -0 height is stored as +0 (it compares equal)
  const float range = sqrtf(p.x * p.x + p.y * p.y);
  const float angle = sc_theta(p.x, p.y);
  if ((double)range > SC_MAX_RADIUS || !(z > -1000.f)) return -1;
  const int ring = max(min(SC_RINGS, (int)ceil(((double)range / SC_MAX_RADIUS) * SC_RINGS)), 1);
  const int sector = max(min(SC_SECTORS, (int)ceil(((double)angle / 360.0) * SC_SECTORS)), 1);
  *v = z;
  return (ring - 1) * SC_SECTORS + (sector - 1);
}

// One CTA per chunk (grid-stride over the chunk table): 1200 keys in shared memory, max-reduced with shared atomics,
// then only the touched bins are flushed into keys[desc * 1200 + bin] with global atomicMax (keys zeroed beforehand).
__global__ void __launch_bounds__(256) k_sc_bins(const KfSeg* __restrict__ segs, const ScChunk* __restrict__ chunks, int n_chunks,
                                                 const float4* __restrict__ src, double lidar_height, unsigned* __restrict__ keys) {
  __shared__ unsigned sk[SC_BINS];
  for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    for (int b = threadIdx.x; b < SC_BINS; b += blockDim.x) sk[b] = 0u;
    __syncthreads();
    const ScChunk ch = chunks[c];
    const KfSeg* s = segs + ch.seg;
    for (int i = ch.begin + threadIdx.x; i < ch.begin + ch.count; i += blockDim.x) {
      long long j;
      float v;
      const int bin = sc_bin(kf_point(s, src, i, &j), lidar_height, &v);
      if (bin >= 0) atomicMax(&sk[bin], sc_key(v));
    }
    __syncthreads();
    unsigned* out = keys + (size_t)ch.desc * SC_BINS;
    for (int b = threadIdx.x; b < SC_BINS; b += blockDim.x)
      if (sk[b]) atomicMax(&out[b], sk[b]);
    __syncthreads();
  }
}

}  // namespace flb

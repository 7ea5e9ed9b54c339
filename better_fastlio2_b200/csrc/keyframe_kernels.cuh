// keyframe_kernels.cuh — assembly of key-frame clouds (SURVEY.md §8f rank 3) as one sm_90a launch:
//   *subMap += *transformPointCloud(surfCloudKeyFrames[k], &cloudKeyPoses6D->points[k])   laserMapping.cpp:636, :1862, :1768
//   *nearKeyframes += *surfCloudKeyFrames[key]  /  += transformPointCloud(.., finalTrans)  laserMapping.cpp:869-877
// over an ordered selection of clouds, whatever the number of key frames.  Per-point streaming work (36 B in, 20 B out).
// The TU is compiled with -fmad=false: t0*x + t1*y + t2*z + t3 rounds after every operation, as the reference does.
#pragma once
#include "frontend_kernels.cuh"

namespace flb {

// One selected key frame: `count` points read from src[src_off..] and written to out[dst_off..].  copy != 0: the record
// is copied verbatim (curvature included); else t (row-major 3x4) is applied and curvature is 0, as transformPointCloud
// writes into freshly resized points (common_lib.h:711-749).
struct KfSeg {
  float t[12];
  long long src_off;
  int dst_off, count, copy, pad;
};

// Output point i's segment: the last one whose dst_off <= i (the host drops empty segments, so dst_off is strictly
// increasing).  Neighbouring threads share a segment, so the search reads the same cached words.
__device__ __forceinline__ const KfSeg* kf_seg_of(const KfSeg* __restrict__ segs, int n_seg, int i) {
  int lo = 0, hi = n_seg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&segs[mid].dst_off) <= i) lo = mid; else hi = mid - 1;
  }
  return segs + lo;
}

// Output point i of segment s: the stored record src[j] (copy) or its affine, x, y, z and intensity.  Every reader of a
// selection (the assembly, the Scan Context bins) goes through this, so they all see the same points.
__device__ __forceinline__ float4 kf_point(const KfSeg* s, const float4* __restrict__ src, int i, long long* j_out) {
  const long long j = s->src_off + (i - s->dst_off);
  *j_out = j;
  const float4 p = src[j];
  if (s->copy) return p;
  const float* a = s->t;
  return make_float4(a[0] * p.x + a[1] * p.y + a[2] * p.z + a[3], a[4] * p.x + a[5] * p.y + a[6] * p.z + a[7],
                     a[8] * p.x + a[9] * p.y + a[10] * p.z + a[11], p.w);
}

// Thread i writes output point i.
__global__ void k_kf_assemble(const KfSeg* __restrict__ segs, int n_seg, const float4* __restrict__ src, const float* __restrict__ src_curv,
                              int n, float4* __restrict__ out, float* __restrict__ out_curv) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const KfSeg* s = kf_seg_of(segs, n_seg, i);
    long long j;
    out[i] = kf_point(s, src, i, &j);
    if (out_curv) out_curv[i] = (s->copy && src_curv) ? src_curv[j] : 0.f;
  }
}

}  // namespace flb

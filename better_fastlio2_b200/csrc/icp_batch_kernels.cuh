// icp_batch_kernels.cuh — the lockstep passes of flb_keyframes_icp_batch (icp_batch_host.cuh): every active pair of a
// round runs flb_keyframes_icp's iteration at once.  Each pair's target has its own grid index (built by the kernels of
// icp_kernels.cuh into its slice of one packed index); a pass is one thread-per-query 1-NN kernel and one far kernel over
// all active pairs' queries, each query reading its pair's grid and transform, then one segmented reduction per sum
// record.  The segmented reduction gives every pair k_reduce's partition for that pair's n (nb = 2 x SMs contiguous
// ranges, strided thread sums, the same tree, block partials summed in block order), so a pair's sums are the bits
// flb_keyframes_icp computes, whatever else the round holds.  Compiled with -fmad=false as icp_kernels.cuh.
#pragma once
#include "icp_kernels.cuh"

namespace flb {

constexpr int ICPB_REC = 17;   // doubles of a pair's sum record: the pairs record (8), then the cross products (9)

// One active pair of a pass.  Source slices (source, moved source, visiting order, matches) start at s_off; the target
// and its sorted finite points at t_off; the CSR offsets at cs_off; the coarse boxes at box_off.  Its queries are
// [q0, q0 + n_s) of the pass.
struct IcpBatchItem {
  IcpGrid g;
  IcpXf xf;
  int q0, n_s, s_off, t_off, cs_off, box_off;
};

// The item of pass query t: the last one whose q0 <= t (q0 strictly increasing: no active pair is empty).
__device__ __forceinline__ int icpb_item(const IcpBatchItem* __restrict__ items, int n_items, int t) {
  int lo = 0, hi = n_items - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].q0 <= t) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// k_icp_nn over every active pair: q = xf(in[i]) into out[i], the fine rings on the pair's grid, results by packed source
// index (idx = the nearest target's index within the pair's target); an open query goes to open_list as (index, item).
__global__ void __launch_bounds__(256) k_icpb_nn(const IcpBatchItem* __restrict__ items, int n_items, int n_q, const int* __restrict__ order,
                                                const float4* in, float4* out, const float4* __restrict__ sorted,
                                                const int* __restrict__ cs_all, int* __restrict__ idx, float* __restrict__ d2,
                                                int2* __restrict__ open_list, int* __restrict__ open_n) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_q; t += gridDim.x * blockDim.x) {
    const int s = icpb_item(items, n_items, t);
    const IcpBatchItem& it = items[s];
    const IcpGrid g = it.g;
    const int i = it.s_off + __ldg(&order[it.s_off + (t - it.q0)]);
    float4 q = in[i];
    if (it.xf.apply) {
      const float* m = it.xf.m;
      q = make_float4(m[0] * q.x + m[1] * q.y + m[2] * q.z + m[3], m[4] * q.x + m[5] * q.y + m[6] * q.z + m[7],
                      m[8] * q.x + m[9] * q.y + m[10] * q.z + m[11], q.w);
    }
    out[i] = q;
    if (!icp_finite(q)) { idx[i] = -1; d2[i] = INFINITY; continue; }
    const float4* pts = sorted + it.t_off;
    const int* cs = cs_all + it.cs_off;
    float best = INFINITY;
    int bi = INT_MAX;
    const bool closed = icp_fine_rings(g, IcpQuery{q}, best, [&](unsigned k) {
      icp_scan(pts, __ldg(&cs[k]), __ldg(&cs[k + 1]), q, best, bi);
    });
    idx[i] = bi;
    d2[i] = best;
    if (!closed) open_list[atomicAdd(open_n, 1)] = make_int2(i, s);
  }
}

// k_icp_nn_far over the open queries of every active pair, each on its pair's grid, boxes and sorted points.
__global__ void __launch_bounds__(256) k_icpb_nn_far(const IcpBatchItem* __restrict__ items, const int2* __restrict__ open_list,
                                                    const int* __restrict__ open_n, const float4* __restrict__ xq,
                                                    const float4* __restrict__ sorted, const int* __restrict__ cs_all,
                                                    const IcpBox* __restrict__ box_all, int* __restrict__ idx, float* __restrict__ d2) {
  const int lane = threadIdx.x & 31;
  const int n_open = *open_n;
  for (int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_open; w += (gridDim.x * blockDim.x) >> 5) {
    const int2 o = open_list[w];
    const int i = o.x;
    const IcpBatchItem& it = items[o.y];
    const IcpGrid g = it.g;
    const float4* pts = sorted + it.t_off;
    const int* cs = cs_all + it.cs_off;
    const float4 q = xq[i];
    float best = d2[i];
    int bi = idx[i];
    icp_coarse_rings<32>(g, box_all + it.box_off, IcpQuery{q}, best, [&](int id) {
      const int bx = (id % g.cx) * ICP_C, by = ((id / g.cx) % g.cy) * ICP_C, bz = (id / (g.cx * g.cy)) * ICP_C;
      for (int l = lane; l < ICP_C3; l += 32) {
        const int k = id * ICP_C3 + l;
        const int s = __ldg(&cs[k]), e = __ldg(&cs[k + 1]);
        if (s < e && icp_box_lb2(g, q, bx + l % ICP_C, by + (l / ICP_C) % ICP_C, bz + l / (ICP_C * ICP_C), 1) <= best)
          icp_scan(pts, s, e, q, best, bi);
      }
      for (int off = 16; off > 0; off >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        icp_take(ob, oi, best, bi);
      }
    });
    if (lane == 0) { idx[i] = bi; d2[i] = best; }
  }
}

// k_reduce per active pair: blocks [s * nb, (s + 1) * nb) reduce item s's n_s elements exactly as k_reduce with nb blocks
// does (op(s, item, i, a) for i in [0, n_s)) into out[s * ICPB_REC + k], k < K.  counters[s] starts at 0 and is left at 0.
template <int K, class Op>
__global__ void __launch_bounds__(256) k_icpb_reduce(const IcpBatchItem* __restrict__ items, int nb, Op op, double* __restrict__ partials_all,
                                                    unsigned* __restrict__ counters, double* __restrict__ out_all) {
  static_assert(K <= ICPB_REC, "a sum record holds ICPB_REC doubles");
  __shared__ double sh[K][256];
  __shared__ bool last;
  const int s = blockIdx.x / nb, blk = blockIdx.x % nb;
  const IcpBatchItem& it = items[s];
  const int n = it.n_s;
  double* partials = partials_all + (size_t)s * nb * K;
  double acc[K], a[K];
  for (int k = 0; k < K; ++k) acc[k] = 0.0;
  const int chunk = (n + nb - 1) / nb;
  const int b0 = blk * chunk, b1 = min(n, b0 + chunk);
  for (int i = b0 + threadIdx.x; i < b1; i += blockDim.x)
    if (op(s, it, i, a))
      for (int k = 0; k < K; ++k) acc[k] += a[k];
  for (int k = 0; k < K; ++k) sh[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int h = blockDim.x / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h)
      for (int k = 0; k < K; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int k = 0; k < K; ++k) partials[(size_t)blk * K + k] = sh[k][0];
    __threadfence();
    last = atomicAdd(&counters[s], 1u) == (unsigned)nb - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int k = 0; k < K; ++k) {
    double v = 0.0;
    for (int b = threadIdx.x; b < nb; b += blockDim.x) v += ((volatile double*)partials)[(size_t)b * K + k];
    sh[k][threadIdx.x] = v;
  }
  __syncthreads();
  for (int h = blockDim.x / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h)
      for (int k = 0; k < K; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int k = 0; k < K; ++k) out_all[(size_t)s * ICPB_REC + k] = sh[k][0];
    counters[s] = 0u;
  }
}

// IcpPairsOp on item s's slices (k_icpb_reduce<8>).
struct IcpBatchPairsOp {
  const int* idx;
  const float* d2;
  const float4* src;
  const float4* tgt;
  double max_d2;
  __device__ bool operator()(int, const IcpBatchItem& it, int i, double* a) const {
    return IcpPairsOp{idx + it.s_off, d2 + it.s_off, src + it.s_off, tgt + it.t_off, max_d2}(i, a);
  }
};

// IcpCrossOp on item s's slices with its own pairs record (k_icpb_reduce<9>, written 8 doubles into the record).
struct IcpBatchCrossOp {
  IcpBatchPairsOp pairs;
  const double* rec;
  __device__ bool operator()(int s, const IcpBatchItem& it, int i, double* a) const {
    const IcpPairsOp p{pairs.idx + it.s_off, pairs.d2 + it.s_off, pairs.src + it.s_off, pairs.tgt + it.t_off, pairs.max_d2};
    return IcpCrossOp{p, rec + (size_t)s * ICPB_REC}(i, a);
  }
};

}  // namespace flb

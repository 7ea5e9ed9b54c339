// fricp_kernels.cuh — the relocaliser's registration (FRICP<3>::point_to_point, include/FRICP-toolkit/FRICP.h:382-543, as
// Registeration::run calls it for regMode 0, 2, 3 and 4) on clouds normalised as registeration.h:47-60 does, in double:
//   the loop ICP's grid index (icp_kernels.cuh), built once per call over the float rounding of the normalised target,
//   with a double copy of the sorted target beside it;
//   an exact double 1-NN pass per iteration with the transform applied in the pass: icp_kernels.cuh's fine and coarse
//   walks with the double query FrQuery, the open queries finished warp-per-query over whole coarse cells;
//   an exact 7-NN self-query over the target (register top-7, thread per point on both walks) for the Welsch scale's
//   end value;
//   k_reduce over the means and over the energy and weighted moments (one fused record).
// The TU is compiled with -fmad=false: d² = (dx*dx + dy*dy) + dz*dz and the affine ((m0 x + m1 y) + m2 z) + m3 round
// after every operation, exactly as tests/cpp/fricp_oracle.cpp computes them.  1-NN tie rule: the smaller double d², then
// the lower target index (the position in the assembled target).
//
// Why the candidate enumeration is conservative for a double query: a target point t (double, |t| <= 1 after
// normalisation) was binned by its float rounding tf, |tf - t| <= 2^-24 |t|, through floor((tf - o) * inv_e) in float,
// whose rounding moves the cell boundary by a few float ulps of |tf - o| * inv_e, i.e. a few ulps of max(|t|, |o|) in
// length.  The grid's slack (IcpGrid::slack = 1e-3 e + 4e-6 (max |coordinate| + extent), icp_host.cuh) is more than 60
// float ulps of the largest coordinate, so every t lies inside its cell (and its coarse cell's float box) widened by
// slack.  The bounds below are computed in double from the query itself, so the query needs no rounding allowance, and a
// cell is skipped only when its widened bound exceeds the current best d² (times 1 - 1e-12, for the bound's own double
// rounding).
#pragma once
#include "icp_kernels.cuh"

namespace flb {

constexpr int FR_RED = 17;   // doubles of a step record: Σw, Σw x (3), Σw q (3), Σw x qᵀ (9, row-major), energy

// Row-major 3x4 double transform of the normalised source.
struct FrXf {
  double m[12];
};

__device__ __forceinline__ void fr_take(double d2, int idx, int pos, double& best, int& bi, int& bp) {
  if (d2 < best || (d2 == best && idx < bi)) { best = d2; bi = idx; bp = pos; }
}

// A double query on the float grid: binned by its float rounding, every bound computed in double from the query itself
// and widened by the grid's slack, a cell or box skipped only when its bound times 1 - 1e-12 exceeds the best d².
struct FrQuery {
  using real = double;
  double q[3];
  __device__ void cell(const IcpGrid& g, int* c) const {
    c[0] = icp_cell1((float)q[0], g.ox, g.inv_e, g.gx);
    c[1] = icp_cell1((float)q[1], g.oy, g.inv_e, g.gy);
    c[2] = icp_cell1((float)q[2], g.oz, g.inv_e, g.gz);
  }
  __device__ double d2(double4 a) const {
    const double dx = a.x - q[0], dy = a.y - q[1], dz = a.z - q[2];
    return (dx * dx + dy * dy) + dz * dz;
  }
  // lower bound of d² to any point binned into fine cell (ix, iy, iz)
  __device__ double cell_lb2(const IcpGrid& g, int ix, int iy, int iz) const {
    const double e = g.e, s = g.slack, o[3] = {g.ox, g.oy, g.oz};
    const int c[3] = {ix, iy, iz};
    double acc[3];
    for (int a = 0; a < 3; ++a) {
      const double lo = o[a] + (double)c[a] * e - s, hi = o[a] + (double)(c[a] + 1) * e + s;
      acc[a] = fmax(fmax(lo - q[a], q[a] - hi), 0.0);
    }
    return (acc[0] * acc[0] + acc[1] * acc[1]) + acc[2] * acc[2];
  }
  __device__ double box_lb2(const IcpGrid& g, const IcpBox& b) const {
    double acc[3];
    for (int a = 0; a < 3; ++a) acc[a] = fmax(fmax(((double)b.lo[a] - g.slack) - q[a], q[a] - ((double)b.hi[a] + g.slack)), 0.0);
    return (acc[0] * acc[0] + acc[1] * acc[1]) + acc[2] * acc[2];
  }
  // icp_ring_lb in double: the distance to every cell of Chebyshev ring r >= 1 around c, INFINITY when the ring has no
  // cell inside the grid
  __device__ bool ring_done(const IcpGrid& g, const int* c, const int* dims, int span, int r, double best) const {
    const double o[3] = {g.ox, g.oy, g.oz}, se = (double)g.e * span, s = g.slack;
    double lb = INFINITY;
    for (int a = 0; a < 3; ++a) {
      if (c[a] - r >= 0) lb = fmin(lb, fmax(q[a] - (o[a] + (double)(c[a] - r + 1) * se + s), 0.0));
      if (c[a] + r < dims[a]) lb = fmin(lb, fmax((o[a] + (double)(c[a] + r) * se - s) - q[a], 0.0));
    }
    return lb == INFINITY || lb * lb * (1.0 - 1e-12) > best;
  }
  __device__ static bool beats(double lb2, double best) { return lb2 * (1.0 - 1e-12) <= best; }
};

// q = T v, ((m0 x + m1 y) + m2 z) + m3 per row
__device__ __forceinline__ FrQuery fr_moved(const FrXf& xf, double4 v) {
  const double* m = xf.m;
  return FrQuery{{((m[0] * v.x + m[1] * v.y) + m[2] * v.z) + m[3], ((m[4] * v.x + m[5] * v.y) + m[6] * v.z) + m[7],
                  ((m[8] * v.x + m[9] * v.y) + m[10] * v.z) + m[11]}};
}

// ------------------------------------------------------------------------------------------------ normalisation
// The finite points' Σ p / scale (k_reduce<3>).
struct FrMeanOp {
  const float4* p;
  double scale;
  __device__ bool operator()(int i, double* a) const {
    const float4 v = p[i];
    if (!icp_finite(v)) return false;
    a[0] = (double)v.x / scale; a[1] = (double)v.y / scale; a[2] = (double)v.z / scale;
    return true;
  }
};

// out[i] = p / scale - mu in double (w = 1 for a finite point, 0 and NaN coordinates otherwise); outf (optional) its float
// rounding, the input of the index build.
__global__ void k_fr_normalise(const float4* __restrict__ p, int n, double scale, const double* __restrict__ mu, double4* __restrict__ out,
                               float4* __restrict__ outf) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 v = p[i];
    double4 o;
    if (icp_finite(v)) o = make_double4((double)v.x / scale - mu[0], (double)v.y / scale - mu[1], (double)v.z / scale - mu[2], 1.0);
    else o = make_double4(NAN, NAN, NAN, 0.0);
    out[i] = o;
    if (outf) outf[i] = make_float4((float)o.x, (float)o.y, (float)o.z, 0.f);
  }
}

// The sorted finite target in double, w = the original index.
__global__ void k_fr_gather(const int* __restrict__ vals, const double4* __restrict__ t, int n_fin, double4* __restrict__ out) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n_fin; j += gridDim.x * blockDim.x) {
    const int i = vals[j];
    const double4 v = t[i];
    out[j] = make_double4(v.x, v.y, v.z, (double)i);
  }
}

// Sort keys of the normalised source on the target grid (its initial visiting order); non-finite points sort last.
__global__ void k_fr_keys(IcpGrid g, const double4* __restrict__ x, int n, unsigned* __restrict__ keys, int* __restrict__ vals) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double4 v = x[i];
    if (v.w != 0.0) {
      int c[3];
      FrQuery{{v.x, v.y, v.z}}.cell(g, c);
      keys[i] = icp_key(g, c[0], c[1], c[2]);
    } else {
      keys[i] = ~0u;
    }
    vals[i] = i;
  }
}

// ------------------------------------------------------------------------------------------------ exact 1-NN
// Thread per query in visiting order: q = T x, then the fine rings.  Results by source index: pos[i] = the nearest
// target's sorted position (-1 for a non-finite source point), d2[i] its double d²; a query the rings do not close is
// appended to the open list for k_fr_nn_far.
__global__ void __launch_bounds__(256, 1) k_fr_nn(IcpGrid g, FrXf xf, const int* __restrict__ order, int n, const double4* __restrict__ x,
                                              const double4* __restrict__ pts, const int* __restrict__ cs, int* __restrict__ pos,
                                              double* __restrict__ d2, int* __restrict__ open_list, int* __restrict__ open_n) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    const int i = order[t];
    const double4 v = x[i];
    if (v.w == 0.0) { pos[i] = -1; d2[i] = INFINITY; continue; }
    const FrQuery q = fr_moved(xf, v);
    double best = INFINITY;
    int bi = INT_MAX, bp = -1;
    const bool closed = icp_fine_rings(g, q, best, [&](unsigned k) {
      const int e = __ldg(&cs[k + 1]);
      for (int j = __ldg(&cs[k]); j < e; ++j) {
        const double4 p = pts[j];
        fr_take(q.d2(p), (int)p.w, j, best, bi, bp);
      }
    });
    pos[i] = bp;
    d2[i] = best;
    if (!closed) open_list[atomicAdd(open_n, 1)] = i;
  }
}

// Warp per open query over the coarse rings, starting from the thread path's partial result.  A visited coarse cell's
// points (one contiguous range of the sorted target) are scanned by the lanes.
__global__ void __launch_bounds__(256) k_fr_nn_far(IcpGrid g, FrXf xf, const int* __restrict__ open_list, const int* __restrict__ open_n,
                                                  const double4* __restrict__ x, const double4* __restrict__ pts, const int* __restrict__ cs,
                                                  const IcpBox* __restrict__ box, int* __restrict__ pos, double* __restrict__ d2) {
  const int lane = threadIdx.x & 31;
  const int n_open = *open_n;
  for (int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_open; w += (gridDim.x * blockDim.x) >> 5) {
    const int i = open_list[w];
    const FrQuery q = fr_moved(xf, x[i]);
    double best = d2[i];
    int bp = pos[i], bi = bp >= 0 ? (int)pts[bp].w : INT_MAX;
    icp_coarse_rings<32>(g, box, q, best, [&](int id) {
      const int s = __ldg(&cs[(size_t)id * ICP_C3]), e = __ldg(&cs[(size_t)(id + 1) * ICP_C3]);
      for (int j = s + lane; j < e; j += 32) {
        const double4 p = pts[j];
        fr_take(q.d2(p), (int)p.w, j, best, bi, bp);
      }
      for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o), op = __shfl_xor_sync(0xffffffffu, bp, o);
        fr_take(ob, oi, op, best, bi, bp);
      }
    });
    if (lane == 0) { pos[i] = bp; d2[i] = best; }
  }
}

// The original target index of every source point's match (-1: none).
__global__ void k_fr_corr_index(const int* __restrict__ pos, const double4* __restrict__ pts, int n, int* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int p = pos[i];
    out[i] = p >= 0 ? (int)pts[p].w : -1;
  }
}

// ------------------------------------------------------------------------------------------------ 7-NN self-query
// igl::median of the k - 1 values after the first of an ascending list top[0..k): the middle one, or the mean of the two
// middle ones for an even count.
__device__ __forceinline__ double fr_median_tail(const double* top, int k) {
  const int n = k - 1, h = n / 2;
  return (n % 2 == 0) ? 0.5 * (top[1 + h] + top[h]) : top[1 + h];
}

__device__ __forceinline__ void fr_insert(double d, double* top, int k) {
  if (!(d < top[k - 1])) return;
  int s = k - 1;
  for (; s > 0 && top[s - 1] > d; --s) top[s] = top[s - 1];
  top[s] = d;
}

// Thread per finite target point j (sorted order): the k = min(7, n_fin) smallest d² to the target points (itself
// included, at 0) over the fine rings; med[j] = the median of the k - 1 after the first.  A point the rings do not close
// goes to the open list for k_fr_knn7_far.
__global__ void __launch_bounds__(256) k_fr_knn7(IcpGrid g, int n_fin, int k, const double4* __restrict__ pts, const int* __restrict__ cs,
                                                double* __restrict__ med, int* __restrict__ open_list,
                                                int* __restrict__ open_n) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n_fin; j += gridDim.x * blockDim.x) {
    const double4 v = pts[j];
    const FrQuery q{{v.x, v.y, v.z}};
    double top[7];
    for (int s = 0; s < 7; ++s) top[s] = INFINITY;
    const bool closed = icp_fine_rings(g, q, top[k - 1], [&](unsigned key) {
      const int e = __ldg(&cs[key + 1]);
      for (int t = __ldg(&cs[key]); t < e; ++t) fr_insert(q.d2(pts[t]), top, k);
    });
    if (!closed) open_list[atomicAdd(open_n, 1)] = j;
    else med[j] = fr_median_tail(top, k);
  }
}

// Thread per open point over the coarse rings, whole coarse cells scanned.  Open points are the isolated ones, whose
// coarse cells hold few points.
__global__ void __launch_bounds__(256) k_fr_knn7_far(IcpGrid g, int k, const int* __restrict__ open_list, const int* __restrict__ open_n,
                                                    const double4* __restrict__ pts, const int* __restrict__ cs, const IcpBox* __restrict__ box,
                                                    double* __restrict__ med) {
  const int n_open = *open_n;
  for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < n_open; w += gridDim.x * blockDim.x) {
    const int j = open_list[w];
    const double4 v = pts[j];
    const FrQuery q{{v.x, v.y, v.z}};
    double top[7];   // from an empty list: the coarse cells hold the fine rings' points again
    for (int s = 0; s < 7; ++s) top[s] = INFINITY;
    icp_coarse_rings<1>(g, box, q, top[k - 1], [&](int id) {
      const int s = __ldg(&cs[(size_t)id * ICP_C3]), e = __ldg(&cs[(size_t)(id + 1) * ICP_C3]);
      for (int p = s; p < e; ++p) fr_insert(q.d2(pts[p]), top, k);
    });
    med[j] = fr_median_tail(top, k);
  }
}

// r = sqrt(d²) of every source point (+inf for a non-finite one), the input of the residual median.
__global__ void k_fr_resid(const double* __restrict__ d2, int n, double* __restrict__ r) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) r[i] = sqrt(d2[i]);
}

// ------------------------------------------------------------------------------------------------ reductions
// Energy and weighted moments of the current pairs (FRICP.h:452 get_energy, :490 robust_weight, :186-194 the weighted
// means and cross-covariance as raw moments): r = sqrt(d²), Welsch weight exp(-r²/(2ν²)) and energy 1 - weight, or
// weight 1 and energy r² without a robust function.
struct FrStepOp {
  const double4* x;
  const double4* pts;
  const int* pos;
  const double* d2;
  double nu;
  int welsch;
  __device__ bool operator()(int i, double* a) const {
    const int p = pos[i];
    if (p < 0) return false;
    const double r = sqrt(d2[i]);
    double w, en;
    if (welsch) {
      w = exp(-r * r / (2 * nu * nu));
      en = 1.0 - w;
    } else {
      w = 1.0;
      en = r * r;
    }
    const double4 s = x[i], t = pts[p];
    const double xs[3] = {s.x, s.y, s.z}, qt[3] = {t.x, t.y, t.z};
    a[0] = w;
    for (int c = 0; c < 3; ++c) { a[1 + c] = w * xs[c]; a[4 + c] = w * qt[c]; }
    for (int r0 = 0; r0 < 3; ++r0)
      for (int c = 0; c < 3; ++c) a[7 + 3 * r0 + c] = w * xs[r0] * qt[c];
    a[16] = en;
    return true;
  }
};

}  // namespace flb

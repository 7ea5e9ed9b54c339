// fricp_kernels.cuh — the relocaliser's registration (FRICP<3>::point_to_point, include/FRICP-toolkit/FRICP.h:382-543, as
// Registeration::run calls it for regMode 0, 2, 3 and 4) on clouds normalised as registeration.h:47-60 does, in double:
//   the loop ICP's index over the target (icp_kernels.cuh: finite points sorted by the cell of a uniform grid, CSR cell
//   offsets, coarse-cell boxes), built once per call over the float rounding of the normalised target;
//   an exact double 1-NN pass per iteration with the transform applied in the pass (thread-per-query fine rings, the few
//   open queries finished warp-per-query over whole coarse cells, nearest ring first, pruned by box distance);
//   an exact 7-NN self-query over the target (register top-7) for the Welsch scale's end value;
//   fixed-order double reductions (means; energy and weighted moments fused in one pass).
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

__device__ __forceinline__ double fr_d2(double4 a, double qx, double qy, double qz) {
  const double dx = a.x - qx, dy = a.y - qy, dz = a.z - qz;
  return (dx * dx + dy * dy) + dz * dz;
}

// Lower bound of d² from q to any point binned into the block of span^3 fine cells at (ix, iy, iz).
__device__ __forceinline__ double fr_box_lb2(const IcpGrid& g, const double* q, int ix, int iy, int iz, int span) {
  const double e = g.e, s = g.slack, o[3] = {g.ox, g.oy, g.oz};
  const int c[3] = {ix, iy, iz};
  double acc[3];
  for (int a = 0; a < 3; ++a) {
    const double lo = o[a] + (double)c[a] * e - s, hi = o[a] + (double)(c[a] + span) * e + s;
    acc[a] = fmax(fmax(lo - q[a], q[a] - hi), 0.0);
  }
  return (acc[0] * acc[0] + acc[1] * acc[1]) + acc[2] * acc[2];
}

// icp_ring_lb in double: the distance from q to every cell of Chebyshev ring r >= 1 around c, INFINITY when the ring has
// no cell inside the grid.
__device__ __forceinline__ double fr_ring_lb(const IcpGrid& g, const double* q, const int* c, const int* dims, int span, int r) {
  const double o[3] = {g.ox, g.oy, g.oz}, se = (double)g.e * span, s = g.slack;
  double lb = INFINITY;
  for (int a = 0; a < 3; ++a) {
    if (c[a] - r >= 0) lb = fmin(lb, fmax(q[a] - (o[a] + (double)(c[a] - r + 1) * se + s), 0.0));
    if (c[a] + r < dims[a]) lb = fmin(lb, fmax((o[a] + (double)(c[a] + r) * se - s) - q[a], 0.0));
  }
  return lb;
}

__device__ __forceinline__ bool fr_done(double lb, double best) { return lb == INFINITY || lb * lb * (1.0 - 1e-12) > best; }

__device__ __forceinline__ void fr_take(double d2, int idx, int pos, double& best, int& bi, int& bp) {
  if (d2 < best || (d2 == best && idx < bi)) { best = d2; bi = idx; bp = pos; }
}

__device__ __forceinline__ void fr_cell(const IcpGrid& g, const double* q, int* c) {
  c[0] = icp_cell1((float)q[0], g.ox, g.inv_e, g.gx);
  c[1] = icp_cell1((float)q[1], g.oy, g.inv_e, g.gy);
  c[2] = icp_cell1((float)q[2], g.oz, g.inv_e, g.gz);
}

// ------------------------------------------------------------------------------------------------ normalisation
// The finite points' Σ p / scale, fixed order (k_fr_reduce's record of 3).
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
      const double q[3] = {v.x, v.y, v.z};
      int c[3];
      fr_cell(g, q, c);
      keys[i] = icp_key(g, c[0], c[1], c[2]);
    } else {
      keys[i] = ~0u;
    }
    vals[i] = i;
  }
}

// ------------------------------------------------------------------------------------------------ exact 1-NN
// Thread per query in visiting order: q = T x, fine rings 0..ICP_RINGS, each cell pruned by its widened bounds.  Results
// by source index: pos[i] = the nearest target's sorted position (-1 for a non-finite source point), d2[i] its double d²;
// a query the rings cannot close is appended to the open list for k_fr_nn_far.
__global__ void __launch_bounds__(256, 1) k_fr_nn(IcpGrid g, FrXf xf, const int* __restrict__ order, int n, const double4* __restrict__ x,
                                              const double4* __restrict__ pts, const int* __restrict__ cs, int* __restrict__ pos,
                                              double* __restrict__ d2, int* __restrict__ open_list, int* __restrict__ open_n) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    const int i = order[t];
    const double4 v = x[i];
    if (v.w == 0.0) { pos[i] = -1; d2[i] = INFINITY; continue; }
    const double* m = xf.m;
    const double q[3] = {((m[0] * v.x + m[1] * v.y) + m[2] * v.z) + m[3], ((m[4] * v.x + m[5] * v.y) + m[6] * v.z) + m[7],
                         ((m[8] * v.x + m[9] * v.y) + m[10] * v.z) + m[11]};
    int c[3];
    fr_cell(g, q, c);
    const int dims[3] = {g.gx, g.gy, g.gz};
    double best = INFINITY;
    int bi = INT_MAX, bp = -1;
    bool open = true;
    for (int r = 0; r <= ICP_RINGS + 1; ++r) {
      if (r > 0 && fr_done(fr_ring_lb(g, q, c, dims, 1, r), best)) { open = false; break; }
      if (r == ICP_RINGS + 1) break;
      for (int dz = -r; dz <= r; ++dz) {
        const int iz = c[2] + dz;
        if (iz < 0 || iz >= g.gz) continue;
        for (int dy = -r; dy <= r; ++dy) {
          const int iy = c[1] + dy;
          if (iy < 0 || iy >= g.gy) continue;
          const bool face = dz == -r || dz == r || dy == -r || dy == r;
          for (int dx = -r; dx <= r; dx += (face ? 1 : 2 * r)) {
            const int ix = c[0] + dx;
            if (ix >= 0 && ix < g.gx && fr_box_lb2(g, q, ix, iy, iz, 1) * (1.0 - 1e-12) <= best) {
              const unsigned k = icp_key(g, ix, iy, iz);
              const int e = __ldg(&cs[k + 1]);
              for (int j = __ldg(&cs[k]); j < e; ++j) {
                const double4 p = pts[j];
                fr_take(fr_d2(p, q[0], q[1], q[2]), (int)p.w, j, best, bi, bp);
              }
            }
            if (r == 0) break;
          }
        }
      }
    }
    pos[i] = bp;
    d2[i] = best;
    if (open) open_list[atomicAdd(open_n, 1)] = i;
  }
}

// Warp per open query: coarse rings from the query's coarse cell, nearest ring first, until a ring cannot hold anything
// closer.  A coarse cell whose widened point box can beat the warp's best has its points (one contiguous range of the
// sorted target) scanned by the lanes.  Starts from the thread path's partial result.
__global__ void __launch_bounds__(256) k_fr_nn_far(IcpGrid g, FrXf xf, const int* __restrict__ open_list, const int* __restrict__ open_n,
                                                  const double4* __restrict__ x, const double4* __restrict__ pts, const int* __restrict__ cs,
                                                  const IcpBox* __restrict__ box, int* __restrict__ pos, double* __restrict__ d2) {
  const int lane = threadIdx.x & 31;
  const int n_open = *open_n;
  const int dims[3] = {g.cx, g.cy, g.cz};
  for (int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_open; w += (gridDim.x * blockDim.x) >> 5) {
    const int i = open_list[w];
    const double4 v = x[i];
    const double* m = xf.m;
    const double q[3] = {((m[0] * v.x + m[1] * v.y) + m[2] * v.z) + m[3], ((m[4] * v.x + m[5] * v.y) + m[6] * v.z) + m[7],
                         ((m[8] * v.x + m[9] * v.y) + m[10] * v.z) + m[11]};
    double best = d2[i];
    int bp = pos[i], bi = bp >= 0 ? (int)pts[bp].w : INT_MAX;
    int c[3];
    fr_cell(g, q, c);
    for (int a = 0; a < 3; ++a) c[a] /= ICP_C;
    for (int R = 0;; ++R) {
      if (R > 0 && fr_done(fr_ring_lb(g, q, c, dims, ICP_C, R), best)) break;
      IcpShell sh;
      sh.init(c, dims, R);
      const int tot = sh.total();
      for (int base = 0; base < tot; base += 32) {
        int cc = -1;
        double lb2 = INFINITY;
        if (base + lane < tot) {
          int o[3];
          sh.cell(base + lane, o);
          const int id = (o[2] * g.cy + o[1]) * g.cx + o[0];
          const IcpBox b = box[id];
          if (b.n > 0) {
            double acc[3];
            for (int a = 0; a < 3; ++a)
              acc[a] = fmax(fmax(((double)b.lo[a] - g.slack) - q[a], q[a] - ((double)b.hi[a] + g.slack)), 0.0);
            lb2 = (acc[0] * acc[0] + acc[1] * acc[1]) + acc[2] * acc[2];
            if (lb2 * (1.0 - 1e-12) <= best) cc = id;
          }
        }
        unsigned mask = __ballot_sync(0xffffffffu, cc >= 0);
        while (mask) {
          const int src = __ffs(mask) - 1;
          mask &= mask - 1;
          const int id = __shfl_sync(0xffffffffu, cc, src);
          if (__shfl_sync(0xffffffffu, lb2, src) * (1.0 - 1e-12) > best) continue;   // best improved since the ballot
          const int s = __ldg(&cs[(size_t)id * ICP_C3]), e = __ldg(&cs[(size_t)(id + 1) * ICP_C3]);
          for (int j = s + lane; j < e; j += 32) {
            const double4 p = pts[j];
            fr_take(fr_d2(p, q[0], q[1], q[2]), (int)p.w, j, best, bi, bp);
          }
          for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o), op = __shfl_xor_sync(0xffffffffu, bp, o);
            fr_take(ob, oi, op, best, bi, bp);
          }
        }
      }
    }
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
// included, at 0) over fine rings 0..ICP_RINGS; med[j] = the median of the k - 1 after the first.  A point the rings
// cannot close goes to the open list for k_fr_knn7_far.
__global__ void __launch_bounds__(256) k_fr_knn7(IcpGrid g, int n_fin, int k, const double4* __restrict__ pts, const int* __restrict__ cs,
                                                double* __restrict__ med, int* __restrict__ open_list,
                                                int* __restrict__ open_n) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n_fin; j += gridDim.x * blockDim.x) {
    const double4 v = pts[j];
    const double q[3] = {v.x, v.y, v.z};
    int c[3];
    fr_cell(g, q, c);
    const int dims[3] = {g.gx, g.gy, g.gz};
    double top[7];
    for (int s = 0; s < 7; ++s) top[s] = INFINITY;
    bool open = true;
    for (int r = 0; r <= ICP_RINGS + 1; ++r) {
      if (r > 0 && fr_done(fr_ring_lb(g, q, c, dims, 1, r), top[k - 1])) { open = false; break; }
      if (r == ICP_RINGS + 1) break;
      for (int dz = -r; dz <= r; ++dz) {
        const int iz = c[2] + dz;
        if (iz < 0 || iz >= g.gz) continue;
        for (int dy = -r; dy <= r; ++dy) {
          const int iy = c[1] + dy;
          if (iy < 0 || iy >= g.gy) continue;
          const bool face = dz == -r || dz == r || dy == -r || dy == r;
          for (int dx = -r; dx <= r; dx += (face ? 1 : 2 * r)) {
            const int ix = c[0] + dx;
            if (ix >= 0 && ix < g.gx && fr_box_lb2(g, q, ix, iy, iz, 1) * (1.0 - 1e-12) <= top[k - 1]) {
              const unsigned key = icp_key(g, ix, iy, iz);
              const int e = __ldg(&cs[key + 1]);
              for (int t = __ldg(&cs[key]); t < e; ++t) fr_insert(fr_d2(pts[t], q[0], q[1], q[2]), top, k);
            }
            if (r == 0) break;
          }
        }
      }
    }
    if (open) open_list[atomicAdd(open_n, 1)] = j;
    else med[j] = fr_median_tail(top, k);
  }
}

// Thread per open point: coarse rings, nearest first, whole coarse cells scanned when their widened box can beat the
// k-th best.  Open points are the isolated ones, whose coarse cells hold few points.
__global__ void __launch_bounds__(256) k_fr_knn7_far(IcpGrid g, int k, const int* __restrict__ open_list, const int* __restrict__ open_n,
                                                    const double4* __restrict__ pts, const int* __restrict__ cs, const IcpBox* __restrict__ box,
                                                    double* __restrict__ med) {
  const int n_open = *open_n;
  const int dims[3] = {g.cx, g.cy, g.cz};
  for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < n_open; w += gridDim.x * blockDim.x) {
    const int j = open_list[w];
    const double4 v = pts[j];
    const double q[3] = {v.x, v.y, v.z};
    double top[7];   // from an empty list: the coarse cells hold the fine rings' points again
    for (int s = 0; s < 7; ++s) top[s] = INFINITY;
    int c[3];
    fr_cell(g, q, c);
    for (int a = 0; a < 3; ++a) c[a] /= ICP_C;
    for (int R = 0;; ++R) {
      if (R > 0 && fr_done(fr_ring_lb(g, q, c, dims, ICP_C, R), top[k - 1])) break;
      IcpShell sh;
      sh.init(c, dims, R);
      const int tot = sh.total();
      for (int t = 0; t < tot; ++t) {
        int o[3];
        sh.cell(t, o);
        const int id = (o[2] * g.cy + o[1]) * g.cx + o[0];
        const IcpBox b = box[id];
        if (b.n == 0) continue;
        double acc[3];
        for (int a = 0; a < 3; ++a) acc[a] = fmax(fmax(((double)b.lo[a] - g.slack) - q[a], q[a] - ((double)b.hi[a] + g.slack)), 0.0);
        if (((acc[0] * acc[0] + acc[1] * acc[1]) + acc[2] * acc[2]) * (1.0 - 1e-12) > top[k - 1]) continue;
        const int s = __ldg(&cs[(size_t)id * ICP_C3]), e = __ldg(&cs[(size_t)(id + 1) * ICP_C3]);
        for (int p = s; p < e; ++p) fr_insert(fr_d2(pts[p], q[0], q[1], q[2]), top, k);
      }
    }
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

// Fixed-order double sums of K values per element: block b takes a fixed contiguous range, each thread sums its strided
// share in index order, the block reduces in a fixed tree, and the last block to finish sums the block partials in block
// order into out[0..K).  Run-to-run bit-identical for a given grid.
template <int K, class Op>
__global__ void __launch_bounds__(256) k_fr_reduce(int n, Op op, double* __restrict__ partials, unsigned* __restrict__ counter,
                                                  double* __restrict__ out) {
  __shared__ double sh[K][256];
  __shared__ bool last;
  double acc[K], a[K];
  for (int k = 0; k < K; ++k) acc[k] = 0.0;
  const int chunk = (n + gridDim.x - 1) / gridDim.x;
  const int b0 = blockIdx.x * chunk, b1 = min(n, b0 + chunk);
  for (int i = b0 + threadIdx.x; i < b1; i += blockDim.x)
    if (op(i, a))
      for (int k = 0; k < K; ++k) acc[k] += a[k];
  for (int k = 0; k < K; ++k) sh[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int k = 0; k < K; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int k = 0; k < K; ++k) partials[(size_t)blockIdx.x * K + k] = sh[k][0];
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int k = 0; k < K; ++k) {
    double v = 0.0;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += blockDim.x) v += ((volatile double*)partials)[(size_t)b * K + k];
    sh[k][threadIdx.x] = v;
  }
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int k = 0; k < K; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int k = 0; k < K; ++k) out[k] = sh[k][0];
    *counter = 0u;
  }
}

}  // namespace flb

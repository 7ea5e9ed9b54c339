// icp_kernels.cuh — the loop-closure registration of performLoopClosure (laserMapping.cpp:946-974,
// pcl::IterativeClosestPoint<PointType, PointType>) between two sub-maps assembled from the key-frame store:
//   an index over the target built once per call (finite points sorted by the cell of a uniform grid, CSR cell offsets,
//   per-coarse-cell point boxes), an exact 1-NN pass per iteration (thread-per-query rings over the fine cells, the few
//   open queries finished warp-per-query over the coarse cells, nearest ring first, pruned by box distance), and two
//   fixed-order double reductions per iteration (count and means, then the demeaned cross products).
// The TU is compiled with -fmad=false: the distance (dx*dx + dy*dy) + dz*dz and the affines round after every operation,
// as the reference's FLANN L2_Simple and transformPointCloud do.  Tie rule of the 1-NN: the smaller float d², then the
// lower target index (the position in the assembled target), so the result does not depend on the visiting order.
#pragma once
#include "keyframe_kernels.cuh"

namespace flb {

constexpr int ICP_C = 8, ICP_C3 = ICP_C * ICP_C * ICP_C;   // fine cells per coarse-cell edge / per coarse cell
constexpr int ICP_RINGS = 2;                                // fine rings a thread searches before the warp path takes over
constexpr int ICP_RED = 9;                                  // doubles per reduction record

// The target's grid: fine cells of edge e from the origin (the finite minimum); gx..gz are multiples of ICP_C.  Fine
// cell (ix, iy, iz) has key coarse * ICP_C3 + local, so every coarse cell's points are one range of the sorted target.
// slack widens every geometric cell bound beyond the rounding of the cell assignment (floor((p - o) * inv_e)).
struct IcpGrid {
  float ox, oy, oz, e, inv_e, slack;
  int gx, gy, gz, cx, cy, cz;
};

// Point box of a coarse cell (n == 0: empty).
struct IcpBox {
  float lo[3], hi[3];
  int n, pad;
};

// count, Σd² and the means of source and target over the pairs (phase 0); Σ (t - μt)(s - μs)ᵀ row-major (phase 1)
struct IcpSums {
  double n, d2, mu_s[3], mu_t[3], h[9];
};

// A float affine (row-major 3x4) applied as transformPointCloud does: ((m0 x + m1 y) + m2 z) + m3.
struct IcpXf {
  float m[12];
  int apply;
};

__device__ __forceinline__ bool icp_finite(float4 p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }

__device__ __forceinline__ int icp_cell1(float p, float o, float inv, int g) {
  const float f = floorf((p - o) * inv);
  return f < 0.f ? 0 : (f >= (float)(g - 1) ? g - 1 : (int)f);   // also maps a far query to the border cell
}

__device__ __forceinline__ unsigned icp_key(const IcpGrid& g, int ix, int iy, int iz) {
  const unsigned coarse = ((unsigned)(iz / ICP_C) * g.cy + (unsigned)(iy / ICP_C)) * g.cx + (unsigned)(ix / ICP_C);
  return coarse * ICP_C3 + (unsigned)(((iz % ICP_C) * ICP_C + iy % ICP_C) * ICP_C + ix % ICP_C);
}

// Lower bound of the float d² from q to any point assigned to the block of span^3 fine cells at (ix, iy, iz).
__device__ __forceinline__ float icp_box_lb2(const IcpGrid& g, float4 q, int ix, int iy, int iz, int span) {
  const float lx = g.ox + (float)ix * g.e - g.slack, hx = g.ox + (float)(ix + span) * g.e + g.slack;
  const float ly = g.oy + (float)iy * g.e - g.slack, hy = g.oy + (float)(iy + span) * g.e + g.slack;
  const float lz = g.oz + (float)iz * g.e - g.slack, hz = g.oz + (float)(iz + span) * g.e + g.slack;
  const float dx = fmaxf(fmaxf(lx - q.x, q.x - hx), 0.f), dy = fmaxf(fmaxf(ly - q.y, q.y - hy), 0.f);
  const float dz = fmaxf(fmaxf(lz - q.z, q.z - hz), 0.f);
  return (dx * dx + dy * dy) + dz * dz;
}

// Lower bound of the distance from q to every cell of Chebyshev ring r >= 1 around cell c (cells of `span` fine cells,
// dims cells per axis), over the directions in which ring r still has cells inside the grid; INFINITY when it has none
// (every cell has been visited).  Monotone in r.
__device__ __forceinline__ float icp_ring_lb(const IcpGrid& g, float4 q, const int* c, const int* dims, int span, int r) {
  const float qa[3] = {q.x, q.y, q.z}, oa[3] = {g.ox, g.oy, g.oz};
  const float se = g.e * (float)span;
  float lb = INFINITY;
  for (int a = 0; a < 3; ++a) {
    if (c[a] - r >= 0) lb = fminf(lb, fmaxf(qa[a] - (oa[a] + (float)(c[a] - r + 1) * se + g.slack), 0.f));
    if (c[a] + r < dims[a]) lb = fminf(lb, fmaxf((oa[a] + (float)(c[a] + r) * se - g.slack) - qa[a], 0.f));
  }
  return lb;
}

// The ring has nothing closer than best: lb² in double with a relative margin over the float rounding of d².
__device__ __forceinline__ bool icp_ring_done(float lb, float best) {
  return lb == INFINITY || (double)lb * (double)lb * (1.0 - 1e-6) > (double)best;
}

__device__ __forceinline__ void icp_take(float d2, int idx, float& best, int& bi) {
  if (d2 < best || (d2 == best && idx < bi)) { best = d2; bi = idx; }
}

// Points [b, e) of the sorted target (w = the original index) against q.
__device__ __forceinline__ void icp_scan(const float4* __restrict__ pts, int b, int e, float4 q, float& best, int& bi) {
  for (int j = b; j < e; ++j) {
    const float4 p = __ldg(&pts[j]);
    const float dx = p.x - q.x, dy = p.y - q.y, dz = p.z - q.z;
    icp_take((dx * dx + dy * dy) + dz * dz, __float_as_int(p.w), best, bi);
  }
}

// ------------------------------------------------------------------------------------------------ index build
// Finite count and the order-preserving keys of the finite bounding box: b[0..2] min (init ~0u), b[3..5] max (init 0),
// b[6] count (init 0).
__device__ __forceinline__ unsigned icp_okey(float v) {
  const unsigned u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(256) k_icp_bounds(const float4* __restrict__ p, int n, unsigned* __restrict__ b) {
  unsigned mn[3] = {~0u, ~0u, ~0u}, mx[3] = {0u, 0u, 0u}, cnt = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 q = p[i];
    if (!icp_finite(q)) continue;
    const unsigned k[3] = {icp_okey(q.x), icp_okey(q.y), icp_okey(q.z)};
    for (int a = 0; a < 3; ++a) { mn[a] = min(mn[a], k[a]); mx[a] = max(mx[a], k[a]); }
    ++cnt;
  }
  for (int o = 16; o > 0; o >>= 1) {
    for (int a = 0; a < 3; ++a) {
      mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
    for (int a = 0; a < 3; ++a) { atomicMin(&b[a], mn[a]); atomicMax(&b[3 + a], mx[a]); }
    atomicAdd(&b[6], cnt);
  }
}

// Sort keys of a cloud on the target grid (a point outside it takes the nearest border cell); non-finite points sort last.
__global__ void k_icp_keys(IcpGrid g, const float4* __restrict__ p, int n, unsigned* __restrict__ keys, int* __restrict__ vals) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 q = p[i];
    keys[i] = icp_finite(q) ? icp_key(g, icp_cell1(q.x, g.ox, g.inv_e, g.gx), icp_cell1(q.y, g.oy, g.inv_e, g.gy),
                                      icp_cell1(q.z, g.oz, g.inv_e, g.gz))
                            : ~0u;
    vals[i] = i;
  }
}

// The first n_fin sorted points with their original index in w.
__global__ void k_icp_gather(const int* __restrict__ vals, const float4* __restrict__ p, int n_fin, float4* __restrict__ out) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n_fin; j += gridDim.x * blockDim.x) {
    const int i = vals[j];
    const float4 q = p[i];
    out[j] = make_float4(q.x, q.y, q.z, __int_as_float(i));
  }
}

// CSR offsets: cs[k] = first sorted position whose key is >= k, for k in [0, n_cells]; every entry written once.
__global__ void k_icp_cell_start(const unsigned* __restrict__ keys, int n_fin, unsigned n_cells, int* __restrict__ cs) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j <= n_fin; j += gridDim.x * blockDim.x) {
    const unsigned from = j == 0 ? 0u : keys[j - 1] + 1u;
    const unsigned to = j == n_fin ? n_cells : keys[j];
    for (unsigned k = from; k <= to; ++k) cs[k] = j;
  }
}

// Warp per coarse cell: the box of its points.
__global__ void __launch_bounds__(256) k_icp_coarse_boxes(const float4* __restrict__ pts, const int* __restrict__ cs, int n_coarse,
                                                         IcpBox* __restrict__ box) {
  const int lane = threadIdx.x & 31;
  for (int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < n_coarse; c += (gridDim.x * blockDim.x) >> 5) {
    const int b = cs[(size_t)c * ICP_C3], e = cs[(size_t)(c + 1) * ICP_C3];
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int j = b + lane; j < e; j += 32) {
      const float4 p = pts[j];
      lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
      hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
    }
    for (int o = 16; o > 0; o >>= 1)
      for (int a = 0; a < 3; ++a) {
        lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
        hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
      }
    if (lane == 0) {
      IcpBox x;
      for (int a = 0; a < 3; ++a) { x.lo[a] = lo[a]; x.hi[a] = hi[a]; }
      x.n = e - b;
      x.pad = 0;
      box[c] = x;
    }
  }
}

// ------------------------------------------------------------------------------------------------ exact 1-NN
// Thread per query, queries in source-cell order (order[t]): q = xf(in[i]) is written to out[i] (in == out allowed), then
// fine rings 0..ICP_RINGS, each cell pruned by its box.  A query is done when the next ring cannot hold anything closer;
// otherwise its partial result is kept and its index appended to the open list for k_icp_nn_far.  Results by source
// index: idx[i] = the nearest target's original index (-1 for a non-finite query), d2[i] its float d².
__global__ void __launch_bounds__(256) k_icp_nn(IcpGrid g, IcpXf xf, const int* __restrict__ order, int n, const float4* in, float4* out,
                                               const float4* __restrict__ pts, const int* __restrict__ cs, int* __restrict__ idx,
                                               float* __restrict__ d2, int* __restrict__ open_list, int* __restrict__ open_n) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    const int i = order[t];
    float4 q = in[i];
    if (xf.apply) {
      const float* m = xf.m;
      q = make_float4(m[0] * q.x + m[1] * q.y + m[2] * q.z + m[3], m[4] * q.x + m[5] * q.y + m[6] * q.z + m[7],
                      m[8] * q.x + m[9] * q.y + m[10] * q.z + m[11], q.w);
    }
    out[i] = q;
    if (!icp_finite(q)) { idx[i] = -1; d2[i] = INFINITY; continue; }
    const int c[3] = {icp_cell1(q.x, g.ox, g.inv_e, g.gx), icp_cell1(q.y, g.oy, g.inv_e, g.gy), icp_cell1(q.z, g.oz, g.inv_e, g.gz)};
    const int dims[3] = {g.gx, g.gy, g.gz};
    float best = INFINITY;
    int bi = INT_MAX;
    bool open = true;
    for (int r = 0; r <= ICP_RINGS + 1; ++r) {
      if (r > 0 && icp_ring_done(icp_ring_lb(g, q, c, dims, 1, r), best)) { open = false; break; }
      if (r == ICP_RINGS + 1) break;
      for (int dz = -r; dz <= r; ++dz) {
        const int iz = c[2] + dz;
        if (iz < 0 || iz >= g.gz) continue;
        for (int dy = -r; dy <= r; ++dy) {
          const int iy = c[1] + dy;
          if (iy < 0 || iy >= g.gy) continue;
          const bool face = dz == -r || dz == r || dy == -r || dy == r;
          for (int dx = -r; dx <= r; dx += (face ? 1 : 2 * r)) {   // interior rows: only the two x faces
            const int ix = c[0] + dx;
            if (ix >= 0 && ix < g.gx && icp_box_lb2(g, q, ix, iy, iz, 1) <= best) {
              const unsigned k = icp_key(g, ix, iy, iz);
              icp_scan(pts, __ldg(&cs[k]), __ldg(&cs[k + 1]), q, best, bi);
            }
            if (r == 0) break;
          }
        }
      }
    }
    idx[i] = bi;
    d2[i] = best;
    if (open) open_list[atomicAdd(open_n, 1)] = i;
  }
}

// The cells of Chebyshev ring R around c clipped to the grid [0, dims): t-th of *count.  Faces: z = c-R, z = c+R (full
// x, y), then y = c∓R (z strictly inside), then x = c∓R (y and z strictly inside).
struct IcpShell {
  int lo[3], hi[3];   // the clipped cube
  int c[3], R;
  int cnt[6];         // cells per face (0 for a face outside the grid or a repeated one)
  __device__ void init(const int* cc, const int* dims, int r) {
    R = r;
    for (int a = 0; a < 3; ++a) { c[a] = cc[a]; lo[a] = max(cc[a] - r, 0); hi[a] = min(cc[a] + r, dims[a] - 1); }
    const int nx = hi[0] - lo[0] + 1, ny = hi[1] - lo[1] + 1;
    const int zi = max(0, min(hi[2], c[2] + R - 1) - max(lo[2], c[2] - R + 1) + 1);
    const int yi = max(0, min(hi[1], c[1] + R - 1) - max(lo[1], c[1] - R + 1) + 1);
    const bool z0 = c[2] - R >= 0, z1 = c[2] + R < dims[2] && R > 0;
    const bool y0 = c[1] - R >= 0, y1 = c[1] + R < dims[1] && R > 0;
    const bool x0 = c[0] - R >= 0, x1 = c[0] + R < dims[0] && R > 0;
    cnt[0] = z0 ? nx * ny : 0;
    cnt[1] = z1 ? nx * ny : 0;
    cnt[2] = (y0 && R > 0) ? nx * zi : 0;
    cnt[3] = y1 ? nx * zi : 0;
    cnt[4] = (x0 && R > 0) ? yi * zi : 0;
    cnt[5] = x1 ? yi * zi : 0;
  }
  __device__ int total() const { return cnt[0] + cnt[1] + cnt[2] + cnt[3] + cnt[4] + cnt[5]; }
  __device__ void cell(int t, int* o) const {
    int f = 0;
    while (t >= cnt[f]) t -= cnt[f++];
    const int nx = hi[0] - lo[0] + 1;
    const int zl = max(lo[2], c[2] - R + 1), yl = max(lo[1], c[1] - R + 1);
    const int yn = max(0, min(hi[1], c[1] + R - 1) - yl + 1);
    if (f < 2) { o[0] = lo[0] + t % nx; o[1] = lo[1] + t / nx; o[2] = f == 0 ? c[2] - R : c[2] + R; }
    else if (f < 4) { o[0] = lo[0] + t % nx; o[1] = f == 2 ? c[1] - R : c[1] + R; o[2] = zl + t / nx; }
    else { o[0] = f == 4 ? c[0] - R : c[0] + R; o[1] = yl + t % yn; o[2] = zl + t / yn; }
  }
};

// Warp per open query: coarse rings from the query's coarse cell, nearest ring first, until a ring cannot hold anything
// closer.  A coarse cell is visited when its point box can beat the warp's best; its non-empty fine cells are then
// pruned by their own boxes and scanned by the lanes.  Starts from the thread path's partial result.
__global__ void __launch_bounds__(256) k_icp_nn_far(IcpGrid g, const int* __restrict__ open_list, const int* __restrict__ open_n,
                                                   const float4* __restrict__ xq, const float4* __restrict__ pts,
                                                   const int* __restrict__ cs, const IcpBox* __restrict__ box, int* __restrict__ idx,
                                                   float* __restrict__ d2) {
  const int lane = threadIdx.x & 31;
  const int n_open = *open_n;
  const int dims[3] = {g.cx, g.cy, g.cz};
  for (int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_open; w += (gridDim.x * blockDim.x) >> 5) {
    const int i = open_list[w];
    const float4 q = xq[i];
    float best = d2[i];
    int bi = idx[i];
    const int c[3] = {icp_cell1(q.x, g.ox, g.inv_e, g.gx) / ICP_C, icp_cell1(q.y, g.oy, g.inv_e, g.gy) / ICP_C,
                      icp_cell1(q.z, g.oz, g.inv_e, g.gz) / ICP_C};
    for (int R = 0;; ++R) {
      if (R > 0 && icp_ring_done(icp_ring_lb(g, q, c, dims, ICP_C, R), best)) break;
      IcpShell sh;
      sh.init(c, dims, R);
      const int tot = sh.total();
      for (int base = 0; base < tot; base += 32) {
        int cc = -1;
        float lb2 = INFINITY;
        if (base + lane < tot) {
          int o[3];
          sh.cell(base + lane, o);
          const int id = (o[2] * g.cy + o[1]) * g.cx + o[0];
          const IcpBox b = box[id];
          if (b.n > 0) {
            const float dx = fmaxf(fmaxf(b.lo[0] - q.x, q.x - b.hi[0]), 0.f), dy = fmaxf(fmaxf(b.lo[1] - q.y, q.y - b.hi[1]), 0.f);
            const float dz = fmaxf(fmaxf(b.lo[2] - q.z, q.z - b.hi[2]), 0.f);
            lb2 = (dx * dx + dy * dy) + dz * dz;
            if (lb2 <= best) cc = id;
          }
        }
        unsigned mask = __ballot_sync(0xffffffffu, cc >= 0);
        while (mask) {
          const int src = __ffs(mask) - 1;
          mask &= mask - 1;
          const int id = __shfl_sync(0xffffffffu, cc, src);
          if (__shfl_sync(0xffffffffu, lb2, src) > best) continue;   // best improved since the ballot
          const int bx = (id % g.cx) * ICP_C, by = ((id / g.cx) % g.cy) * ICP_C, bz = (id / (g.cx * g.cy)) * ICP_C;
          for (int l = lane; l < ICP_C3; l += 32) {
            const int k = id * ICP_C3 + l;
            const int s = __ldg(&cs[k]), e = __ldg(&cs[k + 1]);
            if (s < e && icp_box_lb2(g, q, bx + l % ICP_C, by + (l / ICP_C) % ICP_C, bz + l / (ICP_C * ICP_C), 1) <= best)
              icp_scan(pts, s, e, q, best, bi);
          }
          for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            icp_take(ob, oi, best, bi);
          }
        }
      }
    }
    if (lane == 0) { idx[i] = bi; d2[i] = best; }
  }
}

// ------------------------------------------------------------------------------------------------ reductions
// Fixed-order double sums over the pairs (idx[i] >= 0 and (double)d2[i] <= max_d2): block b takes a fixed contiguous
// range of sources, each thread sums its strided share in index order, the block reduces in a fixed tree, and the last
// block to finish sums the block partials in block order.  Phase 0: count, Σd², means of source and target (into out);
// phase 1 (after phase 0, reading its means): the 9 cross products.  Run-to-run bit-identical for a given grid.
__global__ void __launch_bounds__(256) k_icp_reduce(int phase, int n, const int* __restrict__ idx, const float* __restrict__ d2,
                                                   const float4* __restrict__ src, const float4* __restrict__ tgt, double max_d2,
                                                   double* __restrict__ partials, unsigned* __restrict__ counter, IcpSums* out) {
  __shared__ double sh[ICP_RED][256];
  __shared__ bool last;
  double acc[ICP_RED];
  for (int k = 0; k < ICP_RED; ++k) acc[k] = 0.0;
  double ms[3] = {0, 0, 0}, mt[3] = {0, 0, 0};
  if (phase == 1)
    for (int a = 0; a < 3; ++a) { ms[a] = out->mu_s[a]; mt[a] = out->mu_t[a]; }
  const int chunk = (n + gridDim.x - 1) / gridDim.x;
  const int b0 = blockIdx.x * chunk, b1 = min(n, b0 + chunk);
  for (int i = b0 + threadIdx.x; i < b1; i += blockDim.x) {
    const int j = idx[i];
    if (j < 0) continue;
    const float dd = d2[i];
    if (!((double)dd <= max_d2)) continue;
    const float4 s = src[i], t = tgt[j];
    if (phase == 0) {
      acc[0] += 1.0;
      acc[1] += (double)dd;
      acc[2] += s.x; acc[3] += s.y; acc[4] += s.z;
      acc[5] += t.x; acc[6] += t.y; acc[7] += t.z;
    } else {
      const double ds[3] = {s.x - ms[0], s.y - ms[1], s.z - ms[2]}, dt[3] = {t.x - mt[0], t.y - mt[1], t.z - mt[2]};
      for (int r = 0; r < 3; ++r)
        for (int cc = 0; cc < 3; ++cc) acc[3 * r + cc] += dt[r] * ds[cc];
    }
  }
  const int K = phase == 0 ? 8 : 9;
  for (int k = 0; k < K; ++k) sh[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int k = 0; k < K; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int k = 0; k < K; ++k) partials[(size_t)blockIdx.x * ICP_RED + k] = sh[k][0];
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int k = 0; k < K; ++k) {
    double v = 0.0;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += blockDim.x) v += ((volatile double*)partials)[(size_t)b * ICP_RED + k];
    sh[k][threadIdx.x] = v;
  }
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int k = 0; k < K; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (phase == 0) {
      const double cnt = sh[0][0];
      out->n = cnt;
      out->d2 = sh[1][0];
      for (int a = 0; a < 3; ++a) {
        out->mu_s[a] = cnt > 0 ? sh[2 + a][0] / cnt : 0.0;
        out->mu_t[a] = cnt > 0 ? sh[5 + a][0] / cnt : 0.0;
      }
    } else {
      for (int k = 0; k < 9; ++k) out->h[k] = sh[k][0];
    }
    *counter = 0u;
  }
}

}  // namespace flb

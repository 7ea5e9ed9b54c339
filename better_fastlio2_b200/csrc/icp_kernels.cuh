// icp_kernels.cuh — the loop-closure registration of performLoopClosure (laserMapping.cpp:946-974,
// pcl::IterativeClosestPoint<PointType, PointType>) between two sub-maps assembled from the key-frame store, and the
// pieces flb_keyframes_fricp (fricp_kernels.cuh) shares with it:
//   the grid index over a float target, built once per call (finite points sorted by the cell of a uniform grid, CSR
//   cell offsets, per-coarse-cell point boxes);
//   the two search walks over it, generic in the query's precision: fine rings 0..ICP_RINGS thread-per-query
//   (icp_fine_rings) and coarse rings nearest first, pruned by box distance, for the queries the fine rings leave open
//   (icp_coarse_rings, warp- or thread-per-query);
//   the fixed-order double reduction k_reduce.
// The loop ICP runs an exact 1-NN pass per iteration (k_icp_nn, k_icp_nn_far) and two reductions (the pairs' count and
// sums, then the demeaned cross products).
// The TU is compiled with -fmad=false: the distance (dx*dx + dy*dy) + dz*dz and the affines round after every operation,
// as the reference's FLANN L2_Simple and transformPointCloud do.  Tie rule of the 1-NN: the smaller float d², then the
// lower target index (the position in the assembled target), so the result does not depend on the visiting order.
#pragma once
#include "keyframe_kernels.cuh"

namespace flb {

constexpr int ICP_C = 8, ICP_C3 = ICP_C * ICP_C * ICP_C;   // fine cells per coarse-cell edge / per coarse cell
constexpr int ICP_RINGS = 2;                                // fine rings a thread searches before the coarse walk takes over

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

// ------------------------------------------------------------------------------------------------ search walks
// The loop ICP's query: float coordinates and d², every bound in float, a ring closed with a 1e-6 relative margin in
// double.  flb_keyframes_fricp's double query (FrQuery, fricp_kernels.cuh) has the same members.
struct IcpQuery {
  using real = float;
  float4 q;
  __device__ void cell(const IcpGrid& g, int* c) const {
    c[0] = icp_cell1(q.x, g.ox, g.inv_e, g.gx);
    c[1] = icp_cell1(q.y, g.oy, g.inv_e, g.gy);
    c[2] = icp_cell1(q.z, g.oz, g.inv_e, g.gz);
  }
  __device__ float cell_lb2(const IcpGrid& g, int ix, int iy, int iz) const { return icp_box_lb2(g, q, ix, iy, iz, 1); }
  __device__ float box_lb2(const IcpGrid&, const IcpBox& b) const {
    const float dx = fmaxf(fmaxf(b.lo[0] - q.x, q.x - b.hi[0]), 0.f), dy = fmaxf(fmaxf(b.lo[1] - q.y, q.y - b.hi[1]), 0.f);
    const float dz = fmaxf(fmaxf(b.lo[2] - q.z, q.z - b.hi[2]), 0.f);
    return (dx * dx + dy * dy) + dz * dz;
  }
  __device__ bool ring_done(const IcpGrid& g, const int* c, const int* dims, int span, int r, float best) const {
    return icp_ring_done(icp_ring_lb(g, q, c, dims, span, r), best);
  }
  __device__ static bool beats(float lb2, float best) { return lb2 <= best; }
};

// Fine rings 0..ICP_RINGS around the query's cell (interior rows only at their two x faces); every cell whose bound can
// beat best goes to visit(key), which may lower best.  Returns whether the query closed: the next ring cannot hold
// anything closer than best.
template <class Q, class Visit>
__device__ __forceinline__ bool icp_fine_rings(const IcpGrid& g, const Q& q, const typename Q::real& best, Visit visit) {
  int c[3];
  q.cell(g, c);
  const int dims[3] = {g.gx, g.gy, g.gz};
  for (int r = 0; r <= ICP_RINGS + 1; ++r) {
    if (r > 0 && q.ring_done(g, c, dims, 1, r, best)) return true;
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
          if (ix >= 0 && ix < g.gx && Q::beats(q.cell_lb2(g, ix, iy, iz), best)) visit(icp_key(g, ix, iy, iz));
          if (r == 0) break;
        }
      }
    }
  }
  return false;
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

// Coarse rings from the query's coarse cell, nearest ring first, until a ring cannot hold anything closer than best
// (every query closes).  A coarse cell whose point box can beat best goes to visit(id), which may lower best.  W = 32:
// warp per query, each lane tests one cell of the ring, and the warp visits the ballot's cells in lane order, each
// tested again against the best the earlier visits left (the visit merges the lanes' bests); W = 1: thread per query.
template <int W, class Q, class Visit>
__device__ __forceinline__ void icp_coarse_rings(const IcpGrid& g, const IcpBox* __restrict__ box, const Q& q,
                                                 const typename Q::real& best, Visit visit) {
  int c[3];
  q.cell(g, c);
  for (int a = 0; a < 3; ++a) c[a] /= ICP_C;
  const int dims[3] = {g.cx, g.cy, g.cz};
  const int lane = W == 1 ? 0 : (int)(threadIdx.x & 31);
  for (int R = 0;; ++R) {
    if (R > 0 && q.ring_done(g, c, dims, ICP_C, R, best)) return;
    IcpShell sh;
    sh.init(c, dims, R);
    const int tot = sh.total();
    for (int base = 0; base < tot; base += W) {
      int cc = -1;
      typename Q::real lb2 = INFINITY;
      if (base + lane < tot) {
        int o[3];
        sh.cell(base + lane, o);
        const int id = (o[2] * g.cy + o[1]) * g.cx + o[0];
        const IcpBox b = box[id];
        if (b.n > 0) {
          lb2 = q.box_lb2(g, b);
          if (Q::beats(lb2, best)) cc = id;
        }
      }
      if constexpr (W == 1) {
        if (cc >= 0) visit(cc);
      } else {
        unsigned mask = __ballot_sync(0xffffffffu, cc >= 0);
        while (mask) {
          const int src = __ffs(mask) - 1;
          mask &= mask - 1;
          const int id = __shfl_sync(0xffffffffu, cc, src);
          if (!Q::beats(__shfl_sync(0xffffffffu, lb2, src), best)) continue;   // best improved since the ballot
          visit(id);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ exact 1-NN
// Thread per query, queries in source-cell order (order[t]): q = xf(in[i]) is written to out[i] (in == out allowed), then
// the fine rings, each cell pruned by its box.  A query the rings do not close keeps its partial result and its index
// goes to the open list for k_icp_nn_far.  Results by source index: idx[i] = the nearest target's original index (-1 for
// a non-finite query), d2[i] its float d².
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
    float best = INFINITY;
    int bi = INT_MAX;
    const bool closed = icp_fine_rings(g, IcpQuery{q}, best, [&](unsigned k) {
      icp_scan(pts, __ldg(&cs[k]), __ldg(&cs[k + 1]), q, best, bi);
    });
    idx[i] = bi;
    d2[i] = best;
    if (!closed) open_list[atomicAdd(open_n, 1)] = i;
  }
}

// Warp per open query over the coarse rings, starting from the thread path's partial result.  A visited coarse cell's
// non-empty fine cells are pruned by their own boxes and scanned by the lanes.
__global__ void __launch_bounds__(256) k_icp_nn_far(IcpGrid g, const int* __restrict__ open_list, const int* __restrict__ open_n,
                                                   const float4* __restrict__ xq, const float4* __restrict__ pts,
                                                   const int* __restrict__ cs, const IcpBox* __restrict__ box, int* __restrict__ idx,
                                                   float* __restrict__ d2) {
  const int lane = threadIdx.x & 31;
  const int n_open = *open_n;
  for (int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_open; w += (gridDim.x * blockDim.x) >> 5) {
    const int i = open_list[w];
    const float4 q = xq[i];
    float best = d2[i];
    int bi = idx[i];
    icp_coarse_rings<32>(g, box, IcpQuery{q}, best, [&](int id) {
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
    });
    if (lane == 0) { idx[i] = bi; d2[i] = best; }
  }
}

// ------------------------------------------------------------------------------------------------ reductions
constexpr int ICP_RED_MAX = 17;   // doubles of the widest record (flb_keyframes_fricp's step record)

// Fixed-order double sums of K values per element (op(i, a) fills a[0..K) and returns whether element i counts): block b
// takes a fixed contiguous range, each thread sums its strided share in index order, the block reduces in a fixed tree,
// and the last block to finish sums the block partials in block order into out[0..K).  Run-to-run bit-identical for a
// given grid.
template <int K, class Op>
__global__ void __launch_bounds__(256) k_reduce(int n, Op op, double* __restrict__ partials, unsigned* __restrict__ counter,
                                               double* __restrict__ out) {
  static_assert(K <= ICP_RED_MAX, "the partials hold ICP_RED_MAX doubles per block");
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

// The pairs of a 1-NN pass (idx[i] >= 0 and (double)d2[i] <= max_d2): count, Σd², Σ source, Σ target (k_reduce<8>).
struct IcpPairsOp {
  const int* idx;
  const float* d2;
  const float4* src;
  const float4* tgt;
  double max_d2;
  __device__ bool operator()(int i, double* a) const {
    const int j = idx[i];
    if (j < 0) return false;
    const float dd = d2[i];
    if (!((double)dd <= max_d2)) return false;
    const float4 s = src[i], t = tgt[j];
    a[0] = 1.0;
    a[1] = (double)dd;
    a[2] = s.x; a[3] = s.y; a[4] = s.z;
    a[5] = t.x; a[6] = t.y; a[7] = t.z;
    return true;
  }
};

// Σ (t - μt)(s - μs)ᵀ row-major over the same pairs (k_reduce<9>), each mean formed as sum / count from the pairs record.
struct IcpCrossOp {
  IcpPairsOp pairs;
  const double* rec;
  __device__ bool operator()(int i, double* a) const {
    const double n = rec[0];
    const double ms[3] = {rec[2] / n, rec[3] / n, rec[4] / n}, mt[3] = {rec[5] / n, rec[6] / n, rec[7] / n};
    double p[8];
    if (!pairs(i, p)) return false;
    const double ds[3] = {p[2] - ms[0], p[3] - ms[1], p[4] - ms[2]}, dt[3] = {p[5] - mt[0], p[6] - mt[1], p[7] - mt[2]};
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) a[3 * r + c] = dt[r] * ds[c];
    return true;
  }
};

}  // namespace flb

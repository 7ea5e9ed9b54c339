// knn_kernels.cuh — K1: exact k-nearest-neighbour search on the hashed voxel map, one warp per query.
// Replaces KD_TREE::Nearest_Search / Search (include/ikd-Tree/ikd_Tree.cpp:366-397, :868-1013) as called from
// h_share_model (src/laserMapping.cpp:1909).  Semantics kept: exact over all valid points, unbounded range
// (max_dist = INFINITY by default, ikd_Tree.h:236), float squared distances ((dx*dx+dy*dy)+dz*dz, no FMA —
// calc_dist ikd_Tree.cpp:1373-1378), ascending output, fewer than k results when the map is small.
// Equal-distance ties are broken by (x,y,z) in the exact kernel and kept in arrival order by the stencil pass (TopKId) —
// the reference's order depends on tree traversal (ikd_Tree.h:102-105).
//
// Search plan per query (all exact, each phase only runs if the previous one could not prove completeness):
//   A  5x5x5 voxel stencil around the query voxel (always inside 2x2x2 blocks; 8 hash probes by lanes 0-7)
//   B  the 3x3x3 coarse cells (8x8x8 blocks each) around the query, block bitmaps prune by box distance
//   C  every other coarse cell in the coarse hash (far queries at the map frontier; rare)
// Completeness test: have k candidates and d_k < (distance from the query to the boundary of the searched region)^2.
// Roofline: HBM/L2-latency bound gather; algorithmic bytes 16 (query) + 80 (5 neighbours) + 80 (cache write).
#pragma once
#include "mask_bits.h"
#include "voxel_map.cuh"
#include <math_constants.h>

namespace flb {

constexpr unsigned FULL = 0xffffffffu;
constexpr int BLOCK_RINGS = 8;  // block shells searched by the exact kernel (= EXACT_RINGS) before it falls back to the coarse levels
// exact-kernel launch shape (threads per CTA, minimum CTAs per SM -> register cap)
#ifndef FLB_KNN_THREADS
#define FLB_KNN_THREADS 128
#endif
#ifndef FLB_KNN_MINB
#define FLB_KNN_MINB 4
#endif
constexpr int KNN_THREADS = FLB_KNN_THREADS;
constexpr int KNN_MIN_CTAS = FLB_KNN_MINB;

// Large K (generic Nearest_Search with k up to 20, off the hot path) keeps its list loops ROLLED: the lists then live
// in local memory, but the fully unrolled lexicographic insert at every inlined call site made that instantiation
// 90 % of the translation unit (minutes of ptxas time) for a path that is never timed.
__host__ __device__ constexpr int topk_unroll(int k) { return k <= 8 ? k : 1; }

template <int K>
struct TopK {
  float d[K], x[K], y[K], z[K];
  __device__ __forceinline__ void clear() {
#pragma unroll (topk_unroll(K))
    for (int j = 0; j < K; ++j) { d[j] = CUDART_INF_F; x[j] = 0.f; y[j] = 0.f; z[j] = 0.f; }
  }
  static __device__ __forceinline__ bool less(float da, float xa, float ya, float za, float db, float xb, float yb, float zb) {
    if (da != db) return da < db;
    if (xa != xb) return xa < xb;
    if (ya != yb) return ya < yb;
    return za < zb;
  }
  __device__ __forceinline__ void insert(float dd, float px, float py, float pz) {
    if (!less(dd, px, py, pz, d[K - 1], x[K - 1], y[K - 1], z[K - 1])) return;
    d[K - 1] = dd; x[K - 1] = px; y[K - 1] = py; z[K - 1] = pz;
#pragma unroll (topk_unroll(K))
    for (int j = K - 1; j > 0; --j) {
      if (less(d[j], x[j], y[j], z[j], d[j - 1], x[j - 1], y[j - 1], z[j - 1])) {
        float t;
        t = d[j]; d[j] = d[j - 1]; d[j - 1] = t;
        t = x[j]; x[j] = x[j - 1]; x[j - 1] = t;
        t = y[j]; y[j] = y[j - 1]; y[j - 1] = t;
        t = z[j]; z[j] = z[j - 1]; z[j - 1] = t;
      }
    }
  }
  __device__ __forceinline__ void pop_front() {
#pragma unroll (topk_unroll(K))
    for (int j = 0; j < K - 1; ++j) { d[j] = d[j + 1]; x[j] = x[j + 1]; y[j] = y[j + 1]; z[j] = z[j + 1]; }
    d[K - 1] = CUDART_INF_F;
  }
};

__device__ __forceinline__ float sqdist(float qx, float qy, float qz, float px, float py, float pz) {
  const float dx = __fsub_rn(qx, px), dy = __fsub_rn(qy, py), dz = __fsub_rn(qz, pz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// Merge the lane-local sorted lists of the lanes in `gmask` (a whole warp, or an aligned group of G lanes working on
// one query) into that query's top-K.  gl = lane index inside the group.  On return: group lane r (< gcount) holds
// result r in (rd,rx,ry,rz); every lane's list is cleared except lane r which re-inserts result r; returns gcount and
// the current k-th distance (INF if fewer than K found) in thr.  All lanes of gmask must call it together.
template <int K>
__device__ __forceinline__ int warp_merge(TopK<K>& t, unsigned gmask, int gl, int lane, float& rd, float& rx, float& ry, float& rz,
                                          float& thr) {
  int gcount = 0;
  float last = CUDART_INF_F;
  rd = CUDART_INF_F; rx = ry = rz = CUDART_NAN_F;
#pragma unroll 1
  for (int r = 0; r < K; ++r) {   // always K rounds (no early exit), so that lane groups sharing a warp stay converged
    const unsigned v = __float_as_uint(t.d[0]);
    const unsigned mn = __reduce_min_sync(gmask, v);
    const bool ok = mn != 0x7f800000u;   // group-uniform: a candidate is left
    unsigned who = __ballot_sync(gmask, v == mn);
    int src = __ffs(who) - 1;
    if (ok && (who & (who - 1))) {  // several lanes tie on distance: lexicographic (x,y,z)
      float bx = __shfl_sync(gmask, t.x[0], src), by = __shfl_sync(gmask, t.y[0], src), bz = __shfl_sync(gmask, t.z[0], src);
      unsigned rest = who & ~(1u << src);
      while (rest) {
        const int c = __ffs(rest) - 1;
        rest &= rest - 1;
        const float cx = __shfl_sync(gmask, t.x[0], c), cy = __shfl_sync(gmask, t.y[0], c), cz = __shfl_sync(gmask, t.z[0], c);
        if (cx < bx || (cx == bx && (cy < by || (cy == by && cz < bz)))) { bx = cx; by = cy; bz = cz; src = c; }
      }
    }
    const float gd = __shfl_sync(gmask, t.d[0], src), gx = __shfl_sync(gmask, t.x[0], src);
    const float gy = __shfl_sync(gmask, t.y[0], src), gz = __shfl_sync(gmask, t.z[0], src);
    if (ok) {
      if (gl == r) { rd = gd; rx = gx; ry = gy; rz = gz; }
      if (lane == src) t.pop_front();
      last = gd;
      ++gcount;
    }
  }
  thr = (gcount == K) ? last : CUDART_INF_F;
  t.clear();
  if (gl < gcount) { t.d[0] = rd; t.x[0] = rx; t.y[0] = ry; t.z[0] = rz; }
  return gcount;
}

// voxels of block (bx,by,bz) that lie inside the 5x5x5 stencil around voxel (cvx,cvy,cvz)
__device__ __forceinline__ unsigned long long block_stencil_mask(int bx, int by, int bz, int cvx, int cvy, int cvz) {
  // most callers' blocks lie outside the stencil: one unsigned compare per axis (stencil_axis_bits) settles them
  const unsigned xm = stencil_axis_bits(bx, cvx);
  if (!xm) return 0ull;
  const unsigned ym = stencil_axis_bits(by, cvy), zm = stencil_axis_bits(bz, cvz);
  if (!(ym && zm)) return 0ull;
  return mask_from_axes(xm, ym, zm);
}

// K0: body -> world transform (laserMapping.cpp:1894-1898): double math (Eigen quaternion * vector form), result
// rounded to float.  R = s.rot, Roff = s.offset_R_L_I.
struct PoseDev {
  double rot[4];   // x,y,z,w
  double offR[4];
  double pos[3];
  double offT[3];
};
__device__ __forceinline__ void qrot_d(const double* q, double vx, double vy, double vz, double& ox, double& oy, double& oz) {
  double ux = __dsub_rn(__dmul_rn(q[1], vz), __dmul_rn(q[2], vy));
  double uy = __dsub_rn(__dmul_rn(q[2], vx), __dmul_rn(q[0], vz));
  double uz = __dsub_rn(__dmul_rn(q[0], vy), __dmul_rn(q[1], vx));
  ux = __dadd_rn(ux, ux); uy = __dadd_rn(uy, uy); uz = __dadd_rn(uz, uz);
  const double cx = __dsub_rn(__dmul_rn(q[1], uz), __dmul_rn(q[2], uy));
  const double cy = __dsub_rn(__dmul_rn(q[2], ux), __dmul_rn(q[0], uz));
  const double cz = __dsub_rn(__dmul_rn(q[0], uy), __dmul_rn(q[1], ux));
  ox = __dadd_rn(__dadd_rn(vx, __dmul_rn(q[3], ux)), cx);
  oy = __dadd_rn(__dadd_rn(vy, __dmul_rn(q[3], uy)), cy);
  oz = __dadd_rn(__dadd_rn(vz, __dmul_rn(q[3], uz)), cz);
}
__device__ __forceinline__ float4 body_to_world(const PoseDev& s, const float4 pb) {
  double ax, ay, az, gx, gy, gz;
  qrot_d(s.offR, (double)pb.x, (double)pb.y, (double)pb.z, ax, ay, az);
  ax = __dadd_rn(ax, s.offT[0]); ay = __dadd_rn(ay, s.offT[1]); az = __dadd_rn(az, s.offT[2]);
  qrot_d(s.rot, ax, ay, az, gx, gy, gz);
  return make_float4((float)__dadd_rn(gx, s.pos[0]), (float)__dadd_rn(gy, s.pos[1]), (float)__dadd_rn(gz, s.pos[2]), pb.w);
}

// Device-resident state of the iterated update (see esikf_device.cuh); the measurement kernels read the pose of the
// current iterate and the loop flags from here when running in device-driven mode (ctl != nullptr).
constexpr int NDOF = 23;
struct EsikfCtl {
  double x[26];        // current iterate x_
  double xp[26];       // x_propagated
  double Pp[NDOF * NDOF];
  double P[NDOF * NDOF];
  double limit[NDOF];
  double R;
  double last_res;
  PoseDev pose;        // pose of the current iterate
  int max_iter, it, t, converge, finished, need_host, passes, searches, lastM, n;
  int flg_inited;      // flg_EKF_inited of this scan (laserMapping.cpp:2317)
  int pad_;
  const float4* body;  // feats_down_body of this scan (travels with the staged inputs: the captured graphs do not depend on it)
  unsigned long long t_begin;   // %globaltimer when this scan's sequence started (k_esikf_begin); k_publish reports the span
};
__device__ __forceinline__ bool ctl_pass_active(const EsikfCtl* c) { return !c->finished && c->it < c->max_iter; }

struct KnnArgs {
  MapDev m;
  const float4* q;     // n world-frame query points (x,y,z,*)
  int n;
  float4* nbr;         // [K][n] : (x,y,z,d2) of the r-th neighbour of query i at nbr[r*n+i]
  unsigned char* cnt;  // [n] number of neighbours found
  float max_d2;        // max_dist^2 (INF: unbounded)
  int* phase_stats;    // optional [4]: queries finishing in phase A / B / C, total candidate points
  int* worklist;       // stencil kernel: indices of queries it could not prove complete; warp kernel: its input list
                       // (WORK_EMPTY between passes; see "work-list hand-over" below)
  int* work_count;     // number of entries in worklist (device)
  int* work_ticket;    // exact kernel: next unclaimed work-list entry (device, zeroed with work_count)
  int* stencil_done;   // stencil CTAs holding queries that have published all of them (device, zeroed with work_count)
  int exact_warps;     // warps of the exact kernel's grid: the stencil kernel closes that many entries past the list's end
  const EsikfCtl* ctl; // device-driven mode: queries = body_to_world(ctl->pose, ctl->body[i]); skipped unless a search pass
  const float4* body;  // (unused: the scan pointer of the device-driven mode is ctl->body)
  int stride;          // leading dimension of nbr (>= n; the session capacity, so launches do not depend on n)
};

// squared distance from q to the axis-aligned cell [lo,hi) per axis, shrunk by mg (conservative lower bound)
__device__ __forceinline__ float box_mind2(float qx, float qy, float qz, float lx, float ly, float lz, float hx, float hy, float hz, float mg) {
  const float gx = fmaxf(fmaxf(lx - qx, qx - hx) - mg, 0.f);
  const float gy = fmaxf(fmaxf(ly - qy, qy - hy) - mg, 0.f);
  const float gz = fmaxf(fmaxf(lz - qz, qz - hz) - mg, 0.f);
  return gx * gx + gy * gy + gz * gz;
}
// squared distance from q (inside) to the nearest face of [lo,hi), shrunk by mg; 0 if outside / too close
__device__ __forceinline__ float cover2(float qx, float qy, float qz, float lx, float ly, float lz, float hx, float hy, float hz, float mg) {
  float c = fminf(fminf(fminf(qx - lx, hx - qx), fminf(qy - ly, hy - qy)), fminf(qz - lz, hz - qz)) - mg;
  return c > 0.f ? c * c : 0.f;
}

constexpr int EXACT_RINGS = 8;     // rings searched through the 27 staged coarse bitmaps: (q_block +- 8) stays inside them
constexpr int CAND_CAP = 512;      // per-warp candidate list capacity (voxel slot ids)

struct ExactSmem {
  unsigned cand[KNN_THREADS / 32][CAND_CAP];
  unsigned long long cbits[KNN_THREADS / 32][27 * 8];
};

// shell position idx (0 .. (2r+1)^3 - (2r-1)^3 - 1) of ring r -> block offset; ring 1 enumerates the full 3x3x3 cube instead
__device__ __forceinline__ void shell_offset(int r, int idx, int& dx, int& dy, int& dz) {
  const int wd = 2 * r + 1, face = wd * wd;
  if (idx < 2 * face) {          // the two full slices dz = -r, +r
    const int sl = idx >= face;
    const int rem = idx - sl * face;
    dz = sl ? r : -r;
    dy = rem / wd - r;
    dx = rem - (dy + r) * wd - r;
    return;
  }
  const int j = idx - 2 * face, per = 8 * r;
  const int zi = j / per, p = j - zi * per;
  dz = zi - (r - 1);
  if (p < wd) { dx = p - r; dy = -r; }
  else if (p < 2 * wd) { dx = p - wd - r; dy = r; }
  else {
    const int q = p - 2 * wd, side = q / (wd - 2);
    dy = q - side * (wd - 2) - (r - 1);
    dx = side ? r : -r;
  }
}

// 4-bit mask of the slabs (local voxel coordinate 0..3 along one axis) of block coordinate b that can hold a point
// within sqrt(bound) of q along this axis (conservative: gaps are shrunk by the rounding margin mg)
__device__ __forceinline__ unsigned axis_slabs_within(int b, float q, float ds, float mg, float bound) {
  unsigned m = 0u;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float lo = (float)(b * 4 + i) * ds;
    const float g = fmaxf(fmaxf(lo - q, q - (lo + ds)) - mg, 0.f);
    m |= (g * g <= bound) ? (1u << i) : 0u;
  }
  return m;
}

// One batch of candidate BLOCKS for one query, processed by the whole warp (the core of the exact kernel): `nb` positions
// (pos(idx, bx, by, bz) -> false to skip one) are taken 128 at a time; each is pruned by its box distance against `bound`,
// ONE round trip fetches the 32-byte hash entries (block index + voxel occupancy) of the survivors, the occupancy words are
// cut down (5^3 stencil already seen when cut_stencil; per-axis slab tests against `bound`), the surviving voxels of ALL
// blocks of the round are compacted into one candidate list in shared memory (warp prefix sum; every lane pushes its
// blocks' voxels) and consumed 128 at a time: four independent 16-byte point loads per lane and round trip, then the
// insertions into the lane-local sorted lists `t`.
template <int K, class PosFn>
__device__ __forceinline__ void exact_block_batch(const MapDev& m, unsigned* cand, int lane, int nb, PosFn pos, float qx, float qy,
                                                  float qz, int cvx, int cvy, int cvz, float mg, float bound, bool cut_stencil,
                                                  TopK<K>& t) {
  const float ds = m.ds, bs4 = 4.f * ds;
#pragma unroll 1
  for (int base = 0; base < nb; base += 128) {
    int blk[4];
    uint4 ent[4];
    unsigned long long mask[4];
    int bxs[4], bys[4], bzs[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int idx = base + 32 * u + lane;
      blk[u] = -2;   // -2: no probe issued
      mask[u] = 0ull;
      bxs[u] = bys[u] = bzs[u] = 0;
      if (idx < nb) {
        int bx, by, bz;
        if (pos(idx, bx, by, bz)) {
          bxs[u] = bx; bys[u] = by; bzs[u] = bz;
          const float lx = (float)bx * bs4, ly = (float)by * bs4, lz = (float)bz * bs4;
          if (!(box_mind2(qx, qy, qz, lx, ly, lz, lx + bs4, ly + bs4, lz + bs4, mg) > bound)) {
            const uint32_t hs = hash_key(pack_key(bx, by, bz)) & m.hash_mask;
            const HEntry* he = &m.hent[hs];
            ent[u] = __ldg(reinterpret_cast<const uint4*>(he));
            mask[u] = __ldg(reinterpret_cast<const unsigned long long*>(&he->mask));   // same 32-B sector
            prefetch_next_entry(m, hs);
            blk[u] = -1;
          }
        }
      }
    }
    int c = 0;   // this lane's candidate voxels of the round
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (blk[u] == -1) {
        const uint64_t key = pack_key(bxs[u], bys[u], bzs[u]);
        const uint64_t k0 = ((uint64_t)ent[u].y << 32) | ent[u].x;
        if (k0 == key) blk[u] = (int)ent[u].z;
        else if (k0 == KEY_EMPTY) { blk[u] = -1; mask[u] = 0ull; }
        else blk[u] = find_block_mask(m, key, mask[u]);   // collision: sequential probe
        if (blk[u] >= 0 && mask[u]) {
          if (cut_stencil) mask[u] &= ~block_stencil_mask(bxs[u], bys[u], bzs[u], cvx, cvy, cvz);
          if (bound < CUDART_INF_F)
            mask[u] &= mask_from_axes(axis_slabs_within(bxs[u], qx, ds, mg, bound), axis_slabs_within(bys[u], qy, ds, mg, bound),
                                      axis_slabs_within(bzs[u], qz, ds, mg, bound));
        } else mask[u] = 0ull;
      } else mask[u] = 0ull;
      c += __popcll(mask[u]);
    }
    // ---- compaction: exclusive prefix of the per-lane candidate counts
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(FULL, incl, o);
      if (lane >= o) incl += v;
    }
    const int T = __shfl_sync(FULL, incl, 31);
    if (T == 0) continue;   // warp-uniform
    const int mybase = incl - c;
#pragma unroll 1
    for (int chunk = 0; chunk < T; chunk += CAND_CAP) {
      int p0 = mybase - chunk;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        unsigned long long mm = mask[u];
        const unsigned pb = (unsigned)blk[u] * 64u;
        while (mm) {
          const int sl = __ffsll((long long)mm) - 1;
          mm &= mm - 1;
          if ((unsigned)p0 < (unsigned)CAND_CAP) cand[p0] = pb + (unsigned)sl;
          ++p0;
        }
      }
      __syncwarp();
      const int n = min(T - chunk, CAND_CAP);
#pragma unroll 1
      for (int j0 = 0; j0 < n; j0 += 128) {
        float4 e[4];
        bool ok[4];
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const int j = j0 + 32 * v + lane;
          ok[v] = j < n;
          if (ok[v]) e[v] = __ldg(&m.slots[cand[j]]);
        }
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          if (ok[v]) {
            const float4 p = e[v];
            const float dd = sqdist(qx, qy, qz, p.x, p.y, p.z);
            if (dd <= bound) t.insert(dd, p.x, p.y, p.z);
            walk_chain(m, __float_as_int(p.w), [&](const float4 o, int) {
              const float d2 = sqdist(qx, qy, qz, o.x, o.y, o.z);
              if (d2 <= bound) t.insert(d2, o.x, o.y, o.z);
            });
          }
        }
      }
      __syncwarp();
    }
  }
}

// All blocks of one coarse cell (slot cs) that can still matter: its 512-bit block bitmap is staged in the warp's shared
// memory (`cb`, 8 words) and the cell's blocks go through exact_block_batch; blocks within BLOCK_RINGS of the query block
// were visited by the rings and are skipped.
template <int K>
__device__ __forceinline__ void scan_coarse_cell(const MapDev& m, unsigned* cand, unsigned long long* cb, int cs, int lane, float qx,
                                                 float qy, float qz, int cvx, int cvy, int cvz, bool have, float thr, float lim,
                                                 float mg, TopK<K>& t) {
  const int qbx = cvx >> 2, qby = cvy >> 2, qbz = cvz >> 2;
  int ccx, ccy, ccz;
  unpack_key(__ldg(&m.ckeys[cs]), ccx, ccy, ccz);
  __syncwarp();
  if (lane < 8) cb[lane] = __ldg(&m.cbits[(size_t)cs * 8 + lane]);
  __syncwarp();
  const float bound = fminf(have ? thr : CUDART_INF_F, lim);
  exact_block_batch<K>(m, cand, lane, 512, [&](int idx, int& bx, int& by, int& bz) -> bool {
    if (!((cb[idx >> 6] >> (idx & 63)) & 1ull)) return false;
    bx = ccx * 8 + (idx & 7); by = ccy * 8 + ((idx >> 3) & 7); bz = ccz * 8 + (idx >> 6);
    return !(abs(bx - qbx) <= BLOCK_RINGS && abs(by - qby) <= BLOCK_RINGS && abs(bz - qbz) <= BLOCK_RINGS);
  }, qx, qy, qz, cvx, cvy, cvz, mg, bound, false, t);
}

// Finish ONE query with the whole warp over the coarse levels (rare: map frontier).  A real call (noinline) so that its
// register needs do not inflate the group kernel; wcount/wthr/seed = state of the query after the block rings (lane r
// passes result r in sd,sx,sy,sz).
template <int K>
__device__ __noinline__ void warp_finish_coarse(MapDev m, unsigned* cand, unsigned long long* cb, float4* nbr, unsigned char* cnt,
                                                int* phase_stats, int stride, float lim,
                                                int qi, float wqx, float wqy, float wqz, int wcount, float wthr, float sd, float sx,
                                                float sy, float sz) {
  const int lane = threadIdx.x & 31;
  const float ds = m.ds;
    TopK<K> tw;
    tw.clear();
    float wd_ = CUDART_INF_F, wx = CUDART_NAN_F, wy = CUDART_NAN_F, wz = CUDART_NAN_F;
    if (lane < wcount) { wd_ = sd; wx = sx; wy = sy; wz = sz; tw.d[0] = sd; tw.x[0] = sx; tw.y[0] = sy; tw.z[0] = sz; }
    const int cvx = voxel_of(wqx, ds), cvy = voxel_of(wqy, ds), cvz = voxel_of(wqz, ds);
    const float mg = 1e-3f * ds + 4.8e-7f * (fabsf(wqx) + fabsf(wqy) + fabsf(wqz));
    const int qbx = cvx >> 2, qby = cvy >> 2, qbz = cvz >> 2;
    int phase = 2;
    {
      // ---------------- phase B: 3x3x3 coarse cells around the query
      const int qcx = qbx >> 3, qcy = qby >> 3, qcz = qbz >> 3;
      int mycs = -1;
      if (lane < 27) mycs = find_coarse(m, pack_key(qcx + (lane % 3) - 1, qcy + ((lane / 3) % 3) - 1, qcz + (lane / 9) - 1));
      // nearest cells first (centre cell), so the bound tightens early
      const unsigned present = __ballot_sync(FULL, mycs >= 0);
      {
        const int cs = __shfl_sync(FULL, mycs, 13);
        if (cs >= 0) scan_coarse_cell<K>(m, cand, cb, cs, lane, wqx, wqy, wqz, cvx, cvy, cvz, wcount == K, wthr, lim, mg, tw);
        if (wcount < K) wcount = warp_merge<K>(tw, FULL, lane, lane, wd_, wx, wy, wz, wthr);  // get a finite bound before the ring
      }
      unsigned rest = present & ~(1u << 13);
      while (rest) {
        const int c = __ffs(rest) - 1;
        rest &= rest - 1;
        const int cs = __shfl_sync(FULL, mycs, c);
        scan_coarse_cell<K>(m, cand, cb, cs, lane, wqx, wqy, wqz, cvx, cvy, cvz, wcount == K, wthr, lim, mg, tw);
      }
      wcount = warp_merge<K>(tw, FULL, lane, lane, wd_, wx, wy, wz, wthr);
      const float cs32 = 32.f * ds;
      const float cov = cover2(wqx, wqy, wqz, (float)(qcx - 1) * cs32, (float)(qcy - 1) * cs32, (float)(qcz - 1) * cs32,
                               (float)(qcx + 2) * cs32, (float)(qcy + 2) * cs32, (float)(qcz + 2) * cs32, mg);
      const bool wdone = (wcount == K && wthr < cov) || cov > lim;
      if (!wdone) {
        // ---------------- phase C: every other coarse cell of the map, pruned by its box distance.  Nearest first: while the
        // query has no k-th distance yet (far outside the map: nothing to prune with), the cell(s) at the smallest box distance
        // not visited so far are scanned and merged — the first one or two give a bound that prunes almost all of the rest —
        // then one sweep over the remaining cells with that bound.
        phase = 3;
        const int ncs = m.counters[CNT_COARSE_USED];   // dense list of occupied coarse cells
        auto cell_md = [&](int li, int& cs) -> float {   // box distance of list entry li (INF: no cell / inside the 3x3x3 already done)
          cs = li < ncs ? (int)__ldg(&m.clist[li]) : -1;
          const uint64_t ck = cs >= 0 ? __ldg(&m.ckeys[cs]) : KEY_EMPTY;
          if (ck == KEY_EMPTY) return CUDART_INF_F;
          int cx, cy, cz;
          unpack_key(ck, cx, cy, cz);
          if (abs(cx - qcx) <= 1 && abs(cy - qcy) <= 1 && abs(cz - qcz) <= 1) return CUDART_INF_F;
          return box_mind2(wqx, wqy, wqz, (float)cx * cs32, (float)cy * cs32, (float)cz * cs32, (float)(cx + 1) * cs32,
                           (float)(cy + 1) * cs32, (float)(cz + 1) * cs32, mg);
        };
        float level = -1.f;   // cells with md <= level have been scanned
#pragma unroll 1
        for (int iter = 0; iter < 16 && wcount < K; ++iter) {
          float best = CUDART_INF_F;
#pragma unroll 1
          for (int base = 0; base < ncs; base += 32) {
            int cs;
            const float md = cell_md(base + lane, cs);
            if (md > level && md <= lim) best = fminf(best, md);
          }
          best = __uint_as_float(__reduce_min_sync(FULL, __float_as_uint(best)));   // (non-negative floats order like their bits)
          if (!(best < CUDART_INF_F)) break;
#pragma unroll 1
          for (int base = 0; base < ncs; base += 32) {
            int cs;
            const float md = cell_md(base + lane, cs);
            unsigned todo = __ballot_sync(FULL, md == best);
            while (todo) {
              const int c = __ffs(todo) - 1;
              todo &= todo - 1;
              scan_coarse_cell<K>(m, cand, cb, __shfl_sync(FULL, cs, c), lane, wqx, wqy, wqz, cvx, cvy, cvz, wcount == K, wthr, lim, mg, tw);
            }
          }
          wcount = warp_merge<K>(tw, FULL, lane, lane, wd_, wx, wy, wz, wthr);
          level = best;
        }
#pragma unroll 1
        for (int base = 0; base < ncs; base += 32) {
          int cs;
          const float md = cell_md(base + lane, cs);
          const bool go = md > level && md < CUDART_INF_F && (wcount < K || md <= wthr) && md <= lim;
          unsigned todo = __ballot_sync(FULL, go);
          if (!todo) continue;
          while (todo) {
            const int c = __ffs(todo) - 1;
            todo &= todo - 1;
            scan_coarse_cell<K>(m, cand, cb, __shfl_sync(FULL, cs, c), lane, wqx, wqy, wqz, cvx, cvy, cvz, wcount == K, wthr, lim, mg, tw);
          }
          wcount = warp_merge<K>(tw, FULL, lane, lane, wd_, wx, wy, wz, wthr);
        }
      }
    }
    if (lane < K) nbr[(size_t)lane * stride + qi] = make_float4(wx, wy, wz, wd_);
    if (lane == 0) {
      cnt[qi] = (unsigned char)wcount;
      if (phase_stats) atomicAdd(&phase_stats[phase], 1);
    }
}

// Work-list hand-over.  The exact kernel is launched as a programmatic dependent of the stencil kernel: its CTAs become
// resident while the stencil kernel's slowest warps are still running, and take unresolved queries as they are published.
//   stencil thread: writes the query's neighbour cache and count, takes an entry with atomicAdd(work_count) and stores the
//     query index into it with a release store.  Each CTA holding queries then counts itself into stencil_done; the CTA
//     that completes the count (every entry is published by then) closes the list: it writes WORK_END into the
//     exact_warps entries past its end.
//   exact warp: holds one ticket (entry index) at a time, waits until its entry is no longer WORK_EMPTY (relaxed polls,
//     then one acquire), resets it to WORK_EMPTY and works on it or, at WORK_END, exits.  Tickets are handed out in order and a warp claims
//     a new one only after finishing one, so when the list is closed the warps hold exactly the closed entries: every
//     entry is consumed and the list is left all WORK_EMPTY for the next pass.
//   Launched the ordinary way (no programmatic edge), the exact kernel finds the whole list published and closed.
constexpr int WORK_EMPTY = -1;
constexpr int WORK_END = -2;
constexpr unsigned long long KNN_WAIT_NS = 1000000000ull;   // a wait longer than 1 s is a protocol failure: ERR_KNN_STALL

// Ticket w of the exact kernel (warp-uniform): the query index of entry w, or -1 at the end of the list.
__device__ __forceinline__ int worklist_take(const KnnArgs& a, int w, int lane) {
  int v = WORK_EMPTY;
  if (lane == 0) {
    v = ld_relaxed(&a.worklist[w]);
    if (v == WORK_EMPTY) {
      // not published yet: back off with sleeps, so that waiting warps leave the issue slots to the stencil kernel's warps
      const unsigned long long t0 = global_timer_ns();
      unsigned ns = 32;
      do {
        __nanosleep(ns);
        ns = min(2u * ns, 512u);
        v = ld_relaxed(&a.worklist[w]);
        if (v == WORK_EMPTY && global_timer_ns() - t0 > KNN_WAIT_NS) {
          atomicOr(&a.m.counters[CNT_ERROR], ERR_KNN_STALL);
          v = WORK_END;
        }
      } while (v == WORK_EMPTY);
    }
    if (v >= 0) v = ld_acquire(&a.worklist[w]);   // the one acquire of this entry (same value: only this warp resets it)
    a.worklist[w] = WORK_EMPTY;   // (this warp is the entry's only reader; its next writer is a later kernel)
  }
  v = __shfl_sync(FULL, v, 0);
  __syncwarp();   // the acquire of lane 0 orders the other lanes' reads of the query's neighbour cache
  return v == WORK_END ? -1 : v;
}

// K1b: exact completion of the queries the stencil kernel could not prove complete (its work list).  The stencil
// kernel has already visited the whole 5x5x5 voxel stencil and left its (up to K) best points in the neighbour cache:
// they seed the search, which then only looks OUTSIDE the stencil.  One WARP per query, work claimed by atomic tickets.
//
// The kernel is a chain of dependent memory round trips per query, so it is built to keep that chain short:
//   ring r (shell of blocks at Chebyshev block distance r around the query block, r = 1..EXACT_RINGS):
//     1. the shell positions are enumerated 128 at a time (4 per lane); each is pruned by its box distance against the
//        current k-th distance, and from ring 3 on by the block-occupancy bitmaps of the 3x3x3 coarse cells around the query
//        (staged once into shared memory), so that only blocks that exist and can matter are probed;
//     2. ONE round trip fetches the 32-byte hash entries (block index + voxel occupancy) of all surviving positions;
//     3. the occupancy words are cut down by the 5^3 stencil (ring 1) and by a separable per-axis slab test against the
//        k-th distance; the surviving voxels of ALL blocks of the round are compacted into one candidate list in shared
//        memory (each lane pushes its blocks' voxels at the offset given by a warp prefix sum);
//     4. the list is consumed 128 candidates at a time: four independent 16-byte point loads per lane and round trip,
//        then the insertions into lane-local sorted lists;
//     5. one K-round warp merge per ring gives the new k-th distance and the completeness test
//        (d_k < distance to the boundary of the searched cube).
//   Queries still open after ring EXACT_RINGS (nothing within ~6 m at 0.2 m voxels: far outside the map) are finished over
//   the coarse levels by warp_finish_coarse (remaining blocks of the 3x3x3 coarse cells, then every coarse cell with
//   box-distance pruning).
// Launched as a programmatic dependent of k_knn_stencil (work-list hand-over above): no griddepcontrol.wait before the
// loop (everything but the work list and the neighbour cache was written before the stencil kernel started), and one
// at the end, so that this grid completes only after the stencil grid and the next kernel sees both grids' writes.
template <int K>
__global__ void __launch_bounds__(KNN_THREADS, KNN_MIN_CTAS) k_knn(KnnArgs a) {
  pdl_trigger();
  __shared__ ExactSmem sm;
  const MapDev& m = a.m;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float ds = m.ds;
  const float lim = a.max_d2;
  unsigned* cand = sm.cand[wid];
  unsigned long long* cb = sm.cbits[wid];
  // (the pass's stencil kernel skips the same passes, and a scan without points publishes nothing)
  const bool active = !(a.ctl && !(ctl_pass_active(a.ctl) && a.ctl->converge)) && (a.ctl ? a.ctl->n : a.n) > 0;
#ifdef FLB_TRACE
  const int tslot = 3 * 8 + (a.ctl ? a.ctl->it + 1 : 0);   // timeline of this kernel: first pick-up -> last warp's exit
  bool first_take = true;
#endif
  // Dynamic distribution: every warp claims the next list entry with one atomic.  Query cost varies by two orders of
  // magnitude (ring 1 vs far outside the map), so a static stride leaves the kernel waiting for the unlucky warp.
  // (the first entry of every warp is static — its global warp index — so that a few thousand warps do not start by queueing
  // on one atomic; only the entries beyond the first wave are claimed by ticket)
  const int nwarps = (int)(gridDim.x * (blockDim.x >> 5));
  int w = (int)(blockIdx.x * (blockDim.x >> 5)) + wid;
  for (; active; ) {
    const int i = worklist_take(a, w, lane);   // warp-uniform
    if (i < 0) break;
#ifdef FLB_TRACE
    if (lane == 0) {
      if (first_take) FLB_TRACE_STAMP(tslot, true);
      if (a.ctl && a.ctl->it == -1) FLB_TRACE_HIST(80, 2 * 8);   // when the first pass's unresolved queries are picked up
    }
    first_take = false;
#endif
    const float4 q4 = a.ctl ? body_to_world(a.ctl->pose, __ldg(&a.ctl->body[i])) : __ldg(&a.q[i]);
    const float qx = q4.x, qy = q4.y, qz = q4.z;
    TopK<K> t;
    t.clear();
    float rd = CUDART_INF_F, rx = CUDART_NAN_F, ry = CUDART_NAN_F, rz = CUDART_NAN_F, thr = CUDART_INF_F;
    // ---------------- seed: the stencil kernel's result (state as after a merge: lane r holds result r)
    int gcount = __ldcg(&a.cnt[i]);   // (L2 loads: written by the stencil kernel while this one runs)
    if (lane < gcount) {
      const float4 sd = __ldcg(&a.nbr[(size_t)lane * a.stride + i]);
      rd = sd.w; rx = sd.x; ry = sd.y; rz = sd.z;
      t.d[0] = rd; t.x[0] = rx; t.y[0] = ry; t.z[0] = rz;
    }
    {
      const float dk = __shfl_sync(FULL, rd, K - 1);
      thr = gcount == K ? dk : CUDART_INF_F;
    }
    const int cvx = voxel_of(qx, ds), cvy = voxel_of(qy, ds), cvz = voxel_of(qz, ds);
    const float mg = 1e-3f * ds + 4.8e-7f * (fabsf(qx) + fabsf(qy) + fabsf(qz));
    const int qbx = cvx >> 2, qby = cvy >> 2, qbz = cvz >> 2;
    const int qcx = qbx >> 3, qcy = qby >> 3, qcz = qbz >> 3;
    const float bs4 = 4.f * ds;
    bool done = false;
    FLB_DBG_CLOCK(e0);
    int dbg_rings = 0;
    (void)dbg_rings;
#ifdef FLB_TRACE
    long long ph_probe = 0, ph_merge = 0, ph_mark = clock64();   // (ph_probe: the block batches = probes + compaction + point loads)
    const long long ph_seed = ph_mark - e0;
#define KPH(acc) { const long long now_ = clock64(); acc += now_ - ph_mark; ph_mark = now_; }
#else
#define KPH(acc)
#endif
#pragma unroll 1
    for (int r = 1; r <= EXACT_RINGS && !done; ++r) {
      if (r == 3) {
        // ---- stage the block-occupancy bitmaps of the 3x3x3 coarse cells around the query (27 x 512 bits)
        int mycs = -1;
        if (lane < 27) mycs = find_coarse(m, pack_key(qcx + (lane % 3) - 1, qcy + ((lane / 3) % 3) - 1, qcz + (lane / 9) - 1));
#pragma unroll
        for (int u = 0; u < 7; ++u) {
          const int wi = lane + 32 * u;
          const int cs = __shfl_sync(FULL, mycs, min(wi >> 3, 26));
          if (wi < 27 * 8) cb[wi] = cs >= 0 ? __ldg(&m.cbits[(size_t)cs * 8 + (wi & 7)]) : 0ull;
        }
        __syncwarp();
        // nothing at all within the 3x3x3 coarse cells (a return far outside the map): rings 3..8 cannot find anything
        if (__ballot_sync(FULL, mycs >= 0) == 0u) break;
      }
      const float bound = fminf(gcount == K ? thr : CUDART_INF_F, lim);
      const int wd = 2 * r + 1;
      const int nb = (r == 1) ? 27 : wd * wd * wd - (wd - 2) * (wd - 2) * (wd - 2);
      exact_block_batch<K>(m, cand, lane, nb, [&](int idx, int& bx, int& by, int& bz) -> bool {
        int dx, dy, dz;
        if (r == 1) { dx = idx % 3 - 1; dy = (idx / 3) % 3 - 1; dz = idx / 9 - 1; }   // incl. the query's own block: its
        else shell_offset(r, idx, dx, dy, dz);                                         // voxels outside the stencil are unseen
        bx = qbx + dx; by = qby + dy; bz = qbz + dz;
        if (r >= 3) {   // (rings 3..8 lie inside the staged 3x3x3 coarse cells: only blocks that exist are probed)
          const int cell = ((bz >> 3) - (qcz - 1)) * 9 + ((by >> 3) - (qcy - 1)) * 3 + ((bx >> 3) - (qcx - 1));
          const int bit = ((bz & 7) << 6) | ((by & 7) << 3) | (bx & 7);
          return (cb[cell * 8 + (bit >> 6)] >> (bit & 63)) & 1ull;
        }
        return true;
      }, qx, qy, qz, cvx, cvy, cvz, mg, bound, r == 1, t);
      KPH(ph_probe);
      // ---- merge the lane-local lists: new k-th distance, completeness of the searched cube
      gcount = warp_merge<K>(t, FULL, lane, lane, rd, rx, ry, rz, thr);
      KPH(ph_merge);
      dbg_rings = r;
      const float cov = cover2(qx, qy, qz, (float)(qbx - r) * bs4, (float)(qby - r) * bs4, (float)(qbz - r) * bs4,
                               (float)(qbx + r + 1) * bs4, (float)(qby + r + 1) * bs4, (float)(qbz + r + 1) * bs4, mg);
      done = (gcount == K && thr < cov) || cov > lim;
    }
    if (done) {
      if (lane < K) a.nbr[(size_t)lane * a.stride + i] = make_float4(rx, ry, rz, rd);
      if (lane == 0) {
        a.cnt[i] = (unsigned char)gcount;
        if (a.phase_stats) atomicAdd(&a.phase_stats[1], 1);
      }
    }
#ifdef FLB_TRACE
    if (lane == 0 && a.ctl && a.ctl->it == -1) {
      const long long e1 = clock64();
      FLB_DBG_ADD(16, 1); FLB_DBG_ADD(17, e1 - e0); FLB_DBG_MAX(18, e1 - e0); FLB_DBG_ADD(18 + min(dbg_rings, 6), 1);
      FLB_DBG_ADD(25, done ? 0 : 1);
      FLB_DBG_ADD(58 + (int)min((e1 - e0) >> 13, 5ll), 1);   // histogram of the per-query cycles, 8192-cycle buckets
      FLB_DBG_ADD(32, ph_seed); FLB_DBG_ADD(33, ph_probe); FLB_DBG_ADD(36, ph_merge);
    }
#endif
    // ---------------- still unresolved after the block rings: finish over the coarse levels (the blocks of the rings
    // are skipped inside scan_coarse_cell)
    if (!done) {
      __syncwarp();
      warp_finish_coarse<K>(m, cand, cb, a.nbr, a.cnt, a.phase_stats, a.stride, lim, i, qx, qy, qz, gcount, thr, rd, rx, ry, rz);
    }
    if (lane == 0) w = nwarps + atomicAdd(a.work_ticket, 1);
    w = __shfl_sync(FULL, w, 0);
  }
  pdl_wait();
#ifdef FLB_TRACE
  if (lane == 0 && active) FLB_TRACE_STAMP(tslot, false);
#endif
}

// K1a: phase A with ONE THREAD per query (the common case: >99 % of LiDAR returns lie on mapped surfaces and are
// resolved by the 5x5x5 stencil).  Per query: 8 block probes (one 16-B hash entry + one 8-B occupancy word each),
// then ONE loop over the occupied stencil voxels of all 8 blocks (per-thread cursor, so a warp iterates
// max-over-lanes of the candidate COUNT, not the sum of per-block maxima) with one 16-B point load per candidate and
// a branch-free insertion into a register-resident (distance, slot-id) top-K.  No cross-lane traffic.
// Queries whose stencil cannot prove completeness are appended to a work list for the exact kernel k_knn.
template <int K>
struct TopKId {
  float d[K];
  unsigned id[K];
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int j = 0; j < K; ++j) { d[j] = CUDART_INF_F; id[j] = 0u; }
  }
  // branch-free sorted insert (equal distances keep their arrival order: exact float ties between distinct map points
  // are not canonicalised on this fast path — the reference's own tie order is traversal dependent, ikd_Tree.h:102-105)
  __device__ __forceinline__ void insert(float dd, unsigned pid) {
    bool c[K];
#pragma unroll
    for (int j = 0; j < K; ++j) c[j] = dd < d[j];
#pragma unroll
    for (int j = K - 1; j > 0; --j) {
      d[j] = c[j - 1] ? d[j - 1] : (c[j] ? dd : d[j]);
      id[j] = c[j - 1] ? id[j - 1] : (c[j] ? pid : id[j]);
    }
    d[0] = c[0] ? dd : d[0];
    id[0] = c[0] ? pid : id[0];
  }
};

constexpr int STENCIL_THREADS = 128;
constexpr int SHELL_LIST = 32;   // per-thread capacity of the surviving-shell-voxel list (bytes of shared memory)

// Occupancy-independent part of the candidate masks.  ax/ay/az are 8-bit per-axis masks over the 2 blocks the stencil
// spans (bits 0..3: local coordinates of the low block, 4..7: of the high block); the result is the 64-bit voxel mask
// of block half b (bit 0: x half, 1: y half, 2: z half) in slot order s = (z*4 + y)*4 + x.
__device__ __forceinline__ unsigned long long stencil_mask(unsigned ax, unsigned ay, unsigned az, int b) {
  return mask_from_axes((ax >> ((b & 1) << 2)) & 15u, (ay >> (((b >> 1) & 1) << 2)) & 15u, (az >> ((b >> 2) << 2)) & 15u);
}

// Per-thread shared-memory columns of the stencil kernel: 220 B per query, so that 7 CTAs of 128 threads (the register
// limit) fit one SM: 118 272 queries per wave on an H100's 132 SMs, slightly less than a cfg2 scan (118-119k points).
struct StencilSmem {
  int blk[8][STENCIL_THREADS];                     // block index of the 8 probed blocks (-1: absent)
  unsigned long long c5[8][STENCIL_THREADS];       // occupied voxels of each block inside the 5x5x5 stencil
  float gap[15][STENCIL_THREADS];                  // squared query-to-slab gaps: x[5], y[5], z[5]
  unsigned char list[SHELL_LIST][STENCIL_THREADS]; // surviving shell voxels, stencil-relative index jx + 5 jy + 25 jz
  unsigned xy3[4][STENCIL_THREADS];                // x&y pattern of the inner 3x3x3 mask per (x half, y half) of the 8 blocks
  unsigned z3[4][STENCIL_THREADS];                 // z pattern of the inner mask: [z half of the block pair * 2 + word (lo, hi)]
};
// inner 3x3x3 mask of block half b (dynamic b): three shared-memory words, two ANDs
__device__ __forceinline__ unsigned long long inner_mask(const StencilSmem& sm, int tid, int b) {
  const unsigned xy = sm.xy3[b & 3][tid];
  const int zq = (b >> 2) << 1;
  return ((unsigned long long)(xy & sm.z3[zq + 1][tid]) << 32) | (unsigned long long)(xy & sm.z3[zq][tid]);
}

// Visit the candidate voxels (c5 & inner mask, or c5 & ~inner mask when OUTER) of the 8 blocks: per-thread cursor over
// the blocks, four independent 16-B point loads in flight, branch-free insertion.
template <int K, bool OUTER>
__device__ __forceinline__ void stencil_pass(const MapDev& m, const StencilSmem& sm, int tid, unsigned ix, unsigned iy, unsigned iz,
                                             float qx, float qy, float qz, float lim, TopKId<K>& t, int& n_head, int& n_chain) {
  int b = -1, blk = 0;
  unsigned long long cand = 0ull;
  for (;;) {
    unsigned pid[4];
    int nc = 0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      pid[u] = 0u;
      while (cand == 0ull && b < 7) {
        ++b;
        const unsigned long long in3 = inner_mask(sm, tid, b);
        cand = sm.c5[b][tid] & (OUTER ? ~in3 : in3);
        blk = sm.blk[b][tid];
      }
      if (cand != 0ull) {
        const int sl = __ffsll((long long)cand) - 1;
        cand &= cand - 1;
        pid[u] = (unsigned)blk * 64u + (unsigned)sl;
        nc = u + 1;
      }
    }
    if (nc == 0) break;
    float4 e[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (u < nc) e[u] = __ldg(&m.slots[pid[u]]);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (u < nc) {
        float dd = sqdist(qx, qy, qz, e[u].x, e[u].y, e[u].z);
        if (dd <= lim && dd < t.d[K - 1]) t.insert(dd, pid[u]);   // (the guard lets a warp skip the insertion network when no lane needs it)
        ++n_head;
        walk_chain(m, __float_as_int(e[u].w), [&](const float4 o, int c) {  // overflow chain of this voxel
          ++n_chain;
          const float d2 = sqdist(qx, qy, qz, o.x, o.y, o.z);
          if (d2 <= lim && d2 < t.d[K - 1]) t.insert(d2, 0x80000000u | (unsigned)c);
        });
      }
    }
    if (nc < 4) break;
  }
}

// Outer-shell pass (the 98 voxels of the 5x5x5 stencil outside the inner 3x3x3).  After the inner pass the k-th distance is
// usually far smaller than the stencil, so the shell is cut down BEFORE any per-voxel work: per axis, the 5 slabs whose gap
// to the query exceeds the k-th distance are dropped (15 compares), the three 5-bit slab masks are expanded to the 8
// blocks with the separable mask builder, and only the occupied voxels inside that box go through (1) a flat, load-free
// loop that applies the exact box lower bound (sum of the three gaps) and compacts the survivors into a small per-thread
// list — lanes only diverge on cheap code — and (2) the loads, four survivors at a time; a full list is drained and the
// walk resumes with the tighter k-th distance.
// (ncu source view, round 1: walking all ~60 occupied shell voxels per query one by one was 30 % of the kernel's instructions.)
template <int K>
__device__ __forceinline__ void stencil_shell_pass(const MapDev& m, StencilSmem& sm, int tid, int ox, int oy, int oz, float qx,
                                                   float qy, float qz, float lim, TopKId<K>& t, int& n_head, int& n_chain) {
  // (no k-th distance yet = fewer than K points in the inner 3x3x3, sparse surroundings: bound = INF keeps every slab and
  // every occupied shell voxel — usually a short list — and the lane stays on the path of its warp's other lanes instead of
  // adding a whole-shell loop as a third divergent phase: those warps were the kernel's tail, 59k vs 37k cycles)
  unsigned wx = 0u, wy = 0u, wz = 0u;
  {
    const float bound0 = t.d[K - 1];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      wx |= (sm.gap[j][tid] <= bound0) ? (1u << j) : 0u;
      wy |= (sm.gap[5 + j][tid] <= bound0) ? (1u << j) : 0u;
      wz |= (sm.gap[10 + j][tid] <= bound0) ? (1u << j) : 0u;
    }
  }
  const unsigned ax = wx << ox, ay = wy << oy, az = wz << oz;   // 8-bit masks over the two blocks per axis
  // fill the list (load-free, cut with the k-th distance SO FAR), drain it (loads + insertions), and go on where the fill
  // stopped if the list was full: a dense shell under a loose bound streams through the same 32 entries, each round with a
  // tighter bound, instead of overflowing into an unpruned walk over all 98 voxels
  int b = 0;
  unsigned long long cand = 0ull;
  bool more = true;
#pragma unroll 1
  while (more) {
    const float bound = t.d[K - 1];
    int ns = 0;
#pragma unroll 1
    while (ns < SHELL_LIST) {
      if (cand == 0ull) {
        if (b == 8) { more = false; break; }
        cand = sm.c5[b][tid] & stencil_mask(ax, ay, az, b);
        if (cand != 0ull) cand &= ~inner_mask(sm, tid, b);
        ++b;
        continue;
      }
      const int sl = __ffsll((long long)cand) - 1;
      cand &= cand - 1;
      const int bb = b - 1;
      // stencil-relative voxel index per axis (0..4): block half * 4 + local coordinate - stencil origin
      const int jx = ((bb & 1) << 2) + (sl & 3) - ox, jy = (((bb >> 1) & 1) << 2) + ((sl >> 2) & 3) - oy, jz = ((bb >> 2) << 2) + (sl >> 4) - oz;
      const float md = sm.gap[jx][tid] + sm.gap[5 + jy][tid] + sm.gap[10 + jz][tid];
      if (!(md > bound)) {  // a point of this voxel could still enter the top-K
        sm.list[ns][tid] = (unsigned char)(jx + 5 * jy + 25 * jz);
        ++ns;
      }
    }
    for (int base = 0; base < ns; base += 4) {
      unsigned pid[4];
      float4 e[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        pid[u] = 0u;
        if (base + u < ns) {
          const int j = sm.list[base + u][tid];
          const int jz = j / 25, r = j - 25 * jz, jy = r / 5, jx = r - 5 * jy;
          const int vx = ox + jx, vy = oy + jy, vz = oz + jz;   // 0..7 across the two blocks per axis
          const int vb = (vx >> 2) | ((vy >> 2) << 1) | ((vz >> 2) << 2);
          pid[u] = (unsigned)sm.blk[vb][tid] * 64u + (unsigned)((vx & 3) | ((vy & 3) << 2) | ((vz & 3) << 4));
          e[u] = __ldg(&m.slots[pid[u]]);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (base + u < ns) {
          float dd = sqdist(qx, qy, qz, e[u].x, e[u].y, e[u].z);
          if (dd <= lim && dd < t.d[K - 1]) t.insert(dd, pid[u]);
          ++n_head;
          walk_chain(m, __float_as_int(e[u].w), [&](const float4 o, int c) {  // overflow chain of this voxel
            ++n_chain;
            const float d2 = sqdist(qx, qy, qz, o.x, o.y, o.z);
            if (d2 <= lim && d2 < t.d[K - 1]) t.insert(d2, 0x80000000u | (unsigned)c);
          });
        }
      }
    }
  }
}

// One query of the stencil kernel: search, write the neighbour cache, publish the query if it is unresolved.
template <int K>
__device__ __forceinline__ void stencil_query(const KnnArgs& a, StencilSmem& sm, int tid, int i) {
  const MapDev& m = a.m;
  const float ds = m.ds;
  const float lim = a.max_d2;
  const float4 q4 = a.ctl ? body_to_world(a.ctl->pose, __ldg(&a.ctl->body[i])) : __ldg(&a.q[i]);
  const float qx = q4.x, qy = q4.y, qz = q4.z;
  const float qlim = 4.0e6f * ds;
  TopKId<K> t;
  t.clear();
  bool done = false;
  FLB_DBG_CLOCK(w0);
  bool dbg_fallback = false;
  (void)dbg_fallback;
  if (fabsf(qx) < qlim && fabsf(qy) < qlim && fabsf(qz) < qlim) {
    const int cvx = voxel_of(qx, ds), cvy = voxel_of(qy, ds), cvz = voxel_of(qz, ds);
    const int bbx = (cvx - 2) >> 2, bby = (cvy - 2) >> 2, bbz = (cvz - 2) >> 2;
    const float mg = 1e-3f * ds + 4.8e-7f * (fabsf(qx) + fabsf(qy) + fabsf(qz));
    // per axis the 5-wide stencil covers local range [o,3] of the low block and [0,o] of the high block; the inner
    // 3-wide one is the same shifted by one voxel
    const int ox = (cvx - 2) & 3, oy = (cvy - 2) & 3, oz = (cvz - 2) & 3;
    const unsigned ax5 = 31u << ox, ay5 = 31u << oy, az5 = 31u << oz;   // 5-wide axis masks over the two blocks
    const unsigned ix = 14u << ox, iy = 14u << oy, iz = 14u << oz;      // inner 3-wide axis masks
    // squared gaps from the query to the 5 voxel slabs per axis (conservative: shrunk by the rounding margin)
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const float lx = (float)(cvx - 2 + j) * ds, ly = (float)(cvy - 2 + j) * ds, lz = (float)(cvz - 2 + j) * ds;
      const float gx = fmaxf(fmaxf(lx - qx, qx - (lx + ds)) - mg, 0.f);
      const float gy = fmaxf(fmaxf(ly - qy, qy - (ly + ds)) - mg, 0.f);
      const float gz = fmaxf(fmaxf(lz - qz, qz - (lz + ds)) - mg, 0.f);
      sm.gap[j][tid] = gx * gx;
      sm.gap[5 + j][tid] = gy * gy;
      sm.gap[10 + j][tid] = gz * gz;
    }
    // ---- the 8 hash probes are INDEPENDENT loads: issue them back to back (memory-level parallelism), then resolve;
    // only a collision (first slot holds another key) falls back to the sequential probe loop
    // (one 32-byte sector per entry: key + block index in the first half, the occupancy word in the second — the block
    // index and the occupied voxels arrive in ONE round trip, the point loads are the second and last dependent level)
    uint4 ent[8];
    unsigned long long occ[8];
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const uint32_t hs = hash_key(pack_key(bbx + (b & 1), bby + ((b >> 1) & 1), bbz + (b >> 2))) & m.hash_mask;
      const HEntry* he = &m.hent[hs];
      ent[b] = __ldg(reinterpret_cast<const uint4*>(he));
      occ[b] = __ldg(reinterpret_cast<const unsigned long long*>(&he->mask));
      prefetch_next_entry(m, hs);
    }
    int blk8[8];
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const uint64_t key = pack_key(bbx + (b & 1), bby + ((b >> 1) & 1), bbz + (b >> 2));
      const uint64_t k0 = ((uint64_t)ent[b].y << 32) | ent[b].x;
      if (k0 == key) blk8[b] = (int)ent[b].z;
      else if (k0 == KEY_EMPTY) { blk8[b] = -1; occ[b] = 0ull; }
      else blk8[b] = find_block_mask(m, key, occ[b]);   // collision: sequential probe
    }
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      sm.blk[b][tid] = blk8[b];
      sm.c5[b][tid] = occ[b] & stencil_mask(ax5, ay5, az5, b);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      sm.xy3[q][tid] = xpat32((ix >> ((q & 1) << 2)) & 15u) & ypat32((iy >> ((q >> 1) << 2)) & 15u);
      sm.z3[q][tid] = zpat32((((iz >> ((q >> 1) << 2)) & 15u) >> ((q & 1) << 1)) & 3u);
    }
    // ---- inner 3x3x3 first (gives a tight k-th distance), then the outer shell with box-distance pruning
    int n_chain = 0, n_head = 0;
    stencil_pass<K, false>(m, sm, tid, ix, iy, iz, qx, qy, qz, lim, t, n_head, n_chain);
    stencil_shell_pass<K>(m, sm, tid, ox, oy, oz, qx, qy, qz, lim, t, n_head, n_chain);
#ifdef FLB_TRACE
    if (a.ctl && a.ctl->it + 1 == 0) {   // first search pass: how the warps' durations spread (the kernel lasts as long as its slowest warp)
      const unsigned act = __activemask();
      const long long w1 = clock64();
      const int nfb = __popc(__ballot_sync(act, dbg_fallback));
      int mxc = n_chain + n_head;
      for (int o = 16; o; o >>= 1) mxc = max(mxc, __shfl_xor_sync(act, mxc, o));
      if ((tid & 31) == __ffs(act) - 1) {
        const long long d = w1 - w0;
        FLB_DBG_ADD(40, 1); FLB_DBG_ADD(41, d); FLB_DBG_MAX(42, d);
        if (nfb) { FLB_DBG_ADD(43, 1); FLB_DBG_ADD(44, d); FLB_DBG_ADD(45, nfb); }
        FLB_DBG_ADD(48 + (int)min(d >> 13, 7ll), 1);          // histogram, 8192-cycle buckets
        FLB_DBG_ADD(56, mxc); FLB_DBG_MAX(57, mxc);
      }
    }
#endif
    if (a.phase_stats) {  // profiling only: candidate statistics
      atomicAdd(&a.phase_stats[4], n_chain);
      atomicMax(&a.phase_stats[5], n_chain);
      atomicAdd(&a.phase_stats[6], n_head);
    }
    const float cov = cover2(qx, qy, qz, (float)(cvx - 2) * ds, (float)(cvy - 2) * ds, (float)(cvz - 2) * ds,
                             (float)(cvx + 3) * ds, (float)(cvy + 3) * ds, (float)(cvz + 3) * ds, mg);
    done = (t.d[K - 1] < CUDART_INF_F && t.d[K - 1] < cov) || cov > lim;
  } else {
    done = true;  // unrepresentable / NaN query: no neighbours
  }
  // results so far (final when `done`; otherwise the seed of the exact kernel, which only looks OUTSIDE the stencil)
  int c = 0;
#pragma unroll
  for (int r = 0; r < K; ++r) {
    const bool ok = t.d[r] < CUDART_INF_F;
    c += ok ? 1 : 0;
    float4 o = make_float4(CUDART_NAN_F, CUDART_NAN_F, CUDART_NAN_F, CUDART_INF_F);
    if (ok) {
      const float4 e = (t.id[r] & 0x80000000u) ? __ldg(&m.ovf[t.id[r] & 0x7FFFFFFFu]) : __ldg(&m.slots[t.id[r]]);
      o = make_float4(e.x, e.y, e.z, t.d[r]);
    }
    a.nbr[(size_t)r * a.stride + i] = o;
  }
  a.cnt[i] = (unsigned char)c;
  if (done) {
    if (a.phase_stats) atomicAdd(&a.phase_stats[0], 1);
  } else {
    // the exact kernel may already be waiting for this entry: the release orders the neighbour cache and count before it
    st_release(&a.worklist[atomicAdd(a.work_count, 1)], i);
#ifdef FLB_TRACE
    if (a.ctl && a.ctl->it == -1) FLB_TRACE_HIST(64, 2 * 8);   // when the first pass's unresolved queries are published
#endif
  }
}

template <int K>
__global__ void __launch_bounds__(STENCIL_THREADS, 7) k_knn_stencil(KnnArgs a) {
  pdl_sync();
  __shared__ StencilSmem sm;
  const int tid = threadIdx.x;
  FLB_TRACE_BEGIN(2 * 8 + (a.ctl ? a.ctl->it + 1 : 0));
  if (a.ctl && !(ctl_pass_active(a.ctl) && a.ctl->converge)) return;   // (the exact kernel skips the same passes)
  const int n = a.ctl ? a.ctl->n : a.n;
  if ((int)blockIdx.x * STENCIL_THREADS >= n) return;   // a CTA without queries is not counted in stencil_done
  const int i = blockIdx.x * STENCIL_THREADS + tid;
  if (i < n) stencil_query<K>(a, sm, tid, i);
  // every query of this CTA is published: count the CTA in; the CTA that completes the count closes the list
  __syncthreads();
  int last = 0;
  if (tid == 0) {
    const int nq = a.ctl ? a.ctl->n : a.n;   // (read again: keeps the search's register budget as it was)
    last = atom_add_release(a.stencil_done, 1) == (nq + STENCIL_THREADS - 1) / STENCIL_THREADS - 1;
    if (last) __threadfence();   // (acquire: every other CTA's entries, hence the final work_count, happened before)
  }
  if (__syncthreads_or(last)) {
    const int nw = ld_relaxed(a.work_count);
    // (no data behind WORK_END: relaxed stores, a release would put a GPU-wide memory barrier before each one)
    for (int j = tid; j < a.exact_warps; j += STENCIL_THREADS) st_relaxed(&a.worklist[nw + j], WORK_END);
  }
  FLB_TRACE_END(2 * 8 + (a.ctl ? a.ctl->it + 1 : 0));
}

__global__ void k_transform(PoseDev s, const float4* __restrict__ body, float4* __restrict__ world, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) world[i] = body_to_world(s, body[i]);
}

}  // namespace flb

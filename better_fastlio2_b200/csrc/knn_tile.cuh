// knn_tile.cuh — EXPERIMENTAL variant of the stencil 5-NN kernel (K1a) for the bulk-copy A/B of BASELINE's north_star
// ("TMA-staged voxel buckets into shared memory"): a CTA of 128 spatially coherent queries first finds the set of distinct
// map blocks its 128 x 8 stencil probes touch (shared-memory hash set), probes the global block hash ONCE per distinct block,
// stages the 1-KB buckets of those blocks into shared memory with cp.async.bulk (the TMA engine's linear bulk copy,
// completion counted on an mbarrier), and then runs the same exact stencil search out of shared memory.  Blocks that do
// not fit the staging area (or the hash set) are read from global memory as in k_knn_stencil, so the result is identical
// for ANY query order; only the speed depends on how many queries of a CTA share their blocks.
// Not on the product path (tools/knn_tile_ab.py drives it through flb_debug_knn_bench); the measured A/B is in
// profiles/r2_tma_ab.txt and discussed in DESIGN.md §3.
#pragma once
#include "knn_kernels.cuh"

namespace flb {

constexpr int TILE_THREADS = 128;
constexpr int TILE_SLOTS = 256;   // shared-memory hash set of distinct block keys (power of two)
constexpr int TILE_CAP = 40;      // staged buckets per CTA (40 KB; ~73 KB of shared memory per CTA -> 3 CTAs per SM)
constexpr int TILE_PROBE = 24;    // hash-set probe limit before a key is declared overflow

struct __align__(128) TileSmem {
  float4 tile[TILE_CAP][64];                  // staged buckets (bulk-copy destinations: 16-B aligned)
  unsigned long long keys[TILE_SLOTS];
  unsigned long long tmask[TILE_SLOTS];
  int tblk[TILE_SLOTS];
  short ttile[TILE_SLOTS];
  unsigned long long mbar;
  int ntile;
  // per-thread columns
  unsigned short slot[8][TILE_THREADS];       // hash-set slot of each of the 8 probed blocks (0xFFFF: overflow -> global path)
  int blk[8][TILE_THREADS];                   // block index (-1 absent)
  short tix[8][TILE_THREADS];                 // staged tile index (-1: read from global)
  unsigned long long c5[8][TILE_THREADS];
  float gap[15][TILE_THREADS];
  unsigned xy3[4][TILE_THREADS];
  unsigned z3[4][TILE_THREADS];
};

__device__ __forceinline__ unsigned smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ float4 tile_point(const MapDev& m, const TileSmem& sm, int tid, int b, int sl) {
  const int t = sm.tix[b][tid];
  if (t >= 0) return sm.tile[t][sl];
  return __ldg(&m.slots[(size_t)sm.blk[b][tid] * 64 + sl]);
}
__device__ __forceinline__ unsigned long long tile_inner_mask(const TileSmem& sm, int tid, int b) {
  const unsigned xy = sm.xy3[b & 3][tid];
  const int zq = (b >> 2) << 1;
  return ((unsigned long long)(xy & sm.z3[zq + 1][tid]) << 32) | (unsigned long long)(xy & sm.z3[zq][tid]);
}

// candidate ids inside the kernel: (b << 6) | slot for head points, 0x80000000 | node for overflow nodes
template <int K, bool OUTER>
__device__ __forceinline__ void tile_pass(const MapDev& m, const TileSmem& sm, int tid, float qx, float qy, float qz, float lim,
                                          TopKId<K>& t) {
  for (int b = 0; b < 8; ++b) {
    const unsigned long long in3 = tile_inner_mask(sm, tid, b);
    unsigned long long cand = sm.c5[b][tid] & (OUTER ? ~in3 : in3);
    while (cand != 0ull) {
      const int sl = __ffsll((long long)cand) - 1;
      cand &= cand - 1;
      const float4 p = tile_point(m, sm, tid, b, sl);
      const float dd = sqdist(qx, qy, qz, p.x, p.y, p.z);
      if (dd <= lim && dd < t.d[K - 1]) t.insert(dd, (unsigned)((b << 6) | sl));
      walk_chain(m, __float_as_int(p.w), [&](const float4 o, int c) {
        const float d2 = sqdist(qx, qy, qz, o.x, o.y, o.z);
        if (d2 <= lim && d2 < t.d[K - 1]) t.insert(d2, 0x80000000u | (unsigned)c);
      });
    }
  }
}

template <int K>
__global__ void __launch_bounds__(TILE_THREADS, 3) k_knn_tile(KnnArgs a) {
  extern __shared__ __align__(128) unsigned char tile_smem_raw[];
  TileSmem& sm = *reinterpret_cast<TileSmem*>(tile_smem_raw);
  const MapDev& m = a.m;
  const int tid = threadIdx.x;
  const int i = blockIdx.x * blockDim.x + tid;
  const int n = a.n;
  const float ds = m.ds;
  const float lim = a.max_d2;
  // ---- init: empty hash set, mbarrier (one arrival per thread)
  for (int s = tid; s < TILE_SLOTS; s += TILE_THREADS) { sm.keys[s] = KEY_EMPTY; sm.ttile[s] = -1; sm.tblk[s] = -1; sm.tmask[s] = 0ull; }
  if (tid == 0) {
    sm.ntile = 0;
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(&sm.mbar)), "r"(TILE_THREADS));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const bool valid = i < n;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  int cvx = 0, cvy = 0, cvz = 0, bbx = 0, bby = 0, bbz = 0;
  bool inrange = false;
  if (valid) {
    const float4 q4 = __ldg(&a.q[i]);
    qx = q4.x; qy = q4.y; qz = q4.z;
    const float qlim = 4.0e6f * ds;
    inrange = fabsf(qx) < qlim && fabsf(qy) < qlim && fabsf(qz) < qlim;
  }
  if (inrange) {
    cvx = voxel_of(qx, ds); cvy = voxel_of(qy, ds); cvz = voxel_of(qz, ds);
    bbx = (cvx - 2) >> 2; bby = (cvy - 2) >> 2; bbz = (cvz - 2) >> 2;
    // ---- A: the 8 block keys of this query go into the CTA's hash set
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const unsigned long long key = pack_key(bbx + (b & 1), bby + ((b >> 1) & 1), bbz + (b >> 2));
      unsigned h = hash_key(key) & (TILE_SLOTS - 1);
      unsigned short got = 0xFFFFu;
      for (int pr = 0; pr < TILE_PROBE; ++pr) {
        const unsigned long long old = atomicCAS(&sm.keys[h], (unsigned long long)KEY_EMPTY, key);
        if (old == KEY_EMPTY || old == key) { got = (unsigned short)h; break; }
        h = (h + 1) & (TILE_SLOTS - 1);
      }
      sm.slot[b][tid] = got;
    }
  }
  __syncthreads();
  // ---- B: one global probe per distinct block; its bucket is staged by a bulk copy counted on the mbarrier
  unsigned tx = 0u;
  for (int s = tid; s < TILE_SLOTS; s += TILE_THREADS) {
    const unsigned long long key = sm.keys[s];
    if (key == KEY_EMPTY) continue;
    unsigned long long mask;
    const int blk = find_block_mask(m, key, mask);
    sm.tblk[s] = blk;
    sm.tmask[s] = mask;
    if (blk >= 0 && mask != 0ull) {
      const int t = atomicAdd(&sm.ntile, 1);
      if (t < TILE_CAP) {
        sm.ttile[s] = (short)t;
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(&sm.tile[t][0])),
                     "l"(reinterpret_cast<const void*>(&m.slots[(size_t)blk * 64])), "r"(1024u), "r"(smem_addr(&sm.mbar))
                     : "memory");
        tx += 1024u;
      }
    }
  }
  if (tx) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(&sm.mbar)), "r"(tx) : "memory");
  else asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(&sm.mbar)) : "memory");
  __syncthreads();   // tblk / tmask / ttile visible
  TopKId<K> t;
  t.clear();
  bool done = !inrange;
  int ox = 0, oy = 0, oz = 0;
  float mg = 0.f;
  if (inrange) {
    mg = 1e-3f * ds + 4.8e-7f * (fabsf(qx) + fabsf(qy) + fabsf(qz));
    ox = (cvx - 2) & 3; oy = (cvy - 2) & 3; oz = (cvz - 2) & 3;
    const unsigned ax5 = 31u << ox, ay5 = 31u << oy, az5 = 31u << oz;
    const unsigned ix = 14u << ox, iy = 14u << oy, iz = 14u << oz;
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
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const unsigned short s = sm.slot[b][tid];
      int blk;
      unsigned long long occ;
      short tix = -1;
      if (s != 0xFFFFu) { blk = sm.tblk[s]; occ = sm.tmask[s]; tix = sm.ttile[s]; }
      else blk = find_block_mask(m, pack_key(bbx + (b & 1), bby + ((b >> 1) & 1), bbz + (b >> 2)), occ);   // set overflow
      sm.blk[b][tid] = blk;
      sm.tix[b][tid] = tix;
      sm.c5[b][tid] = (blk >= 0 ? occ : 0ull) & stencil_mask(ax5, ay5, az5, b);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      sm.xy3[q][tid] = xpat32((ix >> ((q & 1) << 2)) & 15u) & ypat32((iy >> ((q >> 1) << 2)) & 15u);
      sm.z3[q][tid] = zpat32((((iz >> ((q >> 1) << 2)) & 15u) >> ((q & 1) << 1)) & 3u);
    }
  }
  // ---- C: wait for the staged buckets (phase 0 of the mbarrier)
  {
    unsigned ok = 0u;
    while (!ok) {
      asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(smem_addr(&sm.mbar)), "r"(0u) : "memory");
    }
  }
  if (inrange) {
    // ---- D: the stencil search out of shared memory: inner 3x3x3, then the shell cut down by the k-th distance
    tile_pass<K, false>(m, sm, tid, qx, qy, qz, lim, t);
    const float bound = t.d[K - 1];
    if (bound < CUDART_INF_F) {
      unsigned wx = 0u, wy = 0u, wz = 0u;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        wx |= (sm.gap[j][tid] <= bound) ? (1u << j) : 0u;
        wy |= (sm.gap[5 + j][tid] <= bound) ? (1u << j) : 0u;
        wz |= (sm.gap[10 + j][tid] <= bound) ? (1u << j) : 0u;
      }
      const unsigned ax = wx << ox, ay = wy << oy, az = wz << oz;
      for (int b = 0; b < 8; ++b) {
        unsigned long long cand = sm.c5[b][tid] & stencil_mask(ax, ay, az, b);
        if (cand == 0ull) continue;
        cand &= ~tile_inner_mask(sm, tid, b);
        while (cand != 0ull) {
          const int sl = __ffsll((long long)cand) - 1;
          cand &= cand - 1;
          const int jx = ((b & 1) << 2) + (sl & 3) - ox, jy = (((b >> 1) & 1) << 2) + ((sl >> 2) & 3) - oy, jz = ((b >> 2) << 2) + (sl >> 4) - oz;
          const float md = sm.gap[jx][tid] + sm.gap[5 + jy][tid] + sm.gap[10 + jz][tid];
          if (md > t.d[K - 1]) continue;
          const float4 p = tile_point(m, sm, tid, b, sl);
          const float dd = sqdist(qx, qy, qz, p.x, p.y, p.z);
          if (dd <= lim && dd < t.d[K - 1]) t.insert(dd, (unsigned)((b << 6) | sl));
          walk_chain(m, __float_as_int(p.w), [&](const float4 o, int c) {
            const float d2 = sqdist(qx, qy, qz, o.x, o.y, o.z);
            if (d2 <= lim && d2 < t.d[K - 1]) t.insert(d2, 0x80000000u | (unsigned)c);
          });
        }
      }
    } else {
      tile_pass<K, true>(m, sm, tid, qx, qy, qz, lim, t);
    }
    const float cov = cover2(qx, qy, qz, (float)(cvx - 2) * ds, (float)(cvy - 2) * ds, (float)(cvz - 2) * ds,
                             (float)(cvx + 3) * ds, (float)(cvy + 3) * ds, (float)(cvz + 3) * ds, mg);
    done = (t.d[K - 1] < CUDART_INF_F && t.d[K - 1] < cov) || cov > lim;
  }
  if (!valid) return;
  int c = 0;
#pragma unroll
  for (int r = 0; r < K; ++r) {
    const bool ok = t.d[r] < CUDART_INF_F;
    c += ok ? 1 : 0;
    float4 o = make_float4(CUDART_NAN_F, CUDART_NAN_F, CUDART_NAN_F, CUDART_INF_F);
    if (ok) {
      const float4 e = (t.id[r] & 0x80000000u) ? __ldg(&m.ovf[t.id[r] & 0x7FFFFFFFu]) : tile_point(m, sm, tid, (int)(t.id[r] >> 6), (int)(t.id[r] & 63u));
      o = make_float4(e.x, e.y, e.z, t.d[r]);
    }
    a.nbr[(size_t)r * a.stride + i] = o;
  }
  a.cnt[i] = (unsigned char)c;
  if (!done) st_release(&a.worklist[atomicAdd(a.work_count, 1)], i);   // (published as k_knn_stencil does)
}

}  // namespace flb

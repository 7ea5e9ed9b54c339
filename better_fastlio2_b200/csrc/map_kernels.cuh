// map_kernels.cuh — map maintenance kernels (K3 insert/downsample, K4 box delete, K5 build, K6 flatten) for the
// hashed voxel map of voxel_map.cuh.  They reproduce the FINAL state of the reference's strictly sequential
// KD_TREE::Add_Points / Delete_Point_Boxes (include/ikd-Tree/ikd_Tree.cpp:413-489, :535-556) with parallel atomics.
// Bounded by HBM (≈40 B per inserted point: 16 read + 16 write + 8 hash-slot RMW); no tensor-core work.
#pragma once
#include "voxel_map.cuh"

namespace flb {

// ---------------------------------------------------------------------------------------------- allocators
// Pops and pushes of one free stack never happen in the same kernel (insert kernels pop, delete/downsample kernels
// push), so plain atomic counters suffice.
__device__ __forceinline__ int alloc_block(const MapDev& m) {
  int f = atomicSub(&m.counters[CNT_BLK_FREE], 1);
  if (f > 0) return (int)m.free_blk[f - 1];
  atomicAdd(&m.counters[CNT_BLK_FREE], 1);
  int b = atomicAdd(&m.counters[CNT_BLK_BUMP], 1);
  if (b >= m.block_cap) {
    atomicOr(&m.counters[CNT_ERROR], ERR_BLOCKS_FULL);
    return -1;
  }
  return b;
}
__device__ __forceinline__ int alloc_ovf(const MapDev& m) {
  int f = atomicSub(&m.counters[CNT_OVF_FREE], 1);
  if (f > 0) return (int)m.free_ovf[f - 1];
  atomicAdd(&m.counters[CNT_OVF_FREE], 1);
  int b = atomicAdd(&m.counters[CNT_OVF_BUMP], 1);
  if (b >= m.ovf_cap) {
    atomicOr(&m.counters[CNT_ERROR], ERR_OVF_FULL);
    return -1;
  }
  return b;
}
__device__ __forceinline__ void free_ovf_node(const MapDev& m, int node) {
  int t = atomicAdd(&m.counters[CNT_OVF_FREE], 1);
  m.free_ovf[t] = (uint32_t)node;
}
__device__ __forceinline__ void free_block_idx(const MapDev& m, int blk) {
  int t = atomicAdd(&m.counters[CNT_BLK_FREE], 1);
  m.free_blk[t] = (uint32_t)blk;
}

__device__ __forceinline__ bool coord_ok(float x, float y, float z, float ds) {
  const float lim = 4.0e6f * ds;  // |voxel| < 2^22  => |block| < 2^20
  return fabsf(x) < lim && fabsf(y) < lim && fabsf(z) < lim;  // also false for NaN
}

// Register block (bx,by,bz) in the coarse level (bitmap + bbox).
__device__ __forceinline__ void coarse_set(const MapDev& m, int bx, int by, int bz) {
  const int cx = bx >> 3, cy = by >> 3, cz = bz >> 3;
  const uint64_t ck = pack_key(cx, cy, cz);
  uint32_t s = hash_key(ck) & m.chash_mask;
  int slot = -1;
  for (uint32_t probe = 0; probe <= m.chash_mask; ++probe) {
    uint64_t k = *((volatile uint64_t*)&m.ckeys[s]);
    if (k == ck) { slot = (int)s; break; }
    if (k == KEY_EMPTY) {
      uint64_t old = atomicCAS((unsigned long long*)&m.ckeys[s], (unsigned long long)KEY_EMPTY, (unsigned long long)ck);
      if (old == KEY_EMPTY) {
        m.clist[atomicAdd(&m.counters[CNT_COARSE_USED], 1)] = s;
        atomicMin(&m.counters[CNT_CMIN_X], cx); atomicMin(&m.counters[CNT_CMIN_Y], cy); atomicMin(&m.counters[CNT_CMIN_Z], cz);
        atomicMax(&m.counters[CNT_CMAX_X], cx); atomicMax(&m.counters[CNT_CMAX_Y], cy); atomicMax(&m.counters[CNT_CMAX_Z], cz);
        slot = (int)s;
        break;
      }
      if (old == ck) { slot = (int)s; break; }
    }
    s = (s + 1) & m.chash_mask;
  }
  if (slot < 0) { atomicOr(&m.counters[CNT_ERROR], ERR_COARSE_FULL); return; }
  const int bit = (((bz & 7) << 3) + (by & 7)) * 8 + (bx & 7);
  atomicOr((unsigned long long*)&m.cbits[(size_t)slot * 8 + (bit >> 6)], 1ull << (bit & 63));
}
__device__ __forceinline__ void coarse_clear(const MapDev& m, int bx, int by, int bz) {
  const uint64_t ck = pack_key(bx >> 3, by >> 3, bz >> 3);
  uint32_t s = hash_key(ck) & m.chash_mask;
  for (uint32_t probe = 0; probe <= m.chash_mask; ++probe) {
    uint64_t k = *((volatile uint64_t*)&m.ckeys[s]);
    if (k == ck) {
      const int bit = (((bz & 7) << 3) + (by & 7)) * 8 + (bx & 7);
      atomicAnd((unsigned long long*)&m.cbits[(size_t)s * 8 + (bit >> 6)], ~(1ull << (bit & 63)));
      return;
    }
    if (k == KEY_EMPTY) return;
    s = (s + 1) & m.chash_mask;
  }
}

// Find-or-create the hash entry of a block key. Only ensures existence (vals[] is read by LATER kernels).
__device__ __forceinline__ void touch_block(const MapDev& m, uint64_t key, int bx, int by, int bz) {
  uint32_t s = hash_key(key) & m.hash_mask;
  for (uint32_t probe = 0; probe <= m.hash_mask; ++probe) {
    uint64_t k = *((volatile uint64_t*)&m.hent[s].key);
    if (k == key) return;
    if (k == KEY_EMPTY) {
      uint64_t old = atomicCAS((unsigned long long*)&m.hent[s].key, (unsigned long long)KEY_EMPTY, (unsigned long long)key);
      if (old == KEY_EMPTY) {
        int blk = alloc_block(m);
        m.hent[s].val = (uint32_t)blk;  // -1 on exhaustion (sticky error already raised)
        if (blk >= 0) {
          m.bkey[blk] = key;
          m.bslot[blk] = s;               // (entry mask is 0: cleared at reset / release)
          coarse_set(m, bx, by, bz);
        }
        atomicAdd(&m.counters[CNT_KEYS_USED], 1);
        return;
      }
      if (old == key) return;
    }
    s = (s + 1) & m.hash_mask;
  }
  atomicOr(&m.counters[CNT_ERROR], ERR_HASH_FULL);
}

// ---------------------------------------------------------------------------------------------- K3a: touch blocks
// cls == nullptr: every point; else only points whose class has its bit in cls_mask (bit1: ToAdd, bit2: NoNeed).
__global__ void k_touch_blocks(MapDev m, const float4* __restrict__ pts, const unsigned char* __restrict__ cls,
                               int cls_mask, int n, const int* __restrict__ skip, const int* __restrict__ n_dev) {
  pdl_sync();
  FLB_TRACE_BEGIN(7 * 8);
  if (skip && *skip) return;
  if (n_dev) n = *n_dev;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (cls && !((1 << cls[i]) & cls_mask)) continue;
    const float4 p = pts[i];
    if (!coord_ok(p.x, p.y, p.z, m.ds)) { atomicOr(&m.counters[CNT_ERROR], ERR_RANGE); continue; }
    const int bx = voxel_of(p.x, m.ds) >> 2, by = voxel_of(p.y, m.ds) >> 2, bz = voxel_of(p.z, m.ds) >> 2;
    touch_block(m, pack_key(bx, by, bz), bx, by, bz);
  }
  FLB_TRACE_END(7 * 8);
}

// ---------------------------------------------------------------------------------------------- K3b: verbatim append
// Add_Points(..., downsample_on=false) (ikd_Tree.cpp:471-472) and Build (ikd_Tree.cpp:352-364): no dedupe.
// Optional epilogue of the LAST kernel of a captured scan sequence: the block that finishes last copies the map counters,
// map_incremental's two counts and the sequence's device span into the (mapped pinned) result record, so that no separate
// publishing kernel — one more launch gap on the critical path between two scans — follows the insert.
struct StepTail {
  int* ticket = nullptr;                         // zero before the launch; the last block leaves it zero again
  const int* counters = nullptr;                 // [32] map counters
  const int* cnt2 = nullptr;                     // [2] map_incremental's counts
  const unsigned long long* t_begin = nullptr;   // %globaltimer at the start of the sequence
  int* out_counters = nullptr;
  int* out_cnt2 = nullptr;
  unsigned long long* out_span = nullptr;
};

__global__ void k_append_points(MapDev m, const float4* __restrict__ pts, const unsigned char* __restrict__ cls,
                                int want_cls, int n, const int* __restrict__ skip, const int* __restrict__ n_dev, StepTail tail) {
  pdl_sync();
  FLB_TRACE_BEGIN(10 * 8);
  const bool skipped = skip && *skip;
  if (n_dev) n = *n_dev;
  if (skipped) n = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (cls && cls[i] != want_cls) continue;
    const float4 p = pts[i];
    if (!coord_ok(p.x, p.y, p.z, m.ds)) continue;
    const int vx = voxel_of(p.x, m.ds), vy = voxel_of(p.y, m.ds), vz = voxel_of(p.z, m.ds);
    const int hs = find_slot(m, pack_key(vx >> 2, vy >> 2, vz >> 2));
    const int blk = hs >= 0 ? (int)m.hent[hs].val : -1;
    if (blk < 0) continue;  // capacity error already flagged
    const int s = (((vz & 3) << 2) + (vy & 3)) * 4 + (vx & 3);
    const unsigned long long bit = 1ull << s;
    const size_t idx = (size_t)blk * 64 + s;
    const unsigned long long old = atomicOr((unsigned long long*)&m.hent[hs].mask, bit);
    if (!(old & bit)) {
      // owner of the head slot: write xyz only — w (= -1 by invariant) may concurrently receive a chain push
      float* f = reinterpret_cast<float*>(&m.slots[idx]);
      f[0] = p.x; f[1] = p.y; f[2] = p.z;
      m.sint[idx] = p.w;
    } else {
      const int node = alloc_ovf(m);
      if (node < 0) continue;
      const int prev = atomicExch(reinterpret_cast<int*>(&m.slots[idx]) + 3, node);
      m.ovf[node] = make_float4(p.x, p.y, p.z, __int_as_float(prev));
      m.oint[node] = p.w;
    }
    atomicAdd(&m.counters[CNT_VALID], 1);
  }
  FLB_TRACE_END(10 * 8);
  if (tail.ticket) {
    __shared__ int s_last;
    __syncthreads();                       // every counter update of this block has been issued
    if (threadIdx.x == 0) {
      __threadfence();
      s_last = atomicAdd(tail.ticket, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {                          // block-uniform
      __threadfence();
      if (threadIdx.x < 32) tail.out_counters[threadIdx.x] = __ldcg(&tail.counters[threadIdx.x]);
      else if (threadIdx.x < 34) tail.out_cnt2[threadIdx.x - 32] = __ldcg(&tail.cnt2[threadIdx.x - 32]);
      else if (threadIdx.x == 34) *tail.out_span = global_timer_ns() - __ldcg(tail.t_begin);
      else if (threadIdx.x == 35) *tail.ticket = 0;
    }
  }
}

// ---------------------------------------------------------------------------------------------- K3b': chain relocation
// After a verbatim insert: every voxel that received one of these points and now has >= 2 overflow nodes gets its chain
// copied into a fresh CONTIGUOUS run of ovf[] (bump allocation; next == this + 1), the old nodes go back to the free
// stack.  Pure layout optimisation — the chain stays a valid linked list for every reader — so that the k-NN kernels
// can fetch four nodes per round trip (walk_chain) instead of chasing one pointer per DRAM latency.  One thread per
// inserted point; the first to set the voxel's bit in the scratch bitmap brel owns the voxel and clears the bit again.
// Only bump allocation and free-stack pushes happen here (no pops), as the allocator contract requires.
__global__ void k_relocate_chains(MapDev m, const float4* __restrict__ pts, const unsigned char* __restrict__ cls, int want_cls,
                                  int n, const int* __restrict__ skip, const int* __restrict__ n_dev) {
  pdl_sync();
  FLB_TRACE_BEGIN(11 * 8);
  if (skip && *skip) return;
  if (n_dev) n = *n_dev;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (cls && cls[i] != want_cls) continue;
    const float4 p = pts[i];
    if (!coord_ok(p.x, p.y, p.z, m.ds)) continue;
    const int vx = voxel_of(p.x, m.ds), vy = voxel_of(p.y, m.ds), vz = voxel_of(p.z, m.ds);
    const int blk = find_block(m, pack_key(vx >> 2, vy >> 2, vz >> 2));
    if (blk < 0) continue;
    const int s = (((vz & 3) << 2) + (vy & 3)) * 4 + (vx & 3);
    const unsigned long long bit = 1ull << s;
    if (atomicOr((unsigned long long*)&m.brel[blk], bit) & bit) continue;   // another point of this batch owns the voxel
    const size_t idx = (size_t)blk * 64 + s;
    // L2-coherent loads (__ldcg): a previous owner of this voxel in this same kernel may have just re-laid the chain
    const int first = __float_as_int(__ldcg(&m.slots[idx]).w);
    int L = 0;
    bool contiguous = true;
    for (int c = first; c >= 0;) {
      const int nx = __float_as_int(__ldcg(&m.ovf[c]).w);
      if (nx >= 0 && nx != c + 1) contiguous = false;
      ++L;
      c = nx;
    }
    if (L >= 2 && !contiguous) {
      const int base = atomicAdd(&m.counters[CNT_OVF_BUMP], L);
      if (base + L <= m.ovf_cap) {
        int c = first;
        for (int j = 0; j < L; ++j) {
          const float4 e = __ldcg(&m.ovf[c]);
          m.ovf[base + j] = make_float4(e.x, e.y, e.z, __int_as_float(j + 1 < L ? base + j + 1 : -1));
          m.oint[base + j] = __ldcg(&m.oint[c]);
          free_ovf_node(m, c);
          c = __float_as_int(e.w);
        }
        reinterpret_cast<int*>(&m.slots[idx])[3] = base;
      } else {
        atomicSub(&m.counters[CNT_OVF_BUMP], L);   // no room for a run: keep the scattered chain (still correct)
      }
    }
    __threadfence();   // the new layout is visible before the voxel can be owned again
    atomicAnd((unsigned long long*)&m.brel[blk], ~bit);
  }
  FLB_TRACE_END(11 * 8);
}

// ---------------------------------------------------------------------------------------------- K3c/d: downsampled insert
// Voxel box and centre exactly as ikd_Tree.cpp:424-432: float floor/mul/add, centre = min + (max-min)/2.0 in double.
__device__ __forceinline__ float dist_to_voxel_centre(const float4 p, float ds) {
  const float bx0 = __fmul_rn(floorf(__fdiv_rn(p.x, ds)), ds), bx1 = __fadd_rn(bx0, ds);
  const float by0 = __fmul_rn(floorf(__fdiv_rn(p.y, ds)), ds), by1 = __fadd_rn(by0, ds);
  const float bz0 = __fmul_rn(floorf(__fdiv_rn(p.z, ds)), ds), bz1 = __fadd_rn(bz0, ds);
  const float mx = (float)__dadd_rn((double)bx0, __ddiv_rn((double)__fsub_rn(bx1, bx0), 2.0));
  const float my = (float)__dadd_rn((double)by0, __ddiv_rn((double)__fsub_rn(by1, by0), 2.0));
  const float mz = (float)__dadd_rn((double)bz0, __ddiv_rn((double)__fsub_rn(bz1, bz0), 2.0));
  const float dx = __fsub_rn(p.x, mx), dy = __fsub_rn(p.y, my), dz = __fsub_rn(p.z, mz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));  // calc_dist :1373-1378
}
__device__ __forceinline__ float dist_pt_to_centre_of(const float4 e, const float4 p, float ds) {
  // distance of an existing point e to the centre of p's voxel box
  const float bx0 = __fmul_rn(floorf(__fdiv_rn(p.x, ds)), ds), bx1 = __fadd_rn(bx0, ds);
  const float by0 = __fmul_rn(floorf(__fdiv_rn(p.y, ds)), ds), by1 = __fadd_rn(by0, ds);
  const float bz0 = __fmul_rn(floorf(__fdiv_rn(p.z, ds)), ds), bz1 = __fadd_rn(bz0, ds);
  const float mx = (float)__dadd_rn((double)bx0, __ddiv_rn((double)__fsub_rn(bx1, bx0), 2.0));
  const float my = (float)__dadd_rn((double)by0, __ddiv_rn((double)__fsub_rn(by1, by0), 2.0));
  const float mz = (float)__dadd_rn((double)bz0, __ddiv_rn((double)__fsub_rn(bz1, bz0), 2.0));
  const float dx = __fsub_rn(e.x, mx), dy = __fsub_rn(e.y, my), dz = __fsub_rn(e.z, mz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// Scratch hash: per voxel touched by this batch, the best NEW point = min (dist to centre, later index wins ties —
// the reference processes points in order and a later point replaces an equal-distance earlier one, :436-447).
__device__ __forceinline__ void ds_scatter_one(const MapDev& m, const float4 p, int i, uint64_t vkey, uint64_t* skeys,
                                               unsigned long long* sbest, uint32_t smask) {
  const float d = dist_to_voxel_centre(p, m.ds);
  const unsigned long long pk = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)i);
  uint32_t s = hash_key(vkey) & smask;
  for (uint32_t probe = 0; probe <= smask; ++probe) {
    uint64_t k = *((volatile uint64_t*)&skeys[s]);
    if (k == KEY_EMPTY) {
      uint64_t old = atomicCAS((unsigned long long*)&skeys[s], (unsigned long long)KEY_EMPTY, (unsigned long long)vkey);
      if (old == KEY_EMPTY || old == vkey) k = vkey;
    }
    if (k == vkey) { atomicMin(&sbest[s], pk); break; }
    s = (s + 1) & smask;
  }
}
__global__ void k_ds_scatter(MapDev m, const float4* __restrict__ pts, const unsigned char* __restrict__ cls, int n,
                             uint64_t* skeys, unsigned long long* sbest, uint32_t smask, const int* __restrict__ skip,
                             const int* __restrict__ n_dev) {
  pdl_sync();
  FLB_TRACE_BEGIN(8 * 8);
  if (skip && *skip) return;
  if (n_dev) n = *n_dev;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (cls && cls[i] != 1) continue;
    const float4 p = pts[i];
    if (!coord_ok(p.x, p.y, p.z, m.ds)) continue;
    ds_scatter_one(m, p, i, pack_key(voxel_of(p.x, m.ds), voxel_of(p.y, m.ds), voxel_of(p.z, m.ds)), skeys, sbest, smask);
  }
  FLB_TRACE_END(8 * 8);
}

// The winning new point of each touched voxel applies the reference's rule against the existing content E of the
// voxel (ikd_Tree.cpp:433-449): result = argmin dist-to-centre over {new} ∪ E (existing must be STRICTLY closer to
// win); if |E| > 1 or the new point is the result (same_point): E is deleted and the result inserted.
// E is taken as the points keyed to this voxel (floor(x/ds)); the reference's float box test min<=p<max can
// disagree with that within 1 ulp of a voxel face (documented deviation, DESIGN.md).
__global__ void k_ds_apply(MapDev m, const float4* __restrict__ pts, const unsigned char* __restrict__ cls, int n,
                           const uint64_t* __restrict__ skeys, const unsigned long long* __restrict__ sbest,
                           uint32_t smask, const int* __restrict__ skip, const int* __restrict__ n_dev) {
  pdl_sync();
  FLB_TRACE_BEGIN(9 * 8);
  if (skip && *skip) return;
  if (n_dev) n = *n_dev;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (cls && cls[i] != 1) continue;
    const float4 p = pts[i];
    if (!coord_ok(p.x, p.y, p.z, m.ds)) continue;
    const int vx = voxel_of(p.x, m.ds), vy = voxel_of(p.y, m.ds), vz = voxel_of(p.z, m.ds);
    const uint64_t vkey = pack_key(vx, vy, vz);
    const float d = dist_to_voxel_centre(p, m.ds);
    const unsigned long long pk = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)i);
    uint32_t s = hash_key(vkey) & smask;
    bool mine = false;
    for (uint32_t probe = 0; probe <= smask; ++probe) {
      const uint64_t k = skeys[s];
      if (k == vkey) { mine = (sbest[s] == pk); break; }
      if (k == KEY_EMPTY) break;
      s = (s + 1) & smask;
    }
    if (!mine) continue;
    const int hs = find_slot(m, pack_key(vx >> 2, vy >> 2, vz >> 2));
    const int blk = hs >= 0 ? (int)m.hent[hs].val : -1;
    if (blk < 0) continue;
    const int sl = (((vz & 3) << 2) + (vy & 3)) * 4 + (vx & 3);
    const unsigned long long bit = 1ull << sl;
    const size_t idx = (size_t)blk * 64 + sl;
    const unsigned long long mask = *reinterpret_cast<volatile unsigned long long*>(&m.hent[hs].mask);
    if (!(mask & bit)) {
      float* f = reinterpret_cast<float*>(&m.slots[idx]);
      f[0] = p.x; f[1] = p.y; f[2] = p.z;  // w stays -1
      m.sint[idx] = p.w;
      atomicOr((unsigned long long*)&m.hent[hs].mask, bit);
      atomicAdd(&m.counters[CNT_VALID], 1);
      atomicAdd(&m.counters[CNT_SCRATCH0], 1);
      continue;
    }
    // walk the chain: count E, best existing (strictly closer than the new point), free overflow nodes on collapse
    float4 head = m.slots[idx];
    int L = 1;
    float bestd = d;
    float4 best = p;
    float besti = p.w;
    bool new_wins = true;
    {
      float de = dist_pt_to_centre_of(head, p, m.ds);
      if (de < bestd) { bestd = de; best = head; besti = m.sint[idx]; new_wins = false; }
    }
    for (int c = __float_as_int(head.w); c >= 0;) {
      const float4 e = m.ovf[c];
      float de = dist_pt_to_centre_of(e, p, m.ds);
      if (de < bestd) { bestd = de; best = e; besti = m.oint[c]; new_wins = false; }
      ++L;
      c = __float_as_int(e.w);
    }
    const bool same = new_wins || (fabsf(p.x - best.x) < 1e-6f && fabsf(p.y - best.y) < 1e-6f && fabsf(p.z - best.z) < 1e-6f);
    if (L > 1 || same) {
      for (int c = __float_as_int(head.w); c >= 0;) {
        const int nx = __float_as_int(m.ovf[c].w);
        free_ovf_node(m, c);
        c = nx;
      }
      m.slots[idx] = make_float4(best.x, best.y, best.z, __int_as_float(-1));
      m.sint[idx] = besti;
      if (L != 1) atomicAdd(&m.counters[CNT_VALID], 1 - L);
      atomicAdd(&m.counters[CNT_SCRATCH0], 1);
    }
  }
  FLB_TRACE_END(9 * 8);
}

// ---------------------------------------------------------------------------------------------- block iteration helpers
__device__ __forceinline__ bool in_box(const float4 p, const float* b) {  // ikd_Tree.cpp:670 half-open
  return p.x >= b[0] && p.x < b[3] && p.y >= b[1] && p.y < b[4] && p.z >= b[2] && p.z < b[5];
}

// Remove the block from the hash (tombstone), the coarse bitmap and return it to the free stack.
__device__ __forceinline__ void release_block(const MapDev& m, int blk, uint64_t key) {
  uint32_t s = hash_key(key) & m.hash_mask;
  for (uint32_t probe = 0; probe <= m.hash_mask; ++probe) {
    uint64_t k = *((volatile uint64_t*)&m.hent[s].key);
    if (k == key) { m.hent[s].mask = 0ull; m.hent[s].key = KEY_TOMB; break; }
    if (k == KEY_EMPTY) break;
    s = (s + 1) & m.hash_mask;
  }
  int bx, by, bz;
  unpack_key(key, bx, by, bz);
  coarse_clear(m, bx, by, bz);
  m.bkey[blk] = KEY_EMPTY;
  free_block_idx(m, blk);
  atomicSub(&m.counters[CNT_KEYS_USED], 1);
  atomicAdd(&m.counters[CNT_KEYS_TOMB], 1);
}

// ---------------------------------------------------------------------------------------------- K4: delete
// mode 0: Delete_Point_Boxes (ikd_Tree.cpp:535-556): params = nb boxes x 6 floats.
// mode 1: Delete_Points (ikd_Tree.cpp:513-533): params = np points x 4 floats, match = same_point (1e-6 per axis).
// One warp per allocated block; lane l owns voxels l and l+32 (single writer per chain).
__global__ void k_delete(MapDev m, const float* __restrict__ params, int np, int mode, int nblk) {
  const int lane = threadIdx.x & 31;
  const int warps_per_grid = (gridDim.x * blockDim.x) >> 5;
  for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < nblk; b += warps_per_grid) {
    const uint64_t key = m.bkey[b];
    if (key == KEY_EMPTY) continue;
    int bx, by, bz;
    unpack_key(key, bx, by, bz);
    const float ds = m.ds;
    const float mg = 1e-3f * ds + 1e-6f * (fabsf((float)bx) + fabsf((float)by) + fabsf((float)bz)) * 4.f * ds;
    const float lo[3] = {(float)(bx * 4) * ds - mg, (float)(by * 4) * ds - mg, (float)(bz * 4) * ds - mg};
    const float hi[3] = {(float)(bx * 4 + 4) * ds + mg, (float)(by * 4 + 4) * ds + mg, (float)(bz * 4 + 4) * ds + mg};
    bool touch = false;
    for (int k = 0; k < np && !touch; ++k) {
      if (mode == 0) {
        const float* bb = params + 6 * k;
        touch = !(bb[3] <= lo[0] || bb[0] > hi[0] || bb[4] <= lo[1] || bb[1] > hi[1] || bb[5] <= lo[2] || bb[2] > hi[2]);
      } else {
        const float* pp = params + 4 * k;
        touch = pp[0] >= lo[0] && pp[0] <= hi[0] && pp[1] >= lo[1] && pp[1] <= hi[1] && pp[2] >= lo[2] && pp[2] <= hi[2];
      }
    }
    if (!touch) continue;  // warp-uniform
    const unsigned long long mask = *block_mask_ptr(m, b);
    unsigned long long clear = 0ull;
    int ndel = 0;
    for (int h = 0; h < 2; ++h) {
      const int s = lane + 32 * h;
      if (!((mask >> s) & 1ull)) continue;
      const size_t idx = (size_t)b * 64 + s;
      auto hit = [&](const float4 q) -> bool {
        for (int k = 0; k < np; ++k) {
          if (mode == 0) { if (in_box(q, params + 6 * k)) return true; }
          else {
            const float* pp = params + 4 * k;
            if (fabsf(q.x - pp[0]) < 1e-6f && fabsf(q.y - pp[1]) < 1e-6f && fabsf(q.z - pp[2]) < 1e-6f) return true;
          }
        }
        return false;
      };
      // overflow chain first
      int* link = reinterpret_cast<int*>(&m.slots[idx]) + 3;
      int cur = *link;
      while (cur >= 0) {
        const float4 e = m.ovf[cur];
        const int nx = __float_as_int(e.w);
        if (hit(e)) { *link = nx; free_ovf_node(m, cur); ++ndel; }
        else link = reinterpret_cast<int*>(&m.ovf[cur]) + 3;
        cur = nx;
      }
      const float4 head = m.slots[idx];
      if (hit(head)) {
        ++ndel;
        const int c = __float_as_int(head.w);
        if (c >= 0) { m.slots[idx] = m.ovf[c]; m.sint[idx] = m.oint[c]; free_ovf_node(m, c); }
        else clear |= 1ull << s;  // w already -1
      }
    }
    for (int o = 16; o; o >>= 1) {
      clear |= __shfl_xor_sync(0xffffffffu, clear, o);
      ndel += __shfl_xor_sync(0xffffffffu, ndel, o);
    }
    if (lane == 0 && ndel) {
      atomicAdd(&m.counters[CNT_SCRATCH0], ndel);
      atomicSub(&m.counters[CNT_VALID], ndel);
      const unsigned long long nm = mask & ~clear;
      *block_mask_ptr(m, b) = nm;
      if (nm == 0ull) release_block(m, b, key);
    }
  }
}

// ---------------------------------------------------------------------------------------------- K6: flatten / searches
// mode 0: all points (flatten, ikd_Tree.cpp:1325-1352); mode 1: half-open box (Box_Search :399-404);
// mode 2: within radius, float calc_dist <= r*r (Radius_Search :406-411, :1065).  Appends to out (cap) and counts.
__global__ void k_collect(MapDev m, int nblk, int mode, const float* __restrict__ params, float4* out, int cap,
                          int* out_count) {
  const int lane = threadIdx.x & 31;
  const int warps_per_grid = (gridDim.x * blockDim.x) >> 5;
  for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < nblk; b += warps_per_grid) {
    if (m.bkey[b] == KEY_EMPTY) continue;
    const unsigned long long mask = *block_mask_ptr(m, b);
    auto pass = [&](const float4 q) -> bool {
      if (mode == 0) return true;
      if (mode == 1) return in_box(q, params);
      const float dx = q.x - params[0], dy = q.y - params[1], dz = q.z - params[2];
      return (dx * dx + dy * dy + dz * dz) <= params[3] * params[3];
    };
    int cnt = 0;
    for (int h = 0; h < 2; ++h) {
      const int s = lane + 32 * h;
      if (!((mask >> s) & 1ull)) continue;
      float4 e = m.slots[(size_t)b * 64 + s];
      for (;;) {
        if (pass(e)) ++cnt;
        const int c = __float_as_int(e.w);
        if (c < 0) break;
        e = m.ovf[c];
      }
    }
    int pre = cnt;
    for (int o = 1; o < 32; o <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, pre, o);
      if (lane >= o) pre += v;
    }
    const int total = __shfl_sync(0xffffffffu, pre, 31);
    if (total == 0) continue;
    int base = 0;
    if (lane == 0) base = atomicAdd(out_count, total);
    base = __shfl_sync(0xffffffffu, base, 0);
    int w = base + pre - cnt;
    for (int h = 0; h < 2; ++h) {
      const int s = lane + 32 * h;
      if (!((mask >> s) & 1ull)) continue;
      float4 e = m.slots[(size_t)b * 64 + s];
      float inten = m.sint[(size_t)b * 64 + s];
      for (;;) {
        if (pass(e)) {
          if (out && w < cap) out[w] = make_float4(e.x, e.y, e.z, inten);
          ++w;
        }
        const int c = __float_as_int(e.w);
        if (c < 0) break;
        e = m.ovf[c];
        inten = m.oint[c];
      }
    }
  }
}

// tree_range: min/max of valid points via float-ordered int atomics on a 6-int scratch.
__device__ __forceinline__ int f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7FFFFFFF; }
__global__ void k_range(MapDev m, int nblk, int* box6ord) {
  const int lane = threadIdx.x & 31;
  const int warps_per_grid = (gridDim.x * blockDim.x) >> 5;
  for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < nblk; b += warps_per_grid) {
    if (m.bkey[b] == KEY_EMPTY) continue;
    const unsigned long long mask = *block_mask_ptr(m, b);
    for (int h = 0; h < 2; ++h) {
      const int s = lane + 32 * h;
      if (!((mask >> s) & 1ull)) continue;
      float4 e = m.slots[(size_t)b * 64 + s];
      for (;;) {
        atomicMin(&box6ord[0], f2ord(e.x)); atomicMin(&box6ord[1], f2ord(e.y)); atomicMin(&box6ord[2], f2ord(e.z));
        atomicMax(&box6ord[3], f2ord(e.x)); atomicMax(&box6ord[4], f2ord(e.y)); atomicMax(&box6ord[5], f2ord(e.z));
        const int c = __float_as_int(e.w);
        if (c < 0) break;
        e = m.ovf[c];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- hash table (re)initialisation
__global__ void k_hent_clear(HEntry* hent, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    HEntry e;
    e.key = KEY_EMPTY; e.val = 0xFFFFFFFFu; e.pad = 0u; e.mask = 0ull; e.pad2 = 0ull;
    hent[i] = e;
  }
}
// rehash (drop tombstones), step 1: park every live block's occupancy word in the per-block scratch brel
__global__ void k_rehash_save(MapDev m, int nblk) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nblk; b += gridDim.x * blockDim.x)
    if (m.bkey[b] != KEY_EMPTY) m.brel[b] = m.hent[m.bslot[b]].mask;
}
// step 2 (after k_hent_clear): re-insert the keys with their occupancy words; brel goes back to all-zero
__global__ void k_rehash_insert(MapDev m, int nblk) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nblk; b += gridDim.x * blockDim.x) {
    const uint64_t key = m.bkey[b];
    if (key == KEY_EMPTY) continue;
    uint32_t s = hash_key(key) & m.hash_mask;
    for (uint32_t probe = 0; probe <= m.hash_mask; ++probe) {
      uint64_t old = atomicCAS((unsigned long long*)&m.hent[s].key, (unsigned long long)KEY_EMPTY, (unsigned long long)key);
      if (old == KEY_EMPTY) { m.hent[s].val = (uint32_t)b; m.hent[s].mask = m.brel[b]; m.bslot[b] = s; m.brel[b] = 0ull; break; }
      s = (s + 1) & m.hash_mask;
    }
  }
}
// coarse level rebuild (after its tables were cleared; also the last step of a rehash): every allocated block registers its
// cell again, so cells that deletes emptied leave ckeys and clist
__global__ void k_coarse_rebuild(MapDev m, int nblk) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nblk; b += gridDim.x * blockDim.x) {
    const uint64_t key = m.bkey[b];
    if (key == KEY_EMPTY) continue;
    int bx, by, bz;
    unpack_key(key, bx, by, bz);
    coarse_set(m, bx, by, bz);
  }
}

// intensity of returned neighbours (API searches only; off the hot path): the neighbour's voxel is re-read and the point with
// exactly these coordinates looked up.  pts: [K][nq] (x, y, z, d2) records, NaN x = no neighbour.  A verbatim insert keeps
// duplicate points, each with its own intensity: the r-th neighbour of a query takes the j-th coordinate match of its
// chain, j = the number of that query's earlier neighbours with the same coordinates, so that every duplicate returned
// carries a different record's intensity, as the reference returns each record.
__global__ void k_lookup_intensity(MapDev m, const float4* __restrict__ pts, float* __restrict__ out, int nq, int K) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nq * K; i += gridDim.x * blockDim.x) {
    const float4 p = pts[i];
    float r = 0.f;
    int skip = 0;
    for (int e = i - nq; e >= 0; e -= nq) {
      const float4 o = pts[e];
      skip += (o.x == p.x && o.y == p.y && o.z == p.z) ? 1 : 0;
    }
    if (p.x == p.x && coord_ok(p.x, p.y, p.z, m.ds)) {
      const int vx = voxel_of(p.x, m.ds), vy = voxel_of(p.y, m.ds), vz = voxel_of(p.z, m.ds);
      const int blk = find_block(m, pack_key(vx >> 2, vy >> 2, vz >> 2));
      if (blk >= 0) {
        const size_t idx = (size_t)blk * 64 + ((((vz & 3) << 2) + (vy & 3)) * 4 + (vx & 3));
        float4 e = m.slots[idx];
        float inten = m.sint[idx];
        for (;;) {
          if (e.x == p.x && e.y == p.y && e.z == p.z && skip-- == 0) { r = inten; break; }
          const int c = __float_as_int(e.w);
          if (c < 0) break;
          e = m.ovf[c];
          inten = m.oint[c];
        }
      }
    }
    out[i] = r;
  }
}

}  // namespace flb

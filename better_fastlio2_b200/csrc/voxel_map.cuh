// voxel_map.cuh — device-side layout of the hashed voxel map that replaces the reference's CPU ikd-Tree
// (include/ikd-Tree/ikd_Tree.{h,cpp}).  sm_90a (H100).
//
// Geometry (all in float, as the reference computes its voxel boxes, ikd_Tree.cpp:424-429):
//   voxel  v = floor(x / ds)           ds = downsample_size = filter_size_map_min
//   block  b = v >> 2   (4x4x4 voxels, 64 head slots = 1 KB, contiguous => one bulk-copyable bucket)
//   coarse c = b >> 3   (8x8x8 blocks; 512-bit block-occupancy bitmap) — only used to bound far searches.
//
// Storage in HBM
//   hent[C]           open-addressing hash  block key -> {block index, 64-bit voxel occupancy of the block}
//                     (C = 2^k >= 2*B, one 32-B entry = one DRAM sector per slot: a k-NN probe learns the block index AND
//                     which of its voxels hold points from ONE memory round trip; the occupancy word lives only here)
//   bslot[B]          hash slot of each allocated block (for the kernels that iterate blocks densely)
//   slots[B*64]       float4 head point of each voxel: x,y,z and w = int index of an overflow node (-1: none).
//                     INVARIANT: w == -1 whenever the voxel has no overflow chain (also while the voxel is empty).
//   sint[B*64], oint[O]  intensity of the head point of each voxel / of each overflow node (the reference tree stores whole
//                     PointType records, ikd_Tree.h:64-86; FAST-LIO map points carry x,y,z,intensity — normals and curvature are
//                     zero, laserMapping.cpp:1101-1110).  Side arrays: the k-NN hot path never touches them.
//   ovf[O]            float4 overflow nodes (x,y,z, w = next) for the rare voxels holding > 1 point
//                     (first Build, no-downsample inserts: SURVEY.md §3.3).  A linked list per voxel; after every
//                     verbatim insert the chains it touched are re-laid CONTIGUOUSLY (k_relocate_chains: next == this + 1),
//                     so readers fetch four consecutive nodes per round trip and only fall back to pointer chasing
//                     when a link does not confirm the guess (walk_chain).
//   bkey[B]           key of each allocated block (EMPTY if free) — lets delete/flatten iterate blocks densely
//   ckeys[CC]/cbits[CC*8]  coarse hash + bitmaps
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "trace.cuh"

namespace flb {

// Programmatic dependent launch (sm_90+): the kernels of a scan are launched with the programmatic-stream-serialization
// attribute, so a kernel's launch (grid setup, CTA scheduling, parameter fetch) overlaps the tail of its predecessor in
// the stream / graph instead of starting only after it has drained.  Every such kernel calls this first: it blocks
// until ALL prerequisite grids have completed and their memory is visible (so nothing below it can see stale data), and
// then allows its own dependents to be scheduled.  A no-op for kernels launched the ordinary way.
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_sync() {
  pdl_wait();
  pdl_trigger();
}
// GPU-scope memory operations of a producer kernel handing data to a consumer kernel running beside it.  An acquire
// (ld.acquire, or a fence after a relaxed read) invalidates the SM's whole L1 (CCTL.IVALL), which the other kernel's
// warps on that SM depend on: poll with relaxed loads and acquire once, when the awaited value has arrived.
__device__ __forceinline__ void st_release(int* p, int v) { asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_relaxed(int* p, int v) { asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ int ld_relaxed(const int* p) {
  int v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ int atom_add_release(int* p, int v) {
  int old;
  asm volatile("atom.release.gpu.global.add.s32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}

constexpr uint64_t KEY_EMPTY = 0xFFFFFFFFFFFFFFFFull;
constexpr uint64_t KEY_TOMB = 0xFFFFFFFFFFFFFFFEull;
constexpr int COORD_BIAS = 1 << 20;  // 21-bit biased coordinates per axis

// counters[] indices
enum Counter : int {
  CNT_BLK_BUMP = 0,   // next never-used block index
  CNT_BLK_FREE,       // size of free_blk stack
  CNT_OVF_BUMP,       // next never-used overflow node
  CNT_OVF_FREE,       // size of free_ovf stack
  CNT_VALID,          // number of valid points
  CNT_KEYS_USED,      // live keys in the block hash
  CNT_KEYS_TOMB,      // tombstones in the block hash
  CNT_COARSE_USED,    // coarse cells ever created since the last rebuild (= length of clist)
  CNT_ERROR,          // sticky device error flags (ERR_*)
  CNT_SCRATCH0,       // per-call scratch (returned counts)
  CNT_SCRATCH1,
  CNT_SCRATCH2,
  CNT_CMIN_X, CNT_CMIN_Y, CNT_CMIN_Z,  // coarse-cell bounding box of everything ever inserted since last rebuild
  CNT_CMAX_X, CNT_CMAX_Y, CNT_CMAX_Z,
  CNT_COUNT = 32
};
// ERR_KNN_STALL: the exact k-NN kernel gave up waiting for its work list (a broken hand-over protocol; never expected)
enum DevError : int { ERR_BLOCKS_FULL = 1, ERR_OVF_FULL = 2, ERR_HASH_FULL = 4, ERR_COARSE_FULL = 8, ERR_RANGE = 16, ERR_KNN_STALL = 32 };

// one hash entry = one 32-byte sector: key, block index and the block's voxel-occupancy word side by side
struct __align__(32) HEntry {
  uint64_t key;
  uint32_t val;
  uint32_t pad;
  uint64_t mask;   // bit s set <=> voxel slot s of the block holds >= 1 point (0 for empty / tombstoned entries)
  uint64_t pad2;
};

struct MapDev {
  HEntry* hent;
  uint32_t* bslot;
  float4* slots;
  float* sint;
  float4* ovf;
  float* oint;
  uint64_t* bkey;
  uint64_t* brel;        // per-block scratch bitmap of k_relocate_chains (all zero between kernels)
  uint32_t* free_blk;
  uint32_t* free_ovf;
  uint64_t* ckeys;
  uint64_t* cbits;
  uint32_t* clist;       // dense list of the occupied slots of ckeys (append order) for exhaustive far searches
  int* counters;
  uint32_t hash_mask;    // C-1
  uint32_t chash_mask;   // CC-1
  int block_cap;         // B
  int ovf_cap;           // O
  float ds;              // voxel size (float, = (float)filter_size_map_min)
};

__host__ __device__ __forceinline__ uint64_t pack_key(int x, int y, int z) {
  return ((uint64_t)(uint32_t)(x + COORD_BIAS) << 42) | ((uint64_t)(uint32_t)(y + COORD_BIAS) << 21) |
         (uint64_t)(uint32_t)(z + COORD_BIAS);
}
__host__ __device__ __forceinline__ void unpack_key(uint64_t k, int& x, int& y, int& z) {
  x = (int)((k >> 42) & 0x1FFFFF) - COORD_BIAS;
  y = (int)((k >> 21) & 0x1FFFFF) - COORD_BIAS;
  z = (int)(k & 0x1FFFFF) - COORD_BIAS;
}
// spatial hash of the three 21-bit biased coordinates (32-bit multiplies only: the lookup is on the k-NN hot path)
__host__ __device__ __forceinline__ uint32_t hash_key(uint64_t k) {
  const uint32_t x = (uint32_t)(k >> 42), y = (uint32_t)(k >> 21) & 0x1FFFFFu, z = (uint32_t)k & 0x1FFFFFu;
  uint32_t h = (x * 73856093u) ^ (y * 19349663u) ^ (z * 83492791u);
  h ^= h >> 15;
  h *= 0x9E3779B1u;
  h ^= h >> 13;
  return h;
}

// voxel index of a coordinate: the reference's floor(x/downsample_size) in float (ikd_Tree.cpp:424).
__device__ __forceinline__ int voxel_of(float x, float ds) { return (int)floorf(__fdiv_rn(x, ds)); }

// Visit every node of the overflow chain starting at node c: f(node, index).  Speculates that the chain is laid out
// contiguously (see MapDev::ovf): nodes c..c+3 are loaded together (64 B, at most two sectors) and consumed while the
// links confirm next == this + 1; otherwise the real link is followed.  Reading past a chain's end stays inside ovf[].
template <class F>
__device__ __forceinline__ void walk_chain(const MapDev& m, int c, F&& f) {
  while (c >= 0) {
    if (c + 3 < m.ovf_cap) {
      const float4 o0 = __ldg(&m.ovf[c]), o1 = __ldg(&m.ovf[c + 1]), o2 = __ldg(&m.ovf[c + 2]), o3 = __ldg(&m.ovf[c + 3]);
      f(o0, c);
      int nx = __float_as_int(o0.w);
      if (nx != c + 1) { c = nx; continue; }
      f(o1, c + 1);
      nx = __float_as_int(o1.w);
      if (nx != c + 2) { c = nx; continue; }
      f(o2, c + 2);
      nx = __float_as_int(o2.w);
      if (nx != c + 3) { c = nx; continue; }
      f(o3, c + 3);
      c = __float_as_int(o3.w);
    } else {
      const float4 o = __ldg(&m.ovf[c]);
      f(o, c);
      c = __float_as_int(o.w);
    }
  }
}

// L2 prefetch of the entry AFTER a probe's home slot.  With linear probing a probe that finds another key in its home slot
// continues in the next one: the k-NN kernels issue the home-slot load and this prefetch together, so that the (5-10 % of)
// probes that collide find their second entry in L2 instead of paying a second DRAM round trip — a warp issues 27-256
// probes at a time and otherwise almost always waits for at least one such chain.
__device__ __forceinline__ void prefetch_next_entry(const MapDev& m, uint32_t s) {
  const HEntry* nx = &m.hent[(s + 1) & m.hash_mask];
  asm volatile("prefetch.global.L2 [%0];" ::"l"(nx));
}

// Block lookup (read-only). Returns block index or -1.
__device__ __forceinline__ int find_block(const MapDev& m, uint64_t key) {
  uint32_t s = hash_key(key) & m.hash_mask;
  for (int probe = 0; probe <= (int)m.hash_mask; ++probe) {
    const uint4 e = __ldg(reinterpret_cast<const uint4*>(&m.hent[s]));
    const uint64_t k = ((uint64_t)e.y << 32) | e.x;
    if (k == key) return (int)e.z;
    if (k == KEY_EMPTY) return -1;
    s = (s + 1) & m.hash_mask;
  }
  return -1;
}
// Same, returning the hash slot (or -1): the entry holds the block index (val) and the occupancy word (mask).
__device__ __forceinline__ int find_slot(const MapDev& m, uint64_t key) {
  uint32_t s = hash_key(key) & m.hash_mask;
  for (int probe = 0; probe <= (int)m.hash_mask; ++probe) {
    const uint64_t k = *reinterpret_cast<const volatile uint64_t*>(&m.hent[s].key);
    if (k == key) return (int)s;
    if (k == KEY_EMPTY) return -1;
    s = (s + 1) & m.hash_mask;
  }
  return -1;
}
// Read-only probe for the k-NN kernels: block index (or -1) and its occupancy word from the entry's sector.
__device__ __forceinline__ int find_block_mask(const MapDev& m, uint64_t key, unsigned long long& mask) {
  uint32_t s = hash_key(key) & m.hash_mask;
  for (int probe = 0; probe <= (int)m.hash_mask; ++probe) {
    const uint4 e = __ldg(reinterpret_cast<const uint4*>(&m.hent[s]));
    const uint64_t k = ((uint64_t)e.y << 32) | e.x;
    if (k == key) {
      mask = __ldg(reinterpret_cast<const unsigned long long*>(&m.hent[s].mask));
      return (int)e.z;
    }
    if (k == KEY_EMPTY) break;
    s = (s + 1) & m.hash_mask;
  }
  mask = 0ull;
  return -1;
}
// occupancy word of an allocated block (block-iterating kernels)
__device__ __forceinline__ unsigned long long* block_mask_ptr(const MapDev& m, int blk) {
  return reinterpret_cast<unsigned long long*>(&m.hent[m.bslot[blk]].mask);
}
// Coarse-cell lookup. Returns slot index in ckeys/cbits or -1.
__device__ __forceinline__ int find_coarse(const MapDev& m, uint64_t key) {
  uint32_t s = hash_key(key) & m.chash_mask;
  for (int probe = 0; probe <= (int)m.chash_mask; ++probe) {
    uint64_t k = __ldg(&m.ckeys[s]);
    if (k == key) return (int)s;
    if (k == KEY_EMPTY) return -1;
    s = (s + 1) & m.chash_mask;
  }
  return -1;
}

}  // namespace flb

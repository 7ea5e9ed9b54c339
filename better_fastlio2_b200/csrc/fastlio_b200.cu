// fastlio_b200.cu — C-ABI implementation (include/fastlio_b200.h): host orchestration of the sm_90a kernels.
// One CUDA stream per map; all calls on a handle are issued by one caller thread (as the reference does,
// SURVEY.md §8b "Threading").  No CPU fallback anywhere: without a usable CUDA device every call returns an error.
#include "../../include/fastlio_b200.h"
#include "map_kernels.cuh"
#include "knn_kernels.cuh"
#include "frontend_kernels.cuh"
#include "meas_kernels.cuh"
#include "esikf_device.cuh"
#include "knn_tile.cuh"
#include "esikf_host.hpp"

#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

using namespace flb;

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
static int set_err(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
#define CU(call)                                                                                          \
  do {                                                                                                    \
    cudaError_t e__ = (call);                                                                             \
    if (e__ != cudaSuccess) return set_err("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

// destroy paths: never leave a stale error behind for the next call's cudaGetLastError(), but say what happened
static void quiet(cudaError_t e, const char* what) {
  if (e != cudaSuccess) {
    fprintf(stderr, "[fastlio_b200] warning: %s: %s\n", what, cudaGetErrorString(e));
    cudaGetLastError();
  }
}
#define Q(call) quiet((call), #call)

// ------------------------------------------------------------------------------------------------ grow-only buffers
// Scratch that is only ever grown and whose contents need not survive a growth.  grow() frees the old allocation, then
// allocates max(need, floor) bytes; a failure leaves the buffer empty.  Every caller keeps its own floor (or headroom):
// how often a buffer is reallocated decides how often the captured scan graphs are re-captured (flb_map::gen).  The
// owner frees it by destroying it, with its device current.
template <typename T, bool Pinned>
struct GrowBuf {
  T* p = nullptr;
  size_t cap = 0;   // bytes
  GrowBuf() = default;
  GrowBuf(const GrowBuf&) = delete;
  GrowBuf& operator=(const GrowBuf&) = delete;
  ~GrowBuf() { release(); }
  void release() {
    if (p) Q(Pinned ? cudaFreeHost(p) : cudaFree(p));
    p = nullptr;
    cap = 0;
  }
};
template <typename T> using DevBuf = GrowBuf<T, false>;
template <typename T> using PinnedBuf = GrowBuf<T, true>;   // page-locked host staging

template <typename T, bool Pinned>
static int grow(GrowBuf<T, Pinned>& b, size_t need, size_t floor) {
  if (need <= b.cap) return 0;
  b.release();
  const size_t cap = std::max(need, floor);
  void* p = nullptr;
  CU(Pinned ? cudaMallocHost(&p, cap) : cudaMalloc(&p, cap));
  b.p = static_cast<T*>(p);
  b.cap = cap;
  return 0;
}

extern "C" const char* flb_last_error(void) { return g_err; }
extern "C" const char* flb_version(void) { return "fastlio_b200 0.1 (sm_90a)"; }
extern "C" int flb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

// Kernel launch with or without the programmatic-stream-serialization attribute (programmatic dependent launch: the
// kernel's CTAs may start once every CTA of its predecessor has run griddepcontrol.launch_dependents; under stream capture
// the attribute becomes a programmatic graph edge).
template <typename... P, typename... A>
static cudaError_t launch_kx(bool programmatic, void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = programmatic ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<P>(args)...);
}
// Kernel launch of the scan sequence.  FLB_PDL=1 launches it programmatically (a kernel's launch overlaps its
// predecessor's tail; the kernels call pdl_sync() before touching anything).  OFF by default, kept as an A/B switch; the
// exact k-NN kernel is always launched programmatically after the stencil kernel (launch_knn).
static bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("FLB_PDL"); return e && atoi(e) != 0; }();
  return on;
}
template <typename... P, typename... A>
static cudaError_t launch_k(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  return launch_kx(pdl_enabled(), kern, grid, block, smem, st, static_cast<A&&>(args)...);
}

static inline uint32_t next_pow2(uint64_t v) {
  uint32_t p = 1;
  while (p < v) p <<= 1;
  return p;
}
static inline int grid_for(int n, int threads, int max_blocks) {
  int g = (n + threads - 1) / threads;
  if (g < 1) g = 1;
  return g > max_blocks ? max_blocks : g;
}
// CTAs of `kern` that are resident on the whole device at once (the grid of a kernel that loops over its work)
template <typename... P>
static cudaError_t resident_ctas(void (*kern)(P...), int threads, size_t smem, int sm_count, int& out) {
  int per_sm = 0;
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem);
  out = std::max(per_sm, 1) * sm_count;
  return e;
}

// ------------------------------------------------------------------------------------------------ map
struct flb_map {
  MapDev d{};
  flb_map_config cfg{};
  cudaStream_t stream = nullptr;
  int sm_count = 148;
  int exact_ctas[2] = {0, 0};    // resident CTAs of k_knn<5>, <20> (the grid of the exact completion)
  uint32_t hash_cap = 0, chash_cap = 0;
  size_t device_bytes = 0;
  bool has_root = false;
  int rehash_count = 0;
  // staging
  DevBuf<float4> stage;          // device float4 staging for host uploads
  DevBuf<unsigned char> raw;     // device raw strided upload buffer
  DevBuf<uint64_t> skeys;        // scratch hash of the downsampled insert (scratch_slots entries)
  DevBuf<unsigned long long> sbest;
  DevBuf<float> dparams;         // small device parameter buffer (boxes / points)
  DevBuf<float4> outbuf;         // collect output
  int* h_counters = nullptr;     // pinned mirror of counters
  int* d_misc = nullptr;         // misc device ints (out counts, range)
  int launches = 0;              // kernel launch counter (cumulative)
  int refs = 1;                  // the map handle + every live session: storage is freed when the last one goes
  // optional per-kernel-class CUDA-event timing (flb_map_profile_*)
  bool prof_on = false;
  bool capturing = false;        // inside cudaStreamBeginCapture: no event timing, no allocations
  struct ProfRec { cudaEvent_t a, b; int cls; int nlaunch; };
  std::vector<ProfRec> prof_pool;
  size_t prof_used = 0;
  int* d_phase = nullptr;        // k-NN phase histogram (device, 4 ints)
  DevBuf<int> worklist;          // unresolved-query list of the stencil k-NN kernel
  bool scratch_clean = false;    // the downsample scratch hash was already cleared off the critical path (scan graph)
  DevBuf<unsigned char> kf_raw;  // flb_map_reconstruct_keyframes scratch
  DevBuf<float4> kf_in, kf_out;
  struct KfWork* kfw = nullptr;      // the rest of the key-frame readers' scratch (keyframe_host.cuh, grow-only)
  int gen = 0;                   // bumped whenever a buffer or parameter baked into a captured scan graph changes (scratch hash,
                                 // work list, voxel size): sessions re-capture their graphs on a mismatch
  bool warned_range = false;
};

struct ProfScope {
  flb_map* m; flb_map::ProfRec* r = nullptr; int l0;
  ProfScope(flb_map* m_, int cls) : m(m_), l0(m_->launches) {
    if (!m->prof_on || m->capturing) return;
    if (m->prof_used == m->prof_pool.size()) {
      flb_map::ProfRec n{};
      if (cudaEventCreate(&n.a) != cudaSuccess || cudaEventCreate(&n.b) != cudaSuccess) return;
      m->prof_pool.push_back(n);
    }
    r = &m->prof_pool[m->prof_used++];
    r->cls = cls;
    cudaEventRecord(r->a, m->stream);
  }
  ~ProfScope() { if (r) { r->nlaunch = m->launches - l0; cudaEventRecord(r->b, m->stream); } }
};

static int dev_alloc(flb_map* m, void** p, size_t bytes) {
  CU(cudaMalloc(p, bytes));
  m->device_bytes += bytes;
  return 0;
}

static int map_reset_storage(flb_map* m) {
  MapDev& d = m->d;
  cudaStream_t st = m->stream;
  k_hent_clear<<<m->sm_count * 8, 256, 0, st>>>(d.hent, m->hash_cap);
  CU(cudaGetLastError());
  CU(cudaMemsetAsync(d.slots, 0xFF, sizeof(float4) * 64 * (size_t)d.block_cap, st));
  CU(cudaMemsetAsync(d.bkey, 0xFF, sizeof(uint64_t) * d.block_cap, st));
  CU(cudaMemsetAsync(d.brel, 0, sizeof(uint64_t) * d.block_cap, st));
  CU(cudaMemsetAsync(d.ckeys, 0xFF, sizeof(uint64_t) * m->chash_cap, st));
  CU(cudaMemsetAsync(d.cbits, 0, sizeof(uint64_t) * 8 * (size_t)m->chash_cap, st));
  int init[CNT_COUNT];
  memset(init, 0, sizeof(init));
  init[CNT_CMIN_X] = init[CNT_CMIN_Y] = init[CNT_CMIN_Z] = INT_MAX;
  init[CNT_CMAX_X] = init[CNT_CMAX_Y] = init[CNT_CMAX_Z] = INT_MIN;
  memcpy(m->h_counters, init, sizeof(init));
  CU(cudaMemcpyAsync(d.counters, m->h_counters, sizeof(init), cudaMemcpyHostToDevice, st));
  CU(cudaStreamSynchronize(st));
  m->has_root = false;
  return 0;
}

// A NaN / out-of-range point is skipped by the insert kernels (the reference keeps running in that situation too): the
// flag is reported once and cleared, so that one bad point does not fail every later call.  Capacity errors stay sticky.
static int absorb_range_flag(flb_map* m) {
  int e = m->h_counters[CNT_ERROR];
  if (!(e & ERR_RANGE)) return e;
  if (!m->warned_range) {
    fprintf(stderr, "[fastlio_b200] warning: point(s) outside the representable range / NaN were skipped by the map insert\n");
    m->warned_range = true;
  }
  e &= ~ERR_RANGE;
  m->h_counters[CNT_ERROR] = e;
  // the stream is drained here (callers synchronised): a plain store of the remaining (sticky) bits is race free
  if (cudaMemcpyAsync(m->d.counters + CNT_ERROR, m->h_counters + CNT_ERROR, sizeof(int), cudaMemcpyHostToDevice, m->stream) == cudaSuccess)
    cudaStreamSynchronize(m->stream);
  return e;
}

static int fetch_counters(flb_map* m) {
  CU(cudaMemcpyAsync(m->h_counters, m->d.counters, sizeof(int) * CNT_COUNT, cudaMemcpyDeviceToHost, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  const int e = absorb_range_flag(m);
  if (e) {
    return set_err("device map error flags 0x%x:%s%s%s%s%s%s", e, (e & ERR_BLOCKS_FULL) ? " block pool exhausted (raise max_blocks)" : "",
                   (e & ERR_OVF_FULL) ? " overflow pool exhausted (raise max_points)" : "", (e & ERR_HASH_FULL) ? " block hash full" : "",
                   (e & ERR_COARSE_FULL) ? " coarse hash full" : "", (e & ERR_RANGE) ? " point outside representable range / NaN" : "",
                   (e & ERR_KNN_STALL) ? " k-NN work-list wait timed out" : "");
  }
  return 0;
}

extern "C" int flb_map_create(const flb_map_config* cfg, flb_map** out) {
  if (!cfg || !out) return set_err("flb_map_create: null argument");
  cudaGetLastError();  // start from a clean error state
  if (!(cfg->voxel_size > 0.f)) return set_err("flb_map_create: voxel_size must be > 0");
  int ndev = flb_device_count();
  if (ndev <= 0) return set_err("flb_map_create: no CUDA device available (this library has no CPU fallback)");
  if (cfg->device < 0 || cfg->device >= ndev) return set_err("flb_map_create: bad device %d", cfg->device);
  CU(cudaSetDevice(cfg->device));
  flb_map* m = new (std::nothrow) flb_map();
  if (!m) return set_err("out of host memory");
  m->cfg = *cfg;
  if (m->cfg.max_points <= 0) m->cfg.max_points = 8 * 1024 * 1024;
  if (m->cfg.max_blocks <= 0) m->cfg.max_blocks = std::max(4096, m->cfg.max_points / 4);
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, cfg->device));
  m->sm_count = prop.multiProcessorCount;
  CU(resident_ctas(k_knn<5>, KNN_THREADS, 0, m->sm_count, m->exact_ctas[0]));
  CU(resident_ctas(k_knn<20>, KNN_THREADS, 0, m->sm_count, m->exact_ctas[1]));
  CU(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
  MapDev& d = m->d;
  d.ds = cfg->voxel_size;
  d.block_cap = m->cfg.max_blocks;
  d.ovf_cap = std::max(1024, m->cfg.max_points / 2);
  // load factor <= 1/4 at full capacity (typically 5-10 % in use): a probe rarely continues past its home slot
  m->hash_cap = next_pow2((uint64_t)d.block_cap * 4);
  // one coarse cell per block in the worst case (sparse content): with maybe_rehash dropping the cells that deletes emptied,
  // a map within max_blocks never fills the coarse table (76 B per entry: ckeys + cbits + clist)
  m->chash_cap = next_pow2(std::max<uint64_t>(1024, (uint64_t)d.block_cap));
  d.hash_mask = m->hash_cap - 1;
  d.chash_mask = m->chash_cap - 1;
  int rc = 0;
  rc |= dev_alloc(m, (void**)&d.hent, sizeof(HEntry) * m->hash_cap);
  rc |= dev_alloc(m, (void**)&d.bslot, sizeof(uint32_t) * d.block_cap);
  rc |= dev_alloc(m, (void**)&d.slots, sizeof(float4) * 64 * (size_t)d.block_cap);
  rc |= dev_alloc(m, (void**)&d.ovf, sizeof(float4) * (size_t)d.ovf_cap);
  rc |= dev_alloc(m, (void**)&d.sint, sizeof(float) * 64 * (size_t)d.block_cap);
  rc |= dev_alloc(m, (void**)&d.oint, sizeof(float) * (size_t)d.ovf_cap);
  rc |= dev_alloc(m, (void**)&d.bkey, sizeof(uint64_t) * d.block_cap);
  rc |= dev_alloc(m, (void**)&d.brel, sizeof(uint64_t) * d.block_cap);
  rc |= dev_alloc(m, (void**)&d.free_blk, sizeof(uint32_t) * d.block_cap);
  rc |= dev_alloc(m, (void**)&d.free_ovf, sizeof(uint32_t) * d.ovf_cap);
  rc |= dev_alloc(m, (void**)&d.ckeys, sizeof(uint64_t) * m->chash_cap);
  rc |= dev_alloc(m, (void**)&d.cbits, sizeof(uint64_t) * 8 * (size_t)m->chash_cap);
  rc |= dev_alloc(m, (void**)&d.clist, sizeof(uint32_t) * (size_t)m->chash_cap);
  rc |= dev_alloc(m, (void**)&d.counters, sizeof(int) * CNT_COUNT);
  // d_misc: [0..3] counts, [4..9] range, [12] work count, [13] ticket, [14] stencil CTAs done, [16..23] per-pass work counts,
  // [24..31] per-pass tickets, [32..39] per-pass stencil CTAs done
  rc |= dev_alloc(m, (void**)&m->d_misc, sizeof(int) * 48);
  rc |= dev_alloc(m, (void**)&m->d_phase, sizeof(int) * 8);
  if (rc) { flb_map_destroy(m); return 1; }
  if (cudaMallocHost((void**)&m->h_counters, sizeof(int) * CNT_COUNT) != cudaSuccess) { flb_map_destroy(m); return set_err("cudaMallocHost failed"); }
  // triangle index tables of the 13x13 augmented normal equations
  unsigned char ti[91], tj[91];
  int e = 0;
  for (int i = 0; i < 13; ++i) for (int j = i; j < 13; ++j) { ti[e] = (unsigned char)i; tj[e] = (unsigned char)j; ++e; }
  CU(cudaMemcpyToSymbol(c_tri_i, ti, sizeof(ti)));
  CU(cudaMemcpyToSymbol(c_tri_j, tj, sizeof(tj)));
  if (map_reset_storage(m)) { flb_map_destroy(m); return 1; }
  *out = m;
  return 0;
}

static void map_release(flb_map* m);
static void kfw_release(KfWork* w);
extern "C" void flb_map_destroy(flb_map* m) {
  if (!m) return;
  map_release(m);  // sessions created on this map keep it alive until they are destroyed too
}
static void map_release(flb_map* m) {
  if (--m->refs > 0) return;
  Q(cudaSetDevice(m->cfg.device));
  if (m->stream) Q(cudaStreamSynchronize(m->stream));
  MapDev& d = m->d;
  void* ptrs[] = {d.clist, d.hent, d.bslot, d.slots, d.sint, d.oint, d.ovf, d.bkey, d.brel, d.free_blk, d.free_ovf, d.ckeys, d.cbits, d.counters,
                  m->d_misc, m->d_phase};
  for (void* p : ptrs) if (p) Q(cudaFree(p));
  if (m->h_counters) Q(cudaFreeHost(m->h_counters));
  kfw_release(m->kfw);
  for (auto& r : m->prof_pool) { Q(cudaEventDestroy(r.a)); Q(cudaEventDestroy(r.b)); }
  if (m->stream) Q(cudaStreamDestroy(m->stream));
  delete m;
}

extern "C" int flb_map_set_downsample_param(flb_map* m, float v) {
  if (!m) return set_err("null map");
  if (!(v > 0.f)) return set_err("voxel size must be > 0");
  if (v == m->d.ds) return 0;
  CU(cudaSetDevice(m->cfg.device));
  if (fetch_counters(m)) return 1;
  if (m->h_counters[CNT_VALID] != 0) return set_err("set_downsample_param: map not empty (voxel hashing depends on the voxel size)");
  m->d.ds = v;
  m->cfg.voxel_size = v;
  m->gen++;
  return 0;
}
extern "C" int flb_map_has_root(const flb_map* m) { return m && m->has_root ? 1 : 0; }

// n > 0 records of `stride` bytes, already on the device at `raw` -> dst (x, y, z, intensity at byte off_i) and, when curv is
// given, curv (curvature at off_c); a negative offset means the field is absent (0).  On `st`.
static int pack_records(flb_map* m, cudaStream_t st, const unsigned char* raw, int n, int stride, int off_i, int off_c, float4* dst,
                        float* curv) {
  k_pack_xyzic<<<grid_for(n, 256, m->sm_count * 8), 256, 0, st>>>(raw, stride, off_i, off_c, dst, curv, n);
  m->launches++;
  CU(cudaGetLastError());
  return 0;
}

// n > 0 host records -> device, staged in `raw` (grown to at least raw_floor bytes) and packed as pack_records does, on `st`.
// Records that are (x, y, z, intensity) already (16 bytes, intensity at 12, no curvature asked for) are copied straight to
// dst: no staging, no launch.  Entry points that read a 16-byte record's 4th float as its intensity pass off_i = 12.
static int upload_records(flb_map* m, cudaStream_t st, DevBuf<unsigned char>& raw, size_t raw_floor, const void* src, int n, int stride,
                          int off_i, int off_c, float4* dst, float* curv) {
  if (stride == 16 && off_i == 12 && !curv) {
    CU(cudaMemcpyAsync(dst, src, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
    return 0;
  }
  if (!curv) off_c = -1;
  // the last record is read only up to the end of its last field used
  const size_t bytes = (size_t)(n - 1) * stride + (size_t)std::max({12, off_i + 4, off_c + 4});
  if (grow(raw, bytes, raw_floor)) return 1;
  CU(cudaMemcpyAsync(raw.p, src, bytes, cudaMemcpyHostToDevice, st));
  return pack_records(m, st, raw.p, n, stride, off_i, off_c, dst, curv);
}

// host strided points -> m->stage (x, y, z, intensity).  off_i: byte offset of the intensity inside a record, < 0 = none
// (0).  16-byte records are taken as (x, y, z, intensity) verbatim.
static int upload_points(flb_map* m, const void* pts, int n, int stride, int off_i = -1) {
  if (n <= 0) return 0;
  if (!pts) return set_err("null point buffer");
  if (stride < 12) return set_err("stride_bytes must be >= 12");
  if (off_i >= 0 && off_i + 4 > stride) return set_err("intensity offset %d outside the %d-byte record", off_i, stride);
  if (stride == 16 && off_i < 0) off_i = 12;
  if (grow(m->stage, sizeof(float4) * (size_t)n, sizeof(float4) << 16)) return 1;
  return upload_records(m, m->stream, m->raw, (size_t)1 << 20, pts, n, stride, off_i, -1, m->stage.p, nullptr);
}

// entries of the downsampled insert's scratch hash for n points (load factor <= 1/2)
static inline uint32_t scratch_slots(int n) { return next_pow2((uint64_t)std::max(n, 512) * 2); }

// the scratch hash (skeys / sbest) for n points; a captured scan graph holds its address
static int ensure_scratch(flb_map* m, int n) {
  const size_t need = sizeof(uint64_t) * scratch_slots(n);
  if (need <= m->skeys.cap && need <= m->sbest.cap) return 0;
  if (grow(m->skeys, need, 0) || grow(m->sbest, need, 0)) return 1;
  m->gen++;
  return 0;
}

// warps of the exact k-NN kernel's grid (launch_knn)
static int exact_warps(const flb_map* m, int K) { return m->exact_ctas[K == 5 ? 0 : 1] * (KNN_THREADS / 32); }

// the stencil k-NN kernel's work list for n queries and the entries that close it (one per exact-kernel warp), all
// WORK_EMPTY (0xFF bytes); a captured scan graph holds its address
static int ensure_worklist(flb_map* m, int n) {
  const size_t need = sizeof(int) * ((size_t)n + std::max(exact_warps(m, 5), exact_warps(m, 20)));
  if (need <= m->worklist.cap) return 0;
  if (grow(m->worklist, need, sizeof(int) << 17)) return 1;
  CU(cudaMemsetAsync(m->worklist.p, 0xFF, m->worklist.cap, m->stream));
  m->gen++;
  return 0;
}

static int maybe_rehash(flb_map* m);

// Insert device points. mode 0: verbatim (Build / Add_Points(false)); 1: downsample (Add_Points(true));
// 2: classified (map_incremental: cls 1 -> downsample, cls 2 -> verbatim). Asynchronous on m->stream.
static int insert_device(flb_map* m, const float4* pts, const unsigned char* cls, int n, int mode, const int* skip = nullptr,
                         const int* n_dev = nullptr, bool prefused = false, StepTail tail = StepTail{}) {
  // n_dev != nullptr: n is an upper bound (capacity) used for launch geometry, the real count is read on the device
  if (n <= 0) return 0;
  const int g = grid_for(n, 256, m->sm_count * 8);
  cudaStream_t st = m->stream;
  const unsigned char* c = (mode == 2) ? cls : nullptr;
  ProfScope ps(m, FLB_K_INSERT);
  // prefused: k_classify already touched the blocks and scattered the downsampled class into the (cleared) scratch hash
  if (!prefused) {
    launch_k(k_touch_blocks, g, 256, 0, st, m->d, pts, c, (1 << 1) | (1 << 2), n, skip, n_dev);
    m->launches++;
  }
  if (mode == 1 || mode == 2) {
    const uint32_t sc = scratch_slots(n);
    if (!prefused) {
      if (ensure_scratch(m, n)) return 1;
      if (!m->scratch_clean) {
        CU(cudaMemsetAsync(m->skeys.p, 0xFF, sizeof(uint64_t) * sc, st));
        CU(cudaMemsetAsync(m->sbest.p, 0xFF, sizeof(unsigned long long) * sc, st));
      }
      launch_k(k_ds_scatter, g, 256, 0, st, m->d, pts, c, n, m->skeys.p, m->sbest.p, sc - 1, skip, n_dev);
      m->launches++;
    }
    m->scratch_clean = false;
    launch_k(k_ds_apply, g, 256, 0, st, m->d, pts, c, n, (const uint64_t*)m->skeys.p, (const unsigned long long*)m->sbest.p, sc - 1, skip, n_dev);
    m->launches++;
  }
  if (mode == 0 || mode == 2) {
    launch_k(k_append_points, g, 256, 0, st, m->d, pts, c, 2, n, skip, n_dev, tail);
    m->launches++;
    // Chain relocation is a pure layout optimisation (contiguous overflow chains for the k-NN readers).  It pays after a bulk
    // verbatim insert (Build, Add_Points(false): many multi-point voxels); map_incremental's verbatim class is a few hundred
    // points per scan that land in (almost always) EMPTY voxels — nothing to re-lay — so the scan path leaves it out
    // (6.4 us + a launch gap per scan on cfg2); chains stay valid linked lists either way.
    if (!prefused) {
      launch_k(k_relocate_chains, g, 256, 0, st, m->d, pts, c, 2, n, skip, n_dev);
      m->launches++;
    }
  }
  CU(cudaGetLastError());
  if (!n_dev) m->has_root = true;
  return 0;
}

static int zero_scratch_counters(flb_map* m) {
  CU(cudaMemsetAsync(m->d.counters + CNT_SCRATCH0, 0, sizeof(int) * 3, m->stream));
  return 0;
}

extern "C" int flb_map_build_pt(flb_map* m, const void* pts, int n, int stride, int off_intensity) {
  if (!m) return set_err("null map");
  if (n < 0) return set_err("negative point count");
  CU(cudaSetDevice(m->cfg.device));
  if (map_reset_storage(m)) return 1;
  if (n == 0) return 0;  // Build with an empty cloud leaves Root_Node == nullptr (ikd_Tree.cpp:357)
  if (upload_points(m, pts, n, stride, off_intensity)) return 1;
  if (insert_device(m, m->stage.p, nullptr, n, 0)) return 1;
  return fetch_counters(m);
}
extern "C" int flb_map_build(flb_map* m, const float* xyz, int n, int stride) { return flb_map_build_pt(m, xyz, n, stride, -1); }
extern "C" int flb_map_reconstruct(flb_map* m, const float* xyz, int n, int stride) { return flb_map_build_pt(m, xyz, n, stride, -1); }
extern "C" int flb_map_reconstruct_pt(flb_map* m, const void* pts, int n, int stride, int off_intensity) {
  return flb_map_build_pt(m, pts, n, stride, off_intensity);
}

extern "C" int flb_map_add_points_pt(flb_map* m, const void* pts, int n, int stride, int off_intensity, int downsample_on, int* n_added) {
  if (!m) return set_err("null map");
  if (n_added) *n_added = 0;
  if (n <= 0) return 0;
  CU(cudaSetDevice(m->cfg.device));
  if (upload_points(m, pts, n, stride, off_intensity)) return 1;
  if (zero_scratch_counters(m)) return 1;
  if (insert_device(m, m->stage.p, nullptr, n, downsample_on ? 1 : 0)) return 1;
  if (fetch_counters(m)) return 1;
  // reference return value: tmp_counter counts downsample add ops only (ikd_Tree.cpp:447,457,488)
  if (n_added) *n_added = downsample_on ? m->h_counters[CNT_SCRATCH0] : 0;
  return 0;
}
extern "C" int flb_map_add_points(flb_map* m, const float* xyz, int n, int stride, int downsample_on, int* n_added) {
  return flb_map_add_points_pt(m, xyz, n, stride, -1, downsample_on, n_added);
}

static int upload_params(flb_map* m, const float* host, int nfloats) {
  if (grow(m->dparams, sizeof(float) * (size_t)nfloats, sizeof(float) * 256)) return 1;
  CU(cudaMemcpyAsync(m->dparams.p, host, sizeof(float) * nfloats, cudaMemcpyHostToDevice, m->stream));
  return 0;
}

static int blocks_bumped(flb_map* m) {
  // number of block indices ever handed out (dense iteration range); needs fresh counters
  int b = m->h_counters[CNT_BLK_BUMP];
  return b > m->d.block_cap ? m->d.block_cap : b;
}

static int delete_common(flb_map* m, const float* params, int np, int floats_per, int mode, int* n_deleted) {
  if (n_deleted) *n_deleted = 0;
  if (np <= 0) return 0;
  CU(cudaSetDevice(m->cfg.device));
  if (fetch_counters(m)) return 1;
  const int nblk = blocks_bumped(m);
  if (nblk == 0) return 0;
  if (upload_params(m, params, np * floats_per)) return 1;
  if (zero_scratch_counters(m)) return 1;
  const int g = grid_for(nblk * 32, 256, m->sm_count * 8);
  {
    ProfScope ps(m, FLB_K_DELETE);
    k_delete<<<g, 256, 0, m->stream>>>(m->d, m->dparams.p, np, mode, nblk);
    m->launches++;
  }
  CU(cudaGetLastError());
  if (fetch_counters(m)) return 1;
  if (n_deleted) *n_deleted = m->h_counters[CNT_SCRATCH0];
  return maybe_rehash(m);
}

extern "C" int flb_map_delete_boxes(flb_map* m, const float* boxes6, int nb, int* n_deleted) {
  if (!m) return set_err("null map");
  if (nb > 0 && !boxes6) return set_err("null boxes");
  return delete_common(m, boxes6, nb, 6, 0, n_deleted);
}
extern "C" int flb_map_delete_points(flb_map* m, const float* xyz, int n, int stride, int* n_deleted) {
  if (!m) return set_err("null map");
  if (n > 0 && (!xyz || stride < 12)) return set_err("bad point buffer");
  std::vector<float> p((size_t)std::max(n, 0) * 4);
  for (int i = 0; i < n; ++i) {
    const float* s = reinterpret_cast<const float*>(reinterpret_cast<const unsigned char*>(xyz) + (size_t)i * stride);
    p[4 * i] = s[0]; p[4 * i + 1] = s[1]; p[4 * i + 2] = s[2]; p[4 * i + 3] = 0.f;
  }
  return delete_common(m, p.data(), n, 4, 1, n_deleted);
}

static int maybe_rehash(flb_map* m) {
  // Tombstones only lengthen probe chains: rebuild the key table (16 MB-ish, no point data moves) when they pile up.
  // Coarse cells are never removed one by one (coarse_clear only clears a block's bit), so cells that deletes emptied stay
  // in ckeys and clist until the coarse level is rebuilt from the live blocks.  Between two deletes a cell is created only
  // together with a new block, so cells - live blocks grows only through deletes, and every delete ends here: keeping
  // cells <= live blocks + (chash_cap - max_blocks) at this point bounds the cells by chash_cap until the next delete.
  const int* c = m->h_counters;
  const int live_blocks = blocks_bumped(m) - c[CNT_BLK_FREE];
  const bool rehash = c[CNT_KEYS_TOMB] > (int)(m->hash_cap / 8);
  const bool coarse = c[CNT_COARSE_USED] - live_blocks > (int)m->chash_cap - m->d.block_cap;
  if (!rehash && !coarse) return 0;
  const int nblk = blocks_bumped(m);
  cudaStream_t st = m->stream;
  if (rehash) {
    k_rehash_save<<<grid_for(nblk, 256, m->sm_count * 8), 256, 0, st>>>(m->d, nblk);
    k_hent_clear<<<m->sm_count * 8, 256, 0, st>>>(m->d.hent, m->hash_cap);
    m->launches += 2;
  }
  CU(cudaMemsetAsync(m->d.ckeys, 0xFF, sizeof(uint64_t) * m->chash_cap, st));
  CU(cudaMemsetAsync(m->d.cbits, 0, sizeof(uint64_t) * 8 * (size_t)m->chash_cap, st));
  int init[8] = {0, 0, INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
  // KEYS_TOMB = 0 (rehash only), COARSE_USED = 0, bbox reset
  if (rehash) CU(cudaMemcpyAsync(m->d.counters + CNT_KEYS_TOMB, &init[0], sizeof(int), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(m->d.counters + CNT_COARSE_USED, &init[1], sizeof(int), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(m->d.counters + CNT_CMIN_X, &init[2], sizeof(int) * 6, cudaMemcpyHostToDevice, st));
  CU(cudaStreamSynchronize(st));  // init[] is a stack buffer
  if (rehash) {
    k_rehash_insert<<<grid_for(nblk, 256, m->sm_count * 8), 256, 0, st>>>(m->d, nblk);
    m->launches++;
  }
  k_coarse_rebuild<<<grid_for(nblk, 256, m->sm_count * 8), 256, 0, st>>>(m->d, nblk);
  m->launches++;
  CU(cudaGetLastError());
  if (rehash) m->rehash_count++;
  return fetch_counters(m);
}

// k-NN = thread-per-query stencil kernel + exact warp-per-query kernel over the (small) unresolved work list.
template <int K>
static int launch_knn(flb_map* m, KnnArgs a) {
  if (ensure_worklist(m, a.n)) return 1;
  a.worklist = m->worklist.p;
  if (a.stride <= 0) a.stride = a.n;
  if (!a.work_count) {   // (device-driven scans use per-pass counters zeroed by k_esikf_begin: no memset node per pass)
    a.work_count = m->d_misc + 12;
    a.work_ticket = m->d_misc + 13;
    a.stencil_done = m->d_misc + 14;
    CU(cudaMemsetAsync(a.work_count, 0, 3 * sizeof(int), m->stream));
  }
  a.exact_warps = exact_warps(m, K);
  // one thread per query (a.n is the session capacity on the device-driven path; CTAs past the scan's size exit at once).
  // A cfg2 scan (~930 CTAs) is a little more than the 924 CTAs an H100 holds at 7 per SM.  Two ways to make it one wave
  // were measured slower (DESIGN.md §3): a resident grid looping over warp-sized chunks claimed by ticket (the loop cost
  // ~250 B of register spills per thread) and a 64-register cap for 8 CTAs per SM (~100 B of spills).
  launch_k(k_knn_stencil<K>, (a.n + 127) / 128, 128, 0, m->stream, a);
  // the exact completion: all CTAs resident (from the occupancy API), looping over the work list.  A programmatic
  // dependent of the stencil kernel: its CTAs start on the SMs the stencil kernel's early CTAs leave, and take the
  // unresolved queries as they are published (work-list hand-over, knn_kernels.cuh)
  launch_kx(true, k_knn<K>, m->exact_ctas[K == 5 ? 0 : 1], KNN_THREADS, 0, m->stream, a);
  m->launches += 2;
  return 0;
}

static int ensure_outbuf(flb_map* m, int n) { return grow(m->outbuf, sizeof(float4) * (size_t)n, sizeof(float4) << 16); }

// The reference accepts a neighbour when its float distance satisfies dist <= max_dist * max_dist evaluated in double
// (ikd_Tree.cpp:872,887).  For a float d2 that is the same as d2 <= the largest float not above the double square;
// fl(max_dist * max_dist) is that float when it rounds down, but when it rounds up (0.1f) it admits a neighbour at
// d2 = fl(max_dist * max_dist) that the reference rejects.
static float max_d2_of(float max_dist) {
  const double sq = (double)max_dist * (double)max_dist;
  const float f = (float)sq;
  return (double)f > sq ? std::nextafter(f, 0.f) : f;
}

static int nearest_search_impl(flb_map* m, const float* q_xyz, int nq, int stride, int k, float max_dist, float* out_pts, int out_w,
                               float* out_d2, int* out_cnt) {
  if (!m) return set_err("null map");
  if (k < 1 || k > 20) return set_err("Nearest_Search: k must be in [1,20]");
  if (nq <= 0) return 0;
  CU(cudaSetDevice(m->cfg.device));
  if (upload_points(m, q_xyz, nq, stride)) return 1;
  const int K = k <= 5 ? 5 : 20;
  if (ensure_outbuf(m, nq * K)) return 1;
  unsigned char* dcnt = nullptr;
  float* dint = nullptr;
  CU(cudaMalloc((void**)&dcnt, nq));
  KnnArgs a;
  a.m = m->d; a.q = m->stage.p; a.n = nq; a.nbr = m->outbuf.p; a.cnt = dcnt;
  a.max_d2 = (max_dist > 0.f && max_dist < 1e18f) ? max_d2_of(max_dist) : INFINITY;
  a.phase_stats = nullptr;
  a.ctl = nullptr; a.body = nullptr; a.stride = nq; a.work_count = nullptr;
  int lrc = (K == 5) ? launch_knn<5>(m, a) : launch_knn<20>(m, a);
  cudaError_t le = lrc ? cudaErrorUnknown : cudaGetLastError();
  std::vector<float4> h((size_t)nq * K);
  std::vector<unsigned char> hc(nq);
  std::vector<float> hi;
  if (le == cudaSuccess && out_w == 4 && out_pts) {
    // the neighbours' intensities (the reference returns whole PointType records, ikd_Tree.cpp:391-395)
    hi.resize((size_t)nq * K);
    le = cudaMalloc((void**)&dint, sizeof(float) * hi.size());
    if (le == cudaSuccess) {
      k_lookup_intensity<<<grid_for(nq * K, 256, m->sm_count * 8), 256, 0, m->stream>>>(m->d, m->outbuf.p, dint, nq, K);
      m->launches++;
      le = cudaMemcpyAsync(hi.data(), dint, sizeof(float) * hi.size(), cudaMemcpyDeviceToHost, m->stream);
    }
  }
  if (le == cudaSuccess) le = cudaMemcpyAsync(h.data(), m->outbuf.p, sizeof(float4) * h.size(), cudaMemcpyDeviceToHost, m->stream);
  if (le == cudaSuccess) le = cudaMemcpyAsync(hc.data(), dcnt, nq, cudaMemcpyDeviceToHost, m->stream);
  if (le == cudaSuccess) le = cudaStreamSynchronize(m->stream);
  cudaFree(dcnt);
  if (dint) cudaFree(dint);
  if (le != cudaSuccess) return set_err("nearest_search failed: %s", cudaGetErrorString(le));
  for (int i = 0; i < nq; ++i) {
    const int c = std::min<int>(hc[i], k);
    if (out_cnt) out_cnt[i] = c;
    for (int j = 0; j < k; ++j) {
      const float4 v = h[(size_t)j * nq + i];
      const bool ok = j < c;
      if (out_pts) {
        float* o = out_pts + ((size_t)i * k + j) * out_w;
        o[0] = ok ? v.x : NAN;
        o[1] = ok ? v.y : NAN;
        o[2] = ok ? v.z : NAN;
        if (out_w == 4) o[3] = ok ? hi[(size_t)j * nq + i] : NAN;
      }
      if (out_d2) out_d2[(size_t)i * k + j] = ok ? v.w : INFINITY;
    }
  }
  return 0;
}
extern "C" int flb_map_nearest_search(flb_map* m, const float* q_xyz, int nq, int stride, int k, float max_dist,
                                      float* out_xyz, float* out_d2, int* out_cnt) {
  return nearest_search_impl(m, q_xyz, nq, stride, k, max_dist, out_xyz, 3, out_d2, out_cnt);
}
extern "C" int flb_map_nearest_search_xyzi(flb_map* m, const float* q_xyz, int nq, int stride, int k, float max_dist,
                                           float* out_xyzi, float* out_d2, int* out_cnt) {
  return nearest_search_impl(m, q_xyz, nq, stride, k, max_dist, out_xyzi, 4, out_d2, out_cnt);
}

static int collect_common(flb_map* m, int mode, const float* params, int nparams, float* out_xyz, int cap, int* n_found, int out_w = 3) {
  if (n_found) *n_found = 0;
  CU(cudaSetDevice(m->cfg.device));
  if (fetch_counters(m)) return 1;
  const int nblk = blocks_bumped(m);
  if (nblk == 0) return 0;
  if (cap < 0) cap = 0;
  if (!out_xyz) cap = 0;
  if (cap > 0 && ensure_outbuf(m, cap)) return 1;
  if (nparams && upload_params(m, params, nparams)) return 1;
  CU(cudaMemsetAsync(m->d_misc, 0, sizeof(int), m->stream));
  k_collect<<<grid_for(nblk * 32, 256, m->sm_count * 8), 256, 0, m->stream>>>(m->d, nblk, mode, m->dparams.p, cap ? m->outbuf.p : nullptr, cap, m->d_misc);
  m->launches++;
  CU(cudaGetLastError());
  int total = 0;
  CU(cudaMemcpyAsync(&total, m->d_misc, sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  if (n_found) *n_found = total;
  const int w = std::min(total, cap);
  if (w > 0) {
    std::vector<float4> h(w);
    CU(cudaMemcpy(h.data(), m->outbuf.p, sizeof(float4) * w, cudaMemcpyDeviceToHost));
    if (out_w == 4) memcpy(out_xyz, h.data(), sizeof(float4) * (size_t)w);
    else for (int i = 0; i < w; ++i) { out_xyz[3 * i] = h[i].x; out_xyz[3 * i + 1] = h[i].y; out_xyz[3 * i + 2] = h[i].z; }
  }
  return 0;
}
extern "C" int flb_map_flatten_xyzi(flb_map* m, float* out_xyzi, int cap, int* n) {
  if (!m) return set_err("null map");
  return collect_common(m, 0, nullptr, 0, out_xyzi, cap, n, 4);
}
extern "C" int flb_map_box_search_xyzi(flb_map* m, const float* box6, float* out_xyzi, int cap, int* n_found) {
  if (!m || !box6) return set_err("null argument");
  return collect_common(m, 1, box6, 6, out_xyzi, cap, n_found, 4);
}
extern "C" int flb_map_radius_search_xyzi(flb_map* m, const float* c, float radius, float* out_xyzi, int cap, int* n_found) {
  if (!m || !c) return set_err("null argument");
  const float p[4] = {c[0], c[1], c[2], radius};
  return collect_common(m, 2, p, 4, out_xyzi, cap, n_found, 4);
}
extern "C" int flb_map_flatten(flb_map* m, float* out_xyz, int cap, int* n) {
  if (!m) return set_err("null map");
  return collect_common(m, 0, nullptr, 0, out_xyz, cap, n);
}
extern "C" int flb_map_box_search(flb_map* m, const float* box6, float* out_xyz, int cap, int* n_found) {
  if (!m || !box6) return set_err("null argument");
  return collect_common(m, 1, box6, 6, out_xyz, cap, n_found);
}
extern "C" int flb_map_radius_search(flb_map* m, const float* c, float radius, float* out_xyz, int cap, int* n_found) {
  if (!m || !c) return set_err("null argument");
  const float p[4] = {c[0], c[1], c[2], radius};
  return collect_common(m, 2, p, 4, out_xyz, cap, n_found);
}
extern "C" int flb_map_validnum(flb_map* m) {
  if (!m) return -1;
  if (cudaSetDevice(m->cfg.device) != cudaSuccess) return -1;
  if (fetch_counters(m)) return -1;
  return m->h_counters[CNT_VALID];
}
extern "C" int flb_map_size(flb_map* m) { return flb_map_validnum(m); }

extern "C" int flb_map_range(flb_map* m, float* box6) {
  if (!m || !box6) return set_err("null argument");
  CU(cudaSetDevice(m->cfg.device));
  if (fetch_counters(m)) return 1;
  const int nblk = blocks_bumped(m);
  int init[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
  CU(cudaMemcpyAsync(m->d_misc + 4, init, sizeof(init), cudaMemcpyHostToDevice, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  if (nblk) {
    k_range<<<grid_for(nblk * 32, 256, m->sm_count * 8), 256, 0, m->stream>>>(m->d, nblk, m->d_misc + 4);
    m->launches++;
  }
  int o[6];
  CU(cudaMemcpyAsync(o, m->d_misc + 4, sizeof(o), cudaMemcpyDeviceToHost, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  for (int i = 0; i < 6; ++i) {
    int v = o[i];
    if (v == INT_MAX || v == INT_MIN) { box6[i] = (i < 3) ? INFINITY : -INFINITY; continue; }
    int bits = v >= 0 ? v : v ^ 0x7FFFFFFF;
    memcpy(&box6[i], &bits, 4);
  }
  return 0;
}

extern "C" int flb_map_get_stats(flb_map* m, flb_map_stats* out) {
  if (!m || !out) return set_err("null argument");
  CU(cudaSetDevice(m->cfg.device));
  if (fetch_counters(m)) return 1;
  const int* c = m->h_counters;
  out->valid_points = c[CNT_VALID];
  out->blocks_in_use = std::min(c[CNT_BLK_BUMP], m->d.block_cap) - c[CNT_BLK_FREE];
  out->block_capacity = m->d.block_cap;
  out->overflow_in_use = std::min(c[CNT_OVF_BUMP], m->d.ovf_cap) - c[CNT_OVF_FREE];
  out->overflow_capacity = m->d.ovf_cap;
  out->hash_capacity = (int)m->hash_cap;
  out->hash_tombstones = c[CNT_KEYS_TOMB];
  out->coarse_cells = c[CNT_COARSE_USED];
  out->rehash_count = m->rehash_count;
  out->device_bytes = m->device_bytes;
  return 0;
}

extern "C" int flb_map_profile_enable(flb_map* m, int on) {
  if (!m) return set_err("null map");
  CU(cudaSetDevice(m->cfg.device));
  CU(cudaStreamSynchronize(m->stream));
  m->prof_on = on != 0;
  m->prof_used = 0;
  CU(cudaMemsetAsync(m->d_phase, 0, sizeof(int) * 8, m->stream));
  return 0;
}
extern "C" int flb_map_profile_read(flb_map* m, flb_profile* out, int reset) {
  if (!m || !out) return set_err("null argument");
  CU(cudaSetDevice(m->cfg.device));
  CU(cudaStreamSynchronize(m->stream));
  memset(out, 0, sizeof(*out));
  for (size_t i = 0; i < m->prof_used; ++i) {
    const auto& r = m->prof_pool[i];
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) != cudaSuccess) continue;
    if (r.cls >= 0 && r.cls < FLB_K_COUNT) { out->ms[r.cls] += ms; out->launches[r.cls] += r.nlaunch; out->regions[r.cls] += 1; }
  }
  int ph[8];
  CU(cudaMemcpy(ph, m->d_phase, sizeof(ph), cudaMemcpyDeviceToHost));
  for (int i = 0; i < 4; ++i) out->knn_phase[i] = ph[i];
  out->knn_chain_nodes = ph[4]; out->knn_chain_max = ph[5]; out->knn_head_candidates = ph[6];
  if (reset) { m->prof_used = 0; CU(cudaMemset(m->d_phase, 0, sizeof(int) * 8)); }
  return 0;
}

// A/B harness of the stencil 5-NN kernel variants (tools/knn_tile_ab.py; not on the product path): nq queries, `iters`
// timed launches (CUDA events on the map's stream) of variant 0 = k_knn_stencil<5>, 1 = k_knn_tile<5> (bulk-copy staged
// buckets).  out_d2[nq*5] / out_cnt[nq] (optional) return the variant's raw result (before the exact completion kernel).
extern "C" int flb_debug_knn_bench(flb_map* m, const float* q_xyz, int nq, int stride, int variant, int iters, float* ms_per_launch,
                                   int* unresolved, float* out_d2, int* out_cnt) {
  if (!m || !q_xyz || nq <= 0 || iters <= 0) return set_err("flb_debug_knn_bench: bad argument");
  CU(cudaSetDevice(m->cfg.device));
  if (upload_points(m, q_xyz, nq, stride)) return 1;
  if (ensure_outbuf(m, nq * 5)) return 1;
  if (ensure_worklist(m, nq)) return 1;
  unsigned char* dcnt = nullptr;
  CU(cudaMalloc((void**)&dcnt, nq));
  KnnArgs a;
  a.m = m->d; a.q = m->stage.p; a.n = nq; a.nbr = m->outbuf.p; a.cnt = dcnt; a.max_d2 = INFINITY; a.phase_stats = nullptr;
  a.worklist = m->worklist.p; a.work_count = m->d_misc + 12; a.work_ticket = m->d_misc + 13; a.stencil_done = m->d_misc + 14;
  a.exact_warps = exact_warps(m, 5); a.ctl = nullptr; a.body = nullptr; a.stride = nq;
  cudaError_t e = cudaFuncSetAttribute(k_knn_tile<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileSmem));
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (e == cudaSuccess) e = cudaEventCreate(&e0);
  if (e == cudaSuccess) e = cudaEventCreate(&e1);
  const int grid = (nq + 127) / 128;
  for (int it = -2; it < iters && e == cudaSuccess; ++it) {
    if (it == 0) e = cudaEventRecord(e0, m->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(a.work_count, 0, 3 * sizeof(int), m->stream);
    if (variant == 0) k_knn_stencil<5><<<grid, 128, 0, m->stream>>>(a);
    else k_knn_tile<5><<<grid, TILE_THREADS, sizeof(TileSmem), m->stream>>>(a);
    if (e == cudaSuccess) e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(e1, m->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
  // nothing consumed the list: leave it empty for the next search
  if (e == cudaSuccess) e = cudaMemsetAsync(m->worklist.p, 0xFF, m->worklist.cap, m->stream);
  float ms = 0.f;
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, e0, e1);
  if (ms_per_launch) *ms_per_launch = ms / (float)iters;
  if (e == cudaSuccess && unresolved) e = cudaMemcpy(unresolved, a.work_count, sizeof(int), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && out_d2) {
    std::vector<float4> h((size_t)nq * 5);
    e = cudaMemcpy(h.data(), m->outbuf.p, sizeof(float4) * h.size(), cudaMemcpyDeviceToHost);
    for (int i = 0; i < nq && e == cudaSuccess; ++i)
      for (int j = 0; j < 5; ++j) out_d2[(size_t)i * 5 + j] = h[(size_t)j * nq + i].w;
  }
  if (e == cudaSuccess && out_cnt) {
    std::vector<unsigned char> hc(nq);
    e = cudaMemcpy(hc.data(), dcnt, nq, cudaMemcpyDeviceToHost);
    for (int i = 0; i < nq; ++i) out_cnt[i] = hc[i];
  }
  cudaFree(dcnt);
  if (e0) cudaEventDestroy(e0);
  if (e1) cudaEventDestroy(e1);
  if (e != cudaSuccess) return set_err("flb_debug_knn_bench: %s", cudaGetErrorString(e));
  return 0;
}

// ------------------------------------------------------------------------------------------------ session
struct flb_session {
  flb_map* map = nullptr;
  flb_session_config cfg{};
  int cap = 0, n = 0;
  float4 *body = nullptr, *world = nullptr, *nbr = nullptr, *normvec = nullptr, *plane = nullptr;
  const float4* body_cur = nullptr;   // the current scan: `body` (uploads, front end) or the caller's device buffer (flb_scan_set_device)
  unsigned char *cnt = nullptr, *sel = nullptr, *cls = nullptr;
  double *partial = nullptr, *dout = nullptr;
  int* offs = nullptr;
  int* selint = nullptr;
  void* cub_tmp = nullptr;
  size_t cub_tmp_bytes = 0;
  DevBuf<double> drows;     // M x 13 export buffer, column-major, leading dimension = its row capacity (drows_ld)
  double* h_out = nullptr;  // pinned NACC
  int* h_cnt2 = nullptr;    // pinned 4 ints
  int* d_cnt2 = nullptr;
  int res_grid = 0;
  PoseDev last_pose{};
  bool have_pass = false;
  DevBuf<unsigned char> raw;     // staging of strided scan records
  // device-driven update
  EsikfCtl* ctl = nullptr;       // device
  EsikfCtl* h_ctl = nullptr;     // pinned scratch (initial upload of ctl)
  bool device_update = true;
  EsikfScratch* d_scr = nullptr;
  cudaStream_t side = nullptr;   // second stream: k_esikf_pre overlaps the measurement kernels of the same pass
  cudaEvent_t ev_fork[9] = {nullptr}, ev_join[9] = {nullptr};   // one pair per pass + [8] = the posterior's publish branch
  int graph_gen = -1;            // flb_map::gen the graphs of both slots were captured at
  // FLB_HOST_TIMING=1: where the host side of a step goes (printed when the session is destroyed)
  bool host_timing = false;
  double ht_begin = 0, ht_launch = 0, ht_wait = 0, ht_finish = 0, ht_between = 0;
  long ht_n = 0;
  std::chrono::steady_clock::time_point ht_last_finish{};
  bool use_graph = true;
  // double-buffered scan upload (flb_scan_prefetch)
  float4* body_alt = nullptr;
  DevBuf<unsigned char> raw_alt; // staging of strided prefetched records (on copy_stream)
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_copy = nullptr;
  int pending_n = -1;            // >= 0: a prefetched scan waits in body_alt
  bool flags_clean = false;      // sel / cnt hold their per-scan initial values (see scan_reset)
  // Up to TWO steps may be in flight (begin, begin, finish, begin, finish, ...): everything of a step that lives on the host —
  // pinned input / result records, the graphs whose copy nodes point at them, timing events, the step's bookkeeping —
  // exists once per slot, and every call works on slot[active] (cur).  Device buffers are shared: the steps execute one
  // after the other on the map's stream.
  struct StepSlot {
    double *h_x0P0 = nullptr, *d_x0P0 = nullptr;     // MAPPED pinned staging of a scan's inputs (k_esikf_begin reads it over
                                                     // PCIe), its device-side address
    StepResult *h_res = nullptr, *d_res = nullptr;   // MAPPED pinned result record written by k_publish, its device address
    cudaGraphExec_t graph[2] = {nullptr, nullptr};   // [0] update only, [1] update + map_incremental (no scan or host pointer
    int graph_kernels[2] = {0, 0};                   //  baked in beyond this slot's own staging / result records)
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
    // flb_scan_step_begin / _finish
    bool device = false, ev2_on = false;
    int l0 = 0, deleted = 0, flg = 1, n = 0;
    double x[26], P[NDOF * NDOF];
  } slot[2];
  int active = 0, head = 0, npending = 0;
};

static inline flb_session::StepSlot& cur(flb_session* s) { return s->slot[s->active]; }

extern "C" void flb_session_default_config(flb_session_config* c) {
  if (!c) return;
  c->max_scan_points = 131072;
  c->extrinsic_est_en = 0;
  c->max_iterations = 4;  // NUM_MAX_ITERATIONS default, laserMapping.cpp:2064
  c->laser_point_cov = 0.001;
  c->filter_size_map_min = 0.2;
  for (int i = 0; i < FLB_STATE_DOF; ++i) c->limit[i] = 0.001;
}

extern "C" int flb_session_create(flb_map* m, const flb_session_config* cfg, flb_session** out) {
  if (!m || !cfg || !out) return set_err("flb_session_create: null argument");
  if (cfg->max_scan_points <= 0) return set_err("max_scan_points must be > 0");
  // the scan sequence holds one pass per iteration plus the first (esekfom.hpp:1636 runs i = -1 .. max_iter-1), at most 8
  if (cfg->max_iterations < 0 || cfg->max_iterations > 7) return set_err("max_iterations must be in 0..7, got %d", cfg->max_iterations);
  CU(cudaSetDevice(m->cfg.device));
  flb_session* s = new (std::nothrow) flb_session();
  if (!s) return set_err("out of host memory");
  s->map = m;
  m->refs++;
  s->cfg = *cfg;
  s->cap = cfg->max_scan_points;
  const size_t N = (size_t)s->cap;
  cudaError_t e = cudaFuncSetAttribute(k_residual<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, meas_smem_bytes<true>());   // > 48 KB
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_residual<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, meas_smem_bytes<false>());
  // one partial per resident CTA (one per SM); the partial buffer and the final reductions follow
  if (e == cudaSuccess) {
    if (cfg->extrinsic_est_en) e = resident_ctas(k_residual<true>, meas_threads<true>(), meas_smem_bytes<true>(), m->sm_count, s->res_grid);
    else e = resident_ctas(k_residual<false>, meas_threads<false>(), meas_smem_bytes<false>(), m->sm_count, s->res_grid);
  }
  auto A = [&](void** p, size_t b) { if (e == cudaSuccess) e = cudaMalloc(p, b); };
  A((void**)&s->body, sizeof(float4) * N);
  A((void**)&s->body_alt, sizeof(float4) * N);
  A((void**)&s->world, sizeof(float4) * N);
  A((void**)&s->nbr, sizeof(float4) * N * 5);
  A((void**)&s->normvec, sizeof(float4) * N);
  A((void**)&s->plane, sizeof(float4) * N);
  A((void**)&s->cnt, N);
  A((void**)&s->sel, N);
  A((void**)&s->cls, N);
  A((void**)&s->partial, sizeof(double) * NACC * (size_t)s->res_grid);
  A((void**)&s->dout, sizeof(double) * NACC);
  A((void**)&s->offs, sizeof(int) * N);
  A((void**)&s->selint, sizeof(int) * N);
  A((void**)&s->d_cnt2, sizeof(int) * 8);
  A((void**)&s->ctl, sizeof(EsikfCtl));
  A((void**)&s->d_scr, sizeof(EsikfScratch));
  if (e == cudaSuccess) e = cudaMemset(s->d_cnt2, 0, sizeof(int) * 8);   // [0..1] map_incremental counts
  if (e == cudaSuccess) e = cudaMallocHost((void**)&s->h_ctl, sizeof(EsikfCtl));
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->side, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->copy_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->ev_copy, cudaEventDisableTiming);
  for (int i = 0; i < 9 && e == cudaSuccess; ++i) {
    e = cudaEventCreateWithFlags(&s->ev_fork[i], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->ev_join[i], cudaEventDisableTiming);
  }
  if (e == cudaSuccess) e = cudaMallocHost((void**)&s->h_out, sizeof(double) * NACC);
  if (e == cudaSuccess) e = cudaMallocHost((void**)&s->h_cnt2, sizeof(int) * 8);
  if (e == cudaSuccess) {
    size_t tb = 0;
    e = cub::DeviceScan::ExclusiveSum(nullptr, tb, s->selint, s->offs, s->cap, m->stream);
    s->cub_tmp_bytes = tb;
    A(&s->cub_tmp, tb ? tb : 16);
  }
  if (e == cudaSuccess) {
    memset(s->h_ctl, 0, sizeof(EsikfCtl));
    for (int i = 0; i < NDOF; ++i) s->h_ctl->limit[i] = cfg->limit[i];
    s->h_ctl->R = cfg->laser_point_cov;
    s->h_ctl->max_iter = cfg->max_iterations;
    s->h_ctl->finished = 1;
    e = cudaMemcpy(s->ctl, s->h_ctl, sizeof(EsikfCtl), cudaMemcpyHostToDevice);
  }
  // per-step host records (two slots: two steps may be in flight): mapped pinned staging + result, timing events
  for (int j = 0; j < 2 && e == cudaSuccess; ++j) {
    flb_session::StepSlot& w = s->slot[j];
    e = cudaHostAlloc((void**)&w.h_x0P0, sizeof(double) * (26 + NDOF * NDOF + 4), cudaHostAllocMapped);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer((void**)&w.d_x0P0, w.h_x0P0, 0);
    if (e == cudaSuccess) e = cudaHostAlloc((void**)&w.h_res, sizeof(StepResult), cudaHostAllocMapped);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer((void**)&w.d_res, w.h_res, 0);
    if (e == cudaSuccess) { memset(w.h_x0P0, 0, sizeof(double) * (26 + NDOF * NDOF + 4)); memset(w.h_res, 0, sizeof(StepResult)); }
    if (e == cudaSuccess) e = cudaEventCreate(&w.ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&w.ev1);
    if (e == cudaSuccess) e = cudaEventCreate(&w.ev2);
    if (e == cudaSuccess) e = cudaEventCreate(&w.ev3);
  }
  s->body_cur = s->body;
  if (e != cudaSuccess) { flb_session_destroy(s); return set_err("flb_session_create: %s", cudaGetErrorString(e)); }
  if (const char* ht = getenv("FLB_HOST_TIMING")) s->host_timing = atoi(ht) != 0;
  *out = s;
  return 0;
}

extern "C" void flb_session_destroy(flb_session* s) {
  if (!s) return;
  if (s->host_timing && s->ht_n > 0)
    fprintf(stderr, "[fastlio_b200] host timing over %ld steps (us/step): begin() %.1f (of which graph launch %.1f), finish(): wait %.1f + rest %.1f, "
            "caller between finish and next begin %.1f\n", s->ht_n, 1e6 * s->ht_begin / s->ht_n, 1e6 * s->ht_launch / s->ht_n,
            1e6 * s->ht_wait / s->ht_n, 1e6 * s->ht_finish / s->ht_n, 1e6 * s->ht_between / s->ht_n);
  Q(cudaSetDevice(s->map->cfg.device));
  Q(cudaStreamSynchronize(s->map->stream));
  if (s->side) Q(cudaStreamSynchronize(s->side));
  if (s->copy_stream) Q(cudaStreamSynchronize(s->copy_stream));
  for (const flb_session::StepSlot& w : s->slot) {
    for (cudaGraphExec_t g : w.graph) if (g) Q(cudaGraphExecDestroy(g));
    if (w.h_x0P0) Q(cudaFreeHost(w.h_x0P0));
    if (w.h_res) Q(cudaFreeHost(w.h_res));
    for (cudaEvent_t e : {w.ev0, w.ev1, w.ev2, w.ev3}) if (e) Q(cudaEventDestroy(e));
  }
  void* ptrs[] = {s->body, s->body_alt, s->world, s->nbr, s->normvec, s->plane, s->cnt, s->sel, s->cls, s->partial, s->dout, s->offs, s->selint,
                  s->cub_tmp, s->d_cnt2, s->ctl, s->d_scr};
  for (void* p : ptrs) if (p) Q(cudaFree(p));
  if (s->h_out) Q(cudaFreeHost(s->h_out));
  if (s->h_cnt2) Q(cudaFreeHost(s->h_cnt2));
  if (s->h_ctl) Q(cudaFreeHost(s->h_ctl));
  if (s->ev_copy) Q(cudaEventDestroy(s->ev_copy));
  for (int i = 0; i < 9; ++i) {
    if (s->ev_fork[i]) Q(cudaEventDestroy(s->ev_fork[i]));
    if (s->ev_join[i]) Q(cudaEventDestroy(s->ev_join[i]));
  }
  if (s->side) Q(cudaStreamDestroy(s->side));
  if (s->copy_stream) Q(cudaStreamDestroy(s->copy_stream));
  flb_map* m = s->map;
  delete s;
  map_release(m);
}

extern "C" int flb_session_set_update_engine(flb_session* s, int device_driven) {
  if (!s) return set_err("null session");
  s->device_update = device_driven != 0;
  return 0;
}
extern "C" void* flb_session_stream(flb_session* s) { return s ? (void*)s->map->stream : nullptr; }
extern "C" int flb_session_sync(flb_session* s) {
  if (!s) return set_err("null session");
  CU(cudaStreamSynchronize(s->map->stream));
  return 0;
}

static int scan_flags_reset(flb_session* s) {
  // memset(point_selected_surf, true) (laserMapping.cpp:2131); Nearest_Points empty
  CU(cudaMemsetAsync(s->sel, 1, (size_t)std::max(s->n, 1), s->map->stream));
  CU(cudaMemsetAsync(s->cnt, 0, (size_t)std::max(s->n, 1), s->map->stream));
  s->flags_clean = true;
  return 0;
}
static int scan_reset(flb_session* s, int n) {
  s->n = n;
  s->body_cur = s->body;
  s->have_pass = false;
  s->flags_clean = false;
  // The device-driven sequence always starts with a search pass (esekfom.hpp:1636: converge = true), which rewrites cnt
  // (k_knn_stencil) and sel (k_residual) for every point: the two memsets are only needed by the host-driven entry points
  // (flb_pass may be asked for a cached pass first), which request them on demand.
  if (!s->device_update) return scan_flags_reset(s);
  return 0;
}

extern "C" int flb_scan_upload_pt(flb_session* s, const void* pts, int n, int stride, int off_i) {
  if (!s) return set_err("null session");
  if (n < 0 || n > s->cap) return set_err("scan of %d points exceeds max_scan_points=%d", n, s->cap);
  if (n > 0 && (!pts || stride < 12)) return set_err("bad scan buffer");
  if (off_i >= 0 && off_i + 4 > stride) return set_err("intensity offset %d outside the %d-byte record", off_i, stride);
  CU(cudaSetDevice(s->map->cfg.device));
  flb_map* m = s->map;
  if (stride == 16 && off_i < 0) off_i = 12;
  // (the staging is sized once for the session capacity)
  if (n > 0 && upload_records(m, m->stream, s->raw, (size_t)s->cap * (size_t)stride, pts, n, stride, off_i, -1, s->body, nullptr)) return 1;
  return scan_reset(s, n);
}
// (the 4th float of a 16-byte record is carried as the point's intensity into the map; other strides: no intensity)
extern "C" int flb_scan_upload(flb_session* s, const float* xyz, int n, int stride) { return flb_scan_upload_pt(s, xyz, n, stride, -1); }

extern "C" int flb_scan_prefetch(flb_session* s, const float* xyz, int n, int stride) {
  if (!s) return set_err("null session");
  if (n < 0 || n > s->cap) return set_err("scan of %d points exceeds max_scan_points=%d", n, s->cap);
  if (n > 0 && (!xyz || (stride != 12 && stride != 16))) return set_err("flb_scan_prefetch: stride must be 12 or 16");
  CU(cudaSetDevice(s->map->cfg.device));
  flb_map* m = s->map;
  if (n > 0) {
    // a 16-byte record carries its intensity, as for flb_scan_upload; the previous prefetch may still read raw_alt
    if (stride == 12 && (size_t)n * 12 > s->raw_alt.cap) CU(cudaStreamSynchronize(s->copy_stream));
    if (upload_records(m, s->copy_stream, s->raw_alt, (size_t)1 << 20, xyz, n, stride, stride == 16 ? 12 : -1, -1, s->body_alt, nullptr))
      return 1;
  }
  CU(cudaEventRecord(s->ev_copy, s->copy_stream));
  s->pending_n = n;
  return 0;
}
// make a prefetched scan current: the processing stream waits for the copy, then the two body buffers swap roles
static int adopt_prefetched(flb_session* s) {
  if (s->pending_n < 0) return 0;
  CU(cudaStreamWaitEvent(s->map->stream, s->ev_copy, 0));
  std::swap(s->body, s->body_alt);
  const int n = s->pending_n;
  s->pending_n = -1;
  return scan_reset(s, n);
}

extern "C" int flb_scan_set_device(flb_session* s, const void* body4_dev, int n) {
  if (!s) return set_err("null session");
  if (n < 0 || n > s->cap) return set_err("scan of %d points exceeds max_scan_points=%d", n, s->cap);
  if (n > 0 && !body4_dev) return set_err("null device buffer");
  CU(cudaSetDevice(s->map->cfg.device));
  // no copy: the scan is read in place (the pointer travels with the staged inputs of the step).  The buffer must stay
  // valid and unmodified until the last call that works on this scan has returned (flb_scan_step_finish / flb_map_incremental).
  if (scan_reset(s, n)) return 1;
  if (n > 0) s->body_cur = static_cast<const float4*>(body4_dev);
  return 0;
}

static PoseDev pose_from(const double* st) {
  PoseDev p;
  for (int i = 0; i < 4; ++i) { p.rot[i] = st[3 + i]; p.offR[i] = st[7 + i]; }
  for (int i = 0; i < 3; ++i) { p.pos[i] = st[i]; p.offT[i] = st[11 + i]; }
  return p;
}

static MeasArgs meas_args(flb_session* s, const PoseDev& pose, int search) {
  MeasArgs a;
  a.pose = pose; a.body = s->body_cur; a.world = s->world; a.nbr = s->nbr; a.cnt = s->cnt; a.sel = s->sel;
  a.normvec = s->normvec; a.plane = s->plane; a.partial = s->partial; a.n = s->n; a.search = search;
  a.ctl = nullptr; a.world_out = s->world; a.stride = s->cap;
  return a;
}

// enqueue one pass (no sync). The reduced result lands in s->h_out after the stream drains.
static int enqueue_pass(flb_session* s, const double* state26, int search) {
  flb_map* m = s->map;
  cudaStream_t st = m->stream;
  const int n = s->n;
  const PoseDev pose = pose_from(state26);
  s->last_pose = pose;
  {
    ProfScope ps(m, FLB_K_TRANSFORM);
    k_transform<<<grid_for(n, 256, m->sm_count * 8), 256, 0, st>>>(pose, s->body_cur, s->world, n);
    m->launches++;
  }
  if (search) {
    ProfScope ps(m, FLB_K_KNN);
    KnnArgs a;
    a.m = m->d; a.q = s->world; a.n = n; a.nbr = s->nbr; a.cnt = s->cnt; a.max_d2 = INFINITY;
    a.phase_stats = m->prof_on ? m->d_phase : nullptr;
    a.ctl = nullptr; a.body = nullptr; a.stride = s->cap; a.work_count = nullptr;
    if (launch_knn<5>(m, a)) return 1;
  }
  const MeasArgs ma = meas_args(s, pose, search);
  {
    ProfScope ps(m, FLB_K_RESIDUAL);
    if (s->cfg.extrinsic_est_en) k_residual<true><<<s->res_grid, meas_threads<true>(), meas_smem_bytes<true>(), st>>>(ma);
    else k_residual<false><<<s->res_grid, meas_threads<false>(), meas_smem_bytes<false>(), st>>>(ma);
    m->launches++;
  }
  {
    ProfScope ps(m, FLB_K_REDUCE);
    k_reduce_final<<<1, 384, 0, st>>>(s->partial, s->res_grid, s->dout);
    m->launches++;
  }
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(s->h_out, s->dout, sizeof(double) * NACC, cudaMemcpyDeviceToHost, st));
  s->have_pass = true;
  return 0;
}

static void unpack_result(const double* o, flb_pass_result* r) {
  auto slot = [](int i, int j) { return i * 13 - i * (i - 1) / 2 + (j - i); };
  for (int i = 0; i < 12; ++i) {
    for (int j = i; j < 12; ++j) { r->HTH[i * 12 + j] = o[slot(i, j)]; r->HTH[j * 12 + i] = o[slot(i, j)]; }
    r->HTh[i] = o[slot(i, 12)];
  }
  r->total_residual = o[91];
  r->effct_feat_num = (int)(o[92] + 0.5);
  r->valid = r->effct_feat_num >= 1;
}

extern "C" int flb_pass(flb_session* s, const double* state26, int search, flb_pass_result* out) {
  if (!s || !state26 || !out) return set_err("flb_pass: null argument");
  CU(cudaSetDevice(s->map->cfg.device));
  memset(out, 0, sizeof(*out));
  if (s->n <= 0) { out->valid = 0; return 0; }
  if (!s->flags_clean && !s->have_pass && scan_flags_reset(s)) return 1;
  if (enqueue_pass(s, state26, search)) return 1;
  CU(cudaStreamSynchronize(s->map->stream));
  unpack_result(s->h_out, out);
  return 0;
}

// rows the export buffer holds: the leading dimension of its columns
static inline int drows_ld(const flb_session* s) { return (int)(s->drows.cap / (sizeof(double) * 13)); }

// device export of rows in index order; returns M
static int export_rows(flb_session* s, int M_expected) {
  flb_map* m = s->map;
  cudaStream_t st = m->stream;
  const int n = s->n;
  if (grow(s->drows, sizeof(double) * 13 * (size_t)M_expected, sizeof(double) * 13 * ((size_t)1 << 14))) return 1;
  const int g = grid_for(n, 256, m->sm_count * 8);
  k_sel_to_int<<<g, 256, 0, st>>>(s->sel, s->selint, n);
  size_t tb = s->cub_tmp_bytes;
  CU(cub::DeviceScan::ExclusiveSum(s->cub_tmp, tb, s->selint, s->offs, n, st));
  const MeasArgs ma = meas_args(s, s->last_pose, 0);
  const int ld = drows_ld(s);
  if (s->cfg.extrinsic_est_en) k_rows<true><<<g, 256, 0, st>>>(ma, s->offs, s->drows.p, ld, s->drows.p + (size_t)12 * ld, ld);
  else k_rows<false><<<g, 256, 0, st>>>(ma, s->offs, s->drows.p, ld, s->drows.p + (size_t)12 * ld, ld);
  m->launches += 3;
  CU(cudaGetLastError());
  return 0;
}

extern "C" int flb_pass_rows(flb_session* s, double* hx, int ld, double* h, int capacity_rows, int* M) {
  if (!s || !M) return set_err("flb_pass_rows: null argument");
  if (!s->have_pass) return set_err("flb_pass_rows: no preceding flb_pass for this scan");
  CU(cudaSetDevice(s->map->cfg.device));
  const int Mexp = (int)(s->h_out[92] + 0.5);
  *M = Mexp;
  if (Mexp == 0) return 0;
  if (capacity_rows < Mexp || ld < Mexp) return set_err("flb_pass_rows: capacity %d / ld %d < M = %d", capacity_rows, ld, Mexp);
  if (export_rows(s, Mexp)) return 1;
  cudaStream_t st = s->map->stream;
  const int dl = drows_ld(s);
  if (hx) CU(cudaMemcpy2DAsync(hx, sizeof(double) * ld, s->drows.p, sizeof(double) * dl, sizeof(double) * Mexp, 12, cudaMemcpyDeviceToHost, st));
  if (h) CU(cudaMemcpyAsync(h, s->drows.p + (size_t)12 * dl, sizeof(double) * Mexp, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return 0;
}

static int run_update(flb_session* s, double* state26, double* P, flb_update_stats* stats) {
  flb_map* m = s->map;
  if (!s->flags_clean && scan_flags_reset(s)) return 1;
  host::IteratedUpdate u(state26, P, s->cfg.laser_point_cov, s->cfg.max_iterations, s->cfg.limit);
  int passes = 0, searches = 0, lastM = 0;
  double lastres = 0;
  const flb_session::StepSlot& w = cur(s);
  CU(cudaEventRecord(w.ev0, m->stream));
  while (u.more()) {
    double cur[26];
    u.current_state(cur);
    const int search = u.need_search() ? 1 : 0;
    flb_pass_result r;
    if (s->n <= 0) { u.skip(); ++passes; continue; }
    if (enqueue_pass(s, cur, search)) return 1;
    CU(cudaStreamSynchronize(m->stream));
    unpack_result(s->h_out, &r);
    ++passes;
    searches += search;
    if (!r.valid) { u.skip(); continue; }
    lastM = r.effct_feat_num;
    lastres = r.total_residual;
    if (r.effct_feat_num >= host::DOF) {
      u.step(r.HTH, r.HTh);
    } else {
      // rare under-determined branch (esekfom.hpp:1720-1750) needs the explicit rows
      const int M = r.effct_feat_num;
      if (export_rows(s, M)) return 1;
      std::vector<double> cm((size_t)13 * M), rows((size_t)12 * M), hv(M);
      const int dl = drows_ld(s);
      CU(cudaMemcpy2DAsync(cm.data(), sizeof(double) * M, s->drows.p, sizeof(double) * dl, sizeof(double) * M, 13, cudaMemcpyDeviceToHost, m->stream));
      CU(cudaStreamSynchronize(m->stream));
      for (int r_ = 0; r_ < M; ++r_) { for (int c = 0; c < 12; ++c) rows[(size_t)r_ * 12 + c] = cm[(size_t)c * M + r_]; hv[r_] = cm[(size_t)12 * M + r_]; }
      u.step_rows(rows.data(), hv.data(), M);
    }
  }
  CU(cudaEventRecord(w.ev1, m->stream));
  u.result(state26, P);
  if (stats) {
    stats->passes = passes; stats->search_passes = searches; stats->effct_feat_num = lastM;
    stats->converged_count = u.converged_count(); stats->total_residual = lastres;
    CU(cudaEventSynchronize(w.ev1));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, w.ev0, w.ev1));
    stats->gpu_ms = ms;
  }
  return 0;
}


static int enqueue_map_incremental(flb_session* s, const double* state26, int flg_EKF_inited, bool from_ctl, bool tail_publish = false);

// Device-driven scan: every pass of the iterated update (and optionally map_incremental) is enqueued up front; kernels
// of passes that turn out not to be needed exit on the device-side loop flags.  No host round trip inside.  Launch
// geometry depends only on the session capacity (the scan size n travels in the staging buffer), so the identical
// sequence can be captured once into a CUDA graph.  k_esikf_pre of each pass runs on the side stream next to the
// measurement kernels of that pass (fork/join by events, which become graph edges under capture).
static int enqueue_scan_device(flb_session* s, bool with_insert) {
  flb_map* m = s->map;
  cudaStream_t st = m->stream;
  const bool overlap = !m->prof_on;  // per-class event timing needs a single in-order stream
  const bool md12 = s->cfg.extrinsic_est_en != 0;   // measured subspace: 12 columns with extrinsic estimation, else 6
  const int cap = s->cap;
  const flb_session::StepSlot& w = cur(s);
  launch_k(k_esikf_begin, 1, 256, 0, st, s->ctl, (const double*)w.d_x0P0, m->d_misc + 16);   // reads the mapped pinned staging record
  m->launches++;
  for (int p = 0; p <= s->cfg.max_iterations; ++p) {
    if (overlap) {
      CU(cudaEventRecord(s->ev_fork[p], st));
      CU(cudaStreamWaitEvent(s->side, s->ev_fork[p], 0));
      if (md12) k_esikf_pre<12><<<1, dev::ESIKF_THREADS, 0, s->side>>>(s->ctl, s->d_scr);
      else k_esikf_pre<6><<<1, dev::ESIKF_THREADS, 0, s->side>>>(s->ctl, s->d_scr);
      if (p == 0 && with_insert) {
        // the insert's scratch hash and counters are cleared here, next to the first pass, instead of between the
        // insert kernels at the end of the scan (three memset nodes off the critical path)
        if (!m->capturing && ensure_scratch(m, cap)) return 1;
        const uint32_t sc = scratch_slots(cap);
        CU(cudaMemsetAsync(m->skeys.p, 0xFF, sizeof(uint64_t) * sc, s->side));
        CU(cudaMemsetAsync(m->sbest.p, 0xFF, sizeof(unsigned long long) * sc, s->side));
        CU(cudaMemsetAsync(s->d_cnt2, 0, sizeof(int) * 2, s->side));
        m->scratch_clean = true;
      }
      CU(cudaEventRecord(s->ev_join[p], s->side));
    } else {
      ProfScope ps(m, FLB_K_REDUCE);
      if (md12) k_esikf_pre<12><<<1, dev::ESIKF_THREADS, 0, st>>>(s->ctl, s->d_scr);
      else k_esikf_pre<6><<<1, dev::ESIKF_THREADS, 0, st>>>(s->ctl, s->d_scr);
    }
    m->launches++;
    {
      ProfScope ps(m, FLB_K_KNN);
      KnnArgs a;
      a.m = m->d; a.q = nullptr; a.n = cap; a.nbr = s->nbr; a.cnt = s->cnt; a.max_d2 = INFINITY;
      a.phase_stats = m->prof_on ? m->d_phase : nullptr;
      a.ctl = s->ctl; a.body = nullptr; a.stride = cap; a.work_count = p < 8 ? m->d_misc + 16 + p : nullptr; a.work_ticket = p < 8 ? m->d_misc + 24 + p : nullptr;
      a.stencil_done = p < 8 ? m->d_misc + 32 + p : nullptr;
      if (launch_knn<5>(m, a)) return 1;
    }
    {
      ProfScope ps(m, FLB_K_RESIDUAL);
      MeasArgs ma = meas_args(s, PoseDev{}, 0);
      ma.ctl = s->ctl;
      if (s->cfg.extrinsic_est_en) launch_k(k_residual<true>, s->res_grid, meas_threads<true>(), meas_smem_bytes<true>(), st, ma);
      else launch_k(k_residual<false>, s->res_grid, meas_threads<false>(), meas_smem_bytes<false>(), st, ma);
      m->launches++;
    }
    if (overlap) CU(cudaStreamWaitEvent(st, s->ev_join[p], 0));
    {
      ProfScope ps(m, FLB_K_REDUCE);
      if (md12) launch_k(k_esikf_post<12>, 1, dev::ESIKF_THREADS, 0, st, s->ctl, (const double*)s->partial, s->res_grid, s->d_scr);
      else launch_k(k_esikf_post<6>, 1, dev::ESIKF_THREADS, 0, st, s->ctl, (const double*)s->partial, s->res_grid, s->d_scr);
      m->launches++;
    }
  }
  CU(cudaGetLastError());
  // results go into ONE mapped pinned record (posterior, statistics, map counters, map_incremental's counts).  With an
  // insert behind the update, the posterior is published on the side branch next to the insert kernels and the counters
  // by the last block of the last insert kernel; otherwise one kernel writes everything.
  const bool tail_publish = overlap && with_insert && s->cap > 0;
  if (tail_publish) {
    CU(cudaEventRecord(s->ev_fork[8], st));
    CU(cudaStreamWaitEvent(s->side, s->ev_fork[8], 0));
    k_publish<<<1, 256, 0, s->side>>>((const EsikfCtl*)s->ctl, nullptr, nullptr, w.d_res, 0);
    CU(cudaEventRecord(s->ev_join[8], s->side));
    m->launches++;
  }
  if (with_insert && enqueue_map_incremental(s, nullptr, 0, true, tail_publish)) return 1;
  if (tail_publish) CU(cudaStreamWaitEvent(st, s->ev_join[8], 0));
  else {
    launch_k(k_publish, 1, 256, 0, st, (const EsikfCtl*)s->ctl, (const int*)m->d.counters, (const int*)(with_insert ? s->d_cnt2 : nullptr), w.d_res, 1);
    m->launches++;
  }
  CU(cudaGetLastError());
  s->have_pass = false;
  return 0;
}

// Stage a scan's inputs and run the device-driven sequence, through a CUDA graph when possible.
static int launch_scan_device(flb_session* s, const double* state26, const double* P, int flg_EKF_inited, bool with_insert) {
  flb_map* m = s->map;
  flb_session::StepSlot& w = cur(s);
  double* x0P0 = w.h_x0P0;
  memcpy(x0P0, state26, sizeof(double) * 26);
  memcpy(x0P0 + 26, P, sizeof(double) * NDOF * NDOF);
  x0P0[26 + NDOF * NDOF] = (double)s->n;
  x0P0[26 + NDOF * NDOF + 1] = (double)flg_EKF_inited;
  {
    const unsigned long long bits = (unsigned long long)reinterpret_cast<uintptr_t>(s->body_cur);
    memcpy(&x0P0[26 + NDOF * NDOF + 2], &bits, sizeof(bits));
  }
  const int gi = with_insert ? 1 : 0;
  if (!s->use_graph || m->prof_on) return enqueue_scan_device(s, with_insert);
  if (s->graph_gen != m->gen) {
    // a buffer baked into the captured sequences was reallocated (or the voxel size changed) since: capture again
    for (flb_session::StepSlot& o : s->slot)
      for (cudaGraphExec_t& g : o.graph)
        if (g) { Q(cudaGraphExecDestroy(g)); g = nullptr; }
    s->graph_gen = m->gen;   // (both slots start over: graphs are re-captured lazily, the first capture stamps this again)
  }
  if (!w.graph[gi]) {
    // everything the captured sequence may allocate lazily must exist before capture
    if (ensure_scratch(m, s->cap) || ensure_worklist(m, s->cap)) return 1;
    CU(cudaStreamSynchronize(m->stream));
    const int l0 = m->launches;
    cudaGraph_t g = nullptr;
    CU(cudaStreamBeginCapture(m->stream, cudaStreamCaptureModeThreadLocal));
    m->capturing = true;
    const int rc = enqueue_scan_device(s, with_insert);
    m->capturing = false;
    cudaError_t ce = cudaStreamEndCapture(m->stream, &g);
    if (rc || ce != cudaSuccess || !g) {
      if (g) cudaGraphDestroy(g);
      cudaGetLastError();
      s->use_graph = false;  // fall back to direct launches (same kernels)
      m->launches = l0;
      return enqueue_scan_device(s, with_insert);
    }
    ce = cudaGraphInstantiate(&w.graph[gi], g, 0);
    cudaGraphDestroy(g);
    if (ce != cudaSuccess) {
      cudaGetLastError();
      w.graph[gi] = nullptr; s->use_graph = false; m->launches = l0;
      return enqueue_scan_device(s, with_insert);
    }
    w.graph_kernels[gi] = m->launches - l0;
    m->launches = l0;
    s->graph_gen = m->gen;
  }
  CU(cudaGraphLaunch(w.graph[gi], m->stream));
  m->launches += w.graph_kernels[gi];
  return 0;
}
static int finish_counters(flb_map* m, const int* snapshot) {  // after the sequence completed: interpret the counters it copied
  memcpy(m->h_counters, snapshot, sizeof(int) * CNT_COUNT);
  const int e = absorb_range_flag(m);
  if (e) return set_err("device map error flags 0x%x (capacity exceeded or point out of range; see flb_map_get_stats)", e);
  return 0;
}
static void stats_from_ctl(const StepResult* c, flb_update_stats* stats) {
  if (!stats) return;
  stats->passes = c->passes; stats->search_passes = c->searches; stats->effct_feat_num = c->lastM;
  stats->converged_count = c->t; stats->total_residual = c->last_res;
}

extern "C" int flb_esikf_update(flb_session* s, double* state26, double* P, flb_update_stats* stats) {
  if (!s || !state26 || !P) return set_err("flb_esikf_update: null argument");
  if (s->npending) return set_err("flb_esikf_update: a flb_scan_step is in flight");
  CU(cudaSetDevice(s->map->cfg.device));
  if (adopt_prefetched(s)) return 1;
  if (!s->device_update) return run_update(s, state26, P, stats);
  flb_map* m = s->map;
  const flb_session::StepSlot& w = cur(s);
  CU(cudaEventRecord(w.ev0, m->stream));
  if (launch_scan_device(s, state26, P, 1, false)) return 1;
  CU(cudaEventRecord(w.ev1, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  if (finish_counters(m, w.h_res->counters)) return 1;
  if (w.h_res->need_host) return run_update(s, state26, P, stats);  // M < 23: explicit-row branch on the host
  memcpy(state26, w.h_res->x, sizeof(double) * 26);
  memcpy(P, w.h_res->P, sizeof(double) * NDOF * NDOF);
  stats_from_ctl(w.h_res, stats);
  if (stats) CU(cudaEventElapsedTime(&stats->gpu_ms, w.ev0, w.ev1));
  return 0;
}

static int enqueue_map_incremental(flb_session* s, const double* state26, int flg_EKF_inited, bool from_ctl, bool tail_publish) {
  flb_map* m = s->map;
  cudaStream_t st = m->stream;
  const int n = s->n;
  if (n <= 0 && !from_ctl) return 0;
  const PoseDev pose = from_ctl ? PoseDev{} : pose_from(state26);
  const int npts = from_ctl ? s->cap : n;   // launch geometry / scratch size (the device count is read by the kernels)
  const uint32_t sc = scratch_slots(npts);
  if (!m->scratch_clean) {
    // (inside the captured scan sequence these clears sit on the side branch of the first pass)
    if (!m->capturing && ensure_scratch(m, npts)) return 1;
    CU(cudaMemsetAsync(s->d_cnt2, 0, sizeof(int) * 2, st));
    CU(cudaMemsetAsync(m->skeys.p, 0xFF, sizeof(uint64_t) * sc, st));
    CU(cudaMemsetAsync(m->sbest.p, 0xFF, sizeof(unsigned long long) * sc, st));
  }
  {
    ProfScope ps(m, FLB_K_CLASSIFY);
    launch_k(k_classify, grid_for(npts, 256, m->sm_count * 8), 256, 0, st, pose, (const EsikfCtl*)(from_ctl ? s->ctl : nullptr),
             (const float4*)s->body_cur, (const float4*)s->nbr, (const unsigned char*)s->cnt, n, s->cap, flg_EKF_inited, s->cfg.filter_size_map_min,
             s->world, s->cls, s->d_cnt2, m->d, m->skeys.p, m->sbest.p, sc - 1);
    m->launches++;
  }
  CU(cudaGetLastError());
  if (from_ctl) {
    StepTail tail{};
    if (tail_publish) {
      // the last block of the last insert kernel writes the map counters, map_incremental's counts and the step's device
      // span into the mapped pinned result record: no separate publishing kernel after the insert
      tail.ticket = s->d_cnt2 + 2; tail.counters = m->d.counters; tail.cnt2 = s->d_cnt2; tail.t_begin = &s->ctl->t_begin;
      StepResult* res = cur(s).d_res;
      tail.out_counters = res->counters; tail.out_cnt2 = res->cnt2; tail.out_span = &res->span_ns;
    }
    if (insert_device(m, s->world, s->cls, s->cap, 2, &s->ctl->need_host, &s->ctl->n, true, tail)) return 1;
  } else if (insert_device(m, s->world, s->cls, n, 2, nullptr, nullptr, true)) return 1;
  if (!from_ctl) CU(cudaMemcpyAsync(s->h_cnt2, s->d_cnt2, sizeof(int) * 2, cudaMemcpyDeviceToHost, st));   // (k_publish carries them otherwise)
  return 0;
}

extern "C" int flb_map_incremental(flb_session* s, const double* state26, int flg_EKF_inited, int* n_to_add, int* n_no_ds) {
  if (!s || !state26) return set_err("flb_map_incremental: null argument");
  CU(cudaSetDevice(s->map->cfg.device));
  if (n_to_add) *n_to_add = 0;
  if (n_no_ds) *n_no_ds = 0;
  if (s->n <= 0) return 0;
  if (enqueue_map_incremental(s, state26, flg_EKF_inited, false)) return 1;
  if (fetch_counters(s->map)) return 1;
  if (n_to_add) *n_to_add = s->h_cnt2[0];
  if (n_no_ds) *n_no_ds = s->h_cnt2[1];
  return 0;
}

extern "C" int flb_neighbors_download(flb_session* s, float* nbr_xyz, float* nbr_d2, int* nbr_cnt, unsigned char* selected,
                                      float* normvec, float* world_xyz) {
  if (!s) return set_err("null session");
  CU(cudaSetDevice(s->map->cfg.device));
  const int n = s->n;
  if (n <= 0) return 0;
  cudaStream_t st = s->map->stream;
  std::vector<float4> h4;
  std::vector<unsigned char> hc(n);
  if (nbr_xyz || nbr_d2) {
    h4.resize((size_t)5 * s->cap);
    CU(cudaMemcpyAsync(h4.data(), s->nbr, sizeof(float4) * h4.size(), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(hc.data(), s->cnt, n, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < 5; ++j) {
        const bool ok = j < hc[i];
        const float4 v = h4[(size_t)j * s->cap + i];
        if (nbr_xyz) { nbr_xyz[((size_t)i * 5 + j) * 3] = ok ? v.x : NAN; nbr_xyz[((size_t)i * 5 + j) * 3 + 1] = ok ? v.y : NAN; nbr_xyz[((size_t)i * 5 + j) * 3 + 2] = ok ? v.z : NAN; }
        if (nbr_d2) nbr_d2[(size_t)i * 5 + j] = ok ? v.w : INFINITY;
      }
  }
  if (nbr_cnt) {
    CU(cudaMemcpyAsync(hc.data(), s->cnt, n, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) nbr_cnt[i] = hc[i];
  }
  if (selected) { CU(cudaMemcpyAsync(selected, s->sel, n, cudaMemcpyDeviceToHost, st)); CU(cudaStreamSynchronize(st)); }
  if (normvec) { CU(cudaMemcpyAsync(normvec, s->normvec, sizeof(float4) * (size_t)n, cudaMemcpyDeviceToHost, st)); CU(cudaStreamSynchronize(st)); }
  if (world_xyz) {
    h4.resize(n);
    CU(cudaMemcpyAsync(h4.data(), s->world, sizeof(float4) * (size_t)n, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) { world_xyz[3 * i] = h4[i].x; world_xyz[3 * i + 1] = h4[i].y; world_xyz[3 * i + 2] = h4[i].z; }
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ fov segment
// Host logic of lasermap_fov_segment (laserMapping.cpp:1136-1200); the delete itself runs on the device.
static int fov_boxes(flb_fov_state* f, const double* pos, float* boxes, int* nb) {
  const float MOV_THRESHOLD = 1.5f;  // laserMapping.cpp:53
  *nb = 0;
  if (!f->initialized) {
    for (int i = 0; i < 3; ++i) {
      f->local_map_min[i] = (float)(pos[i] - f->cube_len / 2.0);
      f->local_map_max[i] = (float)(pos[i] + f->cube_len / 2.0);
    }
    f->initialized = 1;
    return 0;
  }
  float edge[3][2];
  bool need_move = false;
  const float lim = MOV_THRESHOLD * f->det_range;
  for (int i = 0; i < 3; ++i) {
    edge[i][0] = (float)std::fabs(pos[i] - (double)f->local_map_min[i]);
    edge[i][1] = (float)std::fabs(pos[i] - (double)f->local_map_max[i]);
    if (edge[i][0] <= lim || edge[i][1] <= lim) need_move = true;
  }
  if (!need_move) return 0;
  float nmin[3], nmax[3];
  for (int i = 0; i < 3; ++i) { nmin[i] = f->local_map_min[i]; nmax[i] = f->local_map_max[i]; }
  const float mov = (float)std::max((f->cube_len - 2.0 * MOV_THRESHOLD * f->det_range) * 0.5 * 0.9,
                                    double(f->det_range * (MOV_THRESHOLD - 1)));
  for (int i = 0; i < 3; ++i) {
    float b[6] = {f->local_map_min[0], f->local_map_min[1], f->local_map_min[2], f->local_map_max[0], f->local_map_max[1], f->local_map_max[2]};
    if (edge[i][0] <= lim) {
      nmax[i] -= mov; nmin[i] -= mov;
      b[i] = f->local_map_max[i] - mov;
      memcpy(boxes + 6 * (*nb), b, sizeof(b));
      ++*nb;
    } else if (edge[i][1] <= lim) {
      nmax[i] += mov; nmin[i] += mov;
      b[3 + i] = f->local_map_min[i] + mov;
      memcpy(boxes + 6 * (*nb), b, sizeof(b));
      ++*nb;
    }
  }
  for (int i = 0; i < 3; ++i) { f->local_map_min[i] = nmin[i]; f->local_map_max[i] = nmax[i]; }
  return 0;
}

extern "C" int flb_fov_segment(flb_map* m, flb_fov_state* fov, const double* pos_lid, float* boxes_out18, int* n_boxes, int* n_deleted) {
  if (!m || !fov || !pos_lid) return set_err("flb_fov_segment: null argument");
  float boxes[18];
  int nb = 0;
  fov_boxes(fov, pos_lid, boxes, &nb);
  if (boxes_out18) memcpy(boxes_out18, boxes, sizeof(float) * 6 * nb);
  if (n_boxes) *n_boxes = nb;
  if (n_deleted) *n_deleted = 0;
  if (nb > 0) return flb_map_delete_boxes(m, boxes, nb, n_deleted);  // :1197-1198
  return 0;
}

// ------------------------------------------------------------------------------------------------ whole scan step
// begin: everything up to (not including) the synchronisation; finish: synchronise and collect.  A streaming caller puts
// flb_scan_prefetch(next scan) between the two so the next upload overlaps this scan's kernels.
extern "C" int flb_scan_step_begin(flb_session* s, flb_fov_state* fov, const float* body, int n, int stride, const double* state26,
                                   const double* P, int flg_EKF_inited) {
  if (!s || !state26 || !P) return set_err("flb_scan_step: null argument");
  flb_map* m = s->map;
  if (s->npending >= 2) return set_err("flb_scan_step_begin: two steps are already in flight (call flb_scan_step_finish first)");
  if (s->npending == 1 && !s->device_update)
    return set_err("flb_scan_step_begin: the host-driven engine runs one step at a time (call flb_scan_step_finish first)");
  s->active = (s->head + s->npending) & 1;
  flb_session::StepSlot& w = cur(s);
  const auto ht0 = std::chrono::steady_clock::now();
  if (s->host_timing && s->ht_n > 0) s->ht_between += std::chrono::duration<double>(ht0 - s->ht_last_finish).count();
  CU(cudaSetDevice(m->cfg.device));
  w.l0 = m->launches;
  w.deleted = 0;
  w.flg = flg_EKF_inited;
  memcpy(w.x, state26, sizeof(w.x));
  memcpy(w.P, P, sizeof(w.P));
  // A device-driven step without an on-stream upload times itself on the device (StepResult::span_ns): no event pair sits
  // on the stream between two steps in flight, only the one event flb_scan_step_finish waits on.
  w.ev2_on = body != nullptr || !s->device_update;
  if (w.ev2_on) CU(cudaEventRecord(w.ev2, m->stream));
  if (body) { if (flb_scan_upload(s, body, n, stride)) return 1; }
  else if (adopt_prefetched(s)) return 1;
  if (fov) {  // laserMapping.cpp:2320 (uses pos_lid of the previous posterior)
    int nb = 0;
    if (flb_fov_segment(m, fov, fov->pos_lid, nullptr, &nb, &w.deleted)) return 1;
  }
  w.device = s->device_update;
  if (w.device) {
    const auto hl0 = std::chrono::steady_clock::now();
    if (launch_scan_device(s, state26, P, flg_EKF_inited, true)) return 1;  // :2380 + :2401, no host round trips inside
    if (s->host_timing) s->ht_launch += std::chrono::duration<double>(std::chrono::steady_clock::now() - hl0).count();
    CU(cudaEventRecord(w.ev3, m->stream));
  }
  w.n = s->n;
  w.l0 = m->launches - w.l0;   // kernels launched by this step so far (a younger step may add its own before finish)
  s->npending++;
  if (s->host_timing) s->ht_begin += std::chrono::duration<double>(std::chrono::steady_clock::now() - ht0).count();
  return 0;
}

extern "C" int flb_scan_step_finish(flb_session* s, flb_fov_state* fov, double* state26, double* P, flb_scan_result* out) {
  if (!s || !state26 || !P) return set_err("flb_scan_step: null argument");
  if (s->npending == 0) return set_err("flb_scan_step_finish without flb_scan_step_begin");
  s->active = s->head;           // the OLDEST step in flight
  const flb_session::StepSlot& w = cur(s);
  s->head ^= 1;
  s->npending--;
  flb_map* m = s->map;
  CU(cudaSetDevice(m->cfg.device));
  flb_scan_result r;
  memset(&r, 0, sizeof(r));
  r.n_deleted = w.deleted;
  bool host_path = !w.device;
  float span_ms = 0.f;   // device-driven step: %globaltimer span of the whole sequence
  const int launches0 = m->launches;
  const auto hf0 = std::chrono::steady_clock::now();
  auto hf1 = hf0;
  if (!host_path) {
    CU(cudaEventSynchronize(w.ev3));                      // the single synchronisation of the step (a younger step may be running on)
    hf1 = std::chrono::steady_clock::now();
    if (finish_counters(m, w.h_res->counters)) return 1;
    m->has_root = m->has_root || m->h_counters[CNT_VALID] > 0;
    if (w.h_res->need_host) {
      if (s->npending)
        return set_err("flb_scan_step_finish: under-determined scan (fewer than 23 rows) while a younger step is already in flight; "
                       "such scans need the host-driven branch: run them with strictly alternating begin / finish");
      host_path = true;                                    // M < 23 branch: redo this scan on the host-driven path
    } else {
      memcpy(state26, w.h_res->x, sizeof(double) * 26);
      memcpy(P, w.h_res->P, sizeof(double) * NDOF * NDOF);
      stats_from_ctl(w.h_res, &r.update);
      s->h_cnt2[0] = w.h_res->cnt2[0];
      s->h_cnt2[1] = w.h_res->cnt2[1];
      r.update.gpu_ms = (float)((double)w.h_res->update_ns * 1e-6);
      span_ms = (float)((double)w.h_res->span_ns * 1e-6);
      if (r.update.gpu_ms > span_ms) r.update.gpu_ms = span_ms;   // (k_publish sits on a parallel branch: never report more than the whole)
    }
  }
  if (host_path) {
    memcpy(state26, w.x, sizeof(w.x));
    memcpy(P, w.P, sizeof(w.P));
    if (run_update(s, state26, P, &r.update)) return 1;  // :2380
    if (w.n > 0 && enqueue_map_incremental(s, state26, w.flg, false)) return 1;  // :2401
    CU(cudaEventRecord(w.ev3, m->stream));
    if (fetch_counters(m)) return 1;
  }
  if (fov) {  // :2383 pos_lid = pos + rot * offset_T_L_I
    host::State x = host::State::from26(state26);
    host::V3 pl = x.pos + host::rotate(x.rot, x.offT);
    for (int i = 0; i < 3; ++i) fov->pos_lid[i] = pl.a[i];
  }
  r.n_to_add = w.n > 0 ? s->h_cnt2[0] : 0;
  r.n_no_downsample = w.n > 0 ? s->h_cnt2[1] : 0;
  r.map_valid = m->h_counters[CNT_VALID];
  if (w.ev2_on) CU(cudaEventElapsedTime(&r.gpu_ms_total, w.ev2, w.ev3));
  else r.gpu_ms_total = span_ms > 0.f ? span_ms : r.update.gpu_ms;
  r.kernel_launches = w.l0 + (m->launches - launches0);
  if (out) *out = r;
  const int rrc = maybe_rehash(m);
  if (s->host_timing) {
    const auto hf2 = std::chrono::steady_clock::now();
    s->ht_wait += std::chrono::duration<double>(hf1 - hf0).count();
    s->ht_finish += std::chrono::duration<double>(hf2 - hf1).count();
    s->ht_last_finish = hf2;
    s->ht_n++;
  }
  return rrc;
}

extern "C" int flb_scan_step(flb_session* s, flb_fov_state* fov, const float* body, int n, int stride, double* state26, double* P,
                             int flg_EKF_inited, flb_scan_result* out) {
  if (flb_scan_step_begin(s, fov, body, n, stride, state26, P, flg_EKF_inited)) return 1;
  return flb_scan_step_finish(s, fov, state26, P, out);
}

#ifdef FLB_TRACE
// Debug-library only (tools/trace_build.sh): read and reset the device-side timeline of trace.cuh.
// out: TRACE_SLOTS x {t0, t1} global-timer ns (t0 = ~0 / t1 = 0 when the slot did not run); phases: TRACE_PHASES clock64 values.
extern "C" int flb_debug_trace_read(unsigned long long* out, long long* phases, unsigned long long* dbg) {
  std::vector<flb::TraceRec> h(flb::TRACE_SLOTS);
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpyFromSymbol(h.data(), flb::g_trace, sizeof(flb::TraceRec) * flb::TRACE_SLOTS));
  if (out) for (int i = 0; i < flb::TRACE_SLOTS; ++i) { out[2 * i] = h[i].t0; out[2 * i + 1] = h[i].t1; }
  if (phases) CU(cudaMemcpyFromSymbol(phases, flb::g_phase_clk, sizeof(long long) * flb::TRACE_PHASES));
  for (auto& r : h) { r.t0 = ~0ull; r.t1 = 0ull; }
  CU(cudaMemcpyToSymbol(flb::g_trace, h.data(), sizeof(flb::TraceRec) * flb::TRACE_SLOTS));
  if (dbg) CU(cudaMemcpyFromSymbol(dbg, flb::g_dbg, sizeof(unsigned long long) * flb::TRACE_DBG));
  std::vector<unsigned long long> zd(flb::TRACE_DBG, 0);
  CU(cudaMemcpyToSymbol(flb::g_dbg, zd.data(), sizeof(unsigned long long) * flb::TRACE_DBG));
  std::vector<long long> z(flb::TRACE_PHASES, 0);
  CU(cudaMemcpyToSymbol(flb::g_phase_clk, z.data(), sizeof(long long) * flb::TRACE_PHASES));
  return 0;
}
#endif

// ------------------------------------------------------------------------------------------------ front-end rows (SURVEY.md §8f)
#include "frontend_host.cuh"
#include "preprocess_host.cuh"
#include "keyframe_host.cuh"
#include "scan_context_host.cuh"
#include "icp_host.cuh"
#include "icp_batch_host.cuh"
#include "fricp_host.cuh"
#include "sicp_host.cuh"
#include "aaicp_host.cuh"
#include "color_host.cuh"
#include "imu_host.cuh"

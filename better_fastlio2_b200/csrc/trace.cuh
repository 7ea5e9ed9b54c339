// trace.cuh — optional device-side timeline (compiled only with -DFLB_TRACE into a separate debug library by
// tools/trace_build.sh; the product library contains none of it).  Each instrumented kernel records the earliest block
// start and the latest block end on the global timer into a slot (kernel id x pass), so the real critical path of a
// graph-launched scan — including launch gaps and side-stream overlap — can be read back without a profiler.
#pragma once
#ifdef FLB_TRACE
namespace flb {
constexpr int TRACE_SLOTS = 128;
constexpr int TRACE_PHASES = 96;
struct TraceRec { unsigned long long t0, t1; };
__device__ TraceRec g_trace[TRACE_SLOTS];
__device__ long long g_phase_clk[TRACE_PHASES];
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void trace_mark(int slot, bool begin) {
  if (threadIdx.x == 0) {
    const unsigned long long t = gtimer();
    if (begin) atomicMin(&g_trace[slot].t0, t);
    else atomicMax(&g_trace[slot].t1, t);
  }
}
// first block start (begin) or last block end of `slot`, stamped by the calling thread itself
__device__ __forceinline__ void trace_stamp(int slot, bool begin) {
  const unsigned long long t = gtimer();
  if (begin) atomicMin(&g_trace[slot].t0, t);
  else atomicMax(&g_trace[slot].t1, t);
}
// 4-us bucket (0..15) of the time elapsed since the earliest block start recorded in `slot`
__device__ __forceinline__ int trace_bucket_since(int slot) {
  const unsigned long long t0 = *(volatile unsigned long long*)&g_trace[slot].t0;
  const unsigned long long t = gtimer();
  return t > t0 ? (int)min((t - t0) / 4000ull, 15ull) : 0;
}
constexpr int TRACE_DBG = 128;
__device__ unsigned long long g_dbg[TRACE_DBG];
__device__ __forceinline__ void dbg_add(int idx, unsigned long long v) { atomicAdd(&g_dbg[idx], v); }
__device__ __forceinline__ void dbg_max(int idx, unsigned long long v) { atomicMax(&g_dbg[idx], v); }
__device__ __forceinline__ void trace_phase(int idx) {
  if (threadIdx.x == 0 && idx < TRACE_PHASES) g_phase_clk[idx] = clock64();
}
}  // namespace flb
#define FLB_TRACE_BEGIN(slot) flb::trace_mark((slot), true)
#define FLB_TRACE_END(slot) flb::trace_mark((slot), false)
#define FLB_TRACE_PHASE(idx) flb::trace_phase(idx)
#define FLB_DBG_ADD(idx, v) flb::dbg_add((idx), (unsigned long long)(v))
#define FLB_DBG_MAX(idx, v) flb::dbg_max((idx), (unsigned long long)(v))
#define FLB_DBG_CLOCK(var) const long long var = clock64()
#define FLB_TRACE_STAMP(slot, begin) flb::trace_stamp((slot), (begin))
#define FLB_TRACE_HIST(idx0, slot) flb::dbg_add((idx0) + flb::trace_bucket_since(slot), 1)
#else
#define FLB_TRACE_BEGIN(slot)
#define FLB_TRACE_END(slot)
#define FLB_TRACE_PHASE(idx)
#define FLB_DBG_ADD(idx, v)
#define FLB_DBG_MAX(idx, v)
#define FLB_DBG_CLOCK(var)
#define FLB_TRACE_STAMP(slot, begin)
#define FLB_TRACE_HIST(idx0, slot)
#endif

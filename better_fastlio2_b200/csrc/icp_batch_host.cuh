// icp_batch_host.cuh — IncreMapping::run's inter-session registrations (multi-session Incremental_mapping.cpp: addSCloops
// :651-696 / doICPVirtualRelative :462-522 and addRSloops :787-837 / doICPGlobalRelative :525-583, run there under
// `omp parallel for`) as one call over every pair.  Set-up goes pair by pair: both selections assembled from the store
// (and VoxelGrid-filtered) into one round's packed arrays, the target's box read back for its grid.  Pairs join the round
// in order while the summed grid cells stay within ICP_MAX_CELLS; then every pair's index is built into its slice of one
// packed index and the round iterates in lockstep: one batched 1-NN pass, two segmented reductions, one copy and one
// synchronisation per iteration, the SVD, the compositions and the convergence test per pair here on the host as
// flb_keyframes_icp runs them, and one batched fitness pass at the end.  The contract is written out in DESIGN.md §9.
// Included after icp_host.cuh.
#pragma once
#include "icp_batch_kernels.cuh"

// A pair of the round being set up: its result slot, sizes, grid and slices.
struct IcpbPair {
  int p, n_s, n_t, n_fin;
  IcpGrid g;
  size_t s_off, t_off, cs_off, box_off;
};

// grow() that keeps the first `used` bytes: a round's packed clouds grow while it is set up.
template <typename T>
static int icpb_grow_keep(flb_map* m, DevBuf<T>& b, size_t used, size_t need) {
  if (need <= b.cap) return 0;
  const size_t cap = need + need / 4;
  void* p = nullptr;
  CU(cudaMalloc(&p, cap));
  if (used) {
    const cudaError_t e = cudaMemcpyAsync(p, b.p, used, cudaMemcpyDeviceToDevice, m->stream);
    if (e != cudaSuccess) {
      Q(cudaFree(p));
      return set_err("icp batch: copy of %zu bytes: %s", used, cudaGetErrorString(e));
    }
  }
  b.release();   // cudaFree waits for the copy
  b.p = static_cast<T*>(p);
  b.cap = cap;
  return 0;
}

// One selection (n_ids key frames with their poses6, n_dense points) as flb_keyframes_assemble writes it with leaf into
// dst from point `used` on: *n points.  A filter costs one synchronisation (its output count).
static int icpb_selection(flb_map* m, const flb_keyframes* k, const int* ids, int n_ids, const float* p6, int n_dense, float leaf,
                          DevBuf<float4>& dst, size_t used, int* n, int* syncs) {
  *n = 0;
  if (n_dense == 0) return 0;
  KfWork& kw = *m->kfw;
  IcpBatchWork& w = kw.icpb;
  if (icpb_grow_keep(m, dst, sizeof(float4) * used, sizeof(float4) * (used + (size_t)n_dense))) return 1;
  float4* out = dst.p + used;
  std::vector<KfSeg> segs;
  kf_selection_segs(k, ids, n_ids, FLB_KF_POSE6, p6, segs);
  if (leaf == 0.f) {   // the dense concatenation
    *n = n_dense;
    return kf_assemble_enqueue(m, segs, k->xyzi, nullptr, n_dense, out, nullptr);
  }
  if (kf_grow(w.raw, sizeof(float4) * (size_t)n_dense) || kf_assemble_enqueue(m, segs, k->xyzi, nullptr, n_dense, w.raw.p, nullptr) ||
      vg_enqueue(m, kw.vg, w.raw.p, nullptr, n_dense, leaf, out, nullptr, n_dense, m->stream))
    return 1;
  CU(cudaStreamSynchronize(m->stream));
  ++*syncs;
  if (kw.vg.h_mm.p[6] != 0) {   // PCL's int32 overflow guard: the assembled cloud unchanged
    CU(cudaMemcpyAsync(out, w.raw.p, sizeof(float4) * (size_t)n_dense, cudaMemcpyDeviceToDevice, m->stream));
    *n = n_dense;
  } else {
    *n = (int)kw.vg.h_mm.p[7];
  }
  return 0;
}

// The 1-NN pass of the first n_items staged items (n_q queries in all) from `in`, and their sums (with cross: also the
// cross products) into w.h_sums; the caller synchronises.  open_n: the open count, after every pair's reduction counter.
static int icpb_pass(flb_map* m, IcpBatchWork& w, int n_items, int n_q, const float4* in, double max_d2, bool cross, int* open_n) {
  const int nb = m->sm_count * 2;   // k_reduce's grid: a pair's partition is the one flb_keyframes_icp uses
  CU(cudaMemcpyAsync(w.items.p, w.h_items.p, sizeof(IcpBatchItem) * (size_t)n_items, cudaMemcpyHostToDevice, m->stream));
  CU(cudaMemsetAsync(open_n, 0, sizeof(int), m->stream));
  k_icpb_nn<<<grid_for(n_q, 256, m->sm_count * 8), 256, 0, m->stream>>>(w.items.p, n_items, n_q, w.order.p, in, w.x.p, w.sorted.p, w.cs.p,
                                                                        w.corr.p, w.corr_d2.p, w.open.p, open_n);
  k_icpb_nn_far<<<m->sm_count * 8, 256, 0, m->stream>>>(w.items.p, w.open.p, open_n, w.x.p, w.sorted.p, w.cs.p, w.box.p, w.corr.p,
                                                        w.corr_d2.p);
  const IcpBatchPairsOp pairs{w.corr.p, w.corr_d2.p, w.x.p, w.tgt.p, max_d2};
  k_icpb_reduce<8><<<n_items * nb, 256, 0, m->stream>>>(w.items.p, nb, pairs, w.partials.p, w.counters.p, w.sums.p);
  if (cross)
    k_icpb_reduce<9><<<n_items * nb, 256, 0, m->stream>>>(w.items.p, nb, IcpBatchCrossOp{pairs, w.sums.p}, w.partials.p, w.counters.p,
                                                          w.sums.p + 8);
  m->launches += cross ? 4 : 3;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(w.h_sums.p, w.sums.p, sizeof(double) * ICPB_REC * (size_t)n_items, cudaMemcpyDeviceToHost, m->stream));
  return 0;
}

static IcpBatchItem icpb_item_of(const IcpbPair& r, const float T[16], bool apply, int q0) {
  IcpBatchItem it{};
  it.g = r.g;
  it.xf = icp_xf(T, apply);
  it.q0 = q0;
  it.n_s = r.n_s;
  it.s_off = (int)r.s_off;
  it.t_off = (int)r.t_off;
  it.cs_off = (int)r.cs_off;
  it.box_off = (int)r.box_off;
  return it;
}

// The round's indices, then its lockstep iterations and the fitness pass; results into out[r.p].
static int icpb_round(flb_map* m, const std::vector<IcpbPair>& R, size_t n_src, size_t n_tgt, size_t n_cs, size_t n_box,
                      const flb_icp_config& cfg, flb_icp_result* out, flb_icp_batch_stats& st) {
  KfWork& kw = *m->kfw;
  IcpBatchWork& w = kw.icpb;
  IcpIndex& x = kw.index;
  const int nr = (int)R.size();
  const size_t ps = sizeof(float4) * n_src, is = sizeof(int) * n_src;
  if (kf_grow(w.x, ps) || kf_grow(w.order, is) || kf_grow(w.corr, is) || kf_grow(w.corr_d2, sizeof(float) * n_src) ||
      kf_grow(w.open, sizeof(int2) * n_src) || kf_grow(w.sorted, sizeof(float4) * n_tgt) || kf_grow(w.cs, sizeof(int) * n_cs) ||
      kf_grow(w.box, sizeof(IcpBox) * n_box) || kf_grow(w.items, sizeof(IcpBatchItem) * nr) || grow(w.h_items, sizeof(IcpBatchItem) * nr, 0) ||
      kf_grow(w.sums, sizeof(double) * ICPB_REC * nr) || grow(w.h_sums, sizeof(double) * ICPB_REC * nr, 0) ||
      kf_grow(w.partials, sizeof(double) * 9 * (size_t)m->sm_count * 2 * nr) || kf_grow(w.counters, sizeof(unsigned) * (nr + 1)))
    return 1;
  CU(cudaMemsetAsync(w.counters.p, 0, sizeof(unsigned) * nr, m->stream));
  int* open_n = (int*)w.counters.p + nr;
  for (const IcpbPair& r : R) {   // each target's index (flb_keyframes_icp's, into its slices), then the source's order
    if (icp_build(m, x, w.tgt.p + r.t_off, r.n_t, r.g, r.n_fin, w.sorted.p + r.t_off, w.cs.p + r.cs_off, w.box.p + r.box_off)) return 1;
    k_icp_keys<<<grid_for(r.n_s, 256, m->sm_count * 8), 256, 0, m->stream>>>(r.g, w.src.p + r.s_off, r.n_s, x.keys_a.p, x.vals_a.p);
    m->launches++;
    if (icp_order(m, x, r.n_s, w.order.p + r.s_off)) return 1;
  }

  // the iterations (icp.hpp computeTransformation), every pair as flb_keyframes_icp runs it
  struct State { float T[16], final_T[16]; double prev_mse; };
  std::vector<State> S(nr);
  std::vector<int> act(nr);
  for (int j = 0; j < nr; ++j) {
    State& s = S[j];
    for (int i = 0; i < 16; ++i) s.final_T[i] = s.T[i] = (i % 5 == 0) ? 1.f : 0.f;
    s.prev_mse = DBL_MAX;
    act[j] = j;
    out[R[j].p].state = FLB_ICP_NOT_CONVERGED;
  }
  const double max_d2 = cfg.max_correspondence_distance * cfg.max_correspondence_distance;
  for (int it = 0; !act.empty(); ++it) {
    int n_q = 0;
    for (size_t a = 0; a < act.size(); ++a) {
      w.h_items.p[a] = icpb_item_of(R[act[a]], S[act[a]].T, it > 0, n_q);
      n_q += R[act[a]].n_s;
    }
    if (icpb_pass(m, w, (int)act.size(), n_q, it == 0 ? w.src.p : w.x.p, max_d2, true, open_n)) return 1;
    CU(cudaStreamSynchronize(m->stream));
    st.iteration_syncs++;
    size_t keep = 0;
    for (size_t a = 0; a < act.size(); ++a) {
      const int j = act[a];
      State& s = S[j];
      flb_icp_result& res = out[R[j].p];
      const double* sm = w.h_sums.p + ICPB_REC * a;
      res.n_correspondences = (int)sm[0];
      if (sm[0] < 3) {   // min_number_correspondences_
        res.state = FLB_ICP_NO_CORRESPONDENCES;
        continue;
      }
      icp_rigid(sm, s.T);
      icp_mul4(s.T, s.final_T, s.final_T);
      res.iterations = it + 1;
      res.state = icp_converged(cfg, res.iterations, s.T, sm[0], sm[1], &s.prev_mse);
      if (res.state != FLB_ICP_NOT_CONVERGED) {
        res.converged = 1;
        continue;
      }
      act[keep++] = j;
    }
    act.resize(keep);
  }

  // getFitnessScore() of every pair: its original source moved once by its final transformation, no cut
  int n_q = 0;
  for (int j = 0; j < nr; ++j) {
    w.h_items.p[j] = icpb_item_of(R[j], S[j].final_T, true, n_q);
    n_q += R[j].n_s;
  }
  if (icpb_pass(m, w, nr, n_q, w.src.p, DBL_MAX, false, open_n)) return 1;
  CU(cudaStreamSynchronize(m->stream));
  st.iteration_syncs++;
  for (int j = 0; j < nr; ++j) {
    flb_icp_result& res = out[R[j].p];
    const double* fs = w.h_sums.p + ICPB_REC * j;
    memcpy(res.final_transformation, S[j].final_T, sizeof(S[j].final_T));
    res.fitness_score = fs[0] > 0 ? fs[1] / fs[0] : DBL_MAX;
  }
  return 0;
}

// One side's selections without the store: offsets from 0 and non-decreasing, ids and poses given, poses finite.
static int icpb_check_shape(int n_pairs, const int* off, const int* ids, const float* p6, const char* side) {
  const char* who = "flb_keyframes_icp_batch";
  if (!off) return set_err("%s: null %s_offsets", who, side);
  if (off[0] != 0) return set_err("%s: %s_offsets[0] is %d, must be 0", who, side, off[0]);
  for (int p = 0; p < n_pairs; ++p)
    if (off[p + 1] < off[p]) return set_err("%s: pair %d: %s_offsets decrease (%d after %d)", who, p, side, off[p + 1], off[p]);
  if (off[n_pairs] > 0 && (!ids || !p6)) return set_err("%s: null %s_ids or %s_poses6", who, side, side);
  for (int p = 0; p < n_pairs; ++p)
    for (int j = off[p]; j < off[p + 1]; ++j)
      for (int c = 0; c < 6; ++c)
        if (!std::isfinite(p6[6 * (size_t)j + c])) return set_err("%s: pair %d: %s_poses6 entry %d is not finite", who, p, side, j);
  return 0;
}

// One side's ids in the store's range; the dense selection sizes into n_dense.
static int icpb_check_ids(const flb_keyframes* k, int n_pairs, const int* off, const int* ids, const char* side, std::vector<int>& n_dense) {
  const char* who = "flb_keyframes_icp_batch";
  n_dense.assign(n_pairs, 0);
  const int n_kf = (int)k->cnt.size();
  for (int p = 0; p < n_pairs; ++p) {
    long long t = 0;
    for (int j = off[p]; j < off[p + 1]; ++j) {
      if (ids[j] < 0 || ids[j] >= n_kf)
        return set_err("%s: pair %d: %s_ids entry %d: key frame %d out of range [0, %d)", who, p, side, j, ids[j], n_kf);
      t += k->cnt[ids[j]];
    }
    if (t > INT_MAX) return set_err("%s: pair %d: %s selection of %lld points is too large", who, p, side, t);
    n_dense[p] = (int)t;
  }
  return 0;
}

extern "C" int flb_keyframes_icp_batch(flb_keyframes* k, int n_pairs, const int* src_offsets, const int* src_ids, const float* src_poses6,
                                       const int* tgt_offsets, const int* tgt_ids, const float* tgt_poses6, float leaf,
                                       const flb_icp_config* cfg, flb_icp_result* out, flb_icp_batch_stats* stats) {
  const char* who = "flb_keyframes_icp_batch";
  if (n_pairs < 0) return set_err("%s: negative n_pairs", who);
  flb_icp_batch_stats st{};
  if (n_pairs == 0) {
    if (stats) *stats = st;
    return 0;
  }
  if (!out) return set_err("%s: null result", who);
  if (!cfg) return set_err("%s: null config", who);
  if (!icp_cfg_ok(cfg))
    return set_err("%s: config values must be finite, max_iterations >= 0 and max_correspondence_distance >= 0", who);
  if (!(std::isfinite(leaf) && leaf >= 0.f)) return set_err("%s: leaf_size must be finite and >= 0 (0: no filter)", who);
  if (icpb_check_shape(n_pairs, src_offsets, src_ids, src_poses6, "src") || icpb_check_shape(n_pairs, tgt_offsets, tgt_ids, tgt_poses6, "tgt"))
    return 1;
  if (!k) return set_err("%s: null key-frame store", who);
  std::vector<int> ns_dense, nt_dense;
  if (icpb_check_ids(k, n_pairs, src_offsets, src_ids, "src", ns_dense) || icpb_check_ids(k, n_pairs, tgt_offsets, tgt_ids, "tgt", nt_dense))
    return 1;

  std::vector<flb_icp_result> res(n_pairs);
  for (flb_icp_result& r : res) {   // initCompute fails: nothing registered
    r = flb_icp_result{};
    for (int i = 0; i < 16; ++i) r.final_transformation[i] = (i % 5 == 0) ? 1.f : 0.f;
    r.state = FLB_ICP_NOT_CONVERGED;
    r.fitness_score = DBL_MAX;
  }
  flb_map* m = k->map;
  CU(cudaSetDevice(m->cfg.device));
  if (kf_work(m)) return 1;
  KfWork& kw = *m->kfw;
  IcpBatchWork& w = kw.icpb;
  std::vector<IcpbPair> R;
  for (int p = 0; p < n_pairs;) {
    R.clear();
    size_t s_used = 0, t_used = 0, cs_used = 0, box_used = 0;
    double cells = 0.0;
    for (; p < n_pairs; ++p) {
      int n_s = 0, n_t = 0;
      const int s0 = src_offsets[p], t0 = tgt_offsets[p];
      if (icp_index_scratch(m, kw.index, ns_dense[p], nt_dense[p], 0) ||
          icpb_selection(m, k, src_ids + s0, src_offsets[p + 1] - s0, src_poses6 + 6 * (size_t)s0, ns_dense[p], leaf, w.src, s_used, &n_s,
                         &st.setup_syncs) ||
          icpb_selection(m, k, tgt_ids + t0, tgt_offsets[p + 1] - t0, tgt_poses6 + 6 * (size_t)t0, nt_dense[p], leaf, w.tgt, t_used, &n_t,
                         &st.setup_syncs))
        return 1;
      res[p].n_source = n_s;
      res[p].n_target = n_t;
      if (n_s == 0 || n_t == 0) continue;
      float lo[3], hi[3];
      int n_fin = 0;
      if (icp_bounds(m, kw.index, w.tgt.p + t_used, n_t, lo, hi, &n_fin)) return 1;
      st.setup_syncs++;
      if (n_fin == 0) continue;   // every target point dropped by KdTreeFLANN: initCompute fails
      IcpbPair r{p, n_s, n_t, n_fin, icp_grid(lo, hi, n_fin), s_used, t_used, cs_used, box_used};
      const double c = (double)r.g.gx * r.g.gy * r.g.gz;
      // p opens the next round and is set up again there (packed offsets are int on the device)
      if (!R.empty() && (cells + c > ICP_MAX_CELLS || s_used + n_s > (size_t)INT_MAX || t_used + n_t > (size_t)INT_MAX)) break;
      R.push_back(r);
      cells += c;
      s_used += n_s;
      t_used += n_t;
      cs_used += (size_t)c + 1;
      box_used += (size_t)r.g.cx * r.g.cy * r.g.cz;
    }
    if (R.empty()) continue;
    if (icpb_round(m, R, s_used, t_used, cs_used, box_used, *cfg, res.data(), st)) return 1;
    st.rounds++;
  }
  memcpy(out, res.data(), sizeof(flb_icp_result) * (size_t)n_pairs);
  if (stats) *stats = st;
  return 0;
}

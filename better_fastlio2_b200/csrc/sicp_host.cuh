// sicp_host.cuh — the relocaliser's Sparse ICP (regMode 7: SICP::point_to_point, include/FRICP-toolkit/ICP.h:275-380, with
// Registeration's SICP::Parameters, registeration.h:67-69 and :143-146): a host source cloud onto a target assembled from
// the device key-frame store.  The set-up (upload, two-stage target assembly, normalisation, grid index) is
// flb_keyframes_fricp's (fr_setup).  Every ICP iteration is one exact double 1-NN pass of the moving source, one
// cooperative launch of k_sicp_admm that runs the whole ADMM loop on the device, one small copy and one synchronisation;
// the μ schedule and its shrinkage thresholds are computed here once per call with the host's pow.  DESIGN.md §9 states
// the contract.  Included after fricp_host.cuh.
#pragma once
#include "sicp_kernels.cuh"

static int sicp_cfg_check(const flb_sicp_config* c, const char* who) {
  if (!(c->p > 0 && c->p <= 1)) return set_err("%s: p must be in (0, 1]", who);
  if (!(std::isfinite(c->mu) && c->mu > 0)) return set_err("%s: mu must be finite and > 0", who);
  if (!(std::isfinite(c->max_mu) && c->max_mu > 0)) return set_err("%s: max_mu must be finite and > 0", who);
  if (!(std::isfinite(c->alpha) && c->alpha >= 1)) return set_err("%s: alpha must be finite and >= 1", who);
  if (c->max_icp < 0) return set_err("%s: max_icp must be >= 0 (got %d)", who, c->max_icp);
  if (c->max_outer < 0) return set_err("%s: max_outer must be >= 0 (got %d)", who, c->max_outer);
  if (!(std::isfinite(c->stop) && c->stop >= 0)) return set_err("%s: stop must be finite and >= 0", who);
  return 0;
}

extern "C" void flb_sicp_default_config(flb_sicp_config* c) {
  if (!c) return;
  c->p = 0.4;
  c->mu = 10.0;
  c->alpha = 1.2;
  c->max_mu = 1e5;
  c->max_icp = 100;
  c->max_outer = 100;
  c->stop = 1e-5;
}

// The μ of every outer iteration of one ICP iteration (μ <- μ α while μ < max_mu, from mu) with Ba = ((2/μ)(1-p))^(1/(2-p))
// and ha = Ba + (p/μ) Ba^(p-1) (shrink, ICP.h:247-248) into sched (3 per iteration); mu_after[k] = μ after k iterations.
static void sicp_schedule(const flb_sicp_config& c, double* sched, double* mu_after) {
  double mu = c.mu;
  mu_after[0] = mu;
  for (int k = 0; k < c.max_outer; ++k) {
    const double Ba = std::pow((2.0 / mu) * (1.0 - c.p), 1.0 / (2.0 - c.p));
    sched[3 * k] = mu;
    sched[3 * k + 1] = Ba;
    sched[3 * k + 2] = Ba + (c.p / mu) * std::pow(Ba, c.p - 1.0);
    if (mu < c.max_mu) mu *= c.alpha;
    mu_after[k + 1] = mu;
  }
}

// Blocks of k_sicp_admm: every block resident (the occupancy of one SM times the SMs), at most one per 256 points.
static int sicp_grid(flb_map* m, int n_s, int* blocks) {
  int per_sm = 0;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_sicp_admm, SICP_BLOCK, 0));
  if (per_sm < 1) return set_err("flb_keyframes_sicp: the ADMM kernel cannot be resident");
  *blocks = std::max(1, std::min(per_sm * m->sm_count, (n_s + SICP_BLOCK - 1) / SICP_BLOCK));
  return 0;
}

static int sicp_scratch(flb_map* m, KfWork& k, int n_s, int blocks, int max_outer) {
  SicpWork& w = k.sicp;
  const size_t pd = sizeof(double4) * (size_t)n_s, sd = sizeof(double) * (3 * (size_t)max_outer + 1);
  if (kf_grow(w.q, pd) || kf_grow(w.z, pd) || kf_grow(w.c, pd) || kf_grow(w.xo2, pd) || kf_grow(w.sched, sd) ||
      grow(w.h_sched, sd, 0) ||
      grow(w.part, sizeof(double) * SICP_SLOTS * SICP_RED * (size_t)blocks, 0) || grow(w.rec, sizeof(double) * SICP_REC_WORDS, 0) ||
      grow(w.h_rec, sizeof(double) * SICP_REC_WORDS, 0))
    return 1;
  return 0;
}

extern "C" int flb_keyframes_sicp(flb_keyframes* k, const void* src_pts, int n_src, int src_stride, int src_off_intensity,
                                  const float* src_pose6, const int* tgt_ids, int n_tgt, const float* tgt_pre_pose6,
                                  const float* tgt_poses6, const flb_sicp_config* cfg, flb_sicp_result* out, int* out_corr_index,
                                  double* out_resid, double* out_log, int log_cap) {
  FrSetup st;
  flb_sicp_result res;
  if (fr_open(k, "flb_keyframes_sicp", cfg, sicp_cfg_check, src_pts, n_src, src_stride, src_off_intensity, src_pose6, tgt_ids, n_tgt,
              tgt_pre_pose6, tgt_poses6, out_corr_index, out_resid, out_log, log_cap, 1, out, res, st))
    return 1;
  if (st.status >= 0) return 0;
  flb_map* m = k->map;
  KfWork& kw = *m->kfw;
  FricpWork& f = kw.fricp;
  SicpWork& w = kw.sicp;
  const int n_s = st.n_s;
  int blocks = 0;
  if (sicp_grid(m, n_s, &blocks) || sicp_scratch(m, kw, n_s, blocks, cfg->max_outer)) return 1;
  res.admm_blocks = blocks;

  // the μ schedule, T = I, C = 0, Xo2 = X (ICP.h:281-290 with init_trans = I)
  std::vector<double> mu_after((size_t)cfg->max_outer + 1);
  sicp_schedule(*cfg, w.h_sched.p, mu_after.data());
  if (cfg->max_outer > 0)
    CU(cudaMemcpyAsync(w.sched.p, w.h_sched.p, sizeof(double) * 3 * (size_t)cfg->max_outer, cudaMemcpyHostToDevice, m->stream));
  double T[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  memcpy(w.h_rec.p + SICP_REC_T, T, sizeof(T));
  CU(cudaMemcpyAsync(w.rec.p, w.h_rec.p, sizeof(double) * SICP_REC_WORDS, cudaMemcpyHostToDevice, m->stream));
  CU(cudaMemsetAsync(w.c.p, 0, sizeof(double4) * (size_t)n_s, m->stream));
  CU(cudaMemcpyAsync(w.xo2.p, f.x.p, sizeof(double4) * (size_t)n_s, cudaMemcpyDeviceToDevice, m->stream));

  SicpArgs a{};
  a.x = f.x.p;
  a.sorted_d = f.sorted_d.p;
  a.pos = f.pos.p;
  a.q = w.q.p;
  a.z = w.z.p;
  a.c = w.c.p;
  a.xo2 = w.xo2.p;
  a.sched = w.sched.p;
  a.part = w.part.p;
  a.rec = w.rec.p;
  a.n = n_s;
  a.max_outer = cfg->max_outer;
  a.n_d = (double)st.n_fs;
  a.inv_n = 1.0 / a.n_d;
  a.p = cfg->p;
  a.stop = cfg->stop;
  void* args[] = {&a};
  const double I[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  int log_n = 0;
  for (int icp = 0; icp < cfg->max_icp; ++icp) {
    // Q = the exact nearest target points of X (the pass's identity transform returns X itself), then the ADMM loop
    if (fr_nn(m, kw, st.g, n_s, I)) return 1;
    CU(cudaLaunchCooperativeKernel((const void*)k_sicp_admm, blocks, SICP_BLOCK, args, 0, m->stream));
    m->launches++;
    CU(cudaMemcpyAsync(w.h_rec.p, w.rec.p, sizeof(double) * SICP_REC_WORDS, cudaMemcpyDeviceToHost, m->stream));
    CU(cudaStreamSynchronize(m->stream));
    res.syncs++;
    const double* r = w.h_rec.p;
    const int outer = (int)r[SICP_REC_OUTER];
    memcpy(T, r + SICP_REC_T, sizeof(T));
    ++res.iterations;
    res.admm_iterations += outer;
    res.primal = r[SICP_REC_PRIMAL];
    res.dual = r[SICP_REC_DUAL];
    res.stop = r[SICP_REC_STOP];
    res.mu_exit = mu_after[outer];
    if (log_n < log_cap) {
      double* row = out_log + 5 * (size_t)log_n++;
      row[0] = outer; row[1] = res.primal; row[2] = res.dual; row[3] = res.stop; row[4] = res.mu_exit;
    }
    if (res.stop < cfg->stop) break;
  }
  res.log_n = log_n;
  if (fr_close(m, st, T, res.iterations > 0, out_corr_index, out_resid, res)) return 1;   // ICP.h:373 and registeration.h:170
  *out = res;
  return 0;
}

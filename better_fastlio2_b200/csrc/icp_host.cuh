// icp_host.cuh — performLoopClosure's ICP (laserMapping.cpp:946-974, pcl::IterativeClosestPoint 1.10 with the settings of
// :947-952 and an identity guess) between two selections of the device key-frame store, and the host side of the grid
// index both registrations use (icp_bounds, icp_index, icp_order, icp_reduce over KfWork's IcpIndex).  Both sub-maps are
// assembled by k_kf_assemble into map-side scratch exactly as flb_keyframes_assemble writes them; the source's
// pre-transform (transformPointCloud(cureKeyframeCloud, &com), :954-962) is one more k_kf_assemble segment over the
// assembled source.  The target index is built once per call; each iteration is one exact 1-NN pass and two fixed-order
// double reductions on the map stream, one small copy and one synchronisation.  The 3x3 SVD, the 4x4 compositions and the
// convergence test run here on the host between iterations.  The contract is written out in DESIGN.md §9.  Included
// after scan_context_host.cuh.
#pragma once
#include <cfloat>
#include <cmath>

#include "icp_kernels.cuh"

constexpr int ICP_MISC_OPEN = 7, ICP_MISC_COUNTER = 8, ICP_MISC_WORDS = 9;   // after the bounds words of k_icp_bounds
constexpr double ICP_CELLS_PER_POINT = 8.0;     // dense fine cells over the target box per finite target point
constexpr double ICP_MAX_CELLS = 134217728.0;   // 2^27 fine cells (512 MB of offsets) at most

// The index's scratch for n_s queries and a target of n_t points (the grid's buffers are grown once the grid is known);
// tmp_bytes: the caller's own CUB temporary storage beside the index's radix sorts.
static int icp_index_scratch(flb_map* m, IcpIndex& x, int n_s, int n_t, size_t tmp_bytes) {
  const int nk = std::max(n_s, n_t);
  const size_t ik = sizeof(int) * (size_t)nk;
  size_t t1 = 0;
  CU(cub::DeviceRadixSort::SortPairs(nullptr, t1, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, nk));
  if (kf_grow(x.sorted, sizeof(float4) * (size_t)n_t) || kf_grow(x.keys_a, ik) || kf_grow(x.keys_b, ik) || kf_grow(x.vals_a, ik) ||
      kf_grow(x.vals_b, ik) || kf_grow(x.order, sizeof(int) * (size_t)n_s) || kf_grow(x.open, ik) ||
      kf_grow(x.tmp, std::max(t1, tmp_bytes) + 256) || grow(x.partials, sizeof(double) * ICP_RED_MAX * (size_t)m->sm_count * 2, 0) ||
      grow(x.misc, sizeof(unsigned) * ICP_MISC_WORDS, 0) || grow(x.h_misc, sizeof(unsigned) * ICP_MISC_WORDS, 0))
    return 1;
  return 0;
}

static float icp_fkey(unsigned k) {   // inverse of icp_okey
  const unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float v;
  memcpy(&v, &u, sizeof(v));
  return v;
}

// The grid over the finite target box [lo, hi]: fine edge from the box volume and the point count, at most
// ICP_MAX_CELLS cells, every axis a multiple of ICP_C.
static IcpGrid icp_grid(const float* lo, const float* hi, int n_fin) {
  double ext[3], L = 0.0, amax = 0.0;
  for (int a = 0; a < 3; ++a) {
    ext[a] = (double)hi[a] - (double)lo[a];
    L = std::max(L, ext[a]);
    amax = std::max(amax, std::max(std::fabs((double)lo[a]), std::fabs((double)hi[a])));
  }
  double e = 1.0;
  if (L > 0.0) {
    const double floor_e = L / 1024.0;
    double V = 1.0;
    for (int a = 0; a < 3; ++a) V *= std::max(ext[a], floor_e);
    e = std::max(std::cbrt(V / (ICP_CELLS_PER_POINT * n_fin)), floor_e);
  }
  IcpGrid g{};
  for (;;) {
    int dims[3];
    double cells = 1.0;
    for (int a = 0; a < 3; ++a) {
      dims[a] = ((int)std::floor(ext[a] / e) + 1 + ICP_C - 1) / ICP_C * ICP_C;
      cells *= dims[a];
    }
    if (cells <= ICP_MAX_CELLS) {
      g.gx = dims[0]; g.gy = dims[1]; g.gz = dims[2];
      break;
    }
    e *= 1.25;
  }
  g.ox = lo[0]; g.oy = lo[1]; g.oz = lo[2];
  g.e = (float)e;
  g.inv_e = 1.0f / g.e;
  g.slack = 1e-3f * g.e + 4e-6f * (float)(amax + L);
  g.cx = g.gx / ICP_C; g.cy = g.gy / ICP_C; g.cz = g.gz / ICP_C;
  return g;
}

// The finite count and box of p[0, n) (k_icp_bounds, read back); resets the open count and the reduction counter too.
static int icp_bounds(flb_map* m, IcpIndex& x, const float4* p, int n, float* lo, float* hi, int* n_fin) {
  const unsigned init[ICP_MISC_WORDS] = {~0u, ~0u, ~0u};
  memcpy(x.h_misc.p, init, sizeof(init));
  CU(cudaMemcpyAsync(x.misc.p, x.h_misc.p, sizeof(init), cudaMemcpyHostToDevice, m->stream));
  k_icp_bounds<<<grid_for(n, 256, m->sm_count * 4), 256, 0, m->stream>>>(p, n, x.misc.p);
  m->launches++;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(x.h_misc.p, x.misc.p, sizeof(unsigned) * 7, cudaMemcpyDeviceToHost, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  for (int a = 0; a < 3; ++a) { lo[a] = icp_fkey(x.h_misc.p[a]); hi[a] = icp_fkey(x.h_misc.p[3 + a]); }
  *n_fin = (int)x.h_misc.p[6];
  return 0;
}

// The grid index over the target t[0, n) on grid g, whose box holds its n_fin finite points: the finite points sorted by
// cell into sorted (w = the original index; x.vals_b the sorted original indices), the CSR offsets cs and the coarse boxes
// box.
static int icp_build(flb_map* m, IcpIndex& x, const float4* t, int n, const IcpGrid& g, int n_fin, float4* sorted, int* cs, IcpBox* box) {
  const unsigned n_cells = (unsigned)g.gx * g.gy * g.gz;
  const int n_coarse = g.cx * g.cy * g.cz;
  size_t tb = x.tmp.cap;
  k_icp_keys<<<grid_for(n, 256, m->sm_count * 8), 256, 0, m->stream>>>(g, t, n, x.keys_a.p, x.vals_a.p);
  CU(cub::DeviceRadixSort::SortPairs(x.tmp.p, tb, (const unsigned*)x.keys_a.p, x.keys_b.p, (const int*)x.vals_a.p, x.vals_b.p, n, 0, 32,
                                     m->stream));
  k_icp_gather<<<grid_for(n_fin, 256, m->sm_count * 8), 256, 0, m->stream>>>(x.vals_b.p, t, n_fin, sorted);
  k_icp_cell_start<<<grid_for(n_fin + 1, 256, m->sm_count * 8), 256, 0, m->stream>>>(x.keys_b.p, n_fin, n_cells, cs);
  k_icp_coarse_boxes<<<grid_for(n_coarse, 8, m->sm_count * 8), 256, 0, m->stream>>>(sorted, cs, n_coarse, box);
  m->launches += 4 + 5;   // + the radix sort's kernels
  CU(cudaGetLastError());
  return 0;
}

// The grid index over the target t[0, n) into x: *n_fin finite points (0: nothing more is built), the grid *g over their
// box, then icp_build into x.sorted, x.cs and x.box.
static int icp_index(flb_map* m, IcpIndex& x, const float4* t, int n, IcpGrid* g, int* n_fin) {
  float lo[3], hi[3];
  if (icp_bounds(m, x, t, n, lo, hi, n_fin)) return 1;
  const int nf = *n_fin;
  if (nf == 0) return 0;
  *g = icp_grid(lo, hi, nf);
  const size_t n_cells = (size_t)g->gx * g->gy * g->gz, n_coarse = (size_t)g->cx * g->cy * g->cz;
  if (grow(x.cs, sizeof(int) * (n_cells + 1), 0) || grow(x.box, sizeof(IcpBox) * n_coarse, 0)) return 1;
  return icp_build(m, x, t, n, *g, nf, x.sorted.p, x.cs.p, x.box.p);
}

// The queries' visiting order: the keys the caller's key kernel wrote to x.keys_a (x.vals_a the identity), sorted into
// order (x.order unless given).
static int icp_order(flb_map* m, IcpIndex& x, int n_s, int* order = nullptr) {
  size_t tb = x.tmp.cap;
  CU(cub::DeviceRadixSort::SortPairs(x.tmp.p, tb, (const unsigned*)x.keys_a.p, x.keys_b.p, (const int*)x.vals_a.p, order ? order : x.order.p,
                                     n_s, 0, 32, m->stream));
  m->launches += 5;   // the radix sort's kernels
  CU(cudaGetLastError());
  return 0;
}

// k_reduce over n elements into out[0..K); the caller copies and synchronises.
template <int K, class Op>
static int icp_reduce(flb_map* m, IcpIndex& x, int n, const Op& op, double* out) {
  k_reduce<K, Op><<<m->sm_count * 2, 256, 0, m->stream>>>(n, op, x.partials.p, x.misc.p + ICP_MISC_COUNTER, out);
  m->launches++;
  CU(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------ host algebra
// One-sided Jacobi SVD of a 3x3 double matrix: A = U diag(s) V^T, s descending.  Columns of U for a zero singular value
// are completed to an orthonormal basis (u3 = u1 x u2).  Host and device (flb_keyframes_sicp solves it in every block of
// its ADMM kernel): only + - * / sqrt, so with -fmad=false both sides give the same bits.  The columns are ordered by a
// stable insertion sort written out as libstdc++'s std::sort runs it for three elements (a move to the front when the new
// element precedes the first, else a linear insert), so host results are those of the std::sort it replaced.
__host__ __device__ inline double icp_max(double a, double b) { return a < b ? b : a; }   // std::max

__host__ __device__ static void icp_svd3(const double A[9], double U[9], double s[3], double V[9]) {
  double B[9];
  memcpy(B, A, sizeof(B));
  for (int i = 0; i < 9; ++i) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double a = 0, b = 0, c = 0;
        for (int r = 0; r < 3; ++r) { a += B[3 * r + p] * B[3 * r + p]; b += B[3 * r + q] * B[3 * r + q]; c += B[3 * r + p] * B[3 * r + q]; }
        if (c == 0.0 || fabs(c) <= 1e-300) continue;
        off = icp_max(off, fabs(c) / sqrt(a * b));
        const double zeta = (b - a) / (2.0 * c);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
        for (int r = 0; r < 3; ++r) {
          const double bp = B[3 * r + p], bq = B[3 * r + q];
          B[3 * r + p] = cs * bp - sn * bq;
          B[3 * r + q] = sn * bp + cs * bq;
          const double vp = V[3 * r + p], vq = V[3 * r + q];
          V[3 * r + p] = cs * vp - sn * vq;
          V[3 * r + q] = sn * vp + cs * vq;
        }
      }
    if (!(off > 1e-15)) break;
  }
  int ord[3] = {0, 1, 2};
  double nrm[3];
  for (int j = 0; j < 3; ++j) nrm[j] = sqrt(B[j] * B[j] + B[3 + j] * B[3 + j] + B[6 + j] * B[6 + j]);
  for (int i = 1; i < 3; ++i) {   // descending by nrm
    const int v = ord[i];
    int j = i;
    if (nrm[v] > nrm[ord[0]]) {
      for (; j > 0; --j) ord[j] = ord[j - 1];
    } else {
      for (; nrm[v] > nrm[ord[j - 1]]; --j) ord[j] = ord[j - 1];
    }
    ord[j] = v;
  }
  double Bs[9], Vs[9];
  for (int j = 0; j < 3; ++j)
    for (int r = 0; r < 3; ++r) { Bs[3 * r + j] = B[3 * r + ord[j]]; Vs[3 * r + j] = V[3 * r + ord[j]]; }
  memcpy(V, Vs, sizeof(Vs));
  for (int j = 0; j < 3; ++j) s[j] = nrm[ord[j]];
  const double tiny = icp_max(s[0], 1e-300) * 1e-13;
  for (int j = 0; j < 3; ++j)
    for (int r = 0; r < 3; ++r) U[3 * r + j] = s[j] > tiny ? Bs[3 * r + j] / s[j] : 0.0;
  if (!(s[1] > tiny)) {   // rank <= 1: any unit vector orthogonal to u1
    const double u0[3] = {U[0], U[3], U[6]};
    double w[3] = {0, 0, 0};
    w[fabs(u0[0]) < 0.6 ? 0 : (fabs(u0[1]) < 0.6 ? 1 : 2)] = 1.0;
    const double d = w[0] * u0[0] + w[1] * u0[1] + w[2] * u0[2];
    double v[3] = {w[0] - d * u0[0], w[1] - d * u0[1], w[2] - d * u0[2]};
    const double nv = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    for (int r = 0; r < 3; ++r) U[3 * r + 1] = v[r] / nv;
  }
  if (!(s[2] > tiny)) {
    U[2] = U[3] * U[7] - U[6] * U[4];
    U[5] = U[6] * U[1] - U[0] * U[7];
    U[8] = U[0] * U[4] - U[3] * U[1];
  }
}

__host__ __device__ static double icp_det3(const double M[9]) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

// TransformationEstimationSVD (Umeyama, no scaling) from the sums S (the pairs record, then H = Σ (t - μt)(s - μs)^T):
// μ = Σ / count as the cross-product op forms it, H = U S V^T, R = U diag(1, 1, det U det V < 0 ? -1 : 1) V^T,
// t = μt - R μs, cast to a float row-major 4x4.
static void icp_rigid(const double* S, float T[16]) {
  double mu_s[3], mu_t[3], U[9], sv[3], V[9], R[9];
  for (int a = 0; a < 3; ++a) { mu_s[a] = S[2 + a] / S[0]; mu_t[a] = S[5 + a] / S[0]; }
  icp_svd3(S + 8, U, sv, V);
  const double d3 = icp_det3(U) * icp_det3(V) < 0 ? -1.0 : 1.0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[3 * r + c] = U[3 * r + 0] * V[3 * c + 0] + U[3 * r + 1] * V[3 * c + 1] + d3 * U[3 * r + 2] * V[3 * c + 2];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[4 * r + c] = (float)R[3 * r + c];
    T[4 * r + 3] = (float)(mu_t[r] - (R[3 * r] * mu_s[0] + R[3 * r + 1] * mu_s[1] + R[3 * r + 2] * mu_s[2]));
  }
  T[12] = T[13] = T[14] = 0.f;
  T[15] = 1.f;
}

// C = A * B in float, each entry ((a0 b0 + a1 b1) + a2 b2) + a3 b3 (final_transformation_ = transformation_ * final_).
static void icp_mul4(const float A[16], const float B[16], float C[16]) {
  float o[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) {
      volatile float acc = A[4 * r] * B[c];   // volatile: no contraction or reassociation by the host compiler
      acc = acc + A[4 * r + 1] * B[4 + c];
      acc = acc + A[4 * r + 2] * B[8 + c];
      acc = acc + A[4 * r + 3] * B[12 + c];
      o[4 * r + c] = acc;
    }
  memcpy(C, o, sizeof(o));
}

static IcpXf icp_xf(const float T[16], bool apply) {
  IcpXf x{};
  for (int i = 0; i < 12; ++i) x.m[i] = T[i];
  x.apply = apply ? 1 : 0;
  return x;
}

// DefaultConvergenceCriteria::hasConverged with max_iterations_similar_transforms_ = 0, after ++nr_iterations, on the
// increment T and the pairs found before it.  Returns the state (FLB_ICP_NOT_CONVERGED: go on); updates *prev_mse.
static int icp_converged(const flb_icp_config& cfg, int iterations, const float T[16], double n, double sum_d2, double* prev_mse) {
  if (iterations >= cfg.max_iterations) return FLB_ICP_ITERATIONS;
  const double cos_angle = 0.5 * ((double)T[0] + (double)T[5] + (double)T[10] - 1.0);
  const double tr2 = (double)T[3] * (double)T[3] + (double)T[7] * (double)T[7] + (double)T[11] * (double)T[11];
  if (cos_angle >= 1.0 - cfg.transformation_epsilon && tr2 <= cfg.transformation_epsilon) return FLB_ICP_TRANSFORM;
  const double mse = sum_d2 / n;
  if (std::fabs(mse - *prev_mse) < 1e-12) return FLB_ICP_ABS_MSE;
  if (std::fabs(mse - *prev_mse) / *prev_mse < cfg.euclidean_fitness_epsilon) return FLB_ICP_REL_MSE;
  *prev_mse = mse;
  return FLB_ICP_NOT_CONVERGED;
}

// ------------------------------------------------------------------------------------------------ device passes
constexpr int ICP_SUM_WORDS = 17;   // the pairs record (8), then the cross products (9)

// Scratch that follows the sizes of the two selections.
static int icp_scratch(flb_map* m, KfWork& k, int n_s, int n_t, bool pre) {
  IcpWork& w = k.icp;
  const size_t ps = sizeof(float4) * (size_t)n_s;
  if (icp_index_scratch(m, k.index, n_s, n_t, 0) || kf_grow(w.src_raw, ps) || (pre && kf_grow(w.src, ps)) || kf_grow(w.x, ps) ||
      kf_grow(w.tgt, sizeof(float4) * (size_t)n_t) || kf_grow(w.corr, sizeof(int) * (size_t)n_s) ||
      kf_grow(w.corr_d2, sizeof(float) * (size_t)n_s) || grow(w.sums, sizeof(double) * ICP_SUM_WORDS, 0) ||
      grow(w.h_sums, sizeof(double) * ICP_SUM_WORDS, 0))
    return 1;
  return 0;
}

// One exact 1-NN pass: q = xf(in[i]) into w.x, nearest target into w.corr / w.corr_d2.
static int icp_nn(flb_map* m, KfWork& k, const IcpGrid& g, const IcpXf& xf, const float4* in, int n_s) {
  IcpIndex& x = k.index;
  IcpWork& w = k.icp;
  unsigned* open_n = x.misc.p + ICP_MISC_OPEN;
  CU(cudaMemsetAsync(open_n, 0, sizeof(unsigned), m->stream));
  k_icp_nn<<<grid_for(n_s, 256, m->sm_count * 8), 256, 0, m->stream>>>(g, xf, x.order.p, n_s, in, w.x.p, x.sorted.p, x.cs.p, w.corr.p,
                                                                      w.corr_d2.p, x.open.p, (int*)open_n);
  k_icp_nn_far<<<m->sm_count * 8, 256, 0, m->stream>>>(g, x.open.p, (const int*)open_n, w.x.p, x.sorted.p, x.cs.p, x.box.p, w.corr.p,
                                                       w.corr_d2.p);
  m->launches += 2;
  CU(cudaGetLastError());
  return 0;
}

// The sums over the pairs of the last pass (with cross: also the cross products) and the copy of their record; the
// caller synchronises.
static int icp_sums(flb_map* m, KfWork& k, int n_s, double max_d2, bool cross) {
  IcpWork& w = k.icp;
  const IcpPairsOp pairs{w.corr.p, w.corr_d2.p, w.x.p, w.tgt.p, max_d2};
  if (icp_reduce<8>(m, k.index, n_s, pairs, w.sums.p) ||
      (cross && icp_reduce<9>(m, k.index, n_s, IcpCrossOp{pairs, w.sums.p}, w.sums.p + 8)))
    return 1;
  CU(cudaMemcpyAsync(w.h_sums.p, w.sums.p, sizeof(double) * ICP_SUM_WORDS, cudaMemcpyDeviceToHost, m->stream));
  return 0;
}

static void icp_no_pairs(int n_s, int* out_idx, float* out_d2) {
  for (int i = 0; i < n_s; ++i) {
    if (out_idx) out_idx[i] = -1;
    if (out_d2) out_d2[i] = INFINITY;
  }
}

static bool icp_cfg_ok(const flb_icp_config* c) {
  return std::isfinite(c->max_correspondence_distance) && std::isfinite(c->transformation_epsilon) &&
         std::isfinite(c->euclidean_fitness_epsilon) && c->max_iterations >= 0 && c->max_correspondence_distance >= 0;
}

extern "C" int flb_keyframes_icp(flb_keyframes* k, const int* src_ids, int n_src, int src_kind, const float* src_transforms,
                                 const float* src_pre_pose6, const int* tgt_ids, int n_tgt, int tgt_kind, const float* tgt_transforms,
                                 const flb_icp_config* cfg, flb_icp_result* out, int* out_corr_index, float* out_corr_d2) {
  const char* who = "flb_keyframes_icp";
  if (!out) return set_err("%s: null result", who);
  if (!cfg) return set_err("%s: null config", who);
  if (!icp_cfg_ok(cfg))
    return set_err("%s: config values must be finite, max_iterations >= 0 and max_correspondence_distance >= 0", who);
  if (n_src < 0 || n_tgt < 0) return set_err("%s: negative n_src or n_tgt", who);
  if ((n_src > 0 && (!src_ids || !src_transforms)) || (n_tgt > 0 && (!tgt_ids || !tgt_transforms)))
    return set_err("%s: null ids or transforms", who);
  for (int kind : {src_kind, tgt_kind})
    if (kind != FLB_KF_POSE6 && kind != FLB_KF_AFFINE)
      return set_err("%s: transform kinds must be FLB_KF_POSE6 (%d) or FLB_KF_AFFINE (%d)", who, FLB_KF_POSE6, FLB_KF_AFFINE);
  if (!k) return set_err("%s: null key-frame store", who);
  int n_s = 0, n_t = 0;
  if (kf_selection(k, src_ids, n_src, who, &n_s) || kf_selection(k, tgt_ids, n_tgt, who, &n_t)) return 1;

  flb_icp_result res{};
  for (int i = 0; i < 16; ++i) res.final_transformation[i] = (i % 5 == 0) ? 1.f : 0.f;
  res.state = FLB_ICP_NOT_CONVERGED;
  res.n_source = n_s;
  res.n_target = n_t;
  res.fitness_score = DBL_MAX;
  if (n_s == 0 || n_t == 0) {   // initCompute fails: nothing registered
    icp_no_pairs(n_s, out_corr_index, out_corr_d2);
    *out = res;
    return 0;
  }
  flb_map* m = k->map;
  CU(cudaSetDevice(m->cfg.device));
  if (kf_work(m) || icp_scratch(m, *m->kfw, n_s, n_t, src_pre_pose6 != nullptr)) return 1;
  KfWork& kw = *m->kfw;
  IcpWork& w = kw.icp;

  // the two loop sub-maps (loopFindNearKeyframes, :918-920), then cureKeyframeCloud = transformPointCloud(.., &com)
  std::vector<KfSeg> segs;
  kf_selection_segs(k, tgt_ids, n_tgt, tgt_kind, tgt_transforms, segs);
  if (kf_assemble_enqueue(m, segs, k->xyzi, nullptr, n_t, w.tgt.p, nullptr)) return 1;
  kf_selection_segs(k, src_ids, n_src, src_kind, src_transforms, segs);
  if (kf_assemble_enqueue(m, segs, k->xyzi, nullptr, n_s, w.src_raw.p, nullptr)) return 1;
  const float4* S = w.src_raw.p;
  if (src_pre_pose6) {
    const std::vector<KfSeg> pre{kf_seg(affine_from_rpy(src_pre_pose6).t, false, 0, 0, n_s)};
    if (kf_assemble_enqueue(m, pre, w.src_raw.p, nullptr, n_s, w.src.p, nullptr)) return 1;
    S = w.src.p;
  }

  // the target's index, then the source's visiting order
  IcpGrid g{};
  int n_fin = 0;
  if (icp_index(m, kw.index, w.tgt.p, n_t, &g, &n_fin)) return 1;
  if (n_fin == 0) {   // every target point dropped by KdTreeFLANN: initCompute fails
    icp_no_pairs(n_s, out_corr_index, out_corr_d2);
    *out = res;
    return 0;
  }
  k_icp_keys<<<grid_for(n_s, 256, m->sm_count * 8), 256, 0, m->stream>>>(g, S, n_s, kw.index.keys_a.p, kw.index.vals_a.p);
  m->launches++;
  if (icp_order(m, kw.index, n_s)) return 1;

  // the iterations (icp.hpp computeTransformation)
  const double max_d2 = cfg->max_correspondence_distance * cfg->max_correspondence_distance;
  float T[16], final_T[16];
  memcpy(final_T, res.final_transformation, sizeof(final_T));
  memcpy(T, final_T, sizeof(T));
  double prev_mse = DBL_MAX;
  for (int it = 0;; ++it) {
    // input_transformed <- T_{k-1} * input_transformed, fused into the pass (iteration 0 reads the source itself)
    if (icp_nn(m, kw, g, icp_xf(T, it > 0), it == 0 ? S : w.x.p, n_s) || icp_sums(m, kw, n_s, max_d2, true)) return 1;
    CU(cudaStreamSynchronize(m->stream));
    const double* sm = w.h_sums.p;
    res.n_correspondences = (int)sm[0];
    if (sm[0] < 3) {   // min_number_correspondences_
      res.state = FLB_ICP_NO_CORRESPONDENCES;
      break;
    }
    icp_rigid(sm, T);
    icp_mul4(T, final_T, final_T);
    res.iterations = it + 1;
    res.state = icp_converged(*cfg, res.iterations, T, sm[0], sm[1], &prev_mse);
    if (res.state != FLB_ICP_NOT_CONVERGED) {
      res.converged = 1;
      break;
    }
  }
  memcpy(res.final_transformation, final_T, sizeof(final_T));
  if (out_corr_index) CU(cudaMemcpyAsync(out_corr_index, w.corr.p, sizeof(int) * (size_t)n_s, cudaMemcpyDeviceToHost, m->stream));
  if (out_corr_d2) CU(cudaMemcpyAsync(out_corr_d2, w.corr_d2.p, sizeof(float) * (size_t)n_s, cudaMemcpyDeviceToHost, m->stream));

  // getFitnessScore(): the original source transformed once by final, every finite point's nearest d², no cut
  if (icp_nn(m, kw, g, icp_xf(final_T, true), S, n_s) || icp_sums(m, kw, n_s, DBL_MAX, false)) return 1;
  CU(cudaStreamSynchronize(m->stream));
  const double* fs = w.h_sums.p;
  res.fitness_score = fs[0] > 0 ? fs[1] / fs[0] : DBL_MAX;
  *out = res;
  return 0;
}

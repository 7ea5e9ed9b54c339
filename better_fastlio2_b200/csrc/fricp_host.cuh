// fricp_host.cuh — the relocaliser's registration (online_relocalization / pose_estimator::run, reg[0].run(curCloud,
// nearCloud) with Registeration(regMode), include/FRICP-toolkit/registeration.h:36-175) for regMode 0, 2, 3 and 4: a host
// source cloud onto a target assembled from the device key-frame store with two transform stages per key frame
// (transformPointCloud(transformPointCloud(cloud, &pose_ext), &poses6D[k]), pose_estimator.cpp:189-194).  The clouds are
// normalised on the device (extent, fixed-order double means), the loop ICP's index (icp_host.cuh) is built once over
// the target, the Welsch scale's end value comes from an exact 7-NN self-query and a device sort, and every iteration is
// one double 1-NN pass, one fused reduction (energy and weighted moments), one small copy and one synchronisation.  The
// 3x3 SVD, the SE(3) log / exp, Anderson acceleration and the stopping tests run here on the host.  DESIGN.md §9 states
// the contract.  Included after icp_host.cuh.
#pragma once
#include <cfloat>
#include <cmath>

#include "fricp_kernels.cuh"

constexpr int FR_SUM_MEAN_S = 0, FR_SUM_MEAN_T = 4, FR_SUM_STEP = 8, FR_SUM_MED = 32, FR_SUM_WORDS = 40;

static int fricp_scratch(flb_map* m, KfWork& k, int n_s, int n_t, bool pre_src, bool two_stage) {
  FricpWork& w = k.fricp;
  const size_t ps = sizeof(float4) * (size_t)n_s, pt = sizeof(float4) * (size_t)n_t;
  const int nk = std::max(n_s, n_t);
  size_t t2 = 0;
  CU(cub::DeviceRadixSort::SortKeys(nullptr, t2, (const double*)nullptr, (double*)nullptr, nk));
  if (icp_index_scratch(m, k.index, n_s, n_t, t2) || kf_grow(w.src_raw, ps) || (pre_src && kf_grow(w.src, ps)) ||
      (two_stage && kf_grow(w.tgt_a, pt)) || kf_grow(w.tgt, pt) || kf_grow(w.tgtf, pt) || kf_grow(w.x, sizeof(double4) * (size_t)n_s) ||
      kf_grow(w.tn, sizeof(double4) * (size_t)n_t) || kf_grow(w.sorted_d, sizeof(double4) * (size_t)n_t) ||
      kf_grow(w.pos, sizeof(int) * (size_t)n_s) || kf_grow(w.d2, sizeof(double) * (size_t)n_s) || kf_grow(w.med, sizeof(double) * (size_t)n_t) ||
      kf_grow(w.sort_a, sizeof(double) * (size_t)nk) || kf_grow(w.sort_b, sizeof(double) * (size_t)nk) ||
      kf_grow(w.corr, sizeof(int) * (size_t)n_s) || grow(w.sums, sizeof(double) * FR_SUM_WORDS, 0) ||
      grow(w.h_sums, sizeof(double) * FR_SUM_WORDS, 0))
    return 1;
  return 0;
}

// ------------------------------------------------------------------------------------------------ host algebra
// SE(3) log / exp in closed form (they replace LogMatrix's RealSchur and Eigen's Padé exp, FRICP.h:41-89, :498).
// T: row-major 3x4 [R | t]; L: the 4x4 log matrix's 16 entries column-major, the vector Anderson works on.
static void fr_log(const double* T, double* L) {
  const double* R = T;
  const double c = std::max(-1.0, std::min(1.0, 0.5 * ((R[0] + R[5] + R[10]) - 1.0)));
  const double a[3] = {R[9] - R[6], R[2] - R[8], R[4] - R[1]};   // 2 sin(th) * axis
  const double th = std::atan2(0.5 * std::sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]), c);   // better than acos(c) near 0, pi
  double w[3];
  if (th < 1e-5) {
    const double f = 0.5 + th * th / 12.0;
    for (int k = 0; k < 3; ++k) w[k] = f * a[k];
  } else if (th < M_PI - 1e-5) {
    const double f = th / (2.0 * std::sin(th));
    for (int k = 0; k < 3; ++k) w[k] = f * a[k];
  } else {   // near pi: axis from (R + R^T)/2 - cos(th) I = (1 - cos th) k k^T, sign from the antisymmetric part
    const double d[3] = {R[0] - c, R[5] - c, R[10] - c};
    int i = 0;
    for (int k = 1; k < 3; ++k) if (d[k] > d[i]) i = k;
    double v[3];
    for (int k = 0; k < 3; ++k) v[k] = 0.5 * (R[4 * i + k] + R[4 * k + i]) - (k == i ? c : 0.0);
    const double n = std::sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
    const double s = ((a[0] * v[0] + a[1] * v[1]) + a[2] * v[2]) < 0 ? -1.0 : 1.0;
    for (int k = 0; k < 3; ++k) w[k] = s * th * v[k] / n;
  }
  const double th2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2], t = std::sqrt(th2);
  const double b = t < 1e-4 ? 1.0 / 12.0 + th2 / 720.0 : (1.0 - t * std::sin(t) / (2.0 * (1.0 - std::cos(t)))) / th2;
  const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  const double tv[3] = {T[3], T[7], T[11]};
  double Wt[3], WWt[3];
  for (int r = 0; r < 3; ++r) Wt[r] = (W[3 * r] * tv[0] + W[3 * r + 1] * tv[1]) + W[3 * r + 2] * tv[2];
  for (int r = 0; r < 3; ++r) WWt[r] = (W[3 * r] * Wt[0] + W[3 * r + 1] * Wt[1]) + W[3 * r + 2] * Wt[2];
  for (int i = 0; i < 16; ++i) L[i] = 0.0;
  for (int r = 0; r < 3; ++r) {
    for (int cc = 0; cc < 3; ++cc) L[4 * cc + r] = W[3 * r + cc];
    L[12 + r] = (tv[r] - 0.5 * Wt[r]) + b * WWt[r];
  }
}

static void fr_exp(const double* L, double* T) {
  const double w[3] = {L[6], L[8], L[1]}, u[3] = {L[12], L[13], L[14]};
  const double th2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2], th = std::sqrt(th2);
  double A, B, C;   // sin th / th, (1 - cos th) / th^2, (th - sin th) / th^3
  if (th < 1e-4) {
    A = 1.0 - th2 / 6.0;
    B = 0.5 - th2 / 24.0;
    C = 1.0 / 6.0 - th2 / 120.0;
  } else {
    A = std::sin(th) / th;
    B = (1.0 - std::cos(th)) / th2;
    C = (th - std::sin(th)) / (th2 * th);
  }
  const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  double W2[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) W2[3 * r + c] = (W[3 * r] * W[c] + W[3 * r + 1] * W[3 + c]) + W[3 * r + 2] * W[6 + c];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[4 * r + c] = ((r == c ? 1.0 : 0.0) + A * W[3 * r + c]) + B * W2[3 * r + c];
    double t = 0;
    for (int c = 0; c < 3; ++c) t += (((r == c ? 1.0 : 0.0) + B * W[3 * r + c]) + C * W2[3 * r + c]) * u[c];
    T[4 * r + 3] = t;
  }
}

// Min-norm solution of the symmetric n x n system M x = b (n <= 5): Jacobi eigen-decomposition, eigenvalues with
// |λ| <= n * DBL_EPSILON * max |λ| treated as zero (the rank threshold of Eigen's CompleteOrthogonalDecomposition).
static void fr_pinv_solve(const double* M, int n, const double* b, double* x) {
  double A[25], V[25];
  memcpy(A, M, sizeof(double) * n * n);
  for (int i = 0; i < n * n; ++i) V[i] = (i % (n + 1) == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 100; ++sweep) {
    double off = 0, diag = 0;
    for (int i = 0; i < n; ++i) {
      diag += A[i * n + i] * A[i * n + i];
      for (int j = i + 1; j < n; ++j) off += A[i * n + j] * A[i * n + j];
    }
    if (!(off > 1e-32 * diag)) break;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = A[p * n + q];
        if (apq == 0.0) continue;
        const double zeta = (A[q * n + q] - A[p * n + p]) / (2.0 * apq);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
        const double cs = 1.0 / std::sqrt(1.0 + t * t), sn = cs * t;
        for (int k = 0; k < n; ++k) {
          const double akp = A[k * n + p], akq = A[k * n + q];
          A[k * n + p] = cs * akp - sn * akq;
          A[k * n + q] = sn * akp + cs * akq;
        }
        for (int k = 0; k < n; ++k) {
          const double apk = A[p * n + k], aqk = A[q * n + k];
          A[p * n + k] = cs * apk - sn * aqk;
          A[q * n + k] = sn * apk + cs * aqk;
        }
        for (int k = 0; k < n; ++k) {
          const double vp = V[k * n + p], vq = V[k * n + q];
          V[k * n + p] = cs * vp - sn * vq;
          V[k * n + q] = sn * vp + cs * vq;
        }
      }
  }
  double lmax = 0;
  for (int i = 0; i < n; ++i) lmax = std::max(lmax, std::fabs(A[i * n + i]));
  const double thr = lmax * n * DBL_EPSILON;
  for (int i = 0; i < n; ++i) x[i] = 0.0;
  for (int e = 0; e < n; ++e) {
    const double l = A[e * n + e];
    if (!(std::fabs(l) > thr)) continue;
    double vb = 0;
    for (int k = 0; k < n; ++k) vb += V[k * n + e] * b[k];
    for (int k = 0; k < n; ++k) x[k] += V[k * n + e] * (vb / l);
  }
}

// AndersonAcceleration.h (m <= 5, dimension 16) with the normal equations solved by fr_pinv_solve.
struct FrAnderson {
  int m = 0, iter = 0, col = 0;
  double u[16], F[16], dG[5][16], dF[5][16], M[5][5], theta[5], scale[5];
  void init(int m_, const double* u0) { m = m_; memcpy(u, u0, sizeof(u)); iter = 0; col = 0; }
  void replace(const double* v) { memcpy(u, v, sizeof(u)); }
  void reset(const double* v) { iter = 0; col = 0; memcpy(u, v, sizeof(u)); }
  const double* compute(const double* g) {
    const int d = 16;
    for (int i = 0; i < d; ++i) F[i] = g[i] - u[i];
    if (iter == 0) {
      for (int i = 0; i < d; ++i) { dF[0][i] = -F[i]; dG[0][i] = -g[i]; u[i] = g[i]; }
    } else {
      for (int i = 0; i < d; ++i) { dF[col][i] += F[i]; dG[col][i] += g[i]; }
      const double eps = 1e-14;
      double nn = 0;
      for (int i = 0; i < d; ++i) nn += dF[col][i] * dF[col][i];
      const double sc = std::max(eps, std::sqrt(nn));
      scale[col] = sc;
      for (int i = 0; i < d; ++i) dF[col][i] /= sc;
      const int mk = std::min(m, iter);
      if (mk == 1) {
        theta[0] = 0;
        double sq = 0;
        for (int i = 0; i < d; ++i) sq += dF[col][i] * dF[col][i];
        M[0][0] = sq;
        const double nrm = std::sqrt(sq);
        if (nrm > eps) {
          double dot = 0;
          for (int i = 0; i < d; ++i) dot += (dF[col][i] / nrm) * (F[i] / nrm);
          theta[0] = dot;
        }
      } else {
        for (int j = 0; j < mk; ++j) {
          double ip = 0;
          for (int i = 0; i < d; ++i) ip += dF[col][i] * dF[j][i];
          M[col][j] = ip;
          M[j][col] = ip;
        }
        double Mk[25], rhs[5];
        for (int r = 0; r < mk; ++r) {
          for (int c = 0; c < mk; ++c) Mk[r * mk + c] = M[r][c];
          double s = 0;
          for (int i = 0; i < d; ++i) s += dF[r][i] * F[i];
          rhs[r] = s;
        }
        fr_pinv_solve(Mk, mk, rhs, theta);
      }
      for (int i = 0; i < d; ++i) {
        double s = 0;
        for (int j = 0; j < mk; ++j) s += dG[j][i] * (theta[j] / scale[j]);
        u[i] = g[i] - s;
      }
      col = (col + 1) % m;
      for (int i = 0; i < d; ++i) { dF[col][i] = -F[i]; dG[col][i] = -g[i]; }
    }
    ++iter;
    return u;
  }
};

// The weighted point-to-point step (FRICP.h:177-209) from the step record: R = V diag(1, 1, ±1) U^T of the SVD of the
// weighted cross-covariance Σ wn (x - x̄)(q - q̄)^T, t = q̄ - R x̄.  T is left as it is when every weight is 0.
static void fr_kabsch(const double* S, double* T) {
  if (!(S[0] > 0)) return;
  double xm[3], qm[3], sig[9], U[9], sv[3], V[9];
  for (int a = 0; a < 3; ++a) { xm[a] = S[1 + a] / S[0]; qm[a] = S[4 + a] / S[0]; }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) sig[3 * r + c] = S[7 + 3 * r + c] / S[0] - xm[r] * qm[c];
  icp_svd3(sig, U, sv, V);
  const double dd = icp_det3(U) * icp_det3(V) < 0 ? -1.0 : 1.0;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[4 * r + c] = (V[3 * r] * U[3 * c] + V[3 * r + 1] * U[3 * c + 1]) + dd * V[3 * r + 2] * U[3 * c + 2];
    T[4 * r + 3] = qm[r] - ((T[4 * r] * xm[0] + T[4 * r + 1] * xm[1]) + T[4 * r + 2] * xm[2]);
  }
}

// ------------------------------------------------------------------------------------------------ device passes
// One exact double 1-NN pass of the normalised source w.x with T applied in the pass: w.pos, w.d2.
static int fr_nn(flb_map* m, KfWork& k, const IcpGrid& g, int n_s, const double* T) {
  IcpIndex& x = k.index;
  FricpWork& w = k.fricp;
  FrXf xf;
  memcpy(xf.m, T, sizeof(xf.m));
  int* open_n = (int*)(x.misc.p + ICP_MISC_OPEN);
  CU(cudaMemsetAsync(open_n, 0, sizeof(int), m->stream));
  k_fr_nn<<<grid_for(n_s, 256, m->sm_count * 8), 256, 0, m->stream>>>(g, xf, x.order.p, n_s, w.x.p, w.sorted_d.p, x.cs.p, w.pos.p,
                                                                      w.d2.p, x.open.p, open_n);
  k_fr_nn_far<<<m->sm_count * 8, 256, 0, m->stream>>>(g, xf, x.open.p, open_n, w.x.p, w.sorted_d.p, x.cs.p, x.box.p, w.pos.p, w.d2.p);
  m->launches += 2;
  CU(cudaGetLastError());
  return 0;
}

// One 1-NN pass (when nn) with T applied in the pass, then the step record (energy and weighted moments at nu) and its
// copy.  The caller synchronises.
static int fr_pass(flb_map* m, KfWork& k, const IcpGrid& g, int n_s, const double* T, bool nn, double nu, bool welsch) {
  IcpIndex& x = k.index;
  FricpWork& w = k.fricp;
  if (nn && fr_nn(m, k, g, n_s, T)) return 1;
  const FrStepOp op{w.x.p, w.sorted_d.p, w.pos.p, w.d2.p, nu, welsch ? 1 : 0};
  if (icp_reduce<FR_RED>(m, x, n_s, op, w.sums.p + FR_SUM_STEP)) return 1;
  CU(cudaMemcpyAsync(w.h_sums.p + FR_SUM_STEP, w.sums.p + FR_SUM_STEP, sizeof(double) * FR_RED, cudaMemcpyDeviceToHost, m->stream));
  return 0;
}

// igl::median of the first n values of `in` (non-finite ones sort last): a device radix sort, then the middle one or two.
static int fr_median(flb_map* m, KfWork& k, const double* in, int n_all, int n, double* out) {
  FricpWork& w = k.fricp;
  size_t tb = k.index.tmp.cap;
  CU(cub::DeviceRadixSort::SortKeys(k.index.tmp.p, tb, in, w.sort_b.p, n_all, 0, 64, m->stream));
  m->launches += 5;   // the radix sort's kernels
  const int h = n / 2;
  const int first = n % 2 == 0 ? h - 1 : h, cnt = n % 2 == 0 ? 2 : 1;
  CU(cudaMemcpyAsync(w.h_sums.p + FR_SUM_MED, w.sort_b.p + first, sizeof(double) * cnt, cudaMemcpyDeviceToHost, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  const double* v = w.h_sums.p + FR_SUM_MED;
  *out = cnt == 2 ? 0.5 * (v[1] + v[0]) : v[0];
  return 0;
}

static bool fr_finite(const float* p, int n) {
  for (int i = 0; i < n; ++i)
    if (!std::isfinite(p[i])) return false;
  return true;
}

static int fr_cfg_check(const flb_fricp_config* c, const char* who) {
  if (c->mode != 0 && c->mode != 2 && c->mode != 3 && c->mode != 4)
    return set_err("%s: regMode %d is not supported (the point-to-point modes 0 ICP, 2 Fast ICP, 3 Robust ICP and 4 Fast and "
                   "Robust ICP are)", who, c->mode);
  if (c->max_icp < 0) return set_err("%s: max_icp must be >= 0 (got %d)", who, c->max_icp);
  if (!(std::isfinite(c->stop) && c->stop >= 0)) return set_err("%s: stop must be finite and >= 0", who);
  if (c->anderson_m < 1 || c->anderson_m > 5) return set_err("%s: anderson_m must be in [1, 5] (got %d)", who, c->anderson_m);
  if (!(std::isfinite(c->nu_begin_k) && c->nu_begin_k > 0) || !(std::isfinite(c->nu_end_k) && c->nu_end_k > 0))
    return set_err("%s: nu_begin_k and nu_end_k must be finite and > 0", who);
  if (!(c->nu_alpha > 0 && c->nu_alpha < 1)) return set_err("%s: nu_alpha must be in (0, 1)", who);
  return 0;
}

extern "C" void flb_fricp_default_config(flb_fricp_config* c) {
  if (!c) return;
  c->mode = FLB_FRICP_FAST_ROBUST;
  c->max_icp = 100;
  c->stop = 1e-5;
  c->anderson_m = 5;
  c->nu_begin_k = 3.0;
  c->nu_end_k = 1.0 / (3.0 * std::sqrt(3.0));
  c->nu_alpha = 0.5;
}

// What fr_setup leaves for the registration: the sizes, the normalisation (p_n = p / scale - mu), the target grid and the
// host synchronisations it made.  status < 0: go on; otherwise the call ends with that FLB_FRICP_* status (the counts,
// and the normalisation once it is known, are filled).
struct FrSetup {
  int status = -1;
  int n_s = 0, n_t = 0, n_fs = 0, n_ft = 0;
  double scale = 1.0, mu_s[3] = {0, 0, 0}, mu_t[3] = {0, 0, 0};
  IcpGrid g{};
  int syncs = 0;
};

// The set-up both relocalisation registrations share (DESIGN.md §9, items 1-2 of flb_keyframes_fricp's contract): the
// argument checks after the config's, the upload of the host source and its pose, the two-stage target assembly, the
// finite counts and boxes, the scale, the fixed-order means, the normalised double clouds in w.x / w.tn, the grid index
// over the float normalised target, the sorted double target w.sorted_d and the source's visiting order.  The optional
// per-source outputs are set to "no match" first.  Ends early (st->status) without a launch for an empty source or
// selection, and after the bounds when there is no finite source point or fewer than min_target finite target points.
static int fr_setup(flb_keyframes* k, const char* who, const void* src_pts, int n_src, int src_stride, int src_off_intensity,
                    const float* src_pose6, const int* tgt_ids, int n_tgt, const float* tgt_pre_pose6, const float* tgt_poses6,
                    int* out_corr_index, double* out_resid, const double* out_log, int log_cap, int min_target, FrSetup* st) {
  if (n_src < 0 || n_tgt < 0) return set_err("%s: negative n_src or n_tgt", who);
  if (n_src > 0 && (!src_pts || src_stride < 12)) return set_err("%s: null source or stride below 12 bytes", who);
  if (src_off_intensity >= 0 && src_off_intensity + 4 > src_stride) return set_err("%s: intensity offset outside the point stride", who);
  if (n_tgt > 0 && (!tgt_ids || !tgt_poses6)) return set_err("%s: null target ids or poses", who);
  if (log_cap < 0 || (log_cap > 0 && !out_log)) return set_err("%s: log_cap must be >= 0, with a log buffer when > 0", who);
  if ((src_pose6 && !fr_finite(src_pose6, 6)) || (tgt_pre_pose6 && !fr_finite(tgt_pre_pose6, 6)) ||
      (n_tgt > 0 && !fr_finite(tgt_poses6, 6 * n_tgt)))
    return set_err("%s: poses must be finite", who);
  if (!k) return set_err("%s: null key-frame store", who);
  int n_t = 0;
  if (kf_selection(k, tgt_ids, n_tgt, who, &n_t)) return 1;
  const int n_s = n_src;
  st->n_s = n_s;
  st->n_t = n_t;
  for (int i = 0; i < n_s; ++i) {
    if (out_corr_index) out_corr_index[i] = -1;
    if (out_resid) out_resid[i] = INFINITY;
  }
  if (n_t == 0 || n_s == 0) {   // nothing to register: no launch
    st->status = n_s == 0 ? FLB_FRICP_NO_SOURCE : FLB_FRICP_FEW_TARGET;
    return 0;
  }
  flb_map* m = k->map;
  CU(cudaSetDevice(m->cfg.device));
  if (kf_work(m) || fricp_scratch(m, *m->kfw, n_s, n_t, src_pose6 != nullptr, tgt_pre_pose6 != nullptr)) return 1;
  KfWork& kw = *m->kfw;
  IcpIndex& x = kw.index;
  FricpWork& w = kw.fricp;

  // curCloud = transformPointCloud(cloud, &initPose) (pose_estimator.cpp:185)
  if (upload_records(m, m->stream, w.raw, 0, src_pts, n_s, src_stride, src_off_intensity, -1, w.src_raw.p, nullptr)) return 1;
  const float4* src = w.src_raw.p;
  if (src_pose6) {
    const std::vector<KfSeg> pre{kf_seg(affine_from_rpy(src_pose6).t, false, 0, 0, n_s)};
    if (kf_assemble_enqueue(m, pre, w.src_raw.p, nullptr, n_s, w.src.p, nullptr)) return 1;
    src = w.src.p;
  }
  // nearCloud = Σ transformPointCloud(transformPointCloud(cloud[k], &pose_ext), &poses6D[k]) (:189-194)
  std::vector<KfSeg> segs;
  int dst = 0;
  for (int j = 0; j < n_tgt; ++j) {
    const int c = k->cnt[tgt_ids[j]];
    if (c == 0) continue;
    segs.push_back(kf_seg(affine_from_rpy(tgt_pre_pose6 ? tgt_pre_pose6 : tgt_poses6 + 6 * j).t, false, k->off[tgt_ids[j]], dst, c));
    dst += c;
  }
  if (kf_assemble_enqueue(m, segs, k->xyzi, nullptr, n_t, tgt_pre_pose6 ? w.tgt_a.p : w.tgt.p, nullptr)) return 1;
  if (tgt_pre_pose6) {
    for (size_t s = 0, j = 0; s < segs.size(); ++j) {
      if (k->cnt[tgt_ids[j]] == 0) continue;
      segs[s] = kf_seg(affine_from_rpy(tgt_poses6 + 6 * j).t, false, segs[s].dst_off, segs[s].dst_off, segs[s].count);
      ++s;
    }
    if (kf_assemble_enqueue(m, segs, w.tgt_a.p, nullptr, n_t, w.tgt.p, nullptr)) return 1;
  }

  // finite counts and boxes of both clouds -> scale (registeration.h:47-53)
  float lo[2][3], hi[2][3];
  int n_fs = 0, n_ft = 0;
  if (icp_bounds(m, x, src, n_s, lo[0], hi[0], &n_fs) || icp_bounds(m, x, w.tgt.p, n_t, lo[1], hi[1], &n_ft)) return 1;
  st->syncs += 2;
  st->n_fs = n_fs;
  st->n_ft = n_ft;
  if (n_ft < min_target || n_fs == 0) {
    st->status = n_fs == 0 ? FLB_FRICP_NO_SOURCE : FLB_FRICP_FEW_TARGET;
    return 0;
  }
  double ext[2];
  for (int c = 0; c < 2; ++c) {
    double e[3];
    for (int a = 0; a < 3; ++a) e[a] = (double)hi[c][a] - (double)lo[c][a];
    ext[c] = std::sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]);
  }
  double scale = std::max(ext[0], ext[1]);
  if (!(scale > 0)) scale = 1.0;   // every finite point of both clouds at one place: nothing to scale

  // means (fixed order), normalised clouds, the float target for the index
  if (icp_reduce<3>(m, x, n_s, FrMeanOp{src, scale}, w.sums.p + FR_SUM_MEAN_S) ||
      icp_reduce<3>(m, x, n_t, FrMeanOp{w.tgt.p, scale}, w.sums.p + FR_SUM_MEAN_T))
    return 1;
  CU(cudaMemcpyAsync(w.h_sums.p, w.sums.p, sizeof(double) * 8, cudaMemcpyDeviceToHost, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  st->syncs++;
  double* mu_s = st->mu_s;
  double* mu_t = st->mu_t;
  for (int a = 0; a < 3; ++a) {
    mu_s[a] = w.h_sums.p[FR_SUM_MEAN_S + a] / (double)n_fs;
    mu_t[a] = w.h_sums.p[FR_SUM_MEAN_T + a] / (double)n_ft;
    w.h_sums.p[FR_SUM_MEAN_S + a] = mu_s[a];
    w.h_sums.p[FR_SUM_MEAN_T + a] = mu_t[a];
  }
  CU(cudaMemcpyAsync(w.sums.p, w.h_sums.p, sizeof(double) * 8, cudaMemcpyHostToDevice, m->stream));
  k_fr_normalise<<<grid_for(n_s, 256, m->sm_count * 8), 256, 0, m->stream>>>(src, n_s, scale, w.sums.p + FR_SUM_MEAN_S, w.x.p, nullptr);
  k_fr_normalise<<<grid_for(n_t, 256, m->sm_count * 8), 256, 0, m->stream>>>(w.tgt.p, n_t, scale, w.sums.p + FR_SUM_MEAN_T, w.tn.p, w.tgtf.p);
  m->launches += 2;
  CU(cudaGetLastError());
  st->scale = scale;

  // the loop ICP's index over the float normalised target (its finite points are the target's), the sorted double
  // target beside it, the source's visiting order
  int n_fin = 0;
  if (icp_index(m, x, w.tgtf.p, n_t, &st->g, &n_fin)) return 1;
  st->syncs++;
  const int gs = grid_for(n_s, 256, m->sm_count * 8);
  k_fr_gather<<<grid_for(n_ft, 256, m->sm_count * 8), 256, 0, m->stream>>>(x.vals_b.p, w.tn.p, n_ft, w.sorted_d.p);
  k_fr_keys<<<gs, 256, 0, m->stream>>>(st->g, w.x.p, n_s, x.keys_a.p, x.vals_a.p);
  m->launches += 2;
  if (icp_order(m, x, n_s)) return 1;
  return 0;
}

// The result's normalisation and counts from the set-up.
template <class R>
static void fr_setup_result(const FrSetup& st, R& res) {
  res.n_source = st.n_s;
  res.n_target = st.n_t;
  res.n_source_finite = st.n_fs;
  res.n_target_finite = st.n_ft;
  res.scale = st.scale;
  for (int a = 0; a < 3; ++a) { res.mu_source[a] = st.mu_s[a]; res.mu_target[a] = st.mu_t[a]; }
  if (st.status >= 0) res.status = st.status;
}

// res_trans from T (row-major 3x4, normalised frame): t <- t - R mu_s + mu_t, then t * scale (FRICP.h:536, ICP.h:373,
// registeration.h:170).
static void fr_res_trans(const FrSetup& st, const double* T, double* out) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) out[4 * r + c] = T[4 * r + c];
    out[4 * r + 3] = (T[4 * r + 3] + (st.mu_t[r] - ((T[4 * r] * st.mu_s[0] + T[4 * r + 1] * st.mu_s[1]) + T[4 * r + 2] * st.mu_s[2]))) *
                     st.scale;
  }
}

// The matched target index and residual of the last 1-NN pass (optional outputs); the caller synchronises.
static int fr_outputs(flb_map* m, KfWork& kw, int n_s, int* out_corr_index, double* out_resid) {
  FricpWork& w = kw.fricp;
  const int gs = grid_for(n_s, 256, m->sm_count * 8);
  if (out_corr_index) {
    k_fr_corr_index<<<gs, 256, 0, m->stream>>>(w.pos.p, w.sorted_d.p, n_s, w.corr.p);
    m->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out_corr_index, w.corr.p, sizeof(int) * (size_t)n_s, cudaMemcpyDeviceToHost, m->stream));
  }
  if (out_resid) {
    k_fr_resid<<<gs, 256, 0, m->stream>>>(w.d2.p, n_s, w.sort_a.p);
    m->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out_resid, w.sort_a.p, sizeof(double) * (size_t)n_s, cudaMemcpyDeviceToHost, m->stream));
  }
  return 0;
}

// Where a result counts its host synchronisations: SICP's and AA-ICP's do, FRICP's has no such count.
static int* fr_syncs(flb_fricp_result&) { return nullptr; }
template <class R>
static int* fr_syncs(R& res) { return &res.syncs; }

// The opening every relocalisation registration shares: the null and config checks, fr_setup, and res as the identity
// with the set-up's counts and normalisation.  When the set-up ends the call (st.status >= 0) res is also written to *out.
template <class C, class R>
static int fr_open(flb_keyframes* k, const char* who, const C* cfg, int (*cfg_check)(const C*, const char*), const void* src_pts,
                   int n_src, int src_stride, int src_off_intensity, const float* src_pose6, const int* tgt_ids, int n_tgt,
                   const float* tgt_pre_pose6, const float* tgt_poses6, int* out_corr_index, double* out_resid, const double* out_log,
                   int log_cap, int min_target, R* out, R& res, FrSetup& st) {
  if (!out) return set_err("%s: null result", who);
  if (!cfg) return set_err("%s: null config", who);
  if (cfg_check(cfg, who) || fr_setup(k, who, src_pts, n_src, src_stride, src_off_intensity, src_pose6, tgt_ids, n_tgt, tgt_pre_pose6,
                                      tgt_poses6, out_corr_index, out_resid, out_log, log_cap, min_target, &st))
    return 1;
  res = R{};
  for (int i = 0; i < 16; ++i) res.res_trans[i] = (i % 5 == 0) ? 1.0 : 0.0;
  fr_setup_result(st, res);
  if (int* syncs = fr_syncs(res)) *syncs = st.syncs;
  if (st.status >= 0) *out = res;
  return 0;
}

// The closing every relocalisation registration shares: res_trans from T (row-major 3x4, normalised frame), the
// per-source outputs of the last 1-NN pass when there was one (`passed`), the synchronisation that ends the call.
template <class R>
static int fr_close(flb_map* m, const FrSetup& st, const double* T, bool passed, int* out_corr_index, double* out_resid, R& res) {
  fr_res_trans(st, T, res.res_trans);
  if (passed && fr_outputs(m, *m->kfw, st.n_s, out_corr_index, out_resid)) return 1;
  CU(cudaStreamSynchronize(m->stream));
  if (int* syncs = fr_syncs(res)) ++*syncs;
  res.status = FLB_FRICP_OK;
  return 0;
}

extern "C" int flb_keyframes_fricp(flb_keyframes* k, const void* src_pts, int n_src, int src_stride, int src_off_intensity,
                                   const float* src_pose6, const int* tgt_ids, int n_tgt, const float* tgt_pre_pose6,
                                   const float* tgt_poses6, const flb_fricp_config* cfg, flb_fricp_result* out, int* out_corr_index,
                                   double* out_resid, double* out_log, int log_cap) {
  FrSetup st;
  flb_fricp_result res;
  if (fr_open(k, "flb_keyframes_fricp", cfg, fr_cfg_check, src_pts, n_src, src_stride, src_off_intensity, src_pose6, tgt_ids, n_tgt,
              tgt_pre_pose6, tgt_poses6, out_corr_index, out_resid, out_log, log_cap, 2, out, res, st))
    return 1;
  if (st.status >= 0) return 0;
  flb_map* m = k->map;
  KfWork& kw = *m->kfw;
  IcpIndex& x = kw.index;
  FricpWork& w = kw.fricp;
  const IcpGrid& g = st.g;
  const int n_s = st.n_s, n_ft = st.n_ft, n_fs = st.n_fs;
  const int gs = grid_for(n_s, 256, m->sm_count * 8);

  // FRICP<3>::point_to_point (FRICP.h:382-543)
  const int mode = cfg->mode;
  const bool welsch = mode == FLB_FRICP_ROBUST || mode == FLB_FRICP_FAST_ROBUST;
  const bool use_aa = mode == FLB_FRICP_FAST || mode == FLB_FRICP_FAST_ROBUST;
  double T[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0}, SVD_T[12], To2[12];
  memcpy(SVD_T, T, sizeof(T));
  memcpy(To2, T, sizeof(T));
  double nu1 = 1, nu2 = 1;
  if (welsch) {   // :421-436: nu_end from the target's 7-NN median spacing, nu_begin from the initial residuals' median
    if (fr_pass(m, kw, g, n_s, T, true, 1.0, false)) return 1;
    int* open_n = (int*)(x.misc.p + ICP_MISC_OPEN);
    CU(cudaMemsetAsync(open_n, 0, sizeof(int), m->stream));
    const int kk = std::min(7, n_ft);
    k_fr_knn7<<<grid_for(n_ft, 256, m->sm_count * 8), 256, 0, m->stream>>>(g, n_ft, kk, w.sorted_d.p, x.cs.p, w.med.p, x.open.p, open_n);
    k_fr_knn7_far<<<grid_for(n_ft, 256, m->sm_count * 8), 256, 0, m->stream>>>(g, kk, x.open.p, open_n, w.sorted_d.p, x.cs.p, x.box.p, w.med.p);
    k_fr_resid<<<gs, 256, 0, m->stream>>>(w.d2.p, n_s, w.sort_a.p);
    m->launches += 3;
    CU(cudaGetLastError());
    double med_t = 0, med_r = 0;
    if (fr_median(m, kw, w.med.p, n_ft, n_ft, &med_t) || fr_median(m, kw, w.sort_a.p, n_s, n_fs, &med_r)) return 1;
    nu2 = cfg->nu_end_k * std::sqrt(med_t);
    nu1 = std::max(cfg->nu_begin_k * med_r, nu2);
    res.nu_begin = nu1;
    res.nu_end = nu2;
    if (fr_pass(m, kw, g, n_s, T, false, nu1, true)) return 1;
  } else {
    if (fr_pass(m, kw, g, n_s, T, true, nu1, false)) return 1;
  }
  CU(cudaStreamSynchronize(m->stream));
  double S[FR_RED];
  memcpy(S, w.h_sums.p + FR_SUM_STEP, sizeof(S));

  FrAnderson aa;
  double L[16];
  fr_log(T, L);
  aa.init(cfg->anderson_m, L);
  double last_energy = DBL_MAX;
  int log_n = 0;
  for (bool stop1 = false; !stop1;) {
    ++res.stages;
    for (int icp = 0; icp < cfg->max_icp; ++icp) {
      const double energy = S[16], prev = last_energy;
      int accepted = 1;
      if (use_aa) {
        if (energy < last_energy) {
          last_energy = energy;
        } else {   // :459-469: back to the plain step's transform
          accepted = 0;
          ++res.rejections;
          fr_log(SVD_T, L);
          aa.replace(L);
          if (fr_pass(m, kw, g, n_s, SVD_T, true, nu1, welsch)) return 1;
          CU(cudaStreamSynchronize(m->stream));
          memcpy(S, w.h_sums.p + FR_SUM_STEP, sizeof(S));
          last_energy = S[16];
        }
      } else {
        last_energy = energy;
      }
      fr_kabsch(S, T);
      memcpy(SVD_T, T, sizeof(T));
      if (use_aa) {
        fr_log(T, L);
        fr_exp(aa.compute(L), T);
      }
      if (fr_pass(m, kw, g, n_s, T, true, nu1, welsch)) return 1;
      CU(cudaStreamSynchronize(m->stream));
      memcpy(S, w.h_sums.p + FR_SUM_STEP, sizeof(S));
      double s2 = 0;
      for (int i = 0; i < 12; ++i) s2 += (T[i] - To2[i]) * (T[i] - To2[i]);
      const double stop2 = std::sqrt(s2);
      memcpy(To2, T, sizeof(T));
      ++res.iterations;
      if (log_n < log_cap) {
        double* row = out_log + 5 * (size_t)log_n++;
        row[0] = res.stages - 1; row[1] = energy; row[2] = prev; row[3] = stop2; row[4] = accepted;
      }
      if (stop2 < cfg->stop) break;
    }
    if (!welsch) {
      stop1 = true;
    } else {   // :518-529: the next, smaller scale
      stop1 = std::fabs(nu1 - nu2) < 1e-6;
      nu1 = nu1 * cfg->nu_alpha > nu2 ? nu1 * cfg->nu_alpha : nu2;
      if (use_aa) {
        fr_log(T, L);
        aa.reset(L);
        last_energy = DBL_MAX;
      }
      if (fr_pass(m, kw, g, n_s, T, false, nu1, true)) return 1;   // the energies and weights at the new scale
      CU(cudaStreamSynchronize(m->stream));
      memcpy(S, w.h_sums.p + FR_SUM_STEP, sizeof(S));
    }
  }
  res.energy = S[16];
  res.log_n = log_n;
  if (fr_close(m, st, T, true, out_corr_index, out_resid, res)) return 1;   // :536 and registeration.h:170
  *out = res;
  return 0;
}

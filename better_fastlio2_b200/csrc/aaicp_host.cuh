// aaicp_host.cuh — the relocaliser's AA-ICP (regMode 1: AAICP::point_to_point_aaicp, include/FRICP-toolkit/ICP.h:841-1033,
// with Registeration's ICP::Parameters, registeration.h:86-91: f = NONE, use_init = false): a host source cloud onto a
// target assembled from the device key-frame store.  The set-up (upload, two-stage target assembly, normalisation, grid
// index) is flb_keyframes_fricp's (fr_setup).  Every iteration is one exact double 1-NN pass of final X0, one fused
// reduction of the step record on the moved source (AaStepOp), one small copy and one synchronisation.  The Kabsch step,
// eulerAngles, the column-pivoting QR solves and the Anderson mixing on 6-vectors run here on the host.  DESIGN.md §9
// states the contract.  Included after fricp_host.cuh.
#pragma once
#include <array>

#include "aaicp_kernels.cuh"

static int aaicp_cfg_check(const flb_aaicp_config* c, const char* who) {
  if (c->max_icp < 0) return set_err("%s: max_icp must be >= 0 (got %d)", who, c->max_icp);
  if (!(std::isfinite(c->stop) && c->stop >= 0)) return set_err("%s: stop must be finite and >= 0", who);
  if (!std::isfinite(c->error_overflow_threshold)) return set_err("%s: error_overflow_threshold must be finite", who);
  return 0;
}

extern "C" void flb_aaicp_default_config(flb_aaicp_config* c) {
  if (!c) return;
  c->max_icp = 100;
  c->stop = 1e-5;
  c->error_overflow_threshold = 0.05;
}

// ------------------------------------------------------------------------------------------------ host algebra
// Eigen 3.3.7's semantics written out (DESIGN.md §9 states the association orders).  Matrices are row-major 4x4.
typedef double AaM4[16];
typedef std::array<double, 6> AaV6;

// Matrix3::eulerAngles(0, 1, 2): the first angle in [0, π]
static void aa_euler(const double* m, double* e) {
  double a = std::atan2(m[5], m[8]);
  const double c2 = std::sqrt(m[0] * m[0] + m[1] * m[1]);
  double b;
  if (a > 0) {
    a -= M_PI;
    b = std::atan2(-m[2], -c2);
  } else {
    b = std::atan2(-m[2], c2);
  }
  const double s1 = std::sin(a), c1 = std::cos(a);
  const double c = std::atan2(s1 * m[6] - c1 * m[3], c1 * m[4] - s1 * m[7]);
  e[0] = -a;
  e[1] = -b;
  e[2] = -c;
}

// Matrix42Vector6: (eulerAngles(0, 1, 2), t)
static AaV6 aa_vec6(const AaM4 T) {
  const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  AaV6 v;
  aa_euler(R, v.data());
  v[3] = T[3];
  v[4] = T[7];
  v[5] = T[11];
  return v;
}

struct AaQuat { double w, x, y, z; };

static AaQuat aa_quat_axis(double angle, int k) {   // Quaternion(AngleAxis(angle, unit axis k))
  const double ha = 0.5 * angle, s = std::sin(ha);
  return AaQuat{std::cos(ha), s * (k == 0 ? 1.0 : 0.0), s * (k == 1 ? 1.0 : 0.0), s * (k == 2 ? 1.0 : 0.0)};
}

static AaQuat aa_qmul(const AaQuat& a, const AaQuat& b) {
  return AaQuat{a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
                a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}

// Vector62Matrix4: (AngleAxis X * AngleAxis Y) * AngleAxis Z as quaternions, toRotationMatrix, translation v[3..5]
static void aa_mat4(const AaV6& v, AaM4 T) {
  const AaQuat q = aa_qmul(aa_qmul(aa_quat_axis(v[0], 0), aa_quat_axis(v[1], 1)), aa_quat_axis(v[2], 2));
  const double tx = 2.0 * q.x, ty = 2.0 * q.y, tz = 2.0 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  const double R[9] = {1.0 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.0 - (txx + tzz), tyz - twx, txz - twy, tyz + twx,
                       1.0 - (txx + tyy)};
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[4 * r + c] = R[3 * r + c];
    T[4 * r + 3] = v[3 + r];
  }
  T[12] = T[13] = T[14] = 0.0;
  T[15] = 1.0;
}

// Matrix4 product, each entry ((a0 b0 + a1 b1) + a2 b2) + a3 b3
static void aa_mul4(const AaM4 A, const AaM4 B, AaM4 C) {
  AaM4 o;
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) o[4 * r + c] = ((A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c]) + A[4 * r + 2] * B[8 + c]) + A[4 * r + 3] * B[12 + c];
  memcpy(C, o, sizeof(o));
}

// Affine3d product: linear A.l B.l, translation A.l B.t + A.t
static void aa_mul_affine(const AaM4 A, const AaM4 B, AaM4 C) {
  AaM4 o;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) o[4 * r + c] = (A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c]) + A[4 * r + 2] * B[8 + c];
    o[4 * r + 3] = ((A[4 * r] * B[3] + A[4 * r + 1] * B[7]) + A[4 * r + 2] * B[11]) + A[4 * r + 3];
  }
  o[12] = o[13] = o[14] = 0.0;
  o[15] = 1.0;
  memcpy(C, o, sizeof(o));
}

// Matrix4::inverse() by the adjugate (each 3x3 minor expanded along its first row, as Eigen's 3x3 determinant), divided by
// ((m00 a00 + m10 a01) + m20 a02) + m30 a03
static void aa_inv4(const AaM4 A, AaM4 out) {
  AaM4 adj;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double m[9];   // minor(j, i)
      for (int r = 0, a = 0; r < 4; ++r) {
        if (r == j) continue;
        for (int c = 0, b = 0; c < 4; ++c)
          if (c != i) m[3 * a + b++] = A[4 * r + c];
        ++a;
      }
      const double d = (m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6])) + m[2] * (m[3] * m[7] - m[4] * m[6]);
      adj[4 * i + j] = ((i + j) % 2) ? -d : d;
    }
  const double det = ((A[0] * adj[0] + A[4] * adj[1]) + A[8] * adj[2]) + A[12] * adj[3];
  for (int k = 0; k < 16; ++k) out[k] = adj[k] / det;
}

// ColPivHouseholderQR<MatrixXd>(A).solve(b) for a 6 x n column-major A: column pivoting on the largest remaining norm
// (ties: the lower index) with LAPACK's norm downdate, the rank = the non-zero pivot count, the basic solution (free
// variables 0).  A is overwritten.
static void aa_qr_solve(double* A, int n, const double* b, double* x) {
  const int rows = 6, size = std::min(rows, n);
  std::vector<double> hc(size), nu(n), nd(n);
  std::vector<int> tr(size);
  auto at = [&](int r, int c) -> double& { return A[(size_t)c * rows + r]; };
  auto col_norm = [&](int c, int r0) {
    double s = 0;
    for (int r = r0; r < rows; ++r) s += at(r, c) * at(r, c);
    return std::sqrt(s);
  };
  for (int k = 0; k < n; ++k) nd[k] = nu[k] = col_norm(k, 0);
  double mx = nu[0];
  for (int k = 1; k < n; ++k) if (nu[k] > mx) mx = nu[k];
  const double thr_helper = (mx * DBL_EPSILON) * (mx * DBL_EPSILON) / (double)rows, downdate = std::sqrt(DBL_EPSILON);
  int nzp = size;
  for (int k = 0; k < size; ++k) {
    int big = k;
    for (int j = k + 1; j < n; ++j) if (nu[j] > nu[big]) big = j;
    if (nzp == size && nu[big] * nu[big] < thr_helper * (double)(rows - k)) nzp = k;
    tr[k] = big;
    if (k != big) {
      for (int r = 0; r < rows; ++r) std::swap(at(r, k), at(r, big));
      std::swap(nu[k], nu[big]);
      std::swap(nd[k], nd[big]);
    }
    double tail = 0;   // makeHouseholderInPlace on rows k..5 of column k
    for (int r = k + 1; r < rows; ++r) tail += at(r, k) * at(r, k);
    const double c0 = at(k, k);
    double tau, beta;
    if (tail <= DBL_MIN) {
      tau = 0.0;
      beta = c0;
      for (int r = k + 1; r < rows; ++r) at(r, k) = 0.0;
    } else {
      beta = std::sqrt(c0 * c0 + tail);
      if (c0 >= 0.0) beta = -beta;
      for (int r = k + 1; r < rows; ++r) at(r, k) = at(r, k) / (c0 - beta);
      tau = (beta - c0) / beta;
    }
    hc[k] = tau;
    at(k, k) = beta;
    if (rows - k == 1) {   // applyHouseholderOnTheLeft on the remaining columns
      for (int c = k + 1; c < n; ++c) at(k, c) = at(k, c) * (1.0 - tau);
    } else if (tau != 0.0) {
      for (int c = k + 1; c < n; ++c) {
        double t = 0;
        for (int r = k + 1; r < rows; ++r) t += at(r, k) * at(r, c);
        t = t + at(k, c);
        at(k, c) = at(k, c) - tau * t;
        for (int r = k + 1; r < rows; ++r) at(r, c) = at(r, c) - (tau * at(r, k)) * t;
      }
    }
    for (int j = k + 1; j < n; ++j) {
      if (nu[j] == 0.0) continue;
      double t = std::fabs(at(k, j)) / nu[j];
      t = (1.0 + t) * (1.0 - t);
      t = t < 0.0 ? 0.0 : t;
      const double q = nu[j] / nd[j];
      if (t * (q * q) <= downdate) {
        nd[j] = col_norm(j, k + 1);
        nu[j] = nd[j];
      } else {
        nu[j] *= std::sqrt(t);
      }
    }
  }
  std::vector<int> perm(n);
  for (int k = 0; k < n; ++k) perm[k] = k;
  for (int k = 0; k < size; ++k) std::swap(perm[k], perm[tr[k]]);
  for (int k = 0; k < n; ++k) x[k] = 0.0;
  if (nzp == 0) return;
  double c[6];
  memcpy(c, b, sizeof(c));
  for (int k = 0; k < nzp; ++k) {   // Q^T b, H_0 first
    if (rows - k == 1) {
      c[k] = c[k] * (1.0 - hc[k]);
    } else if (hc[k] != 0.0) {
      double t = 0;
      for (int r = k + 1; r < rows; ++r) t += at(r, k) * c[r];
      t = t + c[k];
      c[k] = c[k] - hc[k] * t;
      for (int r = k + 1; r < rows; ++r) c[r] = c[r] - (hc[k] * at(r, k)) * t;
    }
  }
  for (int i = nzp - 1; i >= 0; --i) {   // column-oriented back substitution
    if (c[i] == 0.0) continue;
    c[i] = c[i] / at(i, i);
    for (int r = 0; r < i; ++r) c[r] = c[r] - c[i] * at(r, i);
  }
  for (int i = 0; i < nzp; ++i) x[perm[i]] = c[i];
}

// get_next_u (ICP.h:812-837) with β = 1 over the whole history; *na: the α count of the result; *margin: the smallest
// margin of the alphas_cond tests made (NaN when a tested α was NaN, +inf when none was made).
static AaV6 aa_next_u(const std::vector<AaV6>& u, const std::vector<AaV6>& g, const std::vector<AaV6>& f, int* na, double* margin) {
  const int m = (int)f.size();
  AaV6 out;
  for (int r = 0; r < 6; ++r) out[r] = 0.0 * u.back()[r] + 1.0 * g.back()[r];
  *na = 1;
  *margin = INFINITY;
  std::vector<double> A, al;
  for (int i = 2; i <= m; ++i) {
    const AaV6& fl = f[m - 1];
    A.assign((size_t)6 * (i - 1), 0.0);
    al.assign(i, 0.0);
    for (int j = 0; j < i - 1; ++j)
      for (int r = 0; r < 6; ++r) A[(size_t)6 * j + r] = -f[m - i + j][r] + fl[r];
    aa_qr_solve(A.data(), i - 1, fl.data(), al.data());
    double s = 0;
    for (int j = 0; j < i - 1; ++j) s += al[j];
    al[i - 1] = 1.0 - (s + 0.0);
    double lo = al[0], hi = al[0];
    bool nan = std::isnan(*margin) || std::isnan(al[0]);
    for (int j = 1; j < i; ++j) {
      if (al[j] < lo) lo = al[j];
      if (al[j] > hi) hi = al[j];
      nan = nan || std::isnan(al[j]);
    }
    const double mg = std::min(std::fabs(lo + 10.0), std::min(std::fabs(10.0 - hi), std::fabs(al[i - 1])));
    *margin = nan ? NAN : std::min(*margin, mg);
    if (!(-10.0 < lo && hi < 10.0 && al[i - 1] > 0)) break;
    for (int r = 0; r < 6; ++r) {
      double su = 0, sg = 0;
      for (int j = 0; j < i; ++j) { su += u[u.size() - i + j][r] * al[j]; sg += g[m - i + j][r] * al[j]; }
      out[r] = 0.0 * su + 1.0 * sg;
    }
    *na = i;
  }
  return out;
}

// The unweighted point-to-point step from the step record (n, Σx, Σq, Σ x qᵀ): R = V diag(1, 1, ±1) Uᵀ of the SVD of
// Σ x qᵀ / n - x̄ q̄ᵀ, t = q̄ - R x̄; a zero cross-covariance (one point) gives R = I, as Eigen's JacobiSVD does.
static void aa_kabsch(const double* S, AaM4 T) {
  double xm[3], qm[3], sig[9], U[9], sv[3], V[9];
  for (int a = 0; a < 3; ++a) { xm[a] = S[1 + a] / S[0]; qm[a] = S[4 + a] / S[0]; }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) sig[3 * r + c] = S[7 + 3 * r + c] / S[0] - xm[r] * qm[c];
  icp_svd3(sig, U, sv, V);
  if (!(sv[0] > 0))
    for (int k = 0; k < 9; ++k) U[k] = V[k] = (k % 4 == 0) ? 1.0 : 0.0;
  const double dd = icp_det3(U) * icp_det3(V) < 0 ? -1.0 : 1.0;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[4 * r + c] = (V[3 * r] * U[3 * c] + V[3 * r + 1] * U[3 * c + 1]) + dd * V[3 * r + 2] * U[3 * c + 2];
    T[4 * r + 3] = qm[r] - ((T[4 * r] * xm[0] + T[4 * r + 1] * xm[1]) + T[4 * r + 2] * xm[2]);
  }
  T[12] = T[13] = T[14] = 0.0;
  T[15] = 1.0;
}

extern "C" int flb_keyframes_aaicp(flb_keyframes* k, const void* src_pts, int n_src, int src_stride, int src_off_intensity,
                                   const float* src_pose6, const int* tgt_ids, int n_tgt, const float* tgt_pre_pose6,
                                   const float* tgt_poses6, const flb_aaicp_config* cfg, flb_aaicp_result* out, int* out_corr_index,
                                   double* out_resid, double* out_log, int log_cap) {
  FrSetup st;
  flb_aaicp_result res;
  if (fr_open(k, "flb_keyframes_aaicp", cfg, aaicp_cfg_check, src_pts, n_src, src_stride, src_off_intensity, src_pose6, tgt_ids,
              n_tgt, tgt_pre_pose6, tgt_poses6, out_corr_index, out_resid, out_log, log_cap, 1, out, res, st))
    return 1;
  if (st.status >= 0) return 0;
  flb_map* m = k->map;
  KfWork& kw = *m->kfw;
  IcpIndex& x = kw.index;
  FricpWork& w = kw.fricp;
  const int n_s = st.n_s;

  // ICP.h:847-882 with use_init = false: T = final = transformation = To2 = I, X = X0
  const AaM4 I4 = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  AaM4 T, To2, tr, fin;
  memcpy(T, I4, sizeof(AaM4));
  memcpy(To2, I4, sizeof(AaM4));
  memcpy(tr, I4, sizeof(AaM4));
  memcpy(fin, I4, sizeof(AaM4));
  std::vector<AaV6> u, g, f;
  AaV6 u_next{}, u_k{};
  double prev_energy = DBL_MAX;
  int icp = 0, passes = 0, log_n = 0;
  for (; icp < cfg->max_icp; ++icp) {
    // Q = the exact nearest target points of X = final X0; the step record on (X, Q)
    if (fr_nn(m, kw, st.g, n_s, fin)) return 1;
    FrXf xf;
    memcpy(xf.m, fin, sizeof(xf.m));
    if (icp_reduce<FR_RED>(m, x, n_s, AaStepOp{xf, w.x.p, w.sorted_d.p, w.pos.p, w.d2.p}, w.sums.p + FR_SUM_STEP)) return 1;
    CU(cudaMemcpyAsync(w.h_sums.p + FR_SUM_STEP, w.sums.p + FR_SUM_STEP, sizeof(double) * FR_RED, cudaMemcpyDeviceToHost, m->stream));
    CU(cudaStreamSynchronize(m->stream));
    res.syncs++;
    ++passes;
    const double* S = w.h_sums.p + FR_SUM_STEP;
    const double energy = S[16];
    AaM4 step, P;
    aa_kabsch(S, step);
    aa_mul_affine(step, T, T);   // T = point_to_point(X, Q, W) * T, final = T
    memcpy(fin, T, sizeof(AaM4));
    aa_mul4(tr, fin, P);
    const AaV6 gk = aa_vec6(P);
    const double prev = prev_energy;
    double margin = INFINITY;
    int outcome = -1, na = 1;
    if (icp) {   // Anderson acceleration (ICP.h:926-959)
      if ((energy - prev_energy) / prev_energy > cfg->error_overflow_threshold) {   // the first heuristic
        u_next = u_k = g.back();
        prev_energy = DBL_MAX;
        u.erase(u.begin(), u.end() - 2);
        g.erase(g.begin(), g.end() - 1);
        f.erase(f.begin(), f.end() - 1);
        outcome = 0;
        ++res.resets;
      } else {
        prev_energy = energy;
        g.push_back(gk);
        AaV6 fk;
        for (int r = 0; r < 6; ++r) fk[r] = gk[r] - u_k[r];
        f.push_back(fk);
        u_next = aa_next_u(u, g, f, &na, &margin);
        u.push_back(u_next);
        u_k = u_next;
        outcome = 1;
        ++res.accepted;
      }
    } else {     // :960-985
      prev_energy = energy;
      const AaV6 u0 = aa_vec6(I4);
      u = {u0, gk};
      g = {gk};
      AaV6 f0;
      for (int r = 0; r < 6; ++r) f0[r] = gk[r] - u0[r];
      f = {f0};
      u_next = u_k = gk;
    }
    // :987-1001: re-seat on u_next, the stopping test
    AaM4 Mu, Fi;
    aa_mat4(u_next, Mu);
    aa_inv4(fin, Fi);
    aa_mul4(Mu, Fi, tr);
    memcpy(fin, Mu, sizeof(AaM4));
    double s2 = 0;
    for (int i = 0; i < 16; ++i) s2 += (fin[i] - To2[i]) * (fin[i] - To2[i]);
    const double stop2 = std::sqrt(s2);
    memcpy(To2, fin, sizeof(AaM4));
    if (log_n < log_cap) {
      double* row = out_log + 6 * (size_t)log_n++;
      row[0] = energy; row[1] = prev; row[2] = outcome; row[3] = na; row[4] = stop2; row[5] = margin;
    }
    if (stop2 < cfg->stop && icp) break;
  }
  // :1004-1015: the convergence energy of the last matches against the re-seated X, res_trans in the caller's frame
  FrXf xf;
  memcpy(xf.m, fin, sizeof(xf.m));
  if (icp_reduce<1>(m, x, n_s, AaEnergyOp{xf, w.x.p, w.sorted_d.p, w.pos.p, passes > 0 ? 1 : 0}, w.sums.p + FR_SUM_MED)) return 1;
  CU(cudaMemcpyAsync(w.h_sums.p + FR_SUM_MED, w.sums.p + FR_SUM_MED, sizeof(double), cudaMemcpyDeviceToHost, m->stream));
  if (fr_close(m, st, fin, passes > 0, out_corr_index, out_resid, res)) return 1;
  res.energy = w.h_sums.p[FR_SUM_MED];
  res.iterations = icp;
  res.history = (int)u.size();
  res.log_n = log_n;
  *out = res;
  return 0;
}

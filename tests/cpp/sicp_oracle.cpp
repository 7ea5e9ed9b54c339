// Sequential restatement of the relocalisation Sparse ICP contract (DESIGN.md §9, "Relocalisation registration, Sparse
// ICP"): SICP::point_to_point (ICP.h:275-380) as Registeration::run calls it for regMode 7, as flb_keyframes_sicp
// implements it, on host clouds.  The normalisation of the relocalisation registration (status FEW_TARGET only without a
// finite target point), the exact 1-NN of that oracle's k-d tree, the ADMM loop with max_inner = 1 and no penalty mode,
// sequential double sums and that oracle's 3x3 SVD.  The k-d tree, the SVD and the point helpers are
// tests/cpp/fricp_oracle.cpp's, included whole so that both restatements share one copy of them; that file's own entry
// points come along with it.  Compiled by tests/sicp_oracle.py with -ffp-contract=off.
#include "fricp_oracle.cpp"

extern "C" {

// shrinkage<3> with the threshold test of shrink<3> (ICP.h:238-256): the factor Z_i is multiplied by
double orc_sicp_shrink(double n, double mu, double p, double Ba, double ha) {
  if (!(n > ha)) return 0.0;
  double s = (Ba / n + 1.0) / 2.0;
  for (int k = 0; k < 3; ++k) s = 1.0 - ((p / mu) * std::pow(n, p - 2.0)) * std::pow(s, p - 1.0);
  return s;
}

// Ba and ha of shrink<3> at mu (ICP.h:247-248)
void orc_sicp_thresholds(double mu, double p, double* Ba_ha) {
  const double Ba = std::pow((2.0 / mu) * (1.0 - p), 1.0 / (2.0 - p));
  Ba_ha[0] = Ba;
  Ba_ha[1] = Ba + (p / mu) * std::pow(Ba, p - 1.0);
}

// src / tgt: x, y, z, w float records.  norm (optional): scale, source mean, target mean.  res12: res_trans rows 0-2.
// info: status, ICP iterations, ADMM iterations, finite source, finite target.  dinfo: scale, mu_s[3], mu_t[3], and the
// last ICP iteration's primal, dual, stop and μ at exit.  corr / resid (n_s): the last ICP iteration's matched target
// index and residual (-1 / +inf: none).  log: per ICP iteration (ADMM iterations, primal, dual, stop, μ at exit).
int orc_sicp(const float* src, int n_s, const float* tgt, int n_t, double p, double mu0, double alpha, double max_mu, int max_icp,
             int max_outer, double stop, const double* norm, double* res12, int* info, double* dinfo, int* corr, double* resid,
             double* log, int log_cap, int* log_n) {
  for (int i = 0; i < 12; ++i) res12[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int i = 0; i < 5; ++i) info[i] = 0;
  for (int i = 0; i < 11; ++i) dinfo[i] = 0;
  *log_n = 0;
  for (int i = 0; i < n_s; ++i) { corr[i] = -1; resid[i] = INFINITY; }
  std::vector<int> si, ti;
  for (int i = 0; i < n_s; ++i) if (finite3(src + 4 * (size_t)i)) si.push_back(i);
  for (int i = 0; i < n_t; ++i) if (finite3(tgt + 4 * (size_t)i)) ti.push_back(i);
  info[3] = (int)si.size();
  info[4] = (int)ti.size();
  dinfo[0] = 1.0;
  if (si.empty()) { info[0] = 2; return 0; }
  if (ti.empty()) { info[0] = 1; return 0; }
  double scale, ms[3] = {0, 0, 0}, mt[3] = {0, 0, 0};
  if (norm) {
    scale = norm[0];
    for (int a = 0; a < 3; ++a) { ms[a] = norm[1 + a]; mt[a] = norm[4 + a]; }
  } else {
    double e[2] = {0, 0};
    for (int c = 0; c < 2; ++c) {
      const float* P = c ? tgt : src;
      const std::vector<int>& I = c ? ti : si;
      double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
      for (int i : I)
        for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], (double)P[4 * i + a]); hi[a] = std::max(hi[a], (double)P[4 * i + a]); }
      const double ex = hi[0] - lo[0], ey = hi[1] - lo[1], ez = hi[2] - lo[2];
      e[c] = std::sqrt((ex * ex + ey * ey) + ez * ez);
    }
    scale = std::max(e[0], e[1]);
    if (!(scale > 0)) scale = 1.0;
    for (int i : si) for (int a = 0; a < 3; ++a) ms[a] += (double)src[4 * i + a] / scale;
    for (int i : ti) for (int a = 0; a < 3; ++a) mt[a] += (double)tgt[4 * i + a] / scale;
    for (int a = 0; a < 3; ++a) { ms[a] /= (double)si.size(); mt[a] /= (double)ti.size(); }
  }
  dinfo[0] = scale;
  for (int a = 0; a < 3; ++a) { dinfo[1 + a] = ms[a]; dinfo[4 + a] = mt[a]; }
  const int ns = (int)si.size();
  std::vector<V3> X(ns), Y(ti.size()), Q(ns), Z(ns), C(ns), Xo2;
  for (int k = 0; k < ns; ++k) for (int a = 0; a < 3; ++a) { X[k].x[a] = (double)src[4 * si[k] + a] / scale - ms[a]; C[k].x[a] = 0.0; }
  for (size_t k = 0; k < ti.size(); ++k) for (int a = 0; a < 3; ++a) Y[k].x[a] = (double)tgt[4 * ti[k] + a] / scale - mt[a];
  Xo2 = X;
  Tree tree;
  tree.init(Y);
  std::vector<int> M(ns, -1);
  std::vector<double> W(ns, INFINITY);
  const double inv_n = 1.0 / (double)ns;
  auto norm3 = [](double x, double y, double z) { return std::sqrt((x * x + y * y) + z * z); };
  double T[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  int icp = 0, admm = 0;
  double primal = 0, dual = 0, stop_v = 0, mu = mu0;
  for (; icp < max_icp;) {
    for (int k = 0; k < ns; ++k) {   // Q_i = the nearest target point of X_i
      double best = INFINITY;
      int bi = INT32_MAX;
      tree.nn(0, X[k].x, best, bi);
      M[k] = bi;
      W[k] = std::sqrt(best);
      Q[k] = Y[bi];
    }
    mu = mu0;
    int outer = 0;
    primal = dual = 0;
    while (outer < max_outer) {
      double BH[2];
      orc_sicp_thresholds(mu, p, BH);
      double xm[3] = {0, 0, 0}, um[3] = {0, 0, 0};
      for (int k = 0; k < ns; ++k) {   // Z = (X - Q) + C/μ, shrunk; U = (Q + Z) - C/μ
        for (int a = 0; a < 3; ++a) Z[k].x[a] = (X[k].x[a] - Q[k].x[a]) + C[k].x[a] / mu;
        const double w = orc_sicp_shrink(norm3(Z[k].x[0], Z[k].x[1], Z[k].x[2]), mu, p, BH[0], BH[1]);
        for (int a = 0; a < 3; ++a) Z[k].x[a] = Z[k].x[a] * w;
      }
      std::vector<V3> U(ns);
      for (int k = 0; k < ns; ++k) for (int a = 0; a < 3; ++a) U[k].x[a] = (Q[k].x[a] + Z[k].x[a]) - C[k].x[a] / mu;
      for (int k = 0; k < ns; ++k) for (int a = 0; a < 3; ++a) { xm[a] += X[k].x[a] * inv_n; um[a] += U[k].x[a] * inv_n; }
      double sig[9] = {0};
      for (int k = 0; k < ns; ++k)
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) sig[3 * r + c] += ((X[k].x[r] - xm[r]) * inv_n) * (U[k].x[c] - um[c]);
      double Us[9], sv[3], Vm[9], R[12];
      svd3(sig, Us, sv, Vm);
      if (!(sv[0] > 0))   // a zero cross-covariance (one point): U = V = I, as Eigen's JacobiSVD gives them
        for (int k = 0; k < 9; ++k) Us[k] = Vm[k] = (k % 4 == 0) ? 1.0 : 0.0;
      const double dd = det3(Us) * det3(Vm) < 0 ? -1.0 : 1.0;
      for (int r = 0; r < 3; ++r) {   // R = V diag(1, 1, dd) U^T, t = ū - R x̄
        for (int c = 0; c < 3; ++c) R[4 * r + c] = (Vm[3 * r] * Us[3 * c] + Vm[3 * r + 1] * Us[3 * c + 1]) + dd * Vm[3 * r + 2] * Us[3 * c + 2];
        R[4 * r + 3] = um[r] - ((R[4 * r] * xm[0] + R[4 * r + 1] * xm[1]) + R[4 * r + 2] * xm[2]);
      }
      double nT[12];   // T <- cur_T T
      for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 4; ++c) nT[4 * r + c] = (R[4 * r] * T[c] + R[4 * r + 1] * T[4 + c]) + R[4 * r + 2] * T[8 + c];
        nT[4 * r + 3] = nT[4 * r + 3] + R[4 * r + 3];
      }
      std::memcpy(T, nT, sizeof(T));
      double ds = 0;
      primal = 0;
      for (int k = 0; k < ns; ++k) {
        double xn[3];
        apply(R, X[k], xn);
        const double dx = xn[0] - X[k].x[0], dy = xn[1] - X[k].x[1], dz = xn[2] - X[k].x[2];
        ds += (dx * dx + dy * dy) + dz * dz;
        double P[3];
        for (int a = 0; a < 3; ++a) { X[k].x[a] = xn[a]; P[a] = (xn[a] - Q[k].x[a]) - Z[k].x[a]; C[k].x[a] = C[k].x[a] + mu * P[a]; }
        primal = std::max(primal, norm3(P[0], P[1], P[2]));
      }
      dual = ds / (double)ns;
      if (mu < max_mu) mu *= alpha;
      ++outer;
      if (primal < stop && dual < stop) break;
    }
    stop_v = 0;
    for (int k = 0; k < ns; ++k) {
      stop_v = std::max(stop_v, norm3(X[k].x[0] - Xo2[k].x[0], X[k].x[1] - Xo2[k].x[1], X[k].x[2] - Xo2[k].x[2]));
      Xo2[k] = X[k];
    }
    admm += outer;
    ++icp;
    if (*log_n < log_cap) {
      double* row = log + 5 * (size_t)*log_n;
      row[0] = outer; row[1] = primal; row[2] = dual; row[3] = stop_v; row[4] = mu;
      ++*log_n;
    }
    if (stop_v < stop) break;
  }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) res12[4 * r + c] = T[4 * r + c];
    res12[4 * r + 3] = (T[4 * r + 3] + (mt[r] - ((T[4 * r] * ms[0] + T[4 * r + 1] * ms[1]) + T[4 * r + 2] * ms[2]))) * scale;
  }
  if (icp > 0)
    for (int k = 0; k < ns; ++k) { corr[si[k]] = ti[M[k]]; resid[si[k]] = W[k]; }
  info[1] = icp;
  info[2] = admm;
  dinfo[7] = primal; dinfo[8] = dual; dinfo[9] = stop_v; dinfo[10] = icp > 0 ? mu : 0.0;
  return 0;
}

}  // extern "C"

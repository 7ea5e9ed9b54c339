// Sequential restatement of the relocalisation registration contract (DESIGN.md §9, "Relocalisation registration"):
// FRICP<3>::point_to_point as Registeration::run calls it for regMode 0 (ICP), 2 (Fast ICP), 3 (Robust ICP) and 4 (Fast
// and Robust ICP), as flb_keyframes_fricp implements it, on host clouds.  Its own exact k-d tree over the normalised
// finite target (double d² = (dx*dx + dy*dy) + dz*dz; 1-NN ties to the lower target index), its own 3x3 SVD, closed-form
// SE(3) log / exp, Anderson acceleration with a min-norm solve, and sequential double sums.  Compiled by
// tests/fricp_oracle.py with -ffp-contract=off.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

struct V3 { double x[3]; };

// ------------------------------------------------------------------------------------------------ k-d tree
struct Tree {
  const std::vector<V3>* p = nullptr;   // normalised finite target points
  std::vector<int> idx;
  struct Node { int b, e, axis, left, right; double split; };
  std::vector<Node> nodes;

  int build(int b, int e) {
    const int id = (int)nodes.size();
    nodes.push_back(Node{b, e, -1, -1, -1, 0.0});
    if (e - b <= 8) return id;
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = b; i < e; ++i)
      for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], (*p)[idx[i]].x[a]); hi[a] = std::max(hi[a], (*p)[idx[i]].x[a]); }
    int axis = 0;
    for (int a = 1; a < 3; ++a) if (hi[a] - lo[a] > hi[axis] - lo[axis]) axis = a;
    const int mid = (b + e) / 2;
    std::nth_element(idx.begin() + b, idx.begin() + mid, idx.begin() + e,
                     [&](int u, int v) { return (*p)[u].x[axis] < (*p)[v].x[axis]; });
    const double split = (*p)[idx[mid]].x[axis];
    const int l = build(b, mid), r = build(mid, e);
    nodes[id].axis = axis;
    nodes[id].split = split;   // left: coordinate <= split, right: >= split
    nodes[id].left = l;
    nodes[id].right = r;
    return id;
  }
  void init(const std::vector<V3>& pts) {
    p = &pts;
    idx.resize(pts.size());
    for (size_t i = 0; i < pts.size(); ++i) idx[i] = (int)i;
    nodes.clear();
    if (!idx.empty()) build(0, (int)idx.size());
  }
  static double d2(const V3& a, const double* q) {
    const double dx = a.x[0] - q[0], dy = a.x[1] - q[1], dz = a.x[2] - q[2];
    return (dx * dx + dy * dy) + dz * dz;
  }
  // 1-NN over positions in pts (the caller maps them to target indices, which are increasing in position)
  void nn(int id, const double* q, double& best, int& bi) const {
    const Node& nd = nodes[id];
    if (nd.axis < 0) {
      for (int i = nd.b; i < nd.e; ++i) {
        const int j = idx[i];
        const double d = d2((*p)[j], q);
        if (d < best || (d == best && j < bi)) { best = d; bi = j; }
      }
      return;
    }
    const double diff = q[nd.axis] - nd.split;
    const int first = diff <= 0 ? nd.left : nd.right, second = diff <= 0 ? nd.right : nd.left;
    nn(first, q, best, bi);
    if (diff * diff <= best) nn(second, q, best, bi);
  }
  // the k smallest d² (ascending) into top[0..k)
  void knn(int id, const double* q, int k, double* top) const {
    const Node& nd = nodes[id];
    if (nd.axis < 0) {
      for (int i = nd.b; i < nd.e; ++i) {
        double d = d2((*p)[idx[i]], q);
        if (d >= top[k - 1]) continue;
        int s = k - 1;
        while (s > 0 && top[s - 1] > d) { top[s] = top[s - 1]; --s; }
        top[s] = d;
      }
      return;
    }
    const double diff = q[nd.axis] - nd.split;
    const int first = diff <= 0 ? nd.left : nd.right, second = diff <= 0 ? nd.right : nd.left;
    knn(first, q, k, top);
    if (diff * diff <= top[k - 1]) knn(second, q, k, top);
  }
};

// igl::median: the middle value, or the mean of the two middle values for an even count
double median(std::vector<double> v) {
  std::sort(v.begin(), v.end());
  const size_t n = v.size() / 2;
  return v.size() % 2 == 0 ? 0.5 * (v[n] + v[n - 1]) : v[n];
}

// ------------------------------------------------------------------------------------------------ 3x3 SVD
// One-sided Jacobi: A = U diag(s) V^T, s descending (the same procedure as the library's icp_svd3).
void svd3(const double A[9], double U[9], double s[3], double V[9]) {
  double B[9];
  std::memcpy(B, A, sizeof(B));
  for (int i = 0; i < 9; ++i) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double a = 0, b = 0, c = 0;
        for (int r = 0; r < 3; ++r) { a += B[3 * r + p] * B[3 * r + p]; b += B[3 * r + q] * B[3 * r + q]; c += B[3 * r + p] * B[3 * r + q]; }
        if (c == 0.0 || std::fabs(c) <= 1e-300) continue;
        off = std::max(off, std::fabs(c) / std::sqrt(a * b));
        const double zeta = (b - a) / (2.0 * c);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
        const double cs = 1.0 / std::sqrt(1.0 + t * t), sn = cs * t;
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
  for (int j = 0; j < 3; ++j) nrm[j] = std::sqrt(B[j] * B[j] + B[3 + j] * B[3 + j] + B[6 + j] * B[6 + j]);
  std::sort(ord, ord + 3, [&](int x, int y) { return nrm[x] > nrm[y]; });
  double Bs[9], Vs[9];
  for (int j = 0; j < 3; ++j)
    for (int r = 0; r < 3; ++r) { Bs[3 * r + j] = B[3 * r + ord[j]]; Vs[3 * r + j] = V[3 * r + ord[j]]; }
  std::memcpy(V, Vs, sizeof(Vs));
  for (int j = 0; j < 3; ++j) s[j] = nrm[ord[j]];
  const double tiny = std::max(s[0], 1e-300) * 1e-13;
  for (int j = 0; j < 3; ++j)
    for (int r = 0; r < 3; ++r) U[3 * r + j] = s[j] > tiny ? Bs[3 * r + j] / s[j] : 0.0;
  if (!(s[1] > tiny)) {
    const double u0[3] = {U[0], U[3], U[6]};
    double w[3] = {0, 0, 0};
    w[std::fabs(u0[0]) < 0.6 ? 0 : (std::fabs(u0[1]) < 0.6 ? 1 : 2)] = 1.0;
    const double d = w[0] * u0[0] + w[1] * u0[1] + w[2] * u0[2];
    double v[3] = {w[0] - d * u0[0], w[1] - d * u0[1], w[2] - d * u0[2]};
    const double nv = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    for (int r = 0; r < 3; ++r) U[3 * r + 1] = v[r] / nv;
  }
  if (!(s[2] > tiny)) {
    U[2] = U[3] * U[7] - U[6] * U[4];
    U[5] = U[6] * U[1] - U[0] * U[7];
    U[8] = U[0] * U[4] - U[3] * U[1];
  }
}

double det3(const double M[9]) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

// ------------------------------------------------------------------------------------------------ SE(3) log / exp
// T: row-major 3x4 [R | t].  L: the 16 entries of the 4x4 log matrix, column-major (Eigen's data() order).
void se3_log(const double* T, double* L) {
  const double* R = T;
  const double c = std::max(-1.0, std::min(1.0, 0.5 * ((R[0] + R[5] + R[10]) - 1.0)));
  const double a[3] = {R[9] - R[6], R[2] - R[8], R[4] - R[1]};   // 2 sin(th) * axis
  const double th = std::atan2(0.5 * std::sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]), c);   // better than acos(c) near 0, pi
  double w[3];
  if (th < 1e-5) {
    const double f = 0.5 + th * th / 12.0;   // th / (2 sin th)
    for (int k = 0; k < 3; ++k) w[k] = f * a[k];
  } else if (th < M_PI - 1e-5) {
    const double f = th / (2.0 * std::sin(th));
    for (int k = 0; k < 3; ++k) w[k] = f * a[k];
  } else {
    // near pi: the axis from the symmetric part (R + R^T)/2 - cos(th) I = (1 - cos th) k k^T, its sign from a
    const double d[3] = {R[0] - c, R[5] - c, R[10] - c};
    int i = 0;
    for (int k = 1; k < 3; ++k) if (d[k] > d[i]) i = k;
    double v[3];
    for (int k = 0; k < 3; ++k) v[k] = 0.5 * (R[4 * i + k] + R[4 * k + i]) - (k == i ? c : 0.0);
    const double n = std::sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
    double s = (a[0] * v[0] + a[1] * v[1]) + a[2] * v[2];
    s = s < 0 ? -1.0 : 1.0;
    for (int k = 0; k < 3; ++k) w[k] = s * th * v[k] / n;
  }
  // u = V^-1 t, V^-1 = I - W/2 + b W^2, b = (1 - th sin th / (2 (1 - cos th))) / th^2
  const double th2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2], t = std::sqrt(th2);
  const double b = t < 1e-4 ? 1.0 / 12.0 + th2 / 720.0 : (1.0 - t * std::sin(t) / (2.0 * (1.0 - std::cos(t)))) / th2;
  const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  const double tv[3] = {T[3], T[7], T[11]};
  double Wt[3], WWt[3], u[3];
  for (int r = 0; r < 3; ++r) Wt[r] = (W[3 * r] * tv[0] + W[3 * r + 1] * tv[1]) + W[3 * r + 2] * tv[2];
  for (int r = 0; r < 3; ++r) WWt[r] = (W[3 * r] * Wt[0] + W[3 * r + 1] * Wt[1]) + W[3 * r + 2] * Wt[2];
  for (int r = 0; r < 3; ++r) u[r] = (tv[r] - 0.5 * Wt[r]) + b * WWt[r];
  for (int i = 0; i < 16; ++i) L[i] = 0.0;
  for (int r = 0; r < 3; ++r) {
    for (int cc = 0; cc < 3; ++cc) L[4 * cc + r] = W[3 * r + cc];
    L[12 + r] = u[r];
  }
}

void se3_exp(const double* L, double* T) {
  const double w[3] = {L[6], L[8], L[1]};   // (2,1), (0,2), (1,0) of the column-major 4x4
  const double u[3] = {L[12], L[13], L[14]};
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

// ------------------------------------------------------------------------------------------------ Anderson
// AndersonAcceleration.h with the m_k x m_k normal equations solved by a min-norm pseudo-inverse: Jacobi eigen-
// decomposition of M, eigenvalues <= m_k * DBL_EPSILON * (largest) treated as zero.
void sym_pinv_solve(const double* M, int n, const double* b, double* x) {
  double A[25], Vv[25];
  std::memcpy(A, M, sizeof(double) * n * n);
  for (int i = 0; i < n * n; ++i) Vv[i] = (i % (n + 1) == 0) ? 1.0 : 0.0;
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
        for (int k = 0; k < n; ++k) {   // A <- A J
          const double akp = A[k * n + p], akq = A[k * n + q];
          A[k * n + p] = cs * akp - sn * akq;
          A[k * n + q] = sn * akp + cs * akq;
        }
        for (int k = 0; k < n; ++k) {   // A <- J^T A
          const double apk = A[p * n + k], aqk = A[q * n + k];
          A[p * n + k] = cs * apk - sn * aqk;
          A[q * n + k] = sn * apk + cs * aqk;
        }
        for (int k = 0; k < n; ++k) {
          const double vp = Vv[k * n + p], vq = Vv[k * n + q];
          Vv[k * n + p] = cs * vp - sn * vq;
          Vv[k * n + q] = sn * vp + cs * vq;
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
    for (int k = 0; k < n; ++k) vb += Vv[k * n + e] * b[k];
    for (int k = 0; k < n; ++k) x[k] += Vv[k * n + e] * (vb / l);
  }
}

struct Anderson {
  int m = 0, d = 16, iter = 0, col = 0;
  double u[16], F[16], dG[5][16], dF[5][16], M[5][5], theta[5], scale[5];
  void init(int m_, const double* u0) { m = m_; std::memcpy(u, u0, sizeof(u)); iter = 0; col = 0; }
  void replace(const double* v) { std::memcpy(u, v, sizeof(u)); }
  void reset(const double* v) { iter = 0; col = 0; std::memcpy(u, v, sizeof(u)); }
  const double* compute(const double* g) {
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
        sym_pinv_solve(Mk, mk, rhs, theta);
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

bool finite3(const float* p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }

void apply(const double* T, const V3& x, double* q) {
  for (int r = 0; r < 3; ++r) q[r] = ((T[4 * r] * x.x[0] + T[4 * r + 1] * x.x[1]) + T[4 * r + 2] * x.x[2]) + T[4 * r + 3];
}

}  // namespace

extern "C" {

int orc_se3_log(const double* T12, double* L16) { se3_log(T12, L16); return 0; }
int orc_se3_exp(const double* L16, double* T12) { se3_exp(L16, T12); return 0; }
double orc_median(const double* v, int n) { return median(std::vector<double>(v, v + n)); }

// ops[k]: 0 compute(g_k), 1 replace(g_k), 2 reset(g_k); out[k] = the current u after op k (d = 16)
int orc_anderson(int m, const double* u0, int n_ops, const int* ops, const double* g, double* out) {
  Anderson a;
  a.init(m, u0);
  for (int k = 0; k < n_ops; ++k) {
    if (ops[k] == 0) a.compute(g + 16 * k);
    else if (ops[k] == 1) a.replace(g + 16 * k);
    else a.reset(g + 16 * k);
    std::memcpy(out + 16 * k, a.u, sizeof(a.u));
  }
  return 0;
}

// The registration.  src / tgt: x, y, z, w float records.  norm (optional): scale, source mean, target mean to use instead
// of the oracle's own sums.  res12: res_trans rows 0-2 (row-major 3x4).  info: status, stages, iterations, rejections,
// finite source, finite target.  dinfo: scale, mu_s[3], mu_t[3], nu_begin, nu_end, energy.  corr (n_s): the last pass's
// matched target index (-1: non-finite source or nothing registered); resid (n_s): its residual.  log: per iteration
// (stage, energy, previous last_energy, |T - T_prev|_F, accepted), up to log_cap rows; *log_n rows written.
int orc_fricp(const float* src, int n_s, const float* tgt, int n_t, int mode, int max_icp, double stop, int anderson_m,
              double nu_begin_k, double nu_end_k, double nu_alpha, const double* norm, double* res12, int* info, double* dinfo,
              int* corr, double* resid, double* log, int log_cap, int* log_n) {
  const bool welsch = mode == 3 || mode == 4, use_aa = mode == 2 || mode == 4;
  for (int i = 0; i < 12; ++i) res12[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int i = 0; i < 6; ++i) info[i] = 0;
  for (int i = 0; i < 10; ++i) dinfo[i] = 0;
  *log_n = 0;
  for (int i = 0; i < n_s; ++i) { corr[i] = -1; resid[i] = INFINITY; }
  std::vector<int> si, ti;
  for (int i = 0; i < n_s; ++i) if (finite3(src + 4 * (size_t)i)) si.push_back(i);
  for (int i = 0; i < n_t; ++i) if (finite3(tgt + 4 * (size_t)i)) ti.push_back(i);
  info[4] = (int)si.size();
  info[5] = (int)ti.size();
  if (si.empty()) { info[0] = 2; return 0; }
  if (ti.size() < 2) { info[0] = 1; return 0; }
  // normalisation
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
  std::vector<V3> X(si.size()), Y(ti.size()), Q(si.size());
  for (size_t k = 0; k < si.size(); ++k) for (int a = 0; a < 3; ++a) X[k].x[a] = (double)src[4 * si[k] + a] / scale - ms[a];
  for (size_t k = 0; k < ti.size(); ++k) for (int a = 0; a < 3; ++a) Y[k].x[a] = (double)tgt[4 * ti[k] + a] / scale - mt[a];
  Tree tree;
  tree.init(Y);
  const int ns = (int)X.size();
  std::vector<double> W(ns);
  std::vector<int> C(ns);
  auto pass = [&](const double* T) {
    for (int k = 0; k < ns; ++k) {
      double q[3];
      apply(T, X[k], q);
      double best = INFINITY;
      int bi = INT32_MAX;
      tree.nn(0, q, best, bi);
      C[k] = bi;
      Q[k] = Y[bi];
      W[k] = std::sqrt(best);
    }
  };
  auto energy_of = [&](double nu) {
    double e = 0;
    for (int k = 0; k < ns; ++k) e += welsch ? 1.0 - std::exp(-W[k] * W[k] / (2 * nu * nu)) : W[k] * W[k];
    return e;
  };
  // weighted point-to-point step (FRICP.h:177-209) from raw weighted moments; T unchanged when every weight is 0
  auto kabsch = [&](double nu, double* T) {
    double S[16] = {0};
    for (int k = 0; k < ns; ++k) {
      const double w = welsch ? std::exp(-W[k] * W[k] / (2 * nu * nu)) : 1.0;
      S[0] += w;
      for (int a = 0; a < 3; ++a) { S[1 + a] += w * X[k].x[a]; S[4 + a] += w * Q[k].x[a]; }
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) S[7 + 3 * r + c] += w * X[k].x[r] * Q[k].x[c];
    }
    if (!(S[0] > 0)) return;
    double xm[3], qm[3], sig[9], U[9], sv[3], Vm[9];
    for (int a = 0; a < 3; ++a) { xm[a] = S[1 + a] / S[0]; qm[a] = S[4 + a] / S[0]; }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) sig[3 * r + c] = S[7 + 3 * r + c] / S[0] - xm[r] * qm[c];
    svd3(sig, U, sv, Vm);
    const double dd = det3(U) * det3(Vm) < 0 ? -1.0 : 1.0;
    for (int r = 0; r < 3; ++r) {   // R = V diag(1, 1, dd) U^T
      for (int c = 0; c < 3; ++c) T[4 * r + c] = (Vm[3 * r] * U[3 * c] + Vm[3 * r + 1] * U[3 * c + 1]) + dd * Vm[3 * r + 2] * U[3 * c + 2];
      T[4 * r + 3] = qm[r] - ((T[4 * r] * xm[0] + T[4 * r + 1] * xm[1]) + T[4 * r + 2] * xm[2]);
    }
  };
  double T[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0}, SVD_T[12], To2[12];
  std::memcpy(SVD_T, T, sizeof(T));
  std::memcpy(To2, T, sizeof(T));
  pass(T);
  double nu1 = 1, nu2 = 1;
  if (welsch) {
    const int k = (int)std::min<size_t>(7, Y.size());
    std::vector<double> med(Y.size());
    for (size_t i = 0; i < Y.size(); ++i) {
      double top[7];
      for (int j = 0; j < 7; ++j) top[j] = INFINITY;
      tree.knn(0, Y[i].x, k, top);
      med[i] = median(std::vector<double>(top + 1, top + k));
    }
    nu2 = nu_end_k * std::sqrt(median(med));
    nu1 = std::max(nu_begin_k * median(W), nu2);
    dinfo[7] = nu1;
    dinfo[8] = nu2;
  }
  Anderson aa;
  double L[16];
  se3_log(T, L);
  aa.init(anderson_m, L);
  double last_energy = DBL_MAX;
  int stages = 0, iters = 0, rejects = 0;
  for (bool stop1 = false; !stop1;) {
    ++stages;
    for (int icp = 0; icp < max_icp; ++icp) {
      const double energy = energy_of(nu1), prev = last_energy;
      int accepted = 1;
      if (use_aa) {
        if (energy < last_energy) {
          last_energy = energy;
        } else {
          accepted = 0;
          ++rejects;
          se3_log(SVD_T, L);
          aa.replace(L);
          pass(SVD_T);
          last_energy = energy_of(nu1);
        }
      } else {
        last_energy = energy;
      }
      kabsch(nu1, T);
      std::memcpy(SVD_T, T, sizeof(T));
      if (use_aa) {
        se3_log(T, L);
        se3_exp(aa.compute(L), T);
      }
      pass(T);
      double s2 = 0;
      for (int i = 0; i < 12; ++i) s2 += (T[i] - To2[i]) * (T[i] - To2[i]);
      const double stop2 = std::sqrt(s2);
      std::memcpy(To2, T, sizeof(T));
      ++iters;
      if (*log_n < log_cap) {
        double* row = log + 5 * (size_t)*log_n;
        row[0] = stages - 1; row[1] = energy; row[2] = prev; row[3] = stop2; row[4] = accepted;
        ++*log_n;
      }
      if (stop2 < stop) break;
    }
    if (!welsch) {
      stop1 = true;
    } else {
      stop1 = std::fabs(nu1 - nu2) < 1e-6;
      nu1 = nu1 * nu_alpha > nu2 ? nu1 * nu_alpha : nu2;
      if (use_aa) {
        se3_log(T, L);
        aa.reset(L);
        last_energy = DBL_MAX;
      }
    }
  }
  dinfo[9] = energy_of(nu1);
  // T.translation() += -R mu_s + mu_t, then the translation times the scale (registeration.h:170)
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) res12[4 * r + c] = T[4 * r + c];
    res12[4 * r + 3] = (T[4 * r + 3] + (mt[r] - ((T[4 * r] * ms[0] + T[4 * r + 1] * ms[1]) + T[4 * r + 2] * ms[2]))) * scale;
  }
  for (int k = 0; k < ns; ++k) { corr[si[k]] = ti[C[k]]; resid[si[k]] = W[k]; }
  info[1] = stages;
  info[2] = iters;
  info[3] = rejects;
  return 0;
}

}  // extern "C"

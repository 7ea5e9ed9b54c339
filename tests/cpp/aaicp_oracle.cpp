// Sequential restatement of the relocalisation AA-ICP contract (DESIGN.md §9, "Relocalisation registration, AA-ICP"):
// AAICP::point_to_point_aaicp (ICP.h:841-1033) as Registeration::run calls it for regMode 1, with par.f = NONE and
// use_init = false, as flb_keyframes_aaicp implements it, on host clouds.  The normalisation of the relocalisation
// registration (status FEW_TARGET only without a finite target point), the exact 1-NN of the FRICP oracle's k-d tree,
// sequential double sums, that oracle's 3x3 SVD, and Eigen 3.3.7's eulerAngles(0, 1, 2), AngleAxis / Quaternion
// products, 4x4 inverse and ColPivHouseholderQR::solve written out in the association order DESIGN.md §9 states.  The
// k-d tree, the SVD and the point helpers are tests/cpp/fricp_oracle.cpp's, included whole; that file's own entry points
// come along with it.  Compiled by tests/aaicp_oracle.py with -ffp-contract=off.
#include <array>
#include <chrono>

#include "fricp_oracle.cpp"

namespace {

typedef double M4[16];   // row-major 4x4

// Matrix3::eulerAngles(0, 1, 2) (Eigen 3.3.7 EulerAngles.h, a0 = 0, a1 = 1, a2 = 2: i = 0, j = 1, k = 2, odd = 0)
void euler012(const double* m /* row-major 3x3 */, double* e) {
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

// Matrix42Vector6 (ICP.h:768-775)
void vec6(const M4 T, double* v) {
  const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  euler012(R, v);
  v[3] = T[3];
  v[4] = T[7];
  v[5] = T[11];
}

struct Quat { double w, x, y, z; };

// Quaternion(AngleAxis(angle, unit axis k)): w = cos(angle / 2), vec = sin(angle / 2) * axis
Quat quat_axis(double angle, int k) {
  const double ha = 0.5 * angle, s = std::sin(ha);
  const double ax[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
  return Quat{std::cos(ha), s * ax[0], s * ax[1], s * ax[2]};
}

// quat_product (Eigen's generic one): every sum left to right
Quat qmul(const Quat& a, const Quat& b) {
  return Quat{a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
              a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}

// Vector62Matrix4 (ICP.h:778-788): (AngleAxis X * AngleAxis Y) * AngleAxis Z as quaternions, toRotationMatrix
void mat4(const double* v, M4 T) {
  const Quat q = qmul(qmul(quat_axis(v[0], 0), quat_axis(v[1], 1)), quat_axis(v[2], 2));
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

// C = A B, each entry ((a0 b0 + a1 b1) + a2 b2) + a3 b3
void mul4(const M4 A, const M4 B, M4 C) {
  M4 o;
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) o[4 * r + c] = ((A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c]) + A[4 * r + 2] * B[8 + c]) + A[4 * r + 3] * B[12 + c];
  std::memcpy(C, o, sizeof(o));
}

// Eigen's 3x3 determinant (along the first row) of the minor of (r, c): m(0,0)(m(1,1)m(2,2) - m(1,2)m(2,1)) - m(0,1)(...) + m(0,2)(...)
double minor_det(const M4 A, int rr, int cc) {
  double m[9];
  for (int r = 0, i = 0; r < 4; ++r) {
    if (r == rr) continue;
    for (int c = 0, j = 0; c < 4; ++c) {
      if (c == cc) continue;
      m[3 * i + j++] = A[4 * r + c];
    }
    ++i;
  }
  auto h = [&](int a, int b, int c) { return m[3 * 0 + a] * (m[3 * 1 + b] * m[3 * 2 + c] - m[3 * 1 + c] * m[3 * 2 + b]); };
  return (h(0, 1, 2) - h(1, 0, 2)) + h(2, 0, 1);
}

// Matrix4::inverse() by the adjugate: res(i, j) = (-1)^(i+j) det(minor(j, i)), divided by
// ((m00 res00 + m10 res01) + m20 res02) + m30 res03
void inv4(const M4 A, M4 out) {
  M4 r;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      const double d = minor_det(A, j, i);
      r[4 * i + j] = ((i + j) % 2) ? -d : d;
    }
  const double det = ((A[0] * r[0] + A[4] * r[1]) + A[8] * r[2]) + A[12] * r[3];
  for (int k = 0; k < 16; ++k) out[k] = r[k] / det;
}

// Affine3d product A B (Transform<Affine> * Transform<Affine>): linear A.l B.l, translation A.l B.t + A.t
void mul_affine(const M4 A, const M4 B, M4 C) {
  M4 o;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) o[4 * r + c] = (A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c]) + A[4 * r + 2] * B[8 + c];
    o[4 * r + 3] = ((A[4 * r] * B[3] + A[4 * r + 1] * B[7]) + A[4 * r + 2] * B[11]) + A[4 * r + 3];
  }
  o[12] = o[13] = o[14] = 0.0;
  o[15] = 1.0;
  std::memcpy(C, o, sizeof(o));
}

// ColPivHouseholderQR<MatrixXd>(A).solve(b) for a 6 x n column-major A (Eigen 3.3.7 ColPivHouseholderQR.h:482-569 and
// :582-602, Householder.h, HouseholderSequence.h, TriangularSolverVector.h), every sum left to right.  x: n entries.
// Returns the rank (the non-zero pivot count).
int qr_solve(const double* A, int n, const double* b, double* x) {
  const int rows = 6, size = std::min(rows, n);
  std::vector<double> qr(A, A + (size_t)rows * n), hc(size), nu(n), nd(n);
  std::vector<int> tr(size);
  auto at = [&](int r, int c) -> double& { return qr[(size_t)c * rows + r]; };
  auto col_norm = [&](int c, int r0) {
    double s = 0;
    for (int r = r0; r < rows; ++r) s += at(r, c) * at(r, c);
    return std::sqrt(s);
  };
  for (int k = 0; k < n; ++k) nd[k] = nu[k] = col_norm(k, 0);
  double mx = nu[0];
  for (int k = 1; k < n; ++k) if (nu[k] > mx) mx = nu[k];
  const double eps = DBL_EPSILON;
  const double thr_helper = (mx * eps) * (mx * eps) / (double)rows;
  const double downdate = std::sqrt(eps);
  int nzp = size;
  for (int k = 0; k < size; ++k) {
    int big = k;
    for (int j = k + 1; j < n; ++j) if (nu[j] > nu[big]) big = j;   // the first largest
    const double big_sq = nu[big] * nu[big];
    if (nzp == size && big_sq < thr_helper * (double)(rows - k)) nzp = k;
    tr[k] = big;
    if (k != big) {
      for (int r = 0; r < rows; ++r) std::swap(at(r, k), at(r, big));
      std::swap(nu[k], nu[big]);
      std::swap(nd[k], nd[big]);
    }
    // makeHouseholderInPlace on column k, rows k..5
    double tail = 0;
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
    // applyHouseholderOnTheLeft on rows k..5, columns k+1..n-1
    if (rows - k == 1) {
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
    for (int j = k + 1; j < n; ++j) {   // the norm downdate (LAPACK xGEQP3)
      if (nu[j] == 0.0) continue;
      double t = std::fabs(at(k, j)) / nu[j];
      t = (1.0 + t) * (1.0 - t);
      t = t < 0.0 ? 0.0 : t;
      const double q = nu[j] / nd[j];
      const double t2 = t * (q * q);
      if (t2 <= downdate) {
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
  if (nzp == 0) return 0;
  double c[6];
  std::memcpy(c, b, sizeof(c));
  for (int k = 0; k < nzp; ++k) {   // Q^T b: H_0 first
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
  return nzp;
}

struct Hist {   // 6 x k column lists
  std::vector<std::array<double, 6>> c;
  void keep_last(int k) { c.erase(c.begin(), c.end() - k); }
};

// get_next_u (ICP.h:812-837) with beta = 1; na: the number of α of the result; margin: the smallest margin of the
// alphas_cond tests made (INFINITY: none).
void next_u(const Hist& u, const Hist& g, const Hist& f, double* out, int* na, double* margin) {
  const int m = (int)f.c.size();
  for (int r = 0; r < 6; ++r) out[r] = 0.0 * u.c.back()[r] + 1.0 * g.c.back()[r];
  *na = 1;
  *margin = INFINITY;
  for (int i = 2; i <= m; ++i) {
    // A = f.last 1^T - f.rightCols(i).leftCols(i-1), solve A α' = f.last, α = (α', 1 - Σα')
    const std::array<double, 6>& fl = f.c[m - 1];
    std::vector<double> A((size_t)6 * (i - 1)), al(i);
    for (int j = 0; j < i - 1; ++j)
      for (int r = 0; r < 6; ++r) A[(size_t)6 * j + r] = -f.c[m - i + j][r] + fl[r];
    qr_solve(A.data(), i - 1, fl.data(), al.data());
    double s = 0;
    for (int j = 0; j < i - 1; ++j) s += al[j];
    al[i - 1] = 1.0 - (s + 0.0);
    double lo = al[0], hi = al[0];
    for (int j = 1; j < i; ++j) { if (al[j] < lo) lo = al[j]; if (al[j] > hi) hi = al[j]; }
    const double mg = std::min(std::fabs(lo + 10.0), std::min(std::fabs(10.0 - hi), std::fabs(al[i - 1])));
    bool nan = std::isnan(*margin);
    for (int j = 0; j < i; ++j) nan = nan || std::isnan(al[j]);
    *margin = nan ? NAN : std::min(*margin, mg);   // a test on a NaN α has no margin
    if (!(-10.0 < lo && hi < 10.0 && al[i - 1] > 0)) break;
    for (int r = 0; r < 6; ++r) {
      double su = 0, sg = 0;
      for (int j = 0; j < i; ++j) { su += u.c[u.c.size() - i + j][r] * al[j]; sg += g.c[m - i + j][r] * al[j]; }
      out[r] = 0.0 * su + 1.0 * sg;
    }
    *na = i;
  }
}

}  // namespace

extern "C" {

void orc_aa_euler(const double* R9, double* e3) { euler012(R9, e3); }
void orc_aa_mat4(const double* v6, double* T16) { mat4(v6, T16); }
void orc_aa_inv4(const double* A16, double* out16) { inv4(A16, out16); }
int orc_aa_qr_solve(const double* A, int n, const double* b, double* x) { return qr_solve(A, n, b, x); }

// The registration.  src / tgt: x, y, z, w float records.  norm (optional): scale, source mean, target mean.  res12:
// res_trans rows 0-2.  info: status, iterations (the loop index at exit), accepted, resets, history (columns of u),
// finite source, finite target.  dinfo: scale, mu_s[3], mu_t[3], energy, and the wall time (ms) spent from the Euler
// angles to the re-seated transform over all iterations (the Anderson work).  corr / resid (n_s): the last pass's matched
// target index and |X - Q| (-1 / +inf: none).  log: per iteration (energy, prev_energy before the test, outcome -1 / 1 /
// 0, α count, stop2, smallest alphas_cond margin).
int orc_aaicp(const float* src, int n_s, const float* tgt, int n_t, int max_icp, double stop, double thr, const double* norm,
              double* res12, int* info, double* dinfo, int* corr, double* resid, double* log, int log_cap, int* log_n) {
  for (int i = 0; i < 12; ++i) res12[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int i = 0; i < 7; ++i) info[i] = 0;
  for (int i = 0; i < 9; ++i) dinfo[i] = 0;
  *log_n = 0;
  for (int i = 0; i < n_s; ++i) { corr[i] = -1; resid[i] = INFINITY; }
  std::vector<int> si, ti;
  for (int i = 0; i < n_s; ++i) if (finite3(src + 4 * (size_t)i)) si.push_back(i);
  for (int i = 0; i < n_t; ++i) if (finite3(tgt + 4 * (size_t)i)) ti.push_back(i);
  info[5] = (int)si.size();
  info[6] = (int)ti.size();
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
  std::vector<V3> X0(ns), Y(ti.size()), X(ns), Q(ns);
  for (int k = 0; k < ns; ++k) for (int a = 0; a < 3; ++a) X0[k].x[a] = (double)src[4 * si[k] + a] / scale - ms[a];
  for (size_t k = 0; k < ti.size(); ++k) for (int a = 0; a < 3; ++a) Y[k].x[a] = (double)tgt[4 * ti[k] + a] / scale - mt[a];
  for (int k = 0; k < ns; ++k) for (int a = 0; a < 3; ++a) Q[k].x[a] = 0.0;   // Matrix3Xd::Zero
  X = X0;
  Tree tree;
  tree.init(Y);
  std::vector<int> M(ns, -1);
  std::vector<double> W(ns, INFINITY);
  const M4 I4 = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  M4 T, To2, tr, fin;
  std::memcpy(T, I4, sizeof(M4));
  std::memcpy(To2, I4, sizeof(M4));
  std::memcpy(tr, I4, sizeof(M4));
  std::memcpy(fin, I4, sizeof(M4));
  Hist u, g, f;
  double u_next[6], u_k[6], prev_energy = DBL_MAX, energy = DBL_MAX;
  int icp = 0, accepted = 0, resets = 0;
  for (; icp < max_icp; ++icp) {
    for (int k = 0; k < ns; ++k) {   // Q = the nearest target points of X
      double best = INFINITY;
      int bi = INT32_MAX;
      tree.nn(0, X[k].x, best, bi);
      M[k] = bi;
      Q[k] = Y[bi];
      const double dx = X[k].x[0] - Q[k].x[0], dy = X[k].x[1] - Q[k].x[1], dz = X[k].x[2] - Q[k].x[2];
      W[k] = std::sqrt((dx * dx + dy * dy) + dz * dz);
    }
    // the unweighted point-to-point step on (X, Q) from raw moments; X is not moved (ICP.h:120)
    double S[16] = {0};
    for (int k = 0; k < ns; ++k) {
      S[0] += 1.0;
      for (int a = 0; a < 3; ++a) { S[1 + a] += X[k].x[a]; S[4 + a] += Q[k].x[a]; }
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) S[7 + 3 * r + c] += X[k].x[r] * Q[k].x[c];
    }
    double xm[3], qm[3], sig[9], Us[9], sv[3], Vm[9];
    for (int a = 0; a < 3; ++a) { xm[a] = S[1 + a] / S[0]; qm[a] = S[4 + a] / S[0]; }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) sig[3 * r + c] = S[7 + 3 * r + c] / S[0] - xm[r] * qm[c];
    svd3(sig, Us, sv, Vm);
    if (!(sv[0] > 0))   // a zero cross-covariance (one point): U = V = I, as Eigen's JacobiSVD gives them
      for (int k = 0; k < 9; ++k) Us[k] = Vm[k] = (k % 4 == 0) ? 1.0 : 0.0;
    const double dd = det3(Us) * det3(Vm) < 0 ? -1.0 : 1.0;
    M4 step;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) step[4 * r + c] = (Vm[3 * r] * Us[3 * c] + Vm[3 * r + 1] * Us[3 * c + 1]) + dd * Vm[3 * r + 2] * Us[3 * c + 2];
      step[4 * r + 3] = qm[r] - ((step[4 * r] * xm[0] + step[4 * r + 1] * xm[1]) + step[4 * r + 2] * xm[2]);
    }
    step[12] = step[13] = step[14] = 0.0;
    step[15] = 1.0;
    mul_affine(step, T, T);
    std::memcpy(fin, T, sizeof(M4));
    energy = 0;
    for (int k = 0; k < ns; ++k) energy += W[k] * W[k];
    const auto t_aa = std::chrono::steady_clock::now();
    double prev = prev_energy, margin = INFINITY;
    int outcome = -1, na = 1;
    M4 P;
    std::array<double, 6> gk;
    mul4(tr, fin, P);
    vec6(P, gk.data());
    if (icp) {
      if ((energy - prev_energy) / prev_energy > thr) {   // the first heuristic
        std::memcpy(u_next, g.c.back().data(), sizeof(u_next));
        std::memcpy(u_k, u_next, sizeof(u_k));
        prev_energy = DBL_MAX;
        u.keep_last(2);
        g.keep_last(1);
        f.keep_last(1);
        outcome = 0;
        ++resets;
      } else {
        prev_energy = energy;
        g.c.push_back(gk);
        std::array<double, 6> fk;
        for (int r = 0; r < 6; ++r) fk[r] = gk[r] - u_k[r];
        f.c.push_back(fk);
        next_u(u, g, f, u_next, &na, &margin);
        std::array<double, 6> un;
        std::memcpy(un.data(), u_next, sizeof(u_next));
        u.c.push_back(un);
        std::memcpy(u_k, u_next, sizeof(u_k));
        outcome = 1;
        ++accepted;
      }
    } else {
      prev_energy = energy;
      std::array<double, 6> u0;
      vec6(I4, u0.data());
      u.c.push_back(u0);
      g.c.push_back(gk);
      u.c.push_back(gk);
      std::array<double, 6> f0;
      for (int r = 0; r < 6; ++r) f0[r] = gk[r] - u0[r];
      f.c.push_back(f0);
      std::memcpy(u_next, gk.data(), sizeof(u_next));
      std::memcpy(u_k, gk.data(), sizeof(u_k));
    }
    M4 Mu, Fi;
    mat4(u_next, Mu);
    inv4(fin, Fi);
    mul4(Mu, Fi, tr);
    std::memcpy(fin, Mu, sizeof(M4));
    dinfo[8] += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_aa).count();
    for (int k = 0; k < ns; ++k) apply(fin, X0[k], X[k].x);
    double s2 = 0;
    for (int i = 0; i < 16; ++i) s2 += (fin[i] - To2[i]) * (fin[i] - To2[i]);
    const double stop2 = std::sqrt(s2);
    std::memcpy(To2, fin, sizeof(M4));
    if (*log_n < log_cap) {
      double* row = log + 6 * (size_t)*log_n;
      row[0] = energy; row[1] = prev; row[2] = outcome; row[3] = na; row[4] = stop2; row[5] = margin;
      ++*log_n;
    }
    if (stop2 < stop && icp) break;
  }
  double e = 0;   // the convergence energy: the last matches against the re-seated X
  for (int k = 0; k < ns; ++k) {
    const double dx = X[k].x[0] - Q[k].x[0], dy = X[k].x[1] - Q[k].x[1], dz = X[k].x[2] - Q[k].x[2];
    const double w = std::sqrt((dx * dx + dy * dy) + dz * dz);
    e += w * w;
  }
  dinfo[7] = e;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) res12[4 * r + c] = fin[4 * r + c];
    res12[4 * r + 3] = (fin[4 * r + 3] + (mt[r] - ((fin[4 * r] * ms[0] + fin[4 * r + 1] * ms[1]) + fin[4 * r + 2] * ms[2]))) * scale;
  }
  if (max_icp > 0)
    for (int k = 0; k < ns; ++k) { corr[si[k]] = ti[M[k]]; resid[si[k]] = W[k]; }
  info[1] = icp;
  info[2] = accepted;
  info[3] = resets;
  info[4] = (int)u.c.size();
  return 0;
}

}  // extern "C"

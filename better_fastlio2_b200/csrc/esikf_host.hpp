// esikf_host.hpp — host side (C++) of the iterated error-state Kalman update: the 23-DOF manifold algebra and the
// 23x23 linear algebra of esekf::update_iterated_dyn_share_modified
// (reference: include/IKFoM_toolkit/esekfom/esekfom.hpp:1620-1938), consuming the GPU-reduced normal equations
// H^T H (12x12) and H^T h instead of the M x 12 row matrix (boundary B3, SURVEY.md §8b).  The reference keeps this
// part on the host too; it is O(23^3) per pass (microseconds) and is not the data-parallel part of the path.
//
// Manifold conventions restated from include/use-ikfom.hpp:21-30 (state_ikfom), mtk/types/SOn.hpp:233-297 (SO3),
// mtk/types/S2.hpp:136-280 (S2, S2_typ = 1, length 9.809), mtk/src/mtkmath.hpp:142-288, including the reference's
// quirk that S2_Mx evaluates exp(.., scalar(1/2)) with an integer 1/2 == 0 (S2.hpp:277).
#pragma once
#include <array>
#include <cmath>
#include <cstring>

namespace flb {
namespace host {

constexpr int DOF = 23;
constexpr double kTol = 1e-11;
constexpr double kS2Len = 98090.0 / 10000.0;

template <int R, int C>
struct Mat {
  double a[R * C];
  double& operator()(int r, int c) { return a[r * C + c]; }
  double operator()(int r, int c) const { return a[r * C + c]; }
  static Mat zero() { Mat m; std::memset(m.a, 0, sizeof(m.a)); return m; }
  static Mat identity() { Mat m = zero(); for (int i = 0; i < (R < C ? R : C); ++i) m(i, i) = 1.0; return m; }
  Mat<C, R> t() const { Mat<C, R> o; for (int r = 0; r < R; ++r) for (int c = 0; c < C; ++c) o(c, r) = (*this)(r, c); return o; }
};
template <int R, int K, int C>
inline Mat<R, C> operator*(const Mat<R, K>& A, const Mat<K, C>& B) {
  Mat<R, C> o;
  for (int r = 0; r < R; ++r)
    for (int c = 0; c < C; ++c) {
      double s = 0;
      for (int k = 0; k < K; ++k) s += A(r, k) * B(k, c);
      o(r, c) = s;
    }
  return o;
}
template <int R, int C>
inline Mat<R, C> operator*(double s, const Mat<R, C>& A) { Mat<R, C> o; for (int i = 0; i < R * C; ++i) o.a[i] = s * A.a[i]; return o; }
template <int R, int C>
inline Mat<R, C> operator+(const Mat<R, C>& A, const Mat<R, C>& B) { Mat<R, C> o; for (int i = 0; i < R * C; ++i) o.a[i] = A.a[i] + B.a[i]; return o; }
template <int R, int C>
inline Mat<R, C> operator-(const Mat<R, C>& A, const Mat<R, C>& B) { Mat<R, C> o; for (int i = 0; i < R * C; ++i) o.a[i] = A.a[i] - B.a[i]; return o; }

using V3 = Mat<3, 1>;
using M3 = Mat<3, 3>;
using Cov = Mat<DOF, DOF>;

struct Quat { double x, y, z, w; };
inline Quat operator*(const Quat& a, const Quat& b) {
  return Quat{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
              a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
inline Quat conj(const Quat& q) { return Quat{-q.x, -q.y, -q.z, q.w}; }
inline M3 rotmat(const Quat& q) {
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  M3 R;
  R(0, 0) = 1 - (tyy + tzz); R(0, 1) = txy - twz; R(0, 2) = txz + twy;
  R(1, 0) = txy + twz; R(1, 1) = 1 - (txx + tzz); R(1, 2) = tyz - twx;
  R(2, 0) = txz - twy; R(2, 1) = tyz + twx; R(2, 2) = 1 - (txx + tyy);
  return R;
}
inline V3 rotate(const Quat& q, const V3& v) {
  V3 uv; uv(0, 0) = q.y * v(2, 0) - q.z * v(1, 0); uv(1, 0) = q.z * v(0, 0) - q.x * v(2, 0); uv(2, 0) = q.x * v(1, 0) - q.y * v(0, 0);
  for (int i = 0; i < 3; ++i) uv.a[i] += uv.a[i];
  V3 o;
  o(0, 0) = v(0, 0) + q.w * uv(0, 0) + (q.y * uv(2, 0) - q.z * uv(1, 0));
  o(1, 0) = v(1, 0) + q.w * uv(1, 0) + (q.z * uv(0, 0) - q.x * uv(2, 0));
  o(2, 0) = v(2, 0) + q.w * uv(2, 0) + (q.x * uv(1, 0) - q.y * uv(0, 0));
  return o;
}
inline M3 skew(const V3& v) {
  M3 H = M3::zero();
  H(0, 1) = -v(2, 0); H(0, 2) = v(1, 0); H(1, 0) = v(2, 0); H(1, 2) = -v(0, 0); H(2, 0) = -v(1, 0); H(2, 1) = v(0, 0);
  return H;
}

// cos(sqrt(x2)), sinc(sqrt(x2)) with the toolkit's 3-term series below eps^(1/4)  (mtkmath.hpp:142-174)
inline void cos_sinc_sqrt(double x2, double& c, double& s) {
  static const double bound = std::sqrt(std::sqrt(2.220446049250313e-16));
  if (x2 >= bound) { const double x = std::sqrt(x2); c = std::cos(x); s = std::sin(x) / x; return; }
  static const double inv[] = {1 / 3., 1 / 4., 1 / 5., 1 / 6., 1 / 7., 1 / 8., 1 / 9.};
  double cosi = 1., sinc = 1., term = -1 / 2. * x2;
  for (int i = 0; i < 3; ++i) { cosi += term; term *= inv[2 * i]; sinc += term; term *= -inv[2 * i + 1] * x2; }
  c = cosi; s = sinc;
}
// quaternion [w = cos(scale*|v|), vec = sinc(scale*|v|)*scale*v]   (mtkmath.hpp:249-256)
inline Quat exp_quat(const V3& v, double scale) {
  const double n2 = v(0, 0) * v(0, 0) + v(1, 0) * v(1, 0) + v(2, 0) * v(2, 0);
  double c, s;
  cos_sinc_sqrt(scale * scale * n2, c, s);
  const double m = s * scale;
  return Quat{m * v(0, 0), m * v(1, 0), m * v(2, 0), c};
}
inline V3 log_quat(const Quat& q) {  // scale 2, atan form (SOn.hpp:293-297, mtkmath.hpp:268-288)
  double nv = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
  if (nv < kTol) nv = kTol;
  const double s = 2.0 / nv * std::atan(nv / q.w);
  V3 o; o(0, 0) = s * q.x; o(1, 0) = s * q.y; o(2, 0) = s * q.z;
  return o;
}
inline M3 A_matrix(const V3& v) {  // mtkmath.hpp:235-247
  const double sq = v(0, 0) * v(0, 0) + v(1, 0) * v(1, 0) + v(2, 0) * v(2, 0);
  const double n = std::sqrt(sq);
  if (n < kTol) return M3::identity();
  const M3 H = skew(v);
  return M3::identity() + ((1 - std::cos(n)) / sq) * H + ((1 - std::sin(n) / n) / sq) * (H * H);
}

struct S2 {
  V3 vec;
  Mat<3, 2> Bx() const {  // S2.hpp:215-231 (S2_typ == 1)
    Mat<3, 2> B;
    const double len = kS2Len, v0 = vec(0, 0), v1 = vec(1, 0), v2 = vec(2, 0);
    if (v0 + len > kTol) {
      B(0, 0) = -v1; B(0, 1) = -v2;
      B(1, 0) = len - v1 * v1 / (len + v0); B(1, 1) = -v2 * v1 / (len + v0);
      B(2, 0) = -v2 * v1 / (len + v0); B(2, 1) = len - v2 * v2 / (len + v0);
      for (double& e : B.a) e /= len;
    } else {
      B = Mat<3, 2>::zero(); B(1, 1) = -1; B(2, 0) = 1;
    }
    return B;
  }
  Mat<2, 3> Nx_yy() const { return ((1 / kS2Len / kS2Len) * Bx().t()) * skew(vec); }  // S2.hpp:259-264
  Mat<3, 2> Mx(const Mat<2, 1>& delta) const {                                        // S2.hpp:266-280
    const Mat<3, 2> B = Bx();
    const double dn = std::sqrt(delta(0, 0) * delta(0, 0) + delta(1, 0) * delta(1, 0));
    if (dn < kTol) return (-1.0 * skew(vec)) * B;
    const V3 Bu = B * delta;
    const M3 E = rotmat(exp_quat(Bu, 0.0));  // scalar(1/2) == 0 in the reference: identity
    return (((-1.0 * E) * skew(vec)) * A_matrix(Bu).t()) * B;
  }
  void boxplus(const Mat<2, 1>& delta) {  // S2.hpp:136-142
    const V3 Bu = Bx() * delta;
    vec = rotmat(exp_quat(Bu, 0.5)) * vec;
  }
  Mat<2, 1> boxminus(const S2& other) const {  // S2.hpp:144-167
    Mat<2, 1> res;
    const V3 cr = skew(vec) * other.vec;
    const double v_sin = std::sqrt(cr(0, 0) * cr(0, 0) + cr(1, 0) * cr(1, 0) + cr(2, 0) * cr(2, 0));
    const double v_cos = vec(0, 0) * other.vec(0, 0) + vec(1, 0) * other.vec(1, 0) + vec(2, 0) * other.vec(2, 0);
    const double theta = std::atan2(v_sin, v_cos);
    if (v_sin < kTol) {
      res(0, 0) = std::fabs(theta) > kTol ? 3.1415926 : 0.0;
      res(1, 0) = 0.0;
      return res;
    }
    return ((theta / v_sin) * other.Bx().t()) * (skew(other.vec) * vec);
  }
};

struct State {
  V3 pos; Quat rot; Quat offR; V3 offT, vel, bg, ba; S2 grav;
  static State from26(const double* s) {
    State x;
    for (int i = 0; i < 3; ++i) { x.pos.a[i] = s[i]; x.offT.a[i] = s[11 + i]; x.vel.a[i] = s[14 + i]; x.bg.a[i] = s[17 + i]; x.ba.a[i] = s[20 + i]; x.grav.vec.a[i] = s[23 + i]; }
    x.rot = Quat{s[3], s[4], s[5], s[6]};
    x.offR = Quat{s[7], s[8], s[9], s[10]};
    return x;
  }
  void to26(double* s) const {
    for (int i = 0; i < 3; ++i) { s[i] = pos.a[i]; s[11 + i] = offT.a[i]; s[14 + i] = vel.a[i]; s[17 + i] = bg.a[i]; s[20 + i] = ba.a[i]; s[23 + i] = grav.vec.a[i]; }
    s[3] = rot.x; s[4] = rot.y; s[5] = rot.z; s[6] = rot.w;
    s[7] = offR.x; s[8] = offR.y; s[9] = offR.z; s[10] = offR.w;
  }
  static V3 seg3(const double* d) { V3 v; v.a[0] = d[0]; v.a[1] = d[1]; v.a[2] = d[2]; return v; }
  void boxplus(const double* d) {  // build_manifold.hpp:188-190
    for (int i = 0; i < 3; ++i) pos.a[i] += d[i];
    rot = rot * exp_quat(seg3(d + 3), 0.5);
    offR = offR * exp_quat(seg3(d + 6), 0.5);
    for (int i = 0; i < 3; ++i) { offT.a[i] += d[9 + i]; vel.a[i] += d[12 + i]; bg.a[i] += d[15 + i]; ba.a[i] += d[18 + i]; }
    Mat<2, 1> dg; dg.a[0] = d[21]; dg.a[1] = d[22];
    grav.boxplus(dg);
  }
  void boxminus(const State& o, double* r) const {  // build_manifold.hpp:194-196
    for (int i = 0; i < 3; ++i) r[i] = pos.a[i] - o.pos.a[i];
    const V3 lr = log_quat(conj(o.rot) * rot), lo = log_quat(conj(o.offR) * offR);
    for (int i = 0; i < 3; ++i) { r[3 + i] = lr.a[i]; r[6 + i] = lo.a[i]; }
    for (int i = 0; i < 3; ++i) { r[9 + i] = offT.a[i] - o.offT.a[i]; r[12 + i] = vel.a[i] - o.vel.a[i]; r[15 + i] = bg.a[i] - o.bg.a[i]; r[18 + i] = ba.a[i] - o.ba.a[i]; }
    const Mat<2, 1> g = grav.boxminus(o.grav);
    r[21] = g.a[0]; r[22] = g.a[1];
  }
};

// LU factorisation with partial pivoting (Eigen's PartialPivLU, esekfom.hpp:1788,1808), then X = A^-1 B for the C
// columns of B.  B = I gives the dense inverse.
template <int N, int C>
inline bool lu_solve(const Mat<N, N>& A, const Mat<N, C>& B, Mat<N, C>& X) {
  Mat<N, N> lu = A;
  int piv[N];
  for (int i = 0; i < N; ++i) piv[i] = i;
  for (int c = 0; c < N; ++c) {
    int p = c;
    double best = std::fabs(lu(c, c));
    for (int r = c + 1; r < N; ++r) if (std::fabs(lu(r, c)) > best) { best = std::fabs(lu(r, c)); p = r; }
    if (best == 0.0) return false;
    if (p != c) { for (int j = 0; j < N; ++j) std::swap(lu(c, j), lu(p, j)); std::swap(piv[c], piv[p]); }
    const double d = 1.0 / lu(c, c);
    for (int r = c + 1; r < N; ++r) {
      const double f = (lu(r, c) *= d);
      if (f != 0.0) for (int j = c + 1; j < N; ++j) lu(r, j) -= f * lu(c, j);
    }
  }
  // solve LU X = P B column by column
  for (int col = 0; col < C; ++col) {
    double y[N];
    for (int i = 0; i < N; ++i) {
      double s = B(piv[i], col);
      for (int k = 0; k < i; ++k) s -= lu(i, k) * y[k];
      y[i] = s;
    }
    for (int i = N - 1; i >= 0; --i) {
      double s = y[i];
      for (int k = i + 1; k < N; ++k) s -= lu(i, k) * X(k, col);
      X(i, col) = s / lu(i, i);
    }
  }
  return true;
}
template <int N>
inline bool inverse(const Mat<N, N>& A, Mat<N, N>& Ai) { return lu_solve(A, Mat<N, N>::identity(), Ai); }

// Block helpers: rows [idx, idx+D) <- J * Src rows ; cols [idx, idx+D) <- cols * J^T.
template <int D>
inline void mul_rows(Cov& Dst, int idx, const Mat<D, D>& J, const Cov& Src) {
  for (int c = 0; c < DOF; ++c) {
    double t[D];
    for (int i = 0; i < D; ++i) { double s = 0; for (int k = 0; k < D; ++k) s += J(i, k) * Src(idx + k, c); t[i] = s; }
    for (int i = 0; i < D; ++i) Dst(idx + i, c) = t[i];
  }
}
template <int D>
inline void mul_cols_T(Cov& M, int idx, const Mat<D, D>& J) {
  for (int r = 0; r < DOF; ++r) {
    double t[D];
    for (int j = 0; j < D; ++j) { double s = 0; for (int k = 0; k < D; ++k) s += M(r, idx + k) * J(j, k); t[j] = s; }
    for (int j = 0; j < D; ++j) M(r, idx + j) = t[j];
  }
}

// The iterated update as a small state machine driven by the caller (who runs the GPU pass between steps).
class IteratedUpdate {
 public:
  IteratedUpdate(const double* state26, const double* P23, double R, int max_iter, const double* limit)
      : x_(State::from26(state26)), x_prop_(x_), R_(R), max_iter_(max_iter) {
    std::memcpy(P_prop_.a, P23, sizeof(P_prop_.a));
    P_ = P_prop_;
    for (int i = 0; i < DOF; ++i) limit_[i] = limit[i];
  }
  // loop variable of esekfom.hpp:1636 runs i = -1 .. max_iter-1
  bool more() const { return !finished_ && it_ < max_iter_; }
  bool need_search() const { return converge_; }        // dyn_share.converge
  void current_state(double* s26) const { x_.to26(s26); }
  int converged_count() const { return t_; }

  // One pass with a valid measurement (M >= 1): HTH 12x12 row-major, HTh 12.  Requires M >= DOF for the
  // information-form branch (esekfom.hpp:1788-1815); the rare M < 23 branch needs the rows (see step_rows).
  // [K_x[:, 0:12] | K_h] = P_temp^-1 [H^T H | H^T h] (rows 12.. zero) is SOLVED from P_temp's LU factors instead of
  // forming P_temp^-1 and multiplying as the reference does: with extrinsic estimation P_temp is ill-conditioned
  // (position and extrinsic translation enter the rows almost alike) and the explicit inverse times the large H^T H
  // loses digits (6.6e-10 in the state against a float64 solve on a dense prior, tests/test_esikf_dense_cpu.py).
  void step(const double* HTH, const double* HTh) {
    double dx[DOF];
    prepare(dx);
    Cov PR;
    for (int i = 0; i < DOF * DOF; ++i) PR.a[i] = P_.a[i] / R_;
    Cov P_temp;
    inverse(PR, P_temp);
    for (int a = 0; a < 12; ++a) for (int b = 0; b < 12; ++b) P_temp(a, b) += HTH[a * 12 + b];
    Mat<DOF, 13> rhs = Mat<DOF, 13>::zero(), sol;
    for (int a = 0; a < 12; ++a) { for (int b = 0; b < 12; ++b) rhs(a, b) = HTH[a * 12 + b]; rhs(a, 12) = HTh[a]; }
    lu_solve(P_temp, rhs, sol);
    K_x_ = Cov::zero();
    for (int i = 0; i < DOF; ++i) {
      K_h_[i] = sol(i, 12);
      for (int b = 0; b < 12; ++b) K_x_(i, b) = sol(i, b);
    }
    finish(dx);
  }
  // M < 23 branch (esekfom.hpp:1720-1750): K = P Hc^T (Hc P Hc^T / R + I)^-1 / R with explicit rows (row-major M x 12).
  void step_rows(const double* hx, const double* h, int M) {
    double dx[DOF];
    prepare(dx);
    // S = H P[0:12,0:12] H^T / R + I  (Hc has zeros beyond column 12)
    double S[22 * 22], Si[22 * 22], PHt[DOF * 22];
    for (int i = 0; i < DOF; ++i) for (int r = 0; r < M; ++r) { double s = 0; for (int k = 0; k < 12; ++k) s += P_(i, k) * hx[r * 12 + k]; PHt[i * M + r] = s; }
    for (int r = 0; r < M; ++r) for (int c = 0; c < M; ++c) { double s = 0; for (int k = 0; k < 12; ++k) s += hx[r * 12 + k] * PHt[k * M + c]; S[r * M + c] = s / R_ + (r == c ? 1.0 : 0.0); }
    inverse_dyn(S, Si, M);
    K_x_ = Cov::zero();
    for (int i = 0; i < DOF; ++i) {
      double Krow[22];
      for (int c = 0; c < M; ++c) { double s = 0; for (int k = 0; k < M; ++k) s += PHt[i * M + k] * Si[k * M + c]; Krow[c] = s / R_; }
      double s = 0;
      for (int k = 0; k < M; ++k) s += Krow[k] * h[k];
      K_h_[i] = s;
      for (int j = 0; j < 12; ++j) { double q = 0; for (int k = 0; k < M; ++k) q += Krow[k] * hx[k * 12 + j]; K_x_(i, j) = q; }
    }
    finish(dx);
  }
  // A pass whose measurement was invalid (valid=false -> `continue`, esekfom.hpp:1641-1644).
  void skip() { ++it_; }

  void result(double* state26, double* P23) const { x_.to26(state26); std::memcpy(P23, P_.a, sizeof(P_.a)); }
  bool touched() const { return touched_; }

 private:
  static void inverse_dyn(const double* A, double* Ai, int n) {
    double a[22 * 22];
    for (int i = 0; i < n * n; ++i) a[i] = A[i];
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) Ai[i * n + j] = i == j ? 1.0 : 0.0;
    for (int c = 0; c < n; ++c) {
      int p = c; double best = std::fabs(a[c * n + c]);
      for (int r = c + 1; r < n; ++r) if (std::fabs(a[r * n + c]) > best) { best = std::fabs(a[r * n + c]); p = r; }
      if (p != c) for (int j = 0; j < n; ++j) { std::swap(a[c * n + j], a[p * n + j]); std::swap(Ai[c * n + j], Ai[p * n + j]); }
      const double d = 1.0 / a[c * n + c];
      for (int j = 0; j < n; ++j) { a[c * n + j] *= d; Ai[c * n + j] *= d; }
      for (int r = 0; r < n; ++r) if (r != c) { const double f = a[r * n + c]; if (f != 0.0) for (int j = 0; j < n; ++j) { a[r * n + j] -= f * a[c * n + j]; Ai[r * n + j] -= f * Ai[c * n + j]; } }
    }
  }
  Mat<2, 2> s2_jac(const double* d2) const {
    Mat<2, 1> dl; dl.a[0] = d2[0]; dl.a[1] = d2[1];
    return x_.grav.Nx_yy() * x_prop_.grav.Mx(dl);
  }
  void prepare(double* dx) {  // esekfom.hpp:1653-1703
    touched_ = true;
    x_.boxminus(x_prop_, dx);
    for (int i = 0; i < DOF; ++i) dx_new_[i] = dx[i];
    P_ = P_prop_;
    for (int idx : {3, 6}) {
      const M3 J = A_matrix(State::seg3(dx + idx)).t();
      const V3 v = J * State::seg3(dx_new_ + idx);
      for (int i = 0; i < 3; ++i) dx_new_[idx + i] = v.a[i];
      mul_rows<3>(P_, idx, J, P_);
      mul_cols_T<3>(P_, idx, J);
    }
    const Mat<2, 2> J = s2_jac(dx + 21);
    const double t0 = J(0, 0) * dx_new_[21] + J(0, 1) * dx_new_[22], t1 = J(1, 0) * dx_new_[21] + J(1, 1) * dx_new_[22];
    dx_new_[21] = t0; dx_new_[22] = t1;
    mul_rows<2>(P_, 21, J, P_);
    mul_cols_T<2>(P_, 21, J);
  }
  void finish(const double*) {  // esekfom.hpp:1821-1935
    double dx_[DOF];
    for (int i = 0; i < DOF; ++i) {
      double s = 0;
      for (int j = 0; j < DOF; ++j) s += (K_x_(i, j) - (i == j ? 1.0 : 0.0)) * dx_new_[j];
      dx_[i] = K_h_[i] + s;
    }
    x_.boxplus(dx_);
    converge_ = true;
    for (int i = 0; i < DOF; ++i) if (std::fabs(dx_[i]) > limit_[i]) { converge_ = false; break; }
    if (converge_) ++t_;
    if (!t_ && it_ == max_iter_ - 2) converge_ = true;
    if (t_ > 1 || it_ == max_iter_ - 1) {
      Cov L = P_;
      for (int idx : {3, 6}) {
        const M3 J = A_matrix(State::seg3(dx_ + idx)).t();
        mul_rows<3>(L, idx, J, P_);
        for (int c = 0; c < 12; ++c) {
          double tv[3];
          for (int i = 0; i < 3; ++i) { double s = 0; for (int k = 0; k < 3; ++k) s += J(i, k) * K_x_(idx + k, c); tv[i] = s; }
          for (int i = 0; i < 3; ++i) K_x_(idx + i, c) = tv[i];
        }
        mul_cols_T<3>(L, idx, J);
        mul_cols_T<3>(P_, idx, J);
      }
      const Mat<2, 2> J = s2_jac(dx_ + 21);
      mul_rows<2>(L, 21, J, P_);
      for (int c = 0; c < 12; ++c) {
        const double a0 = J(0, 0) * K_x_(21, c) + J(0, 1) * K_x_(22, c), a1 = J(1, 0) * K_x_(21, c) + J(1, 1) * K_x_(22, c);
        K_x_(21, c) = a0; K_x_(22, c) = a1;
      }
      mul_cols_T<2>(L, 21, J);
      mul_cols_T<2>(P_, 21, J);
      Cov Pn;
      for (int i = 0; i < DOF; ++i)
        for (int j = 0; j < DOF; ++j) { double s = 0; for (int k = 0; k < 12; ++k) s += K_x_(i, k) * P_(k, j); Pn(i, j) = L(i, j) - s; }
      P_ = Pn;
      finished_ = true;
    }
    ++it_;
  }

  State x_, x_prop_;
  Cov P_prop_, P_, K_x_;
  double K_h_[DOF], dx_new_[DOF] = {0}, limit_[DOF];
  double R_;
  int max_iter_, it_ = -1, t_ = 0;
  bool converge_ = true, finished_ = false, touched_ = false;
};

}  // namespace host
}  // namespace flb

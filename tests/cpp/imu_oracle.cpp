// imu_oracle.cpp — sequential CPU restatement of ImuProcess::Process up to the forward propagation, for the tests of
// flb_imu_process (libfastlio_b200.so).  Written from the formulas, dense and in double:
//   IMU_init                     src/IMU_Processing.hpp:174-233, MAX_INI_COUNT logic of Process :393-427, Reset :90-102
//   forward loop of UndistortPcl :241-331 (midpoint inputs, acc * G_m_s2 / |mean_acc|, the dt rules, angvel_last /
//                                acc_s_last, IMUpose, the final predict to the lidar end time)
//   esekf::predict               esekfom.hpp:280-384 with get_f / df_dx / df_dw (use-ikfom.hpp:56-97) and the MTK
//                                manifolds: SO3 exp (SOn.hpp:284-288, mtkmath.hpp:249-256), A_matrix (mtkmath.hpp:235-247),
//                                S2<98090, 10000, 1> (S2.hpp: constructor, oplus, Bx, Nx_yy, Mx)
// Every matrix product is dense and sums over k in ascending order from 0.  The backward pass (undistortion) is the
// front-end oracle's (oracle/frontend_oracle.cpp).  Compiled by tests/imu_oracle.py with g++ -O2 -ffp-contract=off.
#include <cmath>
#include <cstring>
#include <initializer_list>

namespace {

constexpr int N = 23;          // state DOF
constexpr int DIM = 24;        // flattened state dimension (S2 has 3)
constexpr int W = 12;          // process noise DOF
constexpr double G_m_s2 = 9.81;
constexpr double S2_LEN = double(98090) / double(10000);
constexpr double TOL = 1e-11;  // MTK::tolerance<double>()
constexpr int MAX_INI_COUNT = 10;

// state26: pos[0:3] rot[3:7] (x,y,z,w) offR[7:11] offT[11:14] vel[14:17] bg[17:20] ba[20:23] grav[23:26]
void matmul(const double* A, const double* B, double* C, int n, int k, int m) {
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < m; ++j) {
      double s = 0.0;
      for (int t = 0; t < k; ++t) s += A[i * k + t] * B[t * m + j];
      C[i * m + j] = s;
    }
}
void hat(const double* v, double* H) {
  H[0] = 0; H[1] = -v[2]; H[2] = v[1]; H[3] = v[2]; H[4] = 0; H[5] = -v[0]; H[6] = -v[1]; H[7] = v[0]; H[8] = 0;
}
void cos_sinc_sqrt(double x2, double& c, double& s) {
  if (x2 >= 1.220703125e-4) { const double x = std::sqrt(x2); c = std::cos(x); s = std::sin(x) / x; return; }
  const double inv[7] = {1 / 3., 1 / 4., 1 / 5., 1 / 6., 1 / 7., 1 / 8., 1 / 9.};
  double cosi = 1., sinc = 1., term = -1 / 2. * x2;
  for (int i = 0; i < 3; ++i) { cosi += term; term *= inv[2 * i]; sinc += term; term *= -inv[2 * i + 1] * x2; }
  c = cosi; s = sinc;
}
// MTK::exp(result, vec, scale): quaternion (x,y,z,w)
void qexp(const double* v, double scale, double* q) {
  const double n2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  double c, s;
  cos_sinc_sqrt(scale * scale * n2, c, s);
  const double m = s * scale;
  q[0] = m * v[0]; q[1] = m * v[1]; q[2] = m * v[2]; q[3] = c;
}
void qmul(const double* a, const double* b, double* r) {
  const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  const double y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  const double z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  r[0] = x; r[1] = y; r[2] = z; r[3] = w;
}
void qmat(const double* q, double* R) {   // toRotationMatrix
  const double tx = 2 * q[0], ty = 2 * q[1], tz = 2 * q[2];
  const double twx = tx * q[3], twy = ty * q[3], twz = tz * q[3], txx = tx * q[0], txy = ty * q[0], txz = tz * q[0];
  const double tyy = ty * q[1], tyz = tz * q[1], tzz = tz * q[2];
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
void qrot(const double* q, const double* v, double* o) {   // q * v: uv = q.vec x v; uv += uv; v + w uv + q.vec x uv
  double u[3] = {q[1] * v[2] - q[2] * v[1], q[2] * v[0] - q[0] * v[2], q[0] * v[1] - q[1] * v[0]};
  for (double& t : u) t += t;
  const double c[3] = {q[1] * u[2] - q[2] * u[1], q[2] * u[0] - q[0] * u[2], q[0] * u[1] - q[1] * u[0]};
  for (int i = 0; i < 3; ++i) o[i] = (v[i] + q[3] * u[i]) + c[i];
}
void A_matrix(const double* v, double* A) {
  const double sq = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  const double n = std::sqrt(sq);
  for (int i = 0; i < 9; ++i) A[i] = (i % 4 == 0) ? 1.0 : 0.0;
  if (n < TOL) return;
  double H[9], HH[9];
  hat(v, H);
  matmul(H, H, HH, 3, 3, 3);
  const double a = (1 - std::cos(n)) / sq, b = (1 - std::sin(n) / n) / sq;
  for (int i = 0; i < 9; ++i) A[i] = (A[i] + a * H[i]) + b * HH[i];
}
void s2_Bx(const double* v, double* B) {   // S2_typ 1, 3x2
  const double L = S2_LEN;
  if (v[0] + L > TOL) {
    B[0] = -v[1]; B[1] = -v[2];
    B[2] = L - v[1] * v[1] / (L + v[0]); B[3] = -v[2] * v[1] / (L + v[0]);
    B[4] = -v[2] * v[1] / (L + v[0]); B[5] = L - v[2] * v[2] / (L + v[0]);
    for (int i = 0; i < 6; ++i) B[i] /= L;
  } else {
    for (int i = 0; i < 6; ++i) B[i] = 0;
    B[3] = -1; B[4] = 1;
  }
}
void s2_Nx_yy(const double* v, double* Nx) {   // 1/len/len * Bx^T * hat(v), 2x3
  double B[6], BT[6], H[9];
  s2_Bx(v, B);
  const double sc = 1 / S2_LEN / S2_LEN;
  for (int i = 0; i < 2; ++i) for (int k = 0; k < 3; ++k) BT[i * 3 + k] = sc * B[k * 2 + i];
  hat(v, H);
  matmul(BT, H, Nx, 2, 3, 3);
}
void s2_Mx0(const double* v, double* Mx) {   // S2_Mx with delta = 0: -hat(v) * Bx, 3x2
  double B[6], H[9];
  s2_Bx(v, B);
  hat(v, H);
  for (double& h : H) h = -h;
  matmul(H, B, Mx, 3, 3, 2);
}

// esekf::predict(dt, Q, in): x (state26), P (23x23), Q (12x12 dense)
void predict(double* x, double* P, const double* Qm, const double* in_acc, const double* in_gyr, double dt) {
  // f, df_dx, df_dw at x_ (use-ikfom.hpp:56-97)
  double f[DIM] = {0}, fx[DIM * N] = {0}, fw[DIM * W] = {0};
  double R[9], omega[3], acc_[3], ai[3];
  qmat(x + 3, R);
  for (int i = 0; i < 3; ++i) { omega[i] = in_gyr[i] - x[17 + i]; acc_[i] = in_acc[i] - x[20 + i]; }
  qrot(x + 3, acc_, ai);
  for (int i = 0; i < 3; ++i) { f[i] = x[14 + i]; f[3 + i] = omega[i]; f[12 + i] = ai[i] + x[23 + i]; }
  double mR[9], H[9], mRH[9], Mx[6];
  for (int i = 0; i < 9; ++i) mR[i] = -R[i];
  hat(acc_, H);
  matmul(mR, H, mRH, 3, 3, 3);
  s2_Mx0(x + 23, Mx);
  for (int i = 0; i < 3; ++i) {
    fx[i * N + 12 + i] = 1.0;
    for (int j = 0; j < 3; ++j) {
      fx[(12 + i) * N + 3 + j] = mRH[3 * i + j];
      fx[(12 + i) * N + 18 + j] = mR[3 * i + j];
      fw[(12 + i) * W + 3 + j] = mR[3 * i + j];
    }
    for (int j = 0; j < 2; ++j) fx[(12 + i) * N + 21 + j] = Mx[2 * i + j];
    fx[(3 + i) * N + 15 + i] = -1.0;
    fw[(3 + i) * W + i] = -1.0;
    fw[(15 + i) * W + 6 + i] = 1.0;
    fw[(18 + i) * W + 9 + i] = 1.0;
  }
  double xb[26];
  std::memcpy(xb, x, sizeof(xb));
  // x_.oplus(f_, dt)
  for (int i = 0; i < 3; ++i) {
    x[i] += dt * f[i]; x[11 + i] += dt * f[9 + i]; x[14 + i] += dt * f[12 + i]; x[17 + i] += dt * f[15 + i]; x[20 + i] += dt * f[18 + i];
  }
  for (int s = 0; s < 2; ++s) {   // rot (f 3..5), offset_R_L_I (f 6..8): x * exp(f, dt)
    double q[4], r[4];
    qexp(f + 3 + 3 * s, dt / 2, q);
    qmul(x + 3 + 4 * s, q, r);
    std::memcpy(x + 3 + 4 * s, r, sizeof(r));
  }
  {   // grav: vec = exp(f 21..23, dt).toRotationMatrix() * vec
    double q[4], Rg[9], g[3];
    qexp(f + 21, dt / 2, q);
    qmat(q, Rg);
    matmul(Rg, x + 23, g, 3, 3, 1);
    std::memcpy(x + 23, g, sizeof(g));
  }
  // F_x1, f_x_final, f_w_final
  double F1[N * N] = {0}, fxf[N * N] = {0}, fwf[N * W] = {0};
  for (int i = 0; i < N; ++i) F1[i * N + i] = 1.0;
  const int vect_idx[5] = {0, 9, 12, 15, 18};
  for (int v : vect_idx)
    for (int j = 0; j < 3; ++j) {
      for (int i = 0; i < N; ++i) fxf[(v + j) * N + i] = fx[(v + j) * N + i];
      for (int i = 0; i < W; ++i) fwf[(v + j) * W + i] = fw[(v + j) * W + i];
    }
  for (int idx : {3, 6}) {   // SO3 states: idx == dim
    double seg[3], q[4], Rs[9], A[9];
    for (int i = 0; i < 3; ++i) seg[i] = -1 * f[idx + i] * dt;
    qexp(seg, 0.0 / 2 /* scalar_type(1/2) == 0 */, q);
    qmat(q, Rs);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) F1[(idx + i) * N + idx + j] = Rs[3 * i + j];
    A_matrix(seg, A);
    for (int c = 0; c < N; ++c) {
      const double col[3] = {fx[idx * N + c], fx[(idx + 1) * N + c], fx[(idx + 2) * N + c]};
      double o[3];
      matmul(A, col, o, 3, 3, 1);
      for (int i = 0; i < 3; ++i) fxf[(idx + i) * N + c] = o[i];
    }
    for (int c = 0; c < W; ++c) {
      const double col[3] = {fw[idx * W + c], fw[(idx + 1) * W + c], fw[(idx + 2) * W + c]};
      double o[3];
      matmul(A, col, o, 3, 3, 1);
      for (int i = 0; i < 3; ++i) fwf[(idx + i) * W + c] = o[i];
    }
  }
  {   // S2 state grav: idx 21, dim 21
    double seg[3], q[4], Rs[9], Nx[6], Mxb[6], NR[6], blk[4], xh[9], At[9], A[9], T1[6], T2[6], rts[6];
    for (int i = 0; i < 3; ++i) seg[i] = f[21 + i] * dt;
    qexp(seg, 0.0 / 2, q);
    qmat(q, Rs);
    s2_Nx_yy(x + 23, Nx);
    s2_Mx0(xb + 23, Mxb);
    matmul(Nx, Rs, NR, 2, 3, 3);
    matmul(NR, Mxb, blk, 2, 3, 2);
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 2; ++j) F1[(21 + i) * N + 21 + j] = blk[2 * i + j];
    hat(xb + 23, xh);
    A_matrix(seg, A);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) At[3 * i + j] = A[3 * j + i];
    double mNR[6];
    for (int i = 0; i < 6; ++i) mNR[i] = -NR[i];
    matmul(mNR, xh, T1, 2, 3, 3);
    matmul(T1, At, T2, 2, 3, 3);
    std::memcpy(rts, T2, sizeof(rts));
    for (int c = 0; c < N; ++c) {
      const double col[3] = {fx[21 * N + c], fx[22 * N + c], fx[23 * N + c]};
      double o[2];
      matmul(rts, col, o, 2, 3, 1);
      fxf[21 * N + c] = o[0]; fxf[22 * N + c] = o[1];
    }
    for (int c = 0; c < W; ++c) {
      const double col[3] = {fw[21 * W + c], fw[22 * W + c], fw[23 * W + c]};
      double o[2];
      matmul(rts, col, o, 2, 3, 1);
      fwf[21 * W + c] = o[0]; fwf[22 * W + c] = o[1];
    }
  }
  // P = F P F^T + (dt G) Q (dt G)^T
  static double F[N * N], Ft[N * N], T[N * N], FPFt[N * N], Gd[N * W], Gdt[W * N], GQ[N * W], GQG[N * N];
  for (int e = 0; e < N * N; ++e) F[e] = F1[e] + fxf[e] * dt;
  for (int i = 0; i < N; ++i) for (int j = 0; j < N; ++j) Ft[j * N + i] = F[i * N + j];
  matmul(F, P, T, N, N, N);
  matmul(T, Ft, FPFt, N, N, N);
  for (int e = 0; e < N * W; ++e) Gd[e] = dt * fwf[e];
  for (int i = 0; i < N; ++i) for (int j = 0; j < W; ++j) Gdt[j * N + i] = Gd[i * W + j];
  matmul(Gd, Qm, GQ, N, W, W);
  matmul(GQ, Gdt, GQG, N, W, N);
  for (int e = 0; e < N * N; ++e) P[e] = FPFt[e] + GQG[e];
}

// Persistent members of ImuProcess, flat (double slots):
enum {
  S_T = 0, S_R = 3, S_GYR_SCALE = 12, S_ACC_SCALE = 15, S_BIAS_GYR = 18, S_BIAS_ACC = 21,   // configuration
  S_MEAN_ACC = 24, S_MEAN_GYR = 27, S_COV_ACC = 30, S_COV_GYR = 33, S_QD = 36, S_ANGVEL = 48, S_ACC_S = 51, S_LAST_IMU = 54,
  S_LAST_END = 61, S_INIT_ITER = 62, S_NEED_INIT = 63, S_FIRST = 64, S_NPOSES = 65, S_SIZE = 66
};

void reset(double* s) {
  s[S_MEAN_ACC] = 0; s[S_MEAN_ACC + 1] = 0; s[S_MEAN_ACC + 2] = -1.0;
  for (int i = 0; i < 3; ++i) { s[S_MEAN_GYR + i] = 0; s[S_ANGVEL + i] = 0; }
  s[S_NEED_INIT] = 1;
  s[S_INIT_ITER] = 1;
  for (int k = 0; k < 7; ++k) s[S_LAST_IMU + k] = 0;
  s[S_NPOSES] = 0;
}

void quat_from_matrix(const double* m, double* q) {
  const double t = m[0] + m[4] + m[8];
  if (t > 0) {
    double r = std::sqrt(t + 1.0);
    q[3] = 0.5 * r;
    r = 0.5 / r;
    q[0] = (m[7] - m[5]) * r; q[1] = (m[2] - m[6]) * r; q[2] = (m[3] - m[1]) * r;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[3 * i + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double r = std::sqrt(m[3 * i + i] - m[3 * j + j] - m[3 * k + k] + 1.0);
    q[i] = 0.5 * r;
    r = 0.5 / r;
    q[3] = (m[3 * k + j] - m[3 * j + k]) * r;
    q[j] = (m[3 * j + i] + m[3 * i + j]) * r;
    q[k] = (m[3 * k + i] + m[3 * i + k]) * r;
  }
}

double norm3(const double* v) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

}  // namespace

extern "C" {

int orc_imu_state_size() { return S_SIZE; }

// ImuProcess() + the setters laserMapping.cpp calls (:2142-2146); cfg = T[3], R[9] row-major, gyr, acc, bias_gyr, bias_acc
void orc_imu_new(const double* cfg, double* s) {
  std::memset(s, 0, sizeof(double) * S_SIZE);
  std::memcpy(s, cfg, sizeof(double) * 24);
  for (int i = 0; i < 3; ++i) { s[S_COV_ACC + i] = 0.1; s[S_COV_GYR + i] = 0.1; }
  for (int i = 0; i < 12; ++i) s[S_QD + i] = i < 6 ? 0.0001 : 0.00001;   // process_noise_cov()
  reset(s);
  s[S_FIRST] = 1;
}

void orc_imu_reset(double* s) { reset(s); }

void orc_imu_predict(double* x, double* P, const double* Qdiag, const double* in_acc, const double* in_gyr, double dt) {
  double Qm[W * W] = {0};
  for (int i = 0; i < W; ++i) Qm[i * W + i] = Qdiag[i];
  predict(x, P, Qm, in_acc, in_gyr, dt);
}

// Process(meas, kf, ...) up to the forward propagation.  Returns the status (0 empty, 1 initialising, 2 propagated);
// poses (>= 256 x 22) receives IMUpose, s[S_NPOSES] its size.
int orc_imu_process(double* s, const double* imu7, int n, double pcl_beg, double pcl_end, double* x, double* P, double* poses) {
  if (n == 0) return 0;
  if (s[S_NEED_INIT] != 0) {
    int Ni = (int)s[S_INIT_ITER];
    if (s[S_FIRST] != 0) {
      reset(s);
      Ni = 1;
      s[S_FIRST] = 0;
      for (int i = 0; i < 3; ++i) { s[S_MEAN_ACC + i] = imu7[1 + i]; s[S_MEAN_GYR + i] = imu7[4 + i]; }
    }
    for (int k = 0; k < n; ++k) {
      const double* r = imu7 + 7 * k;
      double* ma = s + S_MEAN_ACC; double* mg = s + S_MEAN_GYR; double* ca = s + S_COV_ACC; double* cg = s + S_COV_GYR;
      for (int i = 0; i < 3; ++i) {
        ma[i] += (r[1 + i] - ma[i]) / Ni;
        mg[i] += (r[4 + i] - mg[i]) / Ni;
      }
      for (int i = 0; i < 3; ++i) {
        const double da = r[1 + i] - ma[i], dg = r[4 + i] - mg[i];
        ca[i] = ca[i] * (Ni - 1.0) / Ni + da * da * (Ni - 1.0) / (Ni * Ni);
        cg[i] = cg[i] * (Ni - 1.0) / Ni + dg * dg * (Ni - 1.0) / (Ni * Ni);
      }
      Ni++;
    }
    const double na = norm3(s + S_MEAN_ACC);
    double g[3];
    for (int i = 0; i < 3; ++i) g[i] = -s[S_MEAN_ACC + i] / na * G_m_s2;
    const double ng = norm3(g);
    for (int i = 0; i < 3; ++i) x[23 + i] = g[i] / ng * S2_LEN;
    for (int i = 0; i < 3; ++i) { x[17 + i] = s[S_MEAN_GYR + i]; x[11 + i] = s[S_T + i]; }
    quat_from_matrix(s + S_R, x + 7);
    for (int e = 0; e < N * N; ++e) P[e] = 0;
    for (int i = 0; i < N; ++i) P[i * N + i] = 1.0;
    P[6 * N + 6] = P[7 * N + 7] = P[8 * N + 8] = 0.00001;
    P[9 * N + 9] = P[10 * N + 10] = P[11 * N + 11] = 0.00001;
    P[15 * N + 15] = P[16 * N + 16] = P[17 * N + 17] = 0.0001;
    P[18 * N + 18] = P[19 * N + 19] = P[20 * N + 20] = 0.001;
    P[21 * N + 21] = P[22 * N + 22] = 0.00001;
    s[S_INIT_ITER] = Ni;
    std::memcpy(s + S_LAST_IMU, imu7 + 7 * (n - 1), sizeof(double) * 7);
    if (Ni > MAX_INI_COUNT) {
      double* ca = s + S_COV_ACC;
      const double sc = std::pow(G_m_s2 / na, 2);
      for (int i = 0; i < 3; ++i) ca[i] *= sc;   // dead: overwritten on the next line
      s[S_NEED_INIT] = 0;
      for (int i = 0; i < 3; ++i) { s[S_COV_ACC + i] = s[S_ACC_SCALE + i]; s[S_COV_GYR + i] = s[S_GYR_SCALE + i]; }
    }
    return 1;
  }
  // UndistortPcl forward loop over v_imu = [last_imu_] + meas.imu
  const int ns = n + 1;
  auto smp = [&](int k) -> const double* { return k == 0 ? s + S_LAST_IMU : imu7 + 7 * (k - 1); };
  const double L = s[S_LAST_END];
  double Qm[W * W] = {0};
  for (int i = 0; i < W; ++i) Qm[i * W + i] = s[S_QD + i];
  int np = 0;
  auto pose = [&](double t, const double* acc, const double* gyr) {
    double* o = poses + 22 * np++;
    o[0] = t;
    for (int i = 0; i < 3; ++i) { o[1 + i] = acc[i]; o[4 + i] = gyr[i]; o[7 + i] = x[14 + i]; o[10 + i] = x[i]; }
    qmat(x + 3, o + 13);
  };
  pose(0.0, s + S_ACC_S, s + S_ANGVEL);
  double in_acc[3] = {0, 0, 0}, in_gyr[3] = {0, 0, 0};
  const double na = norm3(s + S_MEAN_ACC);
  for (int k = 0; k + 1 < ns; ++k) {
    const double* head = smp(k);
    const double* tail = smp(k + 1);
    if (tail[0] < L) continue;
    double ga[3], aa[3];
    for (int i = 0; i < 3; ++i) { ga[i] = 0.5 * (head[4 + i] + tail[4 + i]); aa[i] = 0.5 * (head[1 + i] + tail[1 + i]); }
    for (int i = 0; i < 3; ++i) aa[i] = aa[i] * G_m_s2 / na;
    const double dt = head[0] < L ? tail[0] - L : tail[0] - head[0];
    for (int i = 0; i < 3; ++i) { in_acc[i] = aa[i]; in_gyr[i] = ga[i]; }
    for (int i = 0; i < 3; ++i) {
      Qm[i * W + i] = s[S_COV_GYR + i];
      Qm[(3 + i) * W + 3 + i] = s[S_COV_ACC + i];
      Qm[(6 + i) * W + 6 + i] = s[S_BIAS_GYR + i];
      Qm[(9 + i) * W + 9 + i] = s[S_BIAS_ACC + i];
    }
    predict(x, P, Qm, in_acc, in_gyr, dt);
    double d[3], a[3];
    for (int i = 0; i < 3; ++i) { s[S_ANGVEL + i] = ga[i] - x[17 + i]; d[i] = aa[i] - x[20 + i]; }
    qrot(x + 3, d, a);
    for (int i = 0; i < 3; ++i) s[S_ACC_S + i] = a[i];
    for (int i = 0; i < 3; ++i) s[S_ACC_S + i] += x[23 + i];
    pose(tail[0] - pcl_beg, s + S_ACC_S, s + S_ANGVEL);
  }
  const double imu_end = smp(ns - 1)[0];
  const double note = pcl_end > imu_end ? 1.0 : -1.0;
  const double dt = note * (pcl_end - imu_end);
  predict(x, P, Qm, in_acc, in_gyr, dt);
  for (int i = 0; i < W; ++i) s[S_QD + i] = Qm[i * W + i];
  std::memcpy(s + S_LAST_IMU, imu7 + 7 * (n - 1), sizeof(double) * 7);
  s[S_LAST_END] = pcl_end;
  s[S_NPOSES] = np;
  return 2;
}

}  // extern "C"

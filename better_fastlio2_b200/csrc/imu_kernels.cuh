// imu_kernels.cuh — the forward propagation of ImuProcess::UndistortPcl (src/IMU_Processing.hpp:241-331) on the device:
// one CTA, double precision, the serial chain of kf.predict (esekfom.hpp:280-384 with get_f / df_dx / df_dw,
// use-ikfom.hpp:56-97) over the span v_imu = [last_imu_] + meas.imu, the Pose6D records (IMUpose) written straight into
// the front end's pose buffer, and the final predict to the lidar end time.  k_undistort then reads its end pose and the
// pose count from the ImuRecord this kernel writes, so nothing passes through the host between the two.
//
// Covariance step P = F P F^T + (dt G) Q (dt G)^T with the structure of this system (scalar_type(1/2) == 0 in predict,
// so the SO3 blocks of F_x1 are the identity and the S2 block is Nx * I * Mx):
//   F rows 0-2   pos:  e_r + dt e_{12+r}
//   F rows 3-5   rot:  e_r - dt A(seg)[r-3][*] on columns 15-17                      (seg = -omega dt)
//   F rows 12-14 vel:  -dt R hat(acc - ba) on 3-5, e_r, -dt R on 18-20, dt Mx on 21-22
//   F rows 21-22 grav: Nx Mx on 21-22
//   every other row is e_r; dt G has -A on rows 3-5 x cols 0-2, -R on 12-14 x 3-5, I on 15-17 x 6-8 and 18-20 x 9-11.
// Each product sums only the non-zero terms, in ascending k: adding an exact zero does not change a sum, so this is
// the dense product in that order bit for bit (tests/cpp/imu_oracle.cpp is the dense restatement).
#pragma once
#include "esikf_device.cuh"

namespace flb {

constexpr int IMU_SAMPLE_DOUBLES = 7;   // stamp, acc x y z, gyro x y z
constexpr int IMU_THREADS = 256;
constexpr double IMU_G_M_S2 = 9.81;     // G_m_s2, common_lib.h:143

struct ImuParams {
  int n_samples;              // v_imu.size() = meas.imu.size() + 1 (last_imu_ first)
  double acc_norm;            // mean_acc.norm()
  double q_init[12];          // diagonal of ImuProcess::Q on entry (process_noise_cov() until a segment overwrote it)
  double q_cov[12];           // cov_gyr, cov_acc, cov_bias_gyr, cov_bias_acc: Q's diagonal blocks once a segment ran
  double last_lidar_end_time; // last_lidar_end_time_
  double pcl_beg, pcl_end;    // meas.lidar_beg_time, meas.lidar_end_time
  double angvel_last[3], acc_s_last[3];
};

struct ImuRecord {            // the propagation's result, read back with the call's one synchronisation
  double x[26];               // kf.get_x() after the last predict (state26)
  double P[NDOF * NDOF];
  double angvel_last[3], acc_s_last[3];
  int n_poses, pad_;
};

namespace dev {

// columns of the non-zero entries of F's row r, ascending
__device__ __forceinline__ int f_row_cols(int r, int* c) {
  if (r < 3) { c[0] = r; c[1] = 12 + r; return 2; }
  if (r < 6) { c[0] = r; c[1] = 15; c[2] = 16; c[3] = 17; return 4; }
  if (r >= 12 && r < 15) { c[0] = 3; c[1] = 4; c[2] = 5; c[3] = r; c[4] = 18; c[5] = 19; c[6] = 20; c[7] = 21; c[8] = 22; return 9; }
  if (r >= 21) { c[0] = 21; c[1] = 22; return 2; }
  c[0] = r;
  return 1;
}
// the columns of dt G (a block of three) that row r of dt G uses; -1: the row is zero
__device__ __forceinline__ int g_row_block(int r) {
  if (r >= 3 && r < 6) return 0;
  if (r >= 12 && r < 15) return 3;
  if (r >= 15 && r < 21) return r < 18 ? 6 : 9;
  return -1;
}

}  // namespace dev

// x (state26) and P in shared memory; F (dense 23x23, rows outside the pattern unused) and dt G (23x12) are built per
// predict.  in_acc / in_gyr: the input_ikfom of this predict.
__device__ __noinline__ void imu_predict(double* x, double* P, double* T, double* F, double* Gd, const double* q,
                                         const double* in_acc, const double* in_gyr, double dt, int tid) {
  using namespace dev;
  __shared__ double A[9], R[9], Mx[6], Nx[6], fvel[3];
  // ---- per-state terms (x is x_before until the barrier)
  if (tid == 0) {                                          // SO3 rot: seg_SO3 = -1 * f * dt, A_matrix(seg)
    double seg[3], At[9];
    for (int i = 0; i < 3; ++i) seg[i] = -1 * (in_gyr[i] - x[17 + i]) * dt;
    A_matrix_T(seg, At);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) A[3 * i + j] = At[3 * j + i];
  } else if (tid == 32) {                                  // S2 grav: Mx(x_before, 0) and Nx_yy(x_after); oplus leaves grav
    const double z2[2] = {0.0, 0.0};                       // unchanged (f's grav rows are 0: exp(0) = identity rotation)
    s2_Mx(x + 23, z2, Mx);
    s2_Nx(x + 23, Nx);
  } else if (tid == 64) {                                  // vel rows: R = rot.toRotationMatrix(), a_inertial + grav
    rotmat(x + 3, R);
    double a0, a1, a2;
    qrot_d(x + 3, in_acc[0] - x[20], in_acc[1] - x[21], in_acc[2] - x[22], a0, a1, a2);
    fvel[0] = a0 + x[23]; fvel[1] = a1 + x[24]; fvel[2] = a2 + x[25];
  }
  __syncthreads();
  // ---- F's pattern rows and dt G
  for (int e = tid; e < NDOF * NDOF; e += IMU_THREADS) {
    const int r = e / NDOF, k = e - r * NDOF;
    double v = r == k ? 1.0 : 0.0;
    if (r < 3) { if (k == 12 + r) v = 0 + 1.0 * dt; }
    else if (r < 6) { if (k >= 15 && k < 18) v = 0 + (-A[3 * (r - 3) + (k - 15)]) * dt; }
    else if (r >= 12 && r < 15) {
      const int i = r - 12;
      if (k >= 3 && k < 6) {                               // (-R) hat(acc - ba)
        const double acc_[3] = {in_acc[0] - x[20], in_acc[1] - x[21], in_acc[2] - x[22]};
        double H[9];
        hat(acc_, H);
        double s = 0;
        for (int m = 0; m < 3; ++m) s += (-R[3 * i + m]) * H[3 * m + (k - 3)];
        v = 0 + s * dt;
      } else if (k >= 18 && k < 21) v = 0 + (-R[3 * i + (k - 18)]) * dt;
      else if (k >= 21) v = 0 + Mx[2 * i + (k - 21)] * dt;
    } else if (r >= 21 && k >= 21) {                       // Nx * I * Mx
      const int i = r - 21, j = k - 21;
      double s = 0;
      for (int m = 0; m < 3; ++m) s += Nx[3 * i + m] * Mx[2 * m + j];
      v = s;
    }
    F[e] = v;
  }
  for (int e = tid; e < NDOF * 12; e += IMU_THREADS) {
    const int r = e / 12, c = e - r * 12;
    double v = 0.0;
    if (r >= 3 && r < 6 && c < 3) v = dt * (-A[3 * (r - 3) + c]);
    else if (r >= 12 && r < 15 && c >= 3 && c < 6) v = dt * (-R[3 * (r - 12) + (c - 3)]);
    else if (r >= 15 && r < 18 && c == r - 9) v = dt * 1.0;
    else if (r >= 18 && r < 21 && c == r - 9) v = dt * 1.0;
    Gd[e] = v;
  }
  __syncthreads();
  // ---- x_.oplus(f_, dt): pos += dt vel, rot = rot * exp(omega, dt / 2), vel += dt (a_inertial + grav); offR / grav see a
  // zero f (identity rotation), offT / bg / ba a zero step
  if (tid == 0) {
    double om[3] = {in_gyr[0] - x[17], in_gyr[1] - x[18], in_gyr[2] - x[19]};
    so3_boxplus(x + 3, om, dt);
  } else if (tid == 32) {
    for (int i = 0; i < 3; ++i) { x[i] += dt * x[14 + i]; x[14 + i] += dt * fvel[i]; }
  }
  // ---- T = F P (sparse rows)
  int cols[9];
  for (int e = tid; e < NDOF * NDOF; e += IMU_THREADS) {
    const int i = e / NDOF, j = e - i * NDOF;
    const int nc = f_row_cols(i, cols);
    double s;
    if (nc == 1) s = P[e];
    else { s = 0; for (int u = 0; u < nc; ++u) s += F[i * NDOF + cols[u]] * P[cols[u] * NDOF + j]; }
    T[e] = s;
  }
  __syncthreads();
  // ---- P = T F^T + (dt G Q) (dt G)^T
  for (int e = tid; e < NDOF * NDOF; e += IMU_THREADS) {
    const int i = e / NDOF, j = e - i * NDOF;
    const int nc = f_row_cols(j, cols);
    double s;
    if (nc == 1) s = T[e];
    else { s = 0; for (int u = 0; u < nc; ++u) s += T[i * NDOF + cols[u]] * F[j * NDOF + cols[u]]; }
    const int bi = g_row_block(i), bj = g_row_block(j);
    double nz = 0;
    if (bi >= 0 && bi == bj)
      for (int c = bi; c < bi + 3; ++c) nz += (Gd[i * 12 + c] * q[c]) * Gd[j * 12 + c];
    P[e] = s + nz;
  }
  __syncthreads();
}

// One CTA of IMU_THREADS threads.  in = [state26 | P (529) | n_samples x 7] (staged in one upload); poses = the front end's
// Pose6D buffer (22 doubles per record); rec = the result.
__global__ void __launch_bounds__(IMU_THREADS) k_imu_propagate(ImuParams p, const double* __restrict__ in, double* __restrict__ poses,
                                                               ImuRecord* __restrict__ rec) {
  using namespace dev;
  __shared__ double x[26], P[NDOF * NDOF], T[NDOF * NDOF], F[NDOF * NDOF], Gd[NDOF * 12], q[12];
  __shared__ double in_acc[3], in_gyr[3], s_dt, avr_g[3], avr_a[3];
  __shared__ int s_np;
  extern __shared__ double smp[];   // n_samples x 7
  const int tid = threadIdx.x;
  for (int e = tid; e < 26 + NDOF * NDOF; e += IMU_THREADS) { if (e < 26) x[e] = in[e]; else P[e - 26] = in[e]; }
  for (int e = tid; e < p.n_samples * IMU_SAMPLE_DOUBLES; e += IMU_THREADS) smp[e] = in[26 + NDOF * NDOF + e];
  if (tid < 12) q[tid] = p.q_init[tid];
  if (tid < 3) { in_acc[tid] = 0.0; in_gyr[tid] = 0.0; }   // input_ikfom in: zero until a segment assigns it (vect.hpp:108)
  if (tid == 0) s_np = 1;
  __syncthreads();
  // IMUpose[0] = set_pose6d(0.0, acc_s_last, angvel_last, vel, pos, rot) of the previous posterior (:258)
  if (tid == 0) {
    double* o = poses;
    o[0] = 0.0;
    for (int i = 0; i < 3; ++i) { o[1 + i] = p.acc_s_last[i]; o[4 + i] = p.angvel_last[i]; o[7 + i] = x[14 + i]; o[10 + i] = x[i]; }
    rotmat(x + 3, o + 13);
  }
  double angvel_last[3] = {p.angvel_last[0], p.angvel_last[1], p.angvel_last[2]};
  double acc_s_last[3] = {p.acc_s_last[0], p.acc_s_last[1], p.acc_s_last[2]};
  const double L = p.last_lidar_end_time;
  for (int s = 0; s + 1 < p.n_samples; ++s) {
    const double* head = smp + s * IMU_SAMPLE_DOUBLES;
    const double* tail = head + IMU_SAMPLE_DOUBLES;
    if (tail[0] < L) continue;                             // uniform: every thread reads the same stamps (:275-276)
    if (tid == 0) {
      for (int i = 0; i < 3; ++i) {
        avr_g[i] = 0.5 * (head[4 + i] + tail[4 + i]);
        avr_a[i] = 0.5 * (head[1 + i] + tail[1 + i]);
        avr_a[i] = avr_a[i] * IMU_G_M_S2 / p.acc_norm;     // acc_avr * G_m_s2 / mean_acc.norm()
        in_acc[i] = avr_a[i];
        in_gyr[i] = avr_g[i];
      }
      s_dt = head[0] < L ? tail[0] - L : tail[0] - head[0];
    }
    if (tid < 12) q[tid] = p.q_cov[tid];                   // Q.block(...).diagonal() = cov_* (:303-306)
    __syncthreads();
    imu_predict(x, P, T, F, Gd, q, in_acc, in_gyr, s_dt, tid);
    if (tid == 0) {                                        // :311-321
      for (int i = 0; i < 3; ++i) angvel_last[i] = avr_g[i] - x[17 + i];
      double a0, a1, a2;
      qrot_d(x + 3, avr_a[0] - x[20], avr_a[1] - x[21], avr_a[2] - x[22], a0, a1, a2);
      acc_s_last[0] = a0; acc_s_last[1] = a1; acc_s_last[2] = a2;
      for (int i = 0; i < 3; ++i) acc_s_last[i] += x[23 + i];
      double* o = poses + (size_t)s_np * IMU_POSE_DOUBLES;
      o[0] = tail[0] - p.pcl_beg;
      for (int i = 0; i < 3; ++i) { o[1 + i] = acc_s_last[i]; o[4 + i] = angvel_last[i]; o[7 + i] = x[14 + i]; o[10 + i] = x[i]; }
      rotmat(x + 3, o + 13);
      s_np++;
    }
  }
  // the final predict to the later of the scan end and the last IMU stamp, with the last `in` (:325-327)
  const double imu_end = smp[(p.n_samples - 1) * IMU_SAMPLE_DOUBLES];
  const double note = p.pcl_end > imu_end ? 1.0 : -1.0;
  const double dt = note * (p.pcl_end - imu_end);
  __syncthreads();
  imu_predict(x, P, T, F, Gd, q, in_acc, in_gyr, dt, tid);
  for (int e = tid; e < NDOF * NDOF; e += IMU_THREADS) rec->P[e] = P[e];
  if (tid < 26) rec->x[tid] = x[tid];
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) { rec->angvel_last[i] = angvel_last[i]; rec->acc_s_last[i] = acc_s_last[i]; }
    rec->n_poses = s_np;
    rec->pad_ = 0;
  }
}

}  // namespace flb

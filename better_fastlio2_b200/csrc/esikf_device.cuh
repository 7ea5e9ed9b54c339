// esikf_device.cuh — the iterated error-state Kalman update (esekfom.hpp:1620-1938) kept RESIDENT ON THE DEVICE so a
// whole scan (<= max_iter+1 measurement passes + map insert) runs as one launch sequence without host round trips.
// One thread block per step: all threads reduce the per-block normal-equation partials in a fixed order, then warp 0
// does the 23-DOF algebra co-operatively on shared-memory matrices (two 23x23 Gauss-Jordan inverses with partial
// pivoting, the SO3 / S2 projections of esekfom.hpp:1663-1703, boxplus, convergence bookkeeping :1824-1838 and the
// final covariance :1841-1931).  Same mathematics as csrc/esikf_host.hpp (which remains the host-driven path and the
// fallback for the under-determined M < 23 branch, esekfom.hpp:1720-1750).
#pragma once
#include "meas_kernels.cuh"

namespace flb {

namespace dev {

constexpr int ESIKF_THREADS = 256;

__device__ __forceinline__ void qmul(const double* a, const double* b, double* r) {  // (x,y,z,w)
  const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  const double y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  const double z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  r[0] = x; r[1] = y; r[2] = z; r[3] = w;
}
__device__ __forceinline__ void rotmat(const double* q, double* R) {
  const double tx = 2 * q[0], ty = 2 * q[1], tz = 2 * q[2];
  const double twx = tx * q[3], twy = ty * q[3], twz = tz * q[3], txx = tx * q[0], txy = ty * q[0], txz = tz * q[0];
  const double tyy = ty * q[1], tyz = tz * q[1], tzz = tz * q[2];
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
__device__ __forceinline__ void hat(const double* v, double* H) {
  H[0] = 0; H[1] = -v[2]; H[2] = v[1]; H[3] = v[2]; H[4] = 0; H[5] = -v[0]; H[6] = -v[1]; H[7] = v[0]; H[8] = 0;
}
__device__ __forceinline__ void mm3(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += A[3 * i + k] * B[3 * k + j]; C[3 * i + j] = s; }
}
__device__ __forceinline__ void cos_sinc_sqrt(double x2, double& c, double& s) {  // mtkmath.hpp:142-174
  const double bound = 1.220703125e-4;  // sqrt(sqrt(eps))
  if (x2 >= bound) { const double x = sqrt(x2); double sn; sincos(x, &sn, &c); s = sn / x; return; }
  const double inv[7] = {1 / 3., 1 / 4., 1 / 5., 1 / 6., 1 / 7., 1 / 8., 1 / 9.};
  double cosi = 1., sinc = 1., term = -1 / 2. * x2;
  for (int i = 0; i < 3; ++i) { cosi += term; term *= inv[2 * i]; sinc += term; term *= -inv[2 * i + 1] * x2; }
  c = cosi; s = sinc;
}
__device__ __forceinline__ void exp_quat(const double* v, double scale, double* q) {  // mtkmath.hpp:249-256
  const double n2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  double c, s;
  cos_sinc_sqrt(scale * scale * n2, c, s);
  const double m = s * scale;
  q[0] = m * v[0]; q[1] = m * v[1]; q[2] = m * v[2]; q[3] = c;
}
__device__ __forceinline__ void log_quat(const double* q, double* r) {  // SOn.hpp:293-297
  double nv = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  if (nv < 1e-11) nv = 1e-11;
  const double s = 2.0 / nv * atan(nv / q[3]);
  r[0] = s * q[0]; r[1] = s * q[1]; r[2] = s * q[2];
}
__device__ __noinline__ void A_matrix_T(const double* v, double* J) {  // A_matrix(v)^T, mtkmath.hpp:235-247
  const double sq = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  const double n = sqrt(sq);
  double A[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (n >= 1e-11) {
    double H[9], HH[9];
    hat(v, H);
    mm3(H, H, HH);
    double sn, cn;
    sincos(n, &sn, &cn);
    const double a = (1 - cn) / sq, b = (1 - sn / n) / sq;
    for (int i = 0; i < 9; ++i) A[i] = A[i] + a * H[i] + b * HH[i];
  }
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) J[3 * i + j] = A[3 * j + i];
}
__device__ __forceinline__ void s2_Bx(const double* vec, double* Bx) {  // S2.hpp:215-231, 3x2 row-major
  const double len = 98090.0 / 10000.0;
  if (vec[0] + len > 1e-11) {
    Bx[0] = -vec[1]; Bx[1] = -vec[2];
    Bx[2] = len - vec[1] * vec[1] / (len + vec[0]); Bx[3] = -vec[2] * vec[1] / (len + vec[0]);
    Bx[4] = -vec[2] * vec[1] / (len + vec[0]); Bx[5] = len - vec[2] * vec[2] / (len + vec[0]);
    for (int i = 0; i < 6; ++i) Bx[i] /= len;
  } else {
    for (int i = 0; i < 6; ++i) Bx[i] = 0;
    Bx[3] = -1; Bx[4] = 1;
  }
}
// Nx_yy(xg) (2x3, S2.hpp:259-264) and Mx(xpg, delta) (3x2, S2.hpp:266-280) separately, so two warps can build them
__device__ __noinline__ void s2_Nx(const double* xg, double* Nx) {
  const double len = 98090.0 / 10000.0;
  double Bx[6], H[9];
  s2_Bx(xg, Bx);
  hat(xg, H);
  const double sc = 1 / len / len;
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += (sc * Bx[2 * k + i]) * H[3 * k + j]; Nx[3 * i + j] = s; }
}
__device__ __noinline__ void s2_Mx(const double* xpg, const double* delta, double* Mx) {
  double Bp[6], Hp[9];
  s2_Bx(xpg, Bp);
  hat(xpg, Hp);
  const double dn = sqrt(delta[0] * delta[0] + delta[1] * delta[1]);
  if (dn < 1e-11) {
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 2; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += (-Hp[3 * i + k]) * Bp[2 * k + j]; Mx[2 * i + j] = s; }
  } else {
    double Bu[3];
    for (int i = 0; i < 3; ++i) Bu[i] = Bp[2 * i] * delta[0] + Bp[2 * i + 1] * delta[1];
    double q[4], E[9], At[9], T1[9], T2[9];
    exp_quat(Bu, 0.0, q);  // scalar(1/2) == 0 in the reference (S2.hpp:277)
    rotmat(q, E);
    A_matrix_T(Bu, At);
    for (int i = 0; i < 9; ++i) E[i] = -E[i];
    mm3(E, Hp, T1);
    mm3(T1, At, T2);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 2; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += T2[3 * i + k] * Bp[2 * k + j]; Mx[2 * i + j] = s; }
  }
}
// Gauss-Jordan inverse of a symmetric positive definite N x N matrix in shared memory, block-wide and COMPACT (a
// rolled N-sweep loop: this kernel runs once per launch, so straight-line unrolled code would be instruction-fetch
// bound).  No pivoting is needed for SPD input.  Ping-pong between buf0 and buf1 (one barrier per sweep); returns the
// buffer holding the result (buf1 for odd N, buf0 for even N).
template <int N>
__device__ __noinline__ double* b_inverse_spd(double* buf0, double* buf1, int tid) {
  static_assert(N * N <= ESIKF_THREADS, "one element per thread");
  double* cur = buf0;
  double* nxt = buf1;
  const int i = tid / N, j = tid - i * N;   // this thread's element (fixed over the sweeps)
  const bool act = tid < N * N;
#pragma unroll 1
  for (int k = 0; k < N; ++k) {
    const double inv = __drcp_rn(cur[k * N + k]);   // IEEE round-to-nearest reciprocal == 1.0 / x, without the division call
    if (act) {
      double v;
      if (i == k) v = (j == k) ? inv : cur[k * N + j] * inv;
      else if (j == k) v = -(cur[i * N + k] * inv);
      else v = cur[tid] - cur[i * N + k] * (cur[k * N + j] * inv);
      nxt[tid] = v;
    }
    __syncthreads();
    double* t = cur; cur = nxt; nxt = t;
  }
  return cur;
}

// ---- the manifold operations piecewise, so that independent sub-manifolds are handled by different warps concurrently
// (x [+] d: build_manifold.hpp:188-190; x [-] o with the S2 part of S2.hpp:144-167)
__device__ __noinline__ void so3_boxminus(const double* xq, const double* oq, double* r) {  // log(o^-1 * x)
  double qc[4] = {-oq[0], -oq[1], -oq[2], oq[3]}, q[4];
  qmul(qc, xq, q);
  log_quat(q, r);
}
__device__ __noinline__ void so3_boxplus(double* xq, const double* d, double scale = 1.0) {   // x * exp(d, scale / 2)
  double q[4];
  exp_quat(d, scale / 2, q);
  qmul(xq, q, xq);
}
__device__ __noinline__ void s2_boxminus(const double* v, const double* ov, double* r) {  // S2.hpp:144-167
  double H[9], t[3];
  hat(v, H);
  for (int i = 0; i < 3; ++i) t[i] = H[3 * i] * ov[0] + H[3 * i + 1] * ov[1] + H[3 * i + 2] * ov[2];
  const double v_sin = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
  const double v_cos = v[0] * ov[0] + v[1] * ov[1] + v[2] * ov[2];
  const double theta = atan2(v_sin, v_cos);
  if (v_sin < 1e-11) {
    r[0] = fabs(theta) > 1e-11 ? 3.1415926 : 0.0;
    r[1] = 0.0;
  } else {
    double Bx[6], Ho[9], u[3];
    s2_Bx(ov, Bx);
    hat(ov, Ho);
    for (int i = 0; i < 3; ++i) u[i] = Ho[3 * i] * v[0] + Ho[3 * i + 1] * v[1] + Ho[3 * i + 2] * v[2];
    const double f = theta / v_sin;
    for (int i = 0; i < 2; ++i) { double s = 0; for (int k = 0; k < 3; ++k) s += (f * Bx[2 * k + i]) * u[k]; r[i] = s; }
  }
}
__device__ __noinline__ void s2_boxplus(double* v, const double* d) {  // S2.hpp:136-142
  double Bx[6], Bu[3], R[9], o[3], q[4];
  s2_Bx(v, Bx);
  for (int i = 0; i < 3; ++i) Bu[i] = Bx[2 * i] * d[0] + Bx[2 * i + 1] * d[1];
  exp_quat(Bu, 0.5, q);
  rotmat(q, R);
  for (int i = 0; i < 3; ++i) o[i] = R[3 * i] * v[0] + R[3 * i + 1] * v[1] + R[3 * i + 2] * v[2];
  v[0] = o[0]; v[1] = o[1]; v[2] = o[2];
}
__device__ __forceinline__ void pose_from_state(const double* x, PoseDev& p) {
  for (int i = 0; i < 4; ++i) { p.rot[i] = x[3 + i]; p.offR[i] = x[7 + i]; }
  for (int i = 0; i < 3; ++i) { p.pos[i] = x[i]; p.offT[i] = x[11 + i]; }
}

// ---- block-cooperative 23x23 helpers on shared memory (row-major, leading dimension NDOF); every thread of the block calls
// them (they contain __syncthreads).  The three projected sub-manifolds together.  The projection Jacobian of esekfom.hpp:1665-1703 / :1841-1918 is block
// diagonal: identity except J3a on rows/cols 3..5 (rot), J3b on 6..8 (offset_R_L_I) and J2 on 21..22 (grav).  The blocks touch
// disjoint rows (columns), so all row products form ONE phase and all column products another: 8 x 23 outputs per phase,
// one per thread, instead of six block-wide phases of 23 busy threads each.  (Entries that sit in the rows of one block and
// the columns of another see "rows, then columns" instead of the reference's block-by-block order: the same products in
// another association, a rounding-level difference.)
struct ProjSel { const double* J; int idx, D, i; };
__device__ __forceinline__ ProjSel proj_sel(int o, const double* J3a, const double* J3b, const double* J2) {
  ProjSel r;
  if (o < 3) { r.J = J3a; r.idx = 3; r.D = 3; r.i = o; }
  else if (o < 6) { r.J = J3b; r.idx = 6; r.D = 3; r.i = o - 3; }
  else { r.J = J2; r.idx = 21; r.D = 2; r.i = o - 6; }
  return r;
}
// value of (J Src)[row of output o][c]
__device__ __forceinline__ double proj_row_value(const double* Src, int ld, const ProjSel& q, int c) {
  double s = 0;
  for (int k = 0; k < q.D; ++k) s += q.J[q.D * q.i + k] * Src[(q.idx + k) * ld + c];
  return s;
}
// value of (M J^T)[r][column of output o]
__device__ __forceinline__ double proj_col_value(const double* M, const ProjSel& q, int r) {
  double s = 0;
  for (int k = 0; k < q.D; ++k) s += M[r * NDOF + q.idx + k] * q.J[q.D * q.i + k];
  return s;
}
constexpr int PROJ_OUT = 8 * NDOF;   // 184 outputs per phase
// M <- Jfull M Jfull^T in place (every thread of the block calls it)
__device__ __forceinline__ void b_project(double* M, const double* J3a, const double* J3b, const double* J2, int tid) {
  const int o = tid / NDOF, c = tid - o * NDOF;
  ProjSel q = proj_sel(o < 8 ? o : 0, J3a, J3b, J2);
  double v = 0;
  if (tid < PROJ_OUT) v = proj_row_value(M, NDOF, q, c);
  __syncthreads();
  if (tid < PROJ_OUT) M[(q.idx + q.i) * NDOF + c] = v;
  __syncthreads();
  if (tid < PROJ_OUT) v = proj_col_value(M, q, c);        // c = row index here
  __syncthreads();
  if (tid < PROJ_OUT) M[c * NDOF + q.idx + q.i] = v;
  __syncthreads();
}
}  // namespace dev

// Load the propagated state / covariance for a new scan.
// staging layout: x0[26] | P0[529] | n | flg_EKF_inited | bits of the device pointer to the scan   (all 8-byte slots).  `stage`
// is MAPPED PINNED HOST memory: the block reads the scan's inputs straight over PCIe (4.5 KB), no copy node in the graph.
__global__ void k_esikf_begin(EsikfCtl* c, const double* __restrict__ stage, int* work_counts) {
  pdl_sync();
  FLB_TRACE_BEGIN(0);
  if (threadIdx.x == 0) c->t_begin = global_timer_ns();
  // the record is 558 doubles: every thread issues its (at most two) 16-byte reads at once — reads of host memory are slow
  // per request, so few wide requests all in flight
  __shared__ double sst[26 + NDOF * NDOF + 4];
  constexpr int NPAIR = (26 + NDOF * NDOF + 4) / 2;
  const double2* st2 = reinterpret_cast<const double2*>(stage);
  for (int i = threadIdx.x; i < NPAIR; i += blockDim.x) {
    const double2 v = st2[i];
    sst[2 * i] = v.x;
    sst[2 * i + 1] = v.y;
  }
  // per-pass k-NN work-list counters [0..7], tickets [8..15] and stencil CTAs done [16..23]
  if (threadIdx.x >= 32 && threadIdx.x < 56) work_counts[threadIdx.x - 32] = 0;
  __syncthreads();
  const double* x0 = sst;
  const double* P0 = sst + 26;
  const int n = (int)sst[26 + NDOF * NDOF];
  for (int i = threadIdx.x; i < NDOF * NDOF; i += blockDim.x) { c->Pp[i] = P0[i]; c->P[i] = P0[i]; }
  if (threadIdx.x < 26) { c->x[threadIdx.x] = x0[threadIdx.x]; c->xp[threadIdx.x] = x0[threadIdx.x]; }
  __syncthreads();
  if (threadIdx.x == 0) {
    c->it = -1; c->t = 0; c->converge = 1; c->finished = 0; c->need_host = 0; c->passes = 0; c->searches = 0;
    c->lastM = 0; c->last_res = 0.0; c->n = n; c->flg_inited = (int)sst[26 + NDOF * NDOF + 1];
    c->body = reinterpret_cast<const float4*>((unsigned long long)__double_as_longlong(sst[26 + NDOF * NDOF + 2]));
    dev::pose_from_state(c->x, c->pose);
  }
  FLB_TRACE_END(0);
}

// Last node of a scan: everything the host reads after a step, written into ONE mapped pinned host record (zero-copy
// stores over PCIe, ~4.7 KB) — posterior state and covariance, loop statistics, the map counters, map_incremental's counts.
struct StepResult {
  double x[26];
  double P[NDOF * NDOF];
  double last_res;
  int passes, searches, lastM, t, need_host, pad_;
  int counters[32];
  int cnt2[2];
  unsigned long long span_ns;   // device time from the start of k_esikf_begin to the end of the sequence (%globaltimer): the step's
                                // own GPU time without an event pair on the stream between two steps in flight
  unsigned long long update_ns; // the same up to k_publish, which starts right behind the last update kernel: the iterated update
                                // without map_incremental
};
__global__ void k_publish(const EsikfCtl* c, const int* __restrict__ counters, const int* __restrict__ cnt2, StepResult* out, int with_tail) {
  pdl_sync();
  const int tid = threadIdx.x;
  for (int i = tid; i < NDOF * NDOF; i += blockDim.x) out->P[i] = c->P[i];
  if (tid < 26) out->x[tid] = c->x[tid];
  if (tid == 64) { out->last_res = c->last_res; out->passes = c->passes; out->searches = c->searches; out->lastM = c->lastM; out->t = c->t; out->need_host = c->need_host; }
  if (tid == 67) out->update_ns = global_timer_ns() - c->t_begin;
  if (!with_tail) return;   // counters, counts and span: written by the last insert kernel (StepTail, map_kernels.cuh)
  if (tid >= 32 && tid < 64) out->counters[tid - 32] = counters[tid - 32];
  if (tid == 65) { out->cnt2[0] = cnt2 ? cnt2[0] : 0; out->cnt2[1] = cnt2 ? cnt2[1] : 0; }
  if (tid == 66) out->span_ns = global_timer_ns() - c->t_begin;
}

// One loop iteration of update_iterated_dyn_share_modified is split in two kernels so that the half that only needs
// the current iterate overlaps with the measurement kernels of the same pass (second stream / graph branch):
//   k_esikf_pre  : dx = x [-] x_prop, projection Jacobians, projected P and (P/R)^-1            (esekfom.hpp:1655-1703,1788)
//   k_esikf_post : reduce the block partials, + H^T H, second inverse, K, dx_, boxplus, convergence bookkeeping and
//                  the final covariance                                                        (:1790-1935)
// Both are latency-oriented: loop flags / state staged in shared memory with parallel loads, transcendental-heavy
// sub-manifold work spread over warps, compact rolled loops (a kernel that runs once per launch is instruction-fetch
// bound on straight-line code).
// The gain is formed in the 12-dimensional subspace the measurement touches instead of through the two 23x23 inverses
// of esekfom.hpp:1788/1808.  With Pr = P/R (projected), U = [I12; 0], S = H^T H (12x12, zero elsewhere):
//   P_inv[:, 0:12] = ((Pr)^-1 + U S U^T)^-1 U = Pr[:, 0:12] (I + S Pr11)^-1 = Q (T11 + S)^-1,
//   T11 = Pr11^-1,  Q = Pr[:, 0:12] T11          (both only depend on the iterate: k_esikf_pre, off the critical path)
// so K_x[:, 0:12] = P_inv[:, 0:12] S and K_h = P_inv[:, 0:12] H^T h (esekfom.hpp:1810-1815) need ONE 12x12 SPD inverse
// after the reduction.  Without extrinsic estimation the Jacobian columns 6..11 are identically zero
// (laserMapping.cpp:1996), so the same identities hold with U = [I6; 0]: MD = 6 and a 6x6 inverse (K_x[:, 6:12] = 0).  Algebraically identical to the reference's information form, better conditioned, and it agrees
// with the host engine (which keeps the reference's two-inverse form) to ~1e-16 (tests/test_gpu_parity.py).
struct EsikfScratch {
  double dxn[NDOF];
  double P[NDOF * NDOF];   // projected P_propagated
  double T11[144];         // (P[0:12,0:12] / R)^-1
  double Q[NDOF * 12];     // (P[:,0:12] / R) T11
};

template <int MD>
__global__ void __launch_bounds__(dev::ESIKF_THREADS) k_esikf_pre(const EsikfCtl* c, EsikfScratch* sc) {
  pdl_sync();
  using namespace dev;
  __shared__ double P[NDOF * NDOF], L[144], T[144];
  __shared__ double dx[NDOF], J3a[9], J3b[9], J2[4], Nx[6], Mx[6], xs[26], xps[26];
  const int tid = threadIdx.x;
  FLB_TRACE_BEGIN(1 * 8 + c->it + 1);
  const int trace_slot = 1 * 8 + c->it + 1;
  const int trace_ph = c->it + 1 == 1 ? 72 : 1 << 20;   // phases of the pass-1 launch (normally a pass without a search: this kernel is its critical path)
  (void)trace_slot; (void)trace_ph;
  FLB_TRACE_PHASE(trace_ph + 0);
  // the loads are issued ahead of the loop flags and complete under them
  double pP[3];
#pragma unroll
  for (int u = 0; u < 3; ++u) { const int e = tid + u * ESIKF_THREADS; pP[u] = e < NDOF * NDOF ? c->Pp[e] : 0.0; }
  double px = 0.0, pxp = 0.0;
  if (tid >= 32 && tid < 58) { px = c->x[tid - 32]; pxp = c->xp[tid - 32]; }
  const double R = c->R;
  if (c->finished || c->it >= c->max_iter || c->n <= 0) return;   // uniform
  if (tid >= 32 && tid < 58) { xs[tid - 32] = px; xps[tid - 32] = pxp; }
#pragma unroll
  for (int u = 0; u < 3; ++u) { const int e = tid + u * ESIKF_THREADS; if (e < NDOF * NDOF) P[e] = pP[u]; }
  __syncthreads();
  FLB_TRACE_PHASE(trace_ph + 1);   // state / covariance staged
  // x_ [-] x_propagated (:1655) and the projection Jacobians, one sub-manifold per warp
  if (tid == 0) {
    so3_boxminus(xs + 3, xps + 3, dx + 3);
    A_matrix_T(dx + 3, J3a);
  } else if (tid == 32) {
    so3_boxminus(xs + 7, xps + 7, dx + 6);
    A_matrix_T(dx + 6, J3b);
  } else if (tid == 64) {
    s2_boxminus(xs + 23, xps + 23, dx + 21);
    s2_Mx(xps + 23, dx + 21, Mx);
  } else if (tid == 96) {
    s2_Nx(xs + 23, Nx);
  } else if (tid == 128) {
    for (int i = 0; i < 3; ++i) {
      dx[i] = xs[i] - xps[i]; dx[9 + i] = xs[11 + i] - xps[11 + i]; dx[12 + i] = xs[14 + i] - xps[14 + i];
      dx[15 + i] = xs[17 + i] - xps[17 + i]; dx[18 + i] = xs[20 + i] - xps[20 + i];
    }
  }
  __syncthreads();
  FLB_TRACE_PHASE(trace_ph + 2);   // boxminus + Jacobians
  if (tid < 4) { const int i = tid >> 1, j = tid & 1; double s = 0; for (int k = 0; k < 3; ++k) s += Nx[3 * i + k] * Mx[2 * k + j]; J2[tid] = s; }
  __syncthreads();
  if (tid < NDOF) {                                     // dx_new with the SO3 / S2 blocks projected (:1671, :1696)
    double v = dx[tid];
    if (tid >= 3 && tid < 6) { const int i = tid - 3; v = J3a[3 * i] * dx[3] + J3a[3 * i + 1] * dx[4] + J3a[3 * i + 2] * dx[5]; }
    else if (tid >= 6 && tid < 9) { const int i = tid - 6; v = J3b[3 * i] * dx[6] + J3b[3 * i + 1] * dx[7] + J3b[3 * i + 2] * dx[8]; }
    else if (tid >= 21) { const int i = tid - 21; v = J2[2 * i] * dx[21] + J2[2 * i + 1] * dx[22]; }
    sc->dxn[tid] = v;
  }
  b_project(P, J3a, J3b, J2, tid);                      // SO3 blocks :1665-1681, S2 block :1683-1703
  FLB_TRACE_PHASE(trace_ph + 3);   // covariance projected
  for (int e = tid; e < NDOF * NDOF; e += ESIKF_THREADS) sc->P[e] = P[e];
  if (tid < MD * MD) L[tid] = P[(tid / MD) * NDOF + (tid % MD)] / R;   // Pr11 (MD x MD)
  __syncthreads();
  FLB_TRACE_PHASE(trace_ph + 4);   // projected covariance stored
  const double* T11 = b_inverse_spd<MD>(L, T, tid);                    // Pr11^-1
  FLB_TRACE_PHASE(trace_ph + 5);   // inverse
  if (tid < MD * MD) sc->T11[tid] = T11[tid];
  for (int e = tid; e < NDOF * MD; e += ESIKF_THREADS) {               // Q = Pr[:, 0:MD] T11
    const int i = e / MD, j = e - i * MD;
    double q = 0;
    for (int k = 0; k < MD; ++k) q += P[i * NDOF + k] * T11[k * MD + j];
    sc->Q[e] = q / R;                                                  // (one division per entry: sum(P T11) / R)
  }
  FLB_TRACE_PHASE(trace_ph + 6);   // Q written
  FLB_TRACE_END(trace_slot);
}

template <int MD>
__global__ void __launch_bounds__(dev::ESIKF_THREADS) k_esikf_post(EsikfCtl* c, const double* __restrict__ partial, int nblocks,
                                                                    const EsikfScratch* __restrict__ sc) {
  pdl_sync();
  using namespace dev;
  __shared__ double acc[96], acc2[96];
  __shared__ double P[NDOF * NDOF], L[NDOF * NDOF], T[144], Q[NDOF * 12], Y[156];
  __shared__ double Kx[NDOF * 12], HTH[144], HTh[12], Kh[NDOF], lim[NDOF];
  __shared__ double dxn[NDOF], dx_[NDOF], J3a[9], J3b[9], J2[4], Nx[6], Mx[6], xs[26], xps[26];
  __shared__ int s_i[8];   // finished, it, max_iter, n, t, converge
  __shared__ int s_fin, s_conv, s_tt;
  const int tid = threadIdx.x;
  const int trace_pass = c->it + 1;
  (void)trace_pass;
  FLB_TRACE_BEGIN(5 * 8 + trace_pass);
  FLB_TRACE_PHASE(trace_pass * 12 + 0);
  if (tid == 0) s_i[0] = c->finished; else if (tid == 1) s_i[1] = c->it; else if (tid == 2) s_i[2] = c->max_iter;
  else if (tid == 3) s_i[3] = c->n; else if (tid == 4) s_i[4] = c->t; else if (tid == 5) s_i[5] = c->converge;
  if (tid >= 32 && tid < 58) { xs[tid - 32] = c->x[tid - 32]; xps[tid - 32] = c->xp[tid - 32]; }
  if (tid >= 64 && tid < 64 + NDOF) { lim[tid - 64] = c->limit[tid - 64]; dxn[tid - 64] = sc->dxn[tid - 64]; }
  // ---- the matrices k_esikf_pre left for this pass: their loads are issued first and complete under the reduction
  double pP[3], pQ[2];
#pragma unroll
  for (int u = 0; u < 3; ++u) { const int e = tid + u * ESIKF_THREADS; pP[u] = e < NDOF * NDOF ? sc->P[e] : 0.0; }
#pragma unroll
  for (int u = 0; u < 2; ++u) { const int e = tid + u * ESIKF_THREADS; pQ[u] = e < NDOF * MD ? sc->Q[e] : 0.0; }
  const double pT = tid < MD * MD ? sc->T11[tid] : 0.0;
  // ---- fixed-order reduction of the per-block partials (role of K2)
  if constexpr (MD == 6) {
    // without extrinsic estimation the measured subspace has 6 columns: only 21 entries of H^T H, 6 of H^T h, the residual
    // sum and the row count are ever read below — 29 of the 93 accumulators.  One warp per eighth of the block range, one
    // lane per entry, every load of a lane in flight at once (a third of the bytes and half the dependent batches of the
    // general form below).
    static_assert(ESIKF_THREADS == 256, "eight warps, one per eighth of the partial rows");
    const int k = tid & 31, w = tid >> 5;
    int e = -1;
    if (k < 21) { int i = 0, r = k; while (r >= 6 - i) { r -= 6 - i; ++i; } e = i * 13 - i * (i - 1) / 2 + r; }   // (i, i + r), both < 6
    else if (k < 27) { const int l = k - 21; e = l * 13 - l * (l - 1) / 2 + (12 - l); }                               // (l, 12)
    else if (k < 29) e = 91 + (k - 27);                                                                             // residual sum, count
    double* part = L;   // [8][32]; L is not used before the second __syncthreads below
    double s = 0.0;
    if (e >= 0) {
      const int per = (nblocks + 7) >> 3;
      const int b0 = min(w * per, nblocks), b1 = min(b0 + per, nblocks);
      for (int b = b0; b < b1; b += 19) {
        double v[19];
#pragma unroll
        for (int u = 0; u < 19; ++u) v[u] = b + u < b1 ? partial[(size_t)(b + u) * NACC + e] : 0.0;
#pragma unroll
        for (int u = 0; u < 19; ++u) s += v[u];
      }
    }
    part[w * 32 + k] = s;
    __syncthreads();
    if (w == 0 && e >= 0) {
      double t = 0.0;
#pragma unroll
      for (int u = 0; u < 8; ++u) t += part[u * 32 + k];
      acc[e] = t;
    }
  } else {
    // 2 threads per entry (halves of the block range, coalesced across the entries), 37 independent loads in flight per thread
    const int e = tid & 127, h = tid >> 7;
    double s = 0.0;
    if (e < NACC) {
      const int half = (nblocks + 1) >> 1;
      const int b0 = h ? half : 0, b1 = h ? nblocks : half;
      for (int b = b0; b < b1; b += 37) {
        double v[37];
#pragma unroll
        for (int u = 0; u < 37; ++u) v[u] = b + u < b1 ? partial[(size_t)(b + u) * NACC + e] : 0.0;
#pragma unroll
        for (int u = 0; u < 37; ++u) s += v[u];
      }
      if (h) acc2[e] = s;
    }
    __syncthreads();
    if (e < NACC && h == 0) acc[e] = s + acc2[e];
  }
  __syncthreads();
  FLB_TRACE_PHASE(trace_pass * 12 + 1);   // partials reduced
  const int it = s_i[1], max_iter = s_i[2];
  if (s_i[0] || it >= max_iter) return;                                          // loop already ended
  if (s_i[3] <= 0) { if (tid == 0) { c->it = it + 1; c->passes++; } return; }    // empty scan: every pass invalid
  const int M = (int)(acc[92] + 0.5);
  if (tid == 0) { c->passes++; if (s_i[5]) c->searches++; }
  if (M < 1) { if (tid == 0) c->it = it + 1; return; }                            // valid = false -> continue (:1641-1644)
  if (M < NDOF) { if (tid == 0) { c->need_host = 1; c->finished = 1; } return; }  // under-determined branch: host path
  if (tid == 0) { c->lastM = M; c->last_res = acc[91]; }
  // gain in the measured subspace (see EsikfScratch): V = (T11 + H^T H)^-1, Y = V [H^T H | H^T h], [K_x | K_h] = Q Y
  if (tid < MD * MD) {
    const int i = tid / MD, j = tid - i * MD;
    const int a = i < j ? i : j, b = i < j ? j : i;
    const double hth = acc[a * 13 - a * (a - 1) / 2 + (b - a)];
    HTH[tid] = hth;                                         // MD x MD
    T[tid] = pT + hth;
  }
  if (tid >= 160 && tid < 160 + MD) { const int l = tid - 160; HTh[l] = acc[l * 13 - l * (l - 1) / 2 + (12 - l)]; }
#pragma unroll
  for (int u = 0; u < 3; ++u) { const int e = tid + u * ESIKF_THREADS; if (e < NDOF * NDOF) P[e] = pP[u]; }
#pragma unroll
  for (int u = 0; u < 2; ++u) { const int e = tid + u * ESIKF_THREADS; if (e < NDOF * MD) Q[e] = pQ[u]; }
  __syncthreads();
  FLB_TRACE_PHASE(trace_pass * 12 + 2);   // matrices staged
  const double* V = b_inverse_spd<MD>(T, L, tid);
  FLB_TRACE_PHASE(trace_pass * 12 + 3);   // inverse done
  if (tid < MD * (MD + 1)) {
    const int i = tid / (MD + 1), j = tid - i * (MD + 1);
    double q = 0;
    for (int k = 0; k < MD; ++k) q += V[i * MD + k] * (j < MD ? HTH[k * MD + j] : HTh[k]);
    Y[tid] = q;
  }
  __syncthreads();
  for (int e = tid; e < NDOF * 13; e += ESIKF_THREADS) {      // K_x (23 x 12, columns >= MD are zero) and K_h
    const int i = e / 13, j = e - i * 13;
    double q = 0;
    if (j < MD || j == 12) {
      const int jj = j == 12 ? MD : j;
      for (int k = 0; k < MD; ++k) q += Q[i * MD + k] * Y[k * (MD + 1) + jj];
    }
    if (j < 12) Kx[i * 12 + j] = q; else Kh[i] = q;
  }
  __syncthreads();
  if (tid < NDOF) {                                     // :1821 dx_ = K_h + (K_x - I) dx_new
    double s = 0;
    for (int j = 0; j < NDOF; ++j) s += ((j < 12 ? Kx[tid * 12 + j] : 0.0) - (tid == j ? 1.0 : 0.0)) * dxn[j];
    dx_[tid] = Kh[tid] + s;
  }
  __syncthreads();
  FLB_TRACE_PHASE(trace_pass * 12 + 4);   // gain and dx_ done
  // convergence test (:1824-1838) first: the Jacobians of the final covariance are only needed on the last pass
  if (tid == 0) {
    int conv = 1, tt = s_i[4];
    for (int i = 0; i < NDOF; ++i) if (fabs(dx_[i]) > lim[i]) { conv = 0; break; }
    if (conv) ++tt;
    if (!tt && it == max_iter - 2) conv = 1;            // :1835-1838
    s_conv = conv; s_tt = tt;
    s_fin = (tt > 1 || it == max_iter - 1) ? 1 : 0;
  }
  __syncthreads();
  // x_ [+] dx_ (:1823) per sub-manifold (+ Jacobians when finishing)
  if (tid == 0) {
    so3_boxplus(xs + 3, dx_ + 3);
    if (s_fin) A_matrix_T(dx_ + 3, J3a);
  } else if (tid == 32) {
    so3_boxplus(xs + 7, dx_ + 6);
    if (s_fin) A_matrix_T(dx_ + 6, J3b);
  } else if (tid == 64) {
    s2_boxplus(xs + 23, dx_ + 21);
    if (s_fin) s2_Nx(xs + 23, Nx);
  } else if (tid == 96) {
    if (s_fin) s2_Mx(xps + 23, dx_ + 21, Mx);
  } else if (tid == 128) {
    for (int i = 0; i < 3; ++i) { xs[i] += dx_[i]; xs[11 + i] += dx_[9 + i]; xs[14 + i] += dx_[12 + i]; xs[17 + i] += dx_[15 + i]; xs[20 + i] += dx_[18 + i]; }
  }
  __syncthreads();
  if (tid < 4 && s_fin) { const int i = tid >> 1, j = tid & 1; double s = 0; for (int k = 0; k < 3; ++k) s += Nx[3 * i + k] * Mx[2 * k + j]; J2[tid] = s; }
  __syncthreads();
  const int fin = s_fin;
  FLB_TRACE_PHASE(trace_pass * 12 + 5);   // boxplus (+ final Jacobians) done
  if (fin) {                                            // :1841-1931, the three sub-manifold blocks together (see b_project)
    // L = Jfull P (rows; L is a separate buffer: no staging), K_x rows <- Jfull K_x rows (in place: staged in registers)
    const int o = tid / NDOF, cc = tid - o * NDOF;
    const ProjSel q = proj_sel(o < 8 ? o : 0, J3a, J3b, J2);
    for (int e = tid; e < NDOF * NDOF; e += ESIKF_THREADS) {
      const int r = e / NDOF;
      if (!((r >= 3 && r < 9) || r >= 21)) L[e] = P[e];
    }
    if (tid < PROJ_OUT) L[(q.idx + q.i) * NDOF + cc] = proj_row_value(P, NDOF, q, cc);
    const int ok = tid / 12, ck = tid - ok * 12;                    // 8 x 12 outputs of the gain
    const ProjSel qk = proj_sel(ok < 8 ? ok : 0, J3a, J3b, J2);
    double kv = 0;
    if (tid < 96) kv = proj_row_value(Kx, 12, qk, ck);
    __syncthreads();
    if (tid < 96) Kx[(qk.idx + qk.i) * 12 + ck] = kv;
    // columns of L and of P (in place, staged in registers)
    double lv = 0, pv = 0;
    if (tid < PROJ_OUT) { lv = proj_col_value(L, q, cc); pv = proj_col_value(P, q, cc); }
    __syncthreads();
    if (tid < PROJ_OUT) { L[cc * NDOF + q.idx + q.i] = lv; P[cc * NDOF + q.idx + q.i] = pv; }
    __syncthreads();
    for (int e = tid; e < NDOF * NDOF; e += ESIKF_THREADS) {      // P_ = L_ - K_x[:, :12] P_[:12, :]
      const int i = e / NDOF, j = e - i * NDOF;
      double s = 0;
      for (int k = 0; k < 12; ++k) s += Kx[i * 12 + k] * P[k * NDOF + j];
      c->P[e] = L[e] - s;
    }
  } else {
    for (int e = tid; e < NDOF * NDOF; e += ESIKF_THREADS) c->P[e] = P[e];  // P_ as last assigned (projected P_propagated)
  }
  if (tid < 26) c->x[tid] = xs[tid];
  if (tid == 32) { c->converge = s_conv; c->t = s_tt; c->finished = fin; c->it = it + 1; }
  if (tid == 64) pose_from_state(xs, c->pose);
  FLB_TRACE_PHASE(trace_pass * 12 + 6);   // covariance / state written
  FLB_TRACE_END(5 * 8 + trace_pass);
}

}  // namespace flb

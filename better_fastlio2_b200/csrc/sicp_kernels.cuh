// sicp_kernels.cuh — the ADMM loop of the relocaliser's Sparse ICP (SICP::point_to_point, include/FRICP-toolkit/ICP.h:275-380,
// as Registeration::run calls it for regMode 7) on the clouds flb_keyframes_fricp's set-up normalises, in double.  One
// persistent cooperative kernel runs every ADMM iteration of one ICP iteration: it grid-strides over the source points and
// separates its three phases with grid-wide barriers.  Each phase ends with per-block partial sums; after the barrier
// every block sums all blocks' partials in the same fixed order and solves the same 3x3 SVD (icp_svd3, shared with the
// host), so every block holds the same means, the same step cur_T and the same stopping decision with no further barrier
// and no host round trip.  The TU is compiled with -fmad=false: every expression below rounds as written, like the
// restatement in tests/cpp/sicp_oracle.cpp (orc_sicp).
#pragma once
#include <cooperative_groups.h>

#include "fricp_kernels.cuh"

namespace flb {

constexpr int SICP_BLOCK = 256;
constexpr int SICP_RED = 9;                  // doubles per block and phase (the widest: the cross-covariance)
constexpr int SICP_SLOTS = 3;                // one partials slot per phase: a slot is rewritten three barriers after it is read
constexpr int SICP_REC_T = 0, SICP_REC_OUTER = 12, SICP_REC_PRIMAL = 13, SICP_REC_DUAL = 14, SICP_REC_STOP = 15,
              SICP_REC_WORDS = 16;           // the record of one ICP iteration: T (row-major 3x4), outer count, primal, dual, stop

// One ICP iteration's ADMM state and parameters.  x: the moving normalised source (w = 1 finite, 0 not), updated in place;
// q: this iteration's matches (w = 1 where x has a match); z, c: the shrunk residuals and the multipliers (c persists
// across ICP iterations); xo2: X at the end of the previous ICP iteration.  sched: per outer iteration μ, Ba and ha.
struct SicpArgs {
  double4* x;
  const double4* sorted_d;
  const int* pos;
  double4 *q, *z, *c, *xo2;
  const double* sched;
  double* part;                              // SICP_SLOTS x gridDim.x x SICP_RED
  double* rec;                               // SICP_REC_WORDS: T in and out, the iteration's exit values out
  int n, max_outer;
  double inv_n, n_d, p, stop;                // 1 / n_finite (the normalised weight), n_finite, p, stop
};

// shrinkage<3> (ICP.h:238-243): s <- 1 - (p/μ) n^(p-2) s^(p-1), three times from s0 = (Ba/n + 1)/2; 0 when n <= ha.
__host__ __device__ inline double sicp_shrink_factor(double n, double mu, double p, double Ba, double ha) {
  if (!(n > ha)) return 0.0;
  double s = (Ba / n + 1.0) / 2.0;
  for (int k = 0; k < 3; ++k) s = 1.0 - ((p / mu) * pow(n, p - 2.0)) * pow(s, p - 1.0);
  return s;
}

__device__ __forceinline__ double sicp_norm(double x, double y, double z) { return sqrt((x * x + y * y) + z * z); }

// Block tree over sh[k][0..256) for k < K (sums for k < n_sum, maxima after); the result in sh[k][0].  Ends synchronised.
template <int K>
__device__ __forceinline__ void sicp_block(double (*sh)[SICP_BLOCK], int n_sum) {
  __syncthreads();
  for (int s = SICP_BLOCK / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int k = 0; k < K; ++k) sh[k][threadIdx.x] = k < n_sum ? sh[k][threadIdx.x] + sh[k][threadIdx.x + s] : fmax(sh[k][threadIdx.x], sh[k][threadIdx.x + s]);
    __syncthreads();
  }
}

// Per-thread values a[K] -> this block's partials in slot `slot`.
template <int K>
__device__ __forceinline__ void sicp_put(double (*sh)[SICP_BLOCK], const double* a, int n_sum, double* part, int slot) {
  for (int k = 0; k < K; ++k) sh[k][threadIdx.x] = a[k];
  sicp_block<K>(sh, n_sum);
  if (threadIdx.x < K) part[((size_t)slot * gridDim.x + blockIdx.x) * SICP_RED + threadIdx.x] = sh[threadIdx.x][0];
}

// Every block: all blocks' partials of slot `slot` in one fixed order (thread t takes blocks t, t + 256, ... in order, then
// the block tree) into out[K].  Every block computes the same bits.
template <int K>
__device__ __forceinline__ void sicp_all(double (*sh)[SICP_BLOCK], int n_sum, const double* part, int slot, double* out) {
  for (int k = 0; k < K; ++k) {
    double v = k < n_sum ? 0.0 : -INFINITY;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += SICP_BLOCK) {
      const double u = __ldcg(&part[((size_t)slot * gridDim.x + b) * SICP_RED + k]);
      v = k < n_sum ? v + u : fmax(v, u);
    }
    sh[k][threadIdx.x] = v;
  }
  sicp_block<K>(sh, n_sum);
  for (int k = 0; k < K; ++k) out[k] = sh[k][0];
  __syncthreads();
}

// The ADMM loop of one ICP iteration (ICP.h:328-358 with max_inner = 1, no penalty mode), then stop = max |X - Xo2| and
// Xo2 <- X (:356-357).  Launched cooperatively with every block resident.
__global__ void __launch_bounds__(SICP_BLOCK) k_sicp_admm(SicpArgs a) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  __shared__ double sh[SICP_RED][SICP_BLOCK];
  __shared__ double sT[12], sC[12];
  const int stride = gridDim.x * SICP_BLOCK;
  const int i0 = blockIdx.x * SICP_BLOCK + threadIdx.x;
  if (threadIdx.x < 12) sT[threadIdx.x] = a.rec[SICP_REC_T + threadIdx.x];
  // Q_i = the matched target point of this iteration's 1-NN pass
  for (int i = i0; i < a.n; i += stride) {
    const int p = a.pos[i];
    a.q[i] = p >= 0 ? make_double4(a.sorted_d[p].x, a.sorted_d[p].y, a.sorted_d[p].z, 1.0) : make_double4(0.0, 0.0, 0.0, 0.0);
  }
  int outer = 0;
  double primal = 0.0, dual = 0.0;
  while (outer < a.max_outer) {
    const double mu = a.sched[3 * outer], Ba = a.sched[3 * outer + 1], ha = a.sched[3 * outer + 2];
    // Z = (X - Q) + C/μ, shrink<3>(Z, μ, p); U = (Q + Z) - C/μ; the normalised means x̄ = Σ x (1/n), ū = Σ u (1/n)
    double acc[SICP_RED];
    for (int k = 0; k < 6; ++k) acc[k] = 0.0;
    for (int i = i0; i < a.n; i += stride) {
      const double4 q = a.q[i];
      if (q.w == 0.0) continue;
      const double4 x = a.x[i], c = a.c[i];
      double z[3] = {(x.x - q.x) + c.x / mu, (x.y - q.y) + c.y / mu, (x.z - q.z) + c.z / mu};
      const double w = sicp_shrink_factor(sicp_norm(z[0], z[1], z[2]), mu, a.p, Ba, ha);
      for (int k = 0; k < 3; ++k) z[k] = z[k] * w;
      a.z[i] = make_double4(z[0], z[1], z[2], 0.0);
      acc[0] += x.x * a.inv_n; acc[1] += x.y * a.inv_n; acc[2] += x.z * a.inv_n;
      acc[3] += ((q.x + z[0]) - c.x / mu) * a.inv_n;
      acc[4] += ((q.y + z[1]) - c.y / mu) * a.inv_n;
      acc[5] += ((q.z + z[2]) - c.z / mu) * a.inv_n;
    }
    sicp_put<6>(sh, acc, 6, a.part, 0);
    grid.sync();
    double mean[6];
    sicp_all<6>(sh, 6, a.part, 0, mean);
    // Σ ((x - x̄)(1/n)) (u - ū)ᵀ, row-major
    for (int k = 0; k < 9; ++k) acc[k] = 0.0;
    for (int i = i0; i < a.n; i += stride) {
      const double4 q = a.q[i];
      if (q.w == 0.0) continue;
      const double4 x = a.x[i], c = a.c[i], z = a.z[i];
      const double xs[3] = {(x.x - mean[0]) * a.inv_n, (x.y - mean[1]) * a.inv_n, (x.z - mean[2]) * a.inv_n};
      const double us[3] = {((q.x + z.x) - c.x / mu) - mean[3], ((q.y + z.y) - c.y / mu) - mean[4], ((q.z + z.z) - c.z / mu) - mean[5]};
      for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) acc[3 * r + k] += xs[r] * us[k];
    }
    sicp_put<9>(sh, acc, 9, a.part, 1);
    grid.sync();
    double sig[9];
    sicp_all<9>(sh, 9, a.part, 1, sig);
    // cur_T = RigidMotionEstimator::point_to_point(X, U) (ICP.h:89-124): R = V diag(1, 1, ±1) Uᵀ, t = ū - R x̄; T <- cur_T T
    if (threadIdx.x == 0) {
      double U[9], sv[3], V[9];
      icp_svd3(sig, U, sv, V);
      if (!(sv[0] > 0))   // a zero cross-covariance (one point): U = V = I as Eigen's JacobiSVD leaves them, R = I
        for (int k = 0; k < 9; ++k) U[k] = V[k] = (k % 4 == 0) ? 1.0 : 0.0;
      const double dd = icp_det3(U) * icp_det3(V) < 0 ? -1.0 : 1.0;
      for (int r = 0; r < 3; ++r) {
        for (int k = 0; k < 3; ++k) sC[4 * r + k] = (V[3 * r] * U[3 * k] + V[3 * r + 1] * U[3 * k + 1]) + dd * V[3 * r + 2] * U[3 * k + 2];
        sC[4 * r + 3] = mean[3 + r] - ((sC[4 * r] * mean[0] + sC[4 * r + 1] * mean[1]) + sC[4 * r + 2] * mean[2]);
      }
      double nT[12];
      for (int r = 0; r < 3; ++r) {
        for (int k = 0; k < 4; ++k) nT[4 * r + k] = (sC[4 * r] * sT[k] + sC[4 * r + 1] * sT[4 + k]) + sC[4 * r + 2] * sT[8 + k];
        nT[4 * r + 3] = nT[4 * r + 3] + sC[4 * r + 3];
      }
      for (int k = 0; k < 12; ++k) sT[k] = nT[k];
    }
    __syncthreads();
    double m[12];
    for (int k = 0; k < 12; ++k) m[k] = sC[k];
    // X <- cur_T X; dual = Σ |X - X_old|² / n; P = (X - Q) - Z, C <- C + μ P; primal = max |P|
    acc[0] = 0.0;
    acc[1] = 0.0;
    for (int i = i0; i < a.n; i += stride) {
      const double4 q = a.q[i];
      if (q.w == 0.0) continue;
      const double4 x = a.x[i], z = a.z[i];
      double4 c = a.c[i];
      const double4 xn = make_double4(((m[0] * x.x + m[1] * x.y) + m[2] * x.z) + m[3], ((m[4] * x.x + m[5] * x.y) + m[6] * x.z) + m[7],
                                      ((m[8] * x.x + m[9] * x.y) + m[10] * x.z) + m[11], x.w);
      const double dx = xn.x - x.x, dy = xn.y - x.y, dz = xn.z - x.z;
      acc[0] += (dx * dx + dy * dy) + dz * dz;
      const double P[3] = {(xn.x - q.x) - z.x, (xn.y - q.y) - z.y, (xn.z - q.z) - z.z};
      c.x = c.x + mu * P[0];
      c.y = c.y + mu * P[1];
      c.z = c.z + mu * P[2];
      acc[1] = fmax(acc[1], sicp_norm(P[0], P[1], P[2]));
      a.x[i] = xn;
      a.c[i] = c;
    }
    sicp_put<2>(sh, acc, 1, a.part, 2);
    grid.sync();
    double dp[2];
    sicp_all<2>(sh, 1, a.part, 2, dp);
    dual = dp[0] / a.n_d;
    primal = dp[1];
    ++outer;
    if (primal < a.stop && dual < a.stop) break;
  }
  // stop = max |X - Xo2|, Xo2 <- X
  double st[1] = {0.0};
  for (int i = i0; i < a.n; i += stride) {
    const double4 x = a.x[i];
    if (x.w == 0.0) continue;
    const double4 o = a.xo2[i];
    st[0] = fmax(st[0], sicp_norm(x.x - o.x, x.y - o.y, x.z - o.z));
    a.xo2[i] = x;
  }
  sicp_put<1>(sh, st, 0, a.part, 0);
  grid.sync();
  if (blockIdx.x != 0) return;
  double sv[1];
  sicp_all<1>(sh, 0, a.part, 0, sv);
  if (threadIdx.x < 12) a.rec[SICP_REC_T + threadIdx.x] = sT[threadIdx.x];
  if (threadIdx.x == 0) {
    a.rec[SICP_REC_OUTER] = outer;
    a.rec[SICP_REC_PRIMAL] = primal;
    a.rec[SICP_REC_DUAL] = dual;
    a.rec[SICP_REC_STOP] = sv[0];
  }
}

}  // namespace flb

// meas_kernels.cuh — K1' point-to-plane residual / Jacobian (+ fused H^T H reduction), K2 final reduce, row export
// and the map_incremental classifier.  Follows h_share_model (src/laserMapping.cpp:1876-2004), esti_plane
// (include/common_lib.h:506-536) and map_incremental (src/laserMapping.cpp:1440-1496) of the reference.
// Precision is kept where the reference has it: world point double->float, plane fit and gates in float (no FMA
// contraction: this TU is compiled with -fmad=false), Jacobian rows and the normal equations in double.
#pragma once
#include "knn_kernels.cuh"
#include "map_kernels.cuh"

namespace flb {

// ---------------------------------------------------------------------------------------------- esti_plane<float>
// Column-pivoted Householder QR least squares of A x = -1 (A = 5x3 neighbour coordinates), Eigen 3.3
// ColPivHouseholderQR restated operation by operation (same sequence as oracle/lio_oracle.cpp::esti_plane_f).
__device__ __forceinline__ bool esti_plane_dev(const float (&P)[5][3], float thr, float& na, float& nb, float& nc, float& nd) {
  float qr[5][3];
#pragma unroll
  for (int r = 0; r < 5; ++r) { qr[r][0] = P[r][0]; qr[r][1] = P[r][1]; qr[r][2] = P[r][2]; }
  float b[5] = {-1.f, -1.f, -1.f, -1.f, -1.f};
  float hc[3];
  int perm[3] = {0, 1, 2};
  float nu[3], nd_[3];
  const float eps = 1.1920929e-07f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < 5; ++r) s += qr[r][k] * qr[r][k];
    nd_[k] = sqrtf(s);
    nu[k] = nd_[k];
  }
  const float th = fmaxf(nu[0], fmaxf(nu[1], nu[2])) * eps;
  const float threshold_helper = (th * th) / 5.f;
  const float norm_downdate_threshold = sqrtf(eps);
  int nonzero_pivots = 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    // biggest remaining column (first maximum wins, as Eigen's maxCoeff)
    int big = k;
    float bigv = nu[k];
#pragma unroll
    for (int j = k + 1; j < 3; ++j)
      if (nu[j] > bigv) { bigv = nu[j]; big = j; }
    if (nonzero_pivots == 3 && (bigv * bigv) < threshold_helper * (float)(5 - k)) nonzero_pivots = k;
    if (big != k) {
#pragma unroll
      for (int j = 1; j < 3; ++j) {
        if (j > k && j == big) {
#pragma unroll
          for (int r = 0; r < 5; ++r) { float t = qr[r][k]; qr[r][k] = qr[r][j]; qr[r][j] = t; }
          float t = nu[k]; nu[k] = nu[j]; nu[j] = t;
          t = nd_[k]; nd_[k] = nd_[j]; nd_[j] = t;
          const int pt = perm[k]; perm[k] = perm[j]; perm[j] = pt;
        }
      }
    }
    float tail = 0.f;
#pragma unroll
    for (int r = 0; r < 5; ++r)
      if (r > k) tail += qr[r][k] * qr[r][k];
    const float c0 = qr[k][k];
    float tau, beta;
    if (tail <= 1.17549435e-38f) {
      tau = 0.f;
      beta = c0;
#pragma unroll
      for (int r = 0; r < 5; ++r)
        if (r > k) qr[r][k] = 0.f;
    } else {
      beta = sqrtf(c0 * c0 + tail);
      if (c0 >= 0.f) beta = -beta;
      const float den = c0 - beta;
#pragma unroll
      for (int r = 0; r < 5; ++r)
        if (r > k) qr[r][k] = qr[r][k] / den;
      tau = (beta - c0) / beta;
    }
    hc[k] = tau;
    qr[k][k] = beta;
    if (tau != 0.f) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        if (j > k) {
          float tmp = 0.f;
#pragma unroll
          for (int r = 0; r < 5; ++r)
            if (r > k) tmp += qr[r][k] * qr[r][j];
          tmp += qr[k][j];
          qr[k][j] -= tau * tmp;
#pragma unroll
          for (int r = 0; r < 5; ++r)
            if (r > k) qr[r][j] -= tau * qr[r][k] * tmp;
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      if (j > k && nu[j] != 0.f) {
        float temp = fabsf(qr[k][j]) / nu[j];
        temp = (1.f + temp) * (1.f - temp);
        temp = temp < 0.f ? 0.f : temp;
        const float ratio = nu[j] / nd_[j];
        const float temp2 = temp * (ratio * ratio);
        if (temp2 <= norm_downdate_threshold) {
          float s = 0.f;
#pragma unroll
          for (int r = 0; r < 5; ++r)
            if (r > k) s += qr[r][j] * qr[r][j];
          nd_[j] = sqrtf(s);
          nu[j] = nd_[j];
        } else {
          nu[j] *= sqrtf(temp);
        }
      }
    }
  }
  float x0 = 0.f, x1 = 0.f, x2 = 0.f;
  if (nonzero_pivots > 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (k < nonzero_pivots && hc[k] != 0.f) {
        float tmp = 0.f;
#pragma unroll
        for (int r = 0; r < 5; ++r)
          if (r > k) tmp += qr[r][k] * b[r];
        tmp += b[k];
        b[k] -= hc[k] * tmp;
#pragma unroll
        for (int r = 0; r < 5; ++r)
          if (r > k) b[r] -= hc[k] * qr[r][k] * tmp;
      }
    }
    float c[3] = {b[0], b[1], b[2]};
#pragma unroll
    for (int i = 2; i >= 0; --i) {
      if (i < nonzero_pivots) {
        c[i] = c[i] / qr[i][i];
#pragma unroll
        for (int r = 0; r < 3; ++r)
          if (r < i) c[r] -= c[i] * qr[r][i];
      }
    }
    float xs[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < nonzero_pivots) {
        if (perm[i] == 0) xs[0] = c[i];
        else if (perm[i] == 1) xs[1] = c[i];
        else xs[2] = c[i];
      }
    }
    x0 = xs[0]; x1 = xs[1]; x2 = xs[2];
  }
  const float n = sqrtf(x0 * x0 + x1 * x1 + x2 * x2);
  na = x0 / n;
  nb = x1 / n;
  nc = x2 / n;
  nd = (float)(1.0 / (double)n);
#pragma unroll
  for (int j = 0; j < 5; ++j)
    if (fabsf(na * P[j][0] + nb * P[j][1] + nc * P[j][2] + nd) > thr) return false;
  return true;
}

// ---------------------------------------------------------------------------------------------- K1': residual + H^T H
// One CTA per SM (one block partial per SM for the update kernel to reduce; the register file holds one such CTA).
// Without extrinsic estimation: 1024 threads = 135 168 over an H100's 132 SMs, so a scan of up to 131 072 points (the
// default session capacity) runs in ONE round of the point loop and no CTA works through a second round while the rest of
// the grid waits at the end; the price is a 64-register cap (a few spilled values in the QR).  With extrinsic estimation
// (13-wide rows) 896 threads at a 72-register cap: at 1024 threads the extra spills made cfg3 (240k-point scans, several
// rounds either way) 3.5 % slower on an H100.
#ifndef FLB_MEAS_THREADS
#define FLB_MEAS_THREADS 1024
#endif
template <bool EXTR>
__host__ __device__ constexpr int meas_threads() { return EXTR ? 896 : FLB_MEAS_THREADS; }
constexpr int NACC = 93;  // 91 upper-triangular entries of [h_x | h]^T [h_x | h] (13x13) + total_residual + M

struct MeasArgs {
  PoseDev pose;
  const float4* body;
  const float4* world;        // feats_down_world for this iterate (K0 output)
  const float4* nbr;          // [5][n]
  const unsigned char* cnt;   // [n]
  unsigned char* sel;         // [n] point_selected_surf (in/out)
  float4* normvec;            // [n] (nx,ny,nz,pd2)
  float4* plane;              // [n] pabcd of the last search pass (valid wherever sel survived it): the plane is a function of
                              // the 5 cached neighbours only, so the passes that re-use Nearest_Points re-use it bit for bit
  double* partial;            // [gridDim.x][NACC]
  int n;
  int search;                 // ekfom_data.converge
  const EsikfCtl* ctl;        // device-driven mode: pose / search flag / early exit come from here
  float4* world_out;          // device-driven mode: feats_down_world is produced here (no separate K0)
  int stride;                 // leading dimension of nbr
};

__constant__ unsigned char c_tri_i[91];
__constant__ unsigned char c_tri_j[91];

// Jacobian row of one selected point (laserMapping.cpp:1970-2001): row[0:12], row[12] = h = -pd2.
template <bool EXTR>
__device__ __forceinline__ void jacobian_row(const PoseDev& s, const float4 pb, const float4 nv, double (&row)[13]) {
  const double nx = (double)nv.x, ny = (double)nv.y, nz = (double)nv.z;
  const double qc[4] = {-s.rot[0], -s.rot[1], -s.rot[2], s.rot[3]};
  double C0, C1, C2;
  qrot_d(qc, nx, ny, nz, C0, C1, C2);                       // C = rot.conjugate() * n
  double p0, p1, p2;
  qrot_d(s.offR, (double)pb.x, (double)pb.y, (double)pb.z, p0, p1, p2);
  p0 = __dadd_rn(p0, s.offT[0]); p1 = __dadd_rn(p1, s.offT[1]); p2 = __dadd_rn(p2, s.offT[2]);  // point_this
  // A = [point_this]x * C
  const double A0 = __dadd_rn(__dmul_rn(-p2, C1), __dmul_rn(p1, C2));
  const double A1 = __dadd_rn(__dmul_rn(p2, C0), __dmul_rn(-p0, C2));
  const double A2 = __dadd_rn(__dmul_rn(-p1, C0), __dmul_rn(p0, C1));
  row[0] = nx; row[1] = ny; row[2] = nz; row[3] = A0; row[4] = A1; row[5] = A2;
  if (EXTR) {
    const double qo[4] = {-s.offR[0], -s.offR[1], -s.offR[2], s.offR[3]};
    double t0, t1, t2;
    qrot_d(qo, C0, C1, C2, t0, t1, t2);                     // offset_R_L_I.conjugate() * C
    const double b0 = (double)pb.x, b1 = (double)pb.y, b2 = (double)pb.z;
    row[6] = __dadd_rn(__dmul_rn(-b2, t1), __dmul_rn(b1, t2));
    row[7] = __dadd_rn(__dmul_rn(b2, t0), __dmul_rn(-b0, t2));
    row[8] = __dadd_rn(__dmul_rn(-b1, t0), __dmul_rn(b0, t1));
    row[9] = C0; row[10] = C1; row[11] = C2;
  } else {
#pragma unroll
    for (int c = 6; c < 12; ++c) row[c] = 0.0;
  }
  row[12] = -(double)nv.w;
}

// Stage A of h_share_model for one point (laserMapping.cpp:1903-1938). Returns selected flag; fills nv.
__device__ __forceinline__ bool select_point(const MeasArgs& a, int i, int search, const float4 pw, float4& nv) {
  bool sel;
  if (search) {
    const int c = a.cnt[i];
    const float d4 = a.nbr[(size_t)4 * a.stride + i].w;
    sel = (c < 5) ? false : (d4 > 5.f ? false : true);        // :1911
  } else {
    sel = a.sel[i] != 0 && a.cnt[i] >= 5;   // (cnt is cleared per scan: a cached pass without a preceding search selects nothing)
  }
  if (!sel) return false;
  float pa, pb_, pc, pd;
  if (search) {
    float P[5][3];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const float4 q = a.nbr[(size_t)j * a.stride + i];
      P[j][0] = q.x; P[j][1] = q.y; P[j][2] = q.z;
    }
    if (!esti_plane_dev(P, 0.1f, pa, pb_, pc, pd)) return false;
    a.plane[i] = make_float4(pa, pb_, pc, pd);
  } else {
    // same Nearest_Points as the last search pass => esti_plane (laserMapping.cpp:1922) returns the same plane: sel[i]
    // can only still be set if that fit was accepted, so the cached coefficients are exactly what it would recompute
    const float4 pl = a.plane[i];
    pa = pl.x; pb_ = pl.y; pc = pl.z; pd = pl.w;
  }
  const float4 pb = (a.ctl ? a.ctl->body : a.body)[i];
  const float pd2 = pa * pw.x + pb_ * pw.y + pc * pw.z + pd;  // :1925 (float, left to right)
  const double bn = sqrt((double)pb.x * (double)pb.x + (double)pb.y * (double)pb.y + (double)pb.z * (double)pb.z);
  const float sc = (float)(1.0 - 0.9 * (double)fabsf(pd2) / sqrt(bn));  // :1927
  if (!((double)sc > 0.9)) return false;
  nv = make_float4(pa, pb_, pc, pd2);
  return true;
}

template <bool EXTR>
constexpr int meas_smem_bytes() { return (meas_threads<EXTR>() / 32) * 32 * (EXTR ? 13 : 7) * (int)sizeof(double); }

template <bool EXTR>
__global__ void __launch_bounds__(meas_threads<EXTR>()) k_residual(MeasArgs a) {
  pdl_sync();
  constexpr int W = EXTR ? 13 : 7;               // augmented row width [cols..., h]
  constexpr int NE = W * (W + 1) / 2;            // 91 or 28
  constexpr int EPL = (NE + 31) / 32;            // entries per lane
  // dynamic shared memory (meas_smem_bytes): the per-warp row tiles; reused for the per-warp totals after the loop
  extern __shared__ double meas_smem[];
  double (*tile)[32][W] = reinterpret_cast<double (*)[32][W]>(meas_smem);
  double (*wacc)[96] = reinterpret_cast<double (*)[96]>(meas_smem);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc[EPL];
#pragma unroll
  for (int e = 0; e < EPL; ++e) acc[e] = 0.0;
  double rsum = 0.0;
  int msum = 0;
  FLB_TRACE_BEGIN(4 * 8 + (a.ctl ? a.ctl->it + 1 : 0));
  if (a.ctl && !ctl_pass_active(a.ctl)) return;   // the iterated update already finished (block-uniform)
  const int search = a.ctl ? a.ctl->converge : a.search;
  const PoseDev pose = a.ctl ? a.ctl->pose : a.pose;
  const float4* __restrict__ body = a.ctl ? a.ctl->body : a.body;
  const int n = a.ctl ? a.ctl->n : a.n;
  const int stride = gridDim.x * blockDim.x;
  const int nround = (n + stride - 1) / stride;
  for (int it = 0; it < nround; ++it) {
    const int i = it * stride + blockIdx.x * blockDim.x + threadIdx.x;
    float4 nv = make_float4(0.f, 0.f, 0.f, 0.f);
    bool sel = false;
    if (i < n) {
      float4 pw;
      if (a.ctl) { pw = body_to_world(pose, body[i]); a.world_out[i] = pw; }
      else pw = a.world[i];
      sel = select_point(a, i, search, pw, nv);
      a.sel[i] = sel ? 1 : 0;
      if (sel) a.normvec[i] = nv;
    }
    double row[13];
    if (sel) jacobian_row<EXTR>(pose, body[i], nv, row);
    const unsigned any = __ballot_sync(FULL, sel);
    if (any == 0u) continue;
    if (EXTR) {
#pragma unroll
      for (int c = 0; c < 13; ++c) tile[warp][lane][c] = sel ? row[c] : 0.0;
    } else {
#pragma unroll
      for (int c = 0; c < 6; ++c) tile[warp][lane][c] = sel ? row[c] : 0.0;
      tile[warp][lane][6] = sel ? row[12] : 0.0;
    }
    if (sel) { rsum += (double)fabsf(nv.w); ++msum; }
    __syncwarp();
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const int ent = lane + 32 * e;
      if (ent < NE) {
        int ci, cj;
        if (EXTR) { ci = c_tri_i[ent]; cj = c_tri_j[ent]; }
        else {
          // upper triangle of 7x7 enumerated row by row
          int r = 0, rem = ent;
          while (rem >= 7 - r) { rem -= 7 - r; ++r; }
          ci = r; cj = r + rem;
        }
        double s = 0.0;
#pragma unroll 8
        for (int r = 0; r < 32; ++r) s += tile[warp][r][ci] * tile[warp][r][cj];
        acc[e] += s;
      }
    }
    __syncwarp();
  }
  // warp totals of rsum / msum (fixed butterfly order)
  for (int o = 16; o; o >>= 1) {
    rsum += __shfl_xor_sync(FULL, rsum, o);
    msum += __shfl_xor_sync(FULL, msum, o);
  }
  __syncthreads();   // every warp is done with its tile: the region now holds the per-warp totals
  for (int e = lane; e < NACC; e += 32) wacc[warp][e] = 0.0;
  __syncwarp();
#pragma unroll
  for (int e = 0; e < EPL; ++e) {
    const int ent = lane + 32 * e;
    if (ent < NE) {
      int slot;
      if (EXTR) slot = ent;
      else {
        int r = 0, rem = ent;
        while (rem >= 7 - r) { rem -= 7 - r; ++r; }
        const int ci = r, cj = r + rem;
        // map the 7-wide indices (0..5 cols, 6 = h) into the 13-wide triangle
        const int gi = ci == 6 ? 12 : ci, gj = cj == 6 ? 12 : cj;
        slot = gi * 13 - gi * (gi - 1) / 2 + (gj - gi);
      }
      wacc[warp][slot] = acc[e];
    }
  }
  if (lane == 0) { wacc[warp][91] = rsum; wacc[warp][92] = (double)msum; }
  __syncthreads();
  for (int e = threadIdx.x; e < NACC; e += blockDim.x) {
    double s = 0.0;
    for (int w = 0; w < meas_threads<EXTR>() / 32; ++w) s += wacc[w][e];
    a.partial[(size_t)blockIdx.x * NACC + e] = s;
  }
  FLB_TRACE_END(4 * 8 + (a.ctl ? a.ctl->it + 1 : 0));
}

// K2: fixed-order final reduction of the per-block partials -> out[NACC]
__global__ void k_reduce_final(const double* __restrict__ partial, int nblocks, double* __restrict__ out) {
  __shared__ double sm[4][NACC];
  const int e = threadIdx.x % 96, part = threadIdx.x / 96;  // 384 threads: 4 slices of the block range
  double s = 0.0;
  if (e < NACC)
    for (int b = part; b < nblocks; b += 4) s += partial[(size_t)b * NACC + e];
  if (e < NACC) sm[part][e] = s;
  __syncthreads();
  if (part == 0 && e < NACC) out[e] = ((sm[0][e] + sm[1][e]) + sm[2][e]) + sm[3][e];
}

// Exact rows for boundary B1: compacted in index order (offs = exclusive scan of sel), h_x COLUMN-major M x 12 (ld).
template <bool EXTR>
__global__ void k_rows(MeasArgs a, const int* __restrict__ offs, double* __restrict__ hx, int ld, double* __restrict__ h, int cap) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    if (!a.sel[i]) continue;
    const int r = offs[i];
    if (r >= cap) continue;
    double row[13];
    jacobian_row<EXTR>(a.pose, a.body[i], a.normvec[i], row);
#pragma unroll
    for (int c = 0; c < 12; ++c) hx[(size_t)c * ld + r] = row[c];
    h[r] = row[12];
  }
}
__global__ void k_sel_to_int(const unsigned char* __restrict__ sel, int* __restrict__ out, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = sel[i] ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------- map_incremental classifier
// laserMapping.cpp:1440-1490. cls: 0 dropped, 1 PointToAdd (downsample), 2 PointNoNeedDownsample.
// counts[0] += #ToAdd, counts[1] += #NoNeed.
// Fused with the first two steps of the insert (K3a touch_block: make sure the block of every point to be added exists;
// K3c scatter: per-voxel best new point of the downsampled class into the scratch hash) when a scratch hash is passed:
// both only need the point and its class, so the points are read once and two launches disappear from the scan's tail.
__global__ void k_classify(PoseDev s_in, const EsikfCtl* ctl, const float4* body, const float4* __restrict__ nbr,
                           const unsigned char* __restrict__ cnt, int n_in, int nbr_stride, int flg_in, double fs,
                           float4* __restrict__ world, unsigned char* __restrict__ cls, int* counts, MapDev m, uint64_t* skeys,
                           unsigned long long* sbest, uint32_t smask) {
  pdl_sync();
  FLB_TRACE_BEGIN(6 * 8);
  if (ctl && ctl->need_host) return;  // the host fallback redoes update + insert for this scan
  const PoseDev s = ctl ? ctl->pose : s_in;
  if (ctl) body = ctl->body;
  const int n = ctl ? ctl->n : n_in;
  const int flg_EKF_inited = ctl ? ctl->flg_inited : flg_in;
  const int lane = threadIdx.x & 31;
  const int stride = gridDim.x * blockDim.x;
  const int nround = (n + stride - 1) / stride;
  for (int it = 0; it < nround; ++it) {
    const int i = it * stride + blockIdx.x * blockDim.x + threadIdx.x;
    int c = 0;
    if (i < n) {
      const float4 pw = body_to_world(s, body[i]);
      world[i] = pw;
      const int k = cnt[i];
      if (k > 0 && flg_EKF_inited) {
        const float hf_x = (float)(floor((double)pw.x / fs) * fs + 0.5 * fs);   // :1459-1461, double arithmetic
        const float hf_y = (float)(floor((double)pw.y / fs) * fs + 0.5 * fs);
        const float hf_z = (float)(floor((double)pw.z / fs) * fs + 0.5 * fs);
        const float dist = sqdist(pw.x, pw.y, pw.z, hf_x, hf_y, hf_z);
        const float4 n0 = nbr[i];
        const double half = 0.5 * fs;
        if ((double)fabsf(n0.x - hf_x) > half && (double)fabsf(n0.y - hf_y) > half && (double)fabsf(n0.z - hf_z) > half) {
          c = 2;
        } else {
          bool need_add = true;
          if (k >= 5) {
#pragma unroll
            for (int j = 0; j < 5; ++j) {
              const float4 q = nbr[(size_t)j * nbr_stride + i];
              if (sqdist(q.x, q.y, q.z, hf_x, hf_y, hf_z) < dist) { need_add = false; break; }
            }
          }
          c = need_add ? 1 : 0;
        }
      } else {
        c = 1;
      }
      cls[i] = (unsigned char)c;
      if (skeys && c != 0) {
        if (!coord_ok(pw.x, pw.y, pw.z, m.ds)) atomicOr(&m.counters[CNT_ERROR], ERR_RANGE);
        else {
          const int vx = voxel_of(pw.x, m.ds), vy = voxel_of(pw.y, m.ds), vz = voxel_of(pw.z, m.ds);
          touch_block(m, pack_key(vx >> 2, vy >> 2, vz >> 2), vx >> 2, vy >> 2, vz >> 2);
          if (c == 1) ds_scatter_one(m, pw, i, pack_key(vx, vy, vz), skeys, sbest, smask);
        }
      }
    }
    const unsigned b1 = __ballot_sync(FULL, c == 1), b2 = __ballot_sync(FULL, c == 2);
    if (lane == 0) {
      if (b1) atomicAdd(&counts[0], __popc(b1));
      if (b2) atomicAdd(&counts[1], __popc(b2));
    }
  }
  FLB_TRACE_END(6 * 8);
}

}  // namespace flb

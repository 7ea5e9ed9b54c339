// lio_gpu_frontend.hpp — drop-in bodies for the hot functions of src/laserMapping.cpp, keeping the
// esekfom::esekf callback signature  void h_share_model(state_ikfom&, esekfom::dyn_share_datastruct<double>&)
// (esekfom.hpp:130, registered at laserMapping.cpp:2151) so that include/IKFoM_toolkit stays byte-identical.
//
//   flb::LioGpu gpu;                                   // next to `KD_TREE<PointType> ikdtree;` (laserMapping.cpp:116)
//   gpu.attach(ikdtree.handle(), extrinsic_est_en, NUM_MAX_ITERATIONS, filter_size_map_min);
//   ... per scan, after downSizeFilterSurf.filter(*feats_down_body) (laserMapping.cpp:2323):
//   gpu.begin_scan(&feats_down_body->points[0].x, feats_down_size, sizeof(PointType));
//   void h_share_model(state_ikfom& s, esekfom::dyn_share_datastruct<double>& d) { gpu.h_share_model(s, d); }
//   void map_incremental() { gpu.map_incremental(state_point, flg_EKF_inited); }
//
// The templates only need the member names of state_ikfom (use-ikfom.hpp:21-30) and dyn_share_datastruct
// (esekfom.hpp:79-89: valid, converge, h_x, h) — Eigen itself is not included here.
#pragma once
#include <cmath>
#include <cstdio>
#include <vector>

#include "../fastlio_b200.h"

namespace flb {

template <class State>
inline void pack_state26(const State& s, double* o) {
  for (int i = 0; i < 3; ++i) {
    o[i] = s.pos[i]; o[11 + i] = s.offset_T_L_I[i]; o[14 + i] = s.vel[i]; o[17 + i] = s.bg[i]; o[20 + i] = s.ba[i]; o[23 + i] = s.grav[i];
  }
  for (int i = 0; i < 4; ++i) { o[3 + i] = s.rot.coeffs()[i]; o[7 + i] = s.offset_R_L_I.coeffs()[i]; }  // Eigen order x,y,z,w
}

// the inverse of pack_state26 (grav is MTK::S2's public `vec`)
template <class State>
inline void unpack_state26(const double* o, State& s) {
  for (int i = 0; i < 3; ++i) {
    s.pos[i] = o[i]; s.offset_T_L_I[i] = o[11 + i]; s.vel[i] = o[14 + i]; s.bg[i] = o[17 + i]; s.ba[i] = o[20 + i]; s.grav.vec[i] = o[23 + i];
  }
  for (int i = 0; i < 4; ++i) { s.rot.coeffs()[i] = o[3 + i]; s.offset_R_L_I.coeffs()[i] = o[7 + i]; }
}

class LioGpu {
 public:
  enum RowMode { EXACT_ROWS /* boundary B1 */, COMPRESSED_ROWS /* boundary B2 */ };
  ~LioGpu() { if (ses_) flb_session_destroy(ses_); }

  bool attach(flb_map* map, bool extrinsic_est_en, int max_iterations, double filter_size_map_min, int max_scan_points = 262144) {
    flb_session_config c;
    flb_session_default_config(&c);
    c.extrinsic_est_en = extrinsic_est_en ? 1 : 0;
    c.max_iterations = max_iterations;
    c.filter_size_map_min = filter_size_map_min;
    c.max_scan_points = max_scan_points;
    if (flb_session_create(map, &c, &ses_)) { std::fprintf(stderr, "[fastlio_b200] %s\n", flb_last_error()); ses_ = nullptr; return false; }
    return true;
  }
  void set_row_mode(RowMode m) { mode_ = m; }

  // feats_down_body (laserMapping.cpp:2322-2325).  off_intensity: byte offset of PointType::intensity inside a record
  // (offsetof(PointType, intensity)); the intensity then travels with the point into the map, as pointBodyToWorld copies it
  // (laserMapping.cpp:1101-1110).  < 0: xyz only.
  bool begin_scan(const float* first_xyz, int n, int stride_bytes, int off_intensity = -1) {
    n_ = n;
    if (flb_scan_upload_pt(ses_, first_xyz, n, stride_bytes, off_intensity)) { std::fprintf(stderr, "[fastlio_b200] %s\n", flb_last_error()); return false; }
    return true;
  }

  // Body of h_share_model (laserMapping.cpp:1876-2004).
  template <class State, class DynShare>
  void h_share_model(State& s, DynShare& ekfom_data) {
    double st[FLB_STATE_DIM];
    pack_state26(s, st);
    flb_pass_result r;
    if (flb_pass(ses_, st, ekfom_data.converge ? 1 : 0, &r)) {
      std::fprintf(stderr, "[fastlio_b200] h_share_model: %s\n", flb_last_error());
      ekfom_data.valid = false;  // the reference's only failure signal on this path (laserMapping.cpp:1956-1961)
      return;
    }
    effct_feat_num = r.effct_feat_num;
    total_residual = r.total_residual;
    res_mean_last = r.effct_feat_num > 0 ? r.total_residual / r.effct_feat_num : 0.0;
    if (!r.valid) { ekfom_data.valid = false; return; }
    const int M = r.effct_feat_num;
    if (mode_ == EXACT_ROWS || M < FLB_STATE_DOF) {
      // B1: the exact M x 12 rows (column-major, the layout of Eigen::MatrixXd) and h = -pd2
      ekfom_data.h_x.resize(M, 12);
      ekfom_data.h.resize(M);
      int Mo = 0;
      if (flb_pass_rows(ses_, ekfom_data.h_x.data(), M, ekfom_data.h.data(), M, &Mo) || Mo != M) {
        std::fprintf(stderr, "[fastlio_b200] h_share_model rows: %s\n", flb_last_error());
        ekfom_data.valid = false;
      }
      return;
    }
    // B2: any h_x' with h_x'^T h_x' = H^T H and h_x'^T h' = H^T h gives the same update when rows >= 23
    // (esekfom.hpp:1788-1815 only uses those products).  h_x' = upper Cholesky factor U of H^T H padded to 24 rows,
    // h' = U^-T (H^T h).
    double U[144] = {0};
    for (int i = 0; i < 12; ++i) {
      for (int j = i; j < 12; ++j) {
        double sum = r.HTH[i * 12 + j];
        for (int k = 0; k < i; ++k) sum -= U[k * 12 + i] * U[k * 12 + j];
        if (i == j) U[i * 12 + i] = sum > 0 ? std::sqrt(sum) : 0.0;
        else U[i * 12 + j] = U[i * 12 + i] > 0 ? sum / U[i * 12 + i] : 0.0;
      }
    }
    double y[12];
    for (int i = 0; i < 12; ++i) {
      double sum = r.HTh[i];
      for (int k = 0; k < i; ++k) sum -= U[k * 12 + i] * y[k];
      y[i] = U[i * 12 + i] > 0 ? sum / U[i * 12 + i] : 0.0;
    }
    const int R = 24;
    ekfom_data.h_x.resize(R, 12);
    ekfom_data.h.resize(R);
    double* hx = ekfom_data.h_x.data();
    double* h = ekfom_data.h.data();
    for (int c = 0; c < 12; ++c)
      for (int rr = 0; rr < R; ++rr) hx[c * R + rr] = rr < 12 ? U[rr * 12 + c] : 0.0;
    for (int rr = 0; rr < R; ++rr) h[rr] = rr < 12 ? y[rr] : 0.0;
  }

  // Body of map_incremental (laserMapping.cpp:1440-1496)
  template <class State>
  int map_incremental(const State& s, bool flg_EKF_inited) {
    double st[FLB_STATE_DIM];
    pack_state26(s, st);
    int a = 0, b = 0;
    if (flb_map_incremental(ses_, st, flg_EKF_inited ? 1 : 0, &a, &b)) std::fprintf(stderr, "[fastlio_b200] map_incremental: %s\n", flb_last_error());
    return a + b;  // add_point_size (laserMapping.cpp:1494)
  }

  // Nearest_Points for callers that keep their own CPU map_incremental (laserMapping.cpp:1453-1481)
  int nearest_points(std::vector<float>& xyz5, std::vector<int>& counts) {
    xyz5.assign((size_t)n_ * 15, 0.f);
    counts.assign(n_, 0);
    return flb_neighbors_download(ses_, xyz5.data(), nullptr, counts.data(), nullptr, nullptr, nullptr);
  }

  flb_session* handle() { return ses_; }
  int effct_feat_num = 0;
  double total_residual = 0.0, res_mean_last = 0.0;

 private:
  flb_session* ses_ = nullptr;
  RowMode mode_ = EXACT_ROWS;
  int n_ = 0;
};

}  // namespace flb

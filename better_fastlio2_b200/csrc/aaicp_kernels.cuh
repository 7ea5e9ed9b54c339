// aaicp_kernels.cuh — the device side of the relocaliser's AA-ICP (AAICP::point_to_point_aaicp, include/FRICP-toolkit/
// ICP.h:841-1033, as Registeration::run calls it for regMode 1): two k_reduce ops over flb_keyframes_fricp's normalised
// source, sorted double target and 1-NN matches (fricp_kernels.cuh).  The search pass itself is fricp's k_fr_nn /
// k_fr_nn_far with the current transform.  In this algorithm the Kabsch step is taken on the moved source X = final X0
// (RigidMotionEstimator::point_to_point does not move X, ICP.h:120), so the ops recompute X with exactly the pass's
// arithmetic (fr_moved: ((m0 x + m1 y) + m2 z) + m3 per row, under -fmad=false).
#pragma once
#include "fricp_kernels.cuh"

namespace flb {

// The step record of one iteration (FR_RED doubles, fr_kabsch's layout): n, Σx, Σq, Σ x qᵀ (row-major) and the energy
// Σ |X - Q|² with |X - Q| = sqrt(d²) of the pass, squared again as get_energy's uniform_energy does.
struct AaStepOp {
  FrXf xf;
  const double4* x;
  const double4* pts;
  const int* pos;
  const double* d2;
  __device__ bool operator()(int i, double* a) const {
    const int p = pos[i];
    if (p < 0) return false;
    const double r = sqrt(d2[i]);
    const FrQuery m = fr_moved(xf, x[i]);
    const double4 t = pts[p];
    const double qt[3] = {t.x, t.y, t.z};
    a[0] = 1.0;
    for (int c = 0; c < 3; ++c) { a[1 + c] = m.q[c]; a[4 + c] = qt[c]; }
    for (int r0 = 0; r0 < 3; ++r0)
      for (int c = 0; c < 3; ++c) a[7 + 3 * r0 + c] = m.q[r0] * qt[c];
    a[16] = r * r;
    return true;
  }
};

// The convergence energy (ICP.h:1004-1005): Σ |final X0 - Q|² against the matches of the last pass, without a search.
// matched = 0 (no pass ran): Q is the zero matrix it was initialised to, the energy is Σ |X0|².
struct AaEnergyOp {
  FrXf xf;
  const double4* x;
  const double4* pts;
  const int* pos;
  int matched;
  __device__ bool operator()(int i, double* a) const {
    const double4 v = x[i];
    if (v.w == 0.0) return false;
    const FrQuery m = fr_moved(xf, v);
    double q[3] = {0.0, 0.0, 0.0};
    if (matched) {
      const double4 t = pts[pos[i]];
      q[0] = t.x; q[1] = t.y; q[2] = t.z;
    }
    const double dx = m.q[0] - q[0], dy = m.q[1] - q[1], dz = m.q[2] - q[2];
    const double w = sqrt((dx * dx + dy * dy) + dz * dz);
    a[0] = w * w;
    return true;
  }
};

}  // namespace flb

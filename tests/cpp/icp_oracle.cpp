// Sequential restatement of the loop-closure ICP contract (DESIGN.md §9, "Loop registration"): PCL 1.10's
// IterativeClosestPoint<PointType, PointType> with an identity guess, as flb_keyframes_icp implements it, on host clouds.
// Its own exact 1-NN (a plain k-d tree over the finite target points, float d² = (dx*dx + dy*dy) + dz*dz, ties to the
// lower target index), its own double 3x3 SVD (Jacobi eigen-decomposition of H^T H) and sequential double sums.
// Compiled by tests/icp_oracle.py with -ffp-contract=off.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

struct Tree {
  const float* p = nullptr;   // x, y, z, w per point
  std::vector<int> idx;       // finite target points, permuted into the tree
  struct Node { int b, e, axis, left, right; float split; };
  std::vector<Node> nodes;

  int build(int b, int e) {
    Node nd{b, e, -1, -1, -1, 0.f};
    const int id = (int)nodes.size();
    nodes.push_back(nd);
    if (e - b <= 8) return id;
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = b; i < e; ++i)
      for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], p[4 * idx[i] + a]); hi[a] = std::max(hi[a], p[4 * idx[i] + a]); }
    int axis = 0;
    for (int a = 1; a < 3; ++a) if (hi[a] - lo[a] > hi[axis] - lo[axis]) axis = a;
    const int mid = (b + e) / 2;
    std::nth_element(idx.begin() + b, idx.begin() + mid, idx.begin() + e,
                     [&](int x, int y) { return p[4 * x + axis] < p[4 * y + axis]; });
    const float split = p[4 * idx[mid] + axis];
    const int l = build(b, mid), r = build(mid, e);
    nodes[id].axis = axis;
    nodes[id].split = split;   // left: coordinate <= split, right: >= split
    nodes[id].left = l;
    nodes[id].right = r;
    return id;
  }
  void init(const float* pts, int n) {
    p = pts;
    for (int i = 0; i < n; ++i)
      if (std::isfinite(pts[4 * i]) && std::isfinite(pts[4 * i + 1]) && std::isfinite(pts[4 * i + 2])) idx.push_back(i);
    nodes.clear();
    if (!idx.empty()) build(0, (int)idx.size());
  }
  void search(int id, const float* q, float& best, int& bi) const {
    const Node& nd = nodes[id];
    if (nd.axis < 0) {
      for (int i = nd.b; i < nd.e; ++i) {
        const int j = idx[i];
        const float dx = p[4 * j] - q[0], dy = p[4 * j + 1] - q[1], dz = p[4 * j + 2] - q[2];
        const float d2 = (dx * dx + dy * dy) + dz * dz;
        if (d2 < best || (d2 == best && j < bi)) { best = d2; bi = j; }
      }
      return;
    }
    const float diff = q[nd.axis] - nd.split;
    const int near = diff <= 0 ? nd.left : nd.right, far = diff <= 0 ? nd.right : nd.left;
    search(near, q, best, bi);
    if (!(diff * diff > best)) search(far, q, best, bi);   // every far point is at least |diff| away along the axis
  }
  // exact nearest finite target point of q: index (-1: none) and float d²
  int nearest(const float* q, float* d2) const {
    float best = INFINITY;
    int bi = INT32_MAX;
    if (!nodes.empty()) search(0, q, best, bi);
    *d2 = best;
    return nodes.empty() ? -1 : bi;
  }
};

bool finite3(const float* q) { return std::isfinite(q[0]) && std::isfinite(q[1]) && std::isfinite(q[2]); }

void apply(const float* T, const float* in, float* out, int n) {   // transformPointCloud with a float 4x4
  for (int i = 0; i < n; ++i) {
    const float x = in[4 * i], y = in[4 * i + 1], z = in[4 * i + 2];
    for (int r = 0; r < 3; ++r) out[4 * i + r] = ((T[4 * r] * x + T[4 * r + 1] * y) + T[4 * r + 2] * z) + T[4 * r + 3];
    out[4 * i + 3] = in[4 * i + 3];
  }
}

void mul4(const float* A, const float* B, float* C) {
  float o[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) o[4 * r + c] = ((A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c]) + A[4 * r + 2] * B[8 + c]) + A[4 * r + 3] * B[12 + c];
  std::memcpy(C, o, sizeof(o));
}

// symmetric 3x3 Jacobi: M = V diag(l) V^T
void jacobi_eig(double M[9], double V[9], double l[3]) {
  for (int i = 0; i < 9; ++i) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 100; ++sweep) {
    const double off = M[1] * M[1] + M[2] * M[2] + M[5] * M[5];
    const double diag = M[0] * M[0] + M[4] * M[4] + M[8] * M[8];
    if (off <= 1e-32 * diag || off == 0.0) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = M[3 * p + q];
        if (apq == 0.0) continue;
        const double theta = (M[3 * q + q] - M[3 * p + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) {   // M <- J^T M J
          const double mkp = M[3 * k + p], mkq = M[3 * k + q];
          M[3 * k + p] = c * mkp - s * mkq;
          M[3 * k + q] = s * mkp + c * mkq;
        }
        for (int k = 0; k < 3; ++k) {
          const double mpk = M[3 * p + k], mqk = M[3 * q + k];
          M[3 * p + k] = c * mpk - s * mqk;
          M[3 * q + k] = s * mpk + c * mqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = V[3 * k + p], vkq = V[3 * k + q];
          V[3 * k + p] = c * vkp - s * vkq;
          V[3 * k + q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < 3; ++i) l[i] = M[4 * i];
}

double det3(const double* M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

// H = U S V^T through H^T H = V S² V^T, u_i = H v_i / s_i; R = U diag(1, 1, det U det V < 0 ? -1 : 1) V^T
void rotation(const double H[9], double R[9]) {
  double M[9], V0[9], l[3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) M[3 * r + c] = H[r] * H[c] + H[3 + r] * H[3 + c] + H[6 + r] * H[6 + c];
  jacobi_eig(M, V0, l);
  int o[3] = {0, 1, 2};
  std::sort(o, o + 3, [&](int a, int b) { return l[a] > l[b]; });
  double V[9], U[9], s[3];
  for (int j = 0; j < 3; ++j) {
    s[j] = std::sqrt(std::max(l[o[j]], 0.0));
    for (int r = 0; r < 3; ++r) V[3 * r + j] = V0[3 * r + o[j]];
  }
  const double tiny = std::max(s[0], 1e-300) * 1e-7;   // s from s² loses half the digits
  for (int j = 0; j < 3; ++j) {
    double u[3] = {0, 0, 0}, nu = 0;
    for (int r = 0; r < 3; ++r) { u[r] = H[3 * r] * V[j] + H[3 * r + 1] * V[3 + j] + H[3 * r + 2] * V[6 + j]; nu += u[r] * u[r]; }
    nu = std::sqrt(nu);
    for (int r = 0; r < 3; ++r) U[3 * r + j] = (s[j] > tiny && nu > 0) ? u[r] / nu : 0.0;
  }
  if (!(s[2] > tiny)) {   // the third left vector completes the basis
    U[2] = U[3] * U[7] - U[6] * U[4];
    U[5] = U[6] * U[1] - U[0] * U[7];
    U[8] = U[0] * U[4] - U[3] * U[1];
  }
  const double d = det3(U) * det3(V) < 0 ? -1.0 : 1.0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[3 * r + c] = U[3 * r] * V[3 * c] + U[3 * r + 1] * V[3 * c + 1] + d * U[3 * r + 2] * V[3 * c + 2];
}

}  // namespace

extern "C" {

// info: converged, iterations, state, n_correspondences; log: per iteration cos_angle, |t|², mse, previous mse (up to
// max(max_iter, 1) rows); corr_idx / corr_d2 (n_s each): the last iteration's nearest target and d² (-1 / inf: none).
int orc_icp(const float* src, int n_s, const float* tgt, int n_t, double max_dist, int max_iter, double teps, double feps,
            float* final16, int* info, double* fitness, int* corr_idx, float* corr_d2, double* log) {
  for (int i = 0; i < 16; ++i) final16[i] = (i % 5 == 0) ? 1.f : 0.f;
  info[0] = 0; info[1] = 0; info[2] = 0; info[3] = 0;
  *fitness = DBL_MAX;
  for (int i = 0; i < n_s; ++i) { corr_idx[i] = -1; corr_d2[i] = INFINITY; }
  Tree tree;
  tree.init(tgt, n_t);
  if (n_s == 0 || tree.idx.empty()) return 0;   // initCompute fails
  std::vector<float> x(src, src + 4 * (size_t)n_s);
  const double max_d2 = max_dist * max_dist;
  float final_T[16], T[16];
  std::memcpy(final_T, final16, sizeof(final_T));
  double prev = DBL_MAX;
  for (int it = 0;; ++it) {
    // determineCorrespondences
    std::vector<int> ps, pt;
    std::vector<float> pd;
    for (int i = 0; i < n_s; ++i) {
      const float* q = &x[4 * (size_t)i];
      if (!finite3(q)) { corr_idx[i] = -1; corr_d2[i] = INFINITY; continue; }
      float d2;
      const int j = tree.nearest(q, &d2);
      corr_idx[i] = j;
      corr_d2[i] = d2;
      if ((double)d2 <= max_d2) { ps.push_back(i); pt.push_back(j); pd.push_back(d2); }
    }
    const int n = (int)ps.size();
    info[3] = n;
    if (n < 3) { info[2] = 5; info[0] = 0; break; }
    // Umeyama: means, then demeaned cross-covariance, sequential double sums
    double ms[3] = {0, 0, 0}, mt[3] = {0, 0, 0};
    for (int k = 0; k < n; ++k)
      for (int a = 0; a < 3; ++a) { ms[a] += x[4 * (size_t)ps[k] + a]; mt[a] += tgt[4 * (size_t)pt[k] + a]; }
    for (int a = 0; a < 3; ++a) { ms[a] /= n; mt[a] /= n; }
    double H[9] = {0};
    for (int k = 0; k < n; ++k) {
      double ds[3], dt[3];
      for (int a = 0; a < 3; ++a) { ds[a] = x[4 * (size_t)ps[k] + a] - ms[a]; dt[a] = tgt[4 * (size_t)pt[k] + a] - mt[a]; }
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) H[3 * r + c] += dt[r] * ds[c];
    }
    double R[9];
    rotation(H, R);
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) T[4 * r + c] = (float)R[3 * r + c];
      T[4 * r + 3] = (float)(mt[r] - (R[3 * r] * ms[0] + R[3 * r + 1] * ms[1] + R[3 * r + 2] * ms[2]));
    }
    T[12] = T[13] = T[14] = 0.f;
    T[15] = 1.f;
    apply(T, x.data(), x.data(), n_s);
    mul4(T, final_T, final_T);
    info[1] = it + 1;
    // DefaultConvergenceCriteria
    const double cosa = 0.5 * ((double)T[0] + (double)T[5] + (double)T[10] - 1.0);
    const double tr2 = (double)T[3] * T[3] + (double)T[7] * T[7] + (double)T[11] * T[11];
    double sd = 0;
    for (int k = 0; k < n; ++k) sd += pd[k];
    const double mse = sd / n;
    if (it < std::max(max_iter, 1)) { log[4 * it] = cosa; log[4 * it + 1] = tr2; log[4 * it + 2] = mse; log[4 * it + 3] = prev; }
    int state = 0;
    if (info[1] >= max_iter) state = 1;
    else if (cosa >= 1.0 - teps && tr2 <= teps) state = 2;
    else if (std::fabs(mse - prev) < 1e-12) state = 3;
    else if (std::fabs(mse - prev) / prev < feps) state = 4;
    else prev = mse;
    if (state) { info[0] = 1; info[2] = state; break; }
  }
  std::memcpy(final16, final_T, sizeof(final_T));
  // getFitnessScore
  std::vector<float> y(4 * (size_t)n_s);
  apply(final_T, src, y.data(), n_s);
  double sum = 0;
  long long cnt = 0;
  for (int i = 0; i < n_s; ++i) {
    if (!finite3(&y[4 * (size_t)i])) continue;
    float d2;
    tree.nearest(&y[4 * (size_t)i], &d2);
    if ((double)d2 <= DBL_MAX) { sum += d2; ++cnt; }
  }
  *fitness = cnt > 0 ? sum / cnt : DBL_MAX;
  return 0;
}

// exact 1-NN of every query (the oracle's tree alone): index (-1: none or non-finite query) and d²
int orc_nn(const float* q, int n_q, const float* tgt, int n_t, int* idx, float* d2) {
  Tree tree;
  tree.init(tgt, n_t);
  for (int i = 0; i < n_q; ++i) {
    if (!finite3(&q[4 * (size_t)i])) { idx[i] = -1; d2[i] = INFINITY; continue; }
    idx[i] = tree.nearest(&q[4 * (size_t)i], &d2[i]);
  }
  return 0;
}

}  // extern "C"

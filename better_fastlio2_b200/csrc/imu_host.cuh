// imu_host.cuh — C-ABI entry points of ImuProcess (src/IMU_Processing.hpp) on a front end.  IMU_init (:174-233) and the
// MAX_INI_COUNT logic of Process (:393-427) stay on the host: a running mean over the first few scans, sequential and
// exact there.  The forward propagation runs in k_imu_propagate (imu_kernels.cuh); the undistortion and the voxel filter
// follow on the same stream, and the call ends in one synchronisation.
// Included at the end of fastlio_b200.cu (uses its flb_frontend definition and error helpers).
#pragma once
#include "imu_kernels.cuh"

constexpr int IMU_MAX_INI_COUNT = 10;   // MAX_INI_COUNT, IMU_Processing.hpp:4
constexpr int IMU_STAGE_DOUBLES = 26 + NDOF * NDOF + MAX_IMU_POSES * IMU_SAMPLE_DOUBLES;

struct flb_imu {
  flb_frontend* fe = nullptr;
  flb_map* map = nullptr;                 // referenced (as the front end does): destroying it never needs the front end
  flb_imu_config cfg{};
  double mean_acc[3] = {0, 0, -1.0}, mean_gyr[3] = {0, 0, 0};
  double cov_acc[3] = {0.1, 0.1, 0.1}, cov_gyr[3] = {0.1, 0.1, 0.1};   // ImuProcess() (:68-69)
  double Qd[12] = {1e-4, 1e-4, 1e-4, 1e-4, 1e-4, 1e-4, 1e-5, 1e-5, 1e-5, 1e-5, 1e-5, 1e-5};   // process_noise_cov()
  double angvel_last[3] = {0, 0, 0};
  double acc_s_last[3] = {0, 0, 0};       // uninitialised in the reference until the first propagation
  double last_imu[IMU_SAMPLE_DOUBLES] = {0, 0, 0, 0, 0, 0, 0};
  double last_lidar_end_time = 0.0;       // uninitialised in the reference until the first propagation
  int init_iter_num = 1;
  bool need_init = true, first_frame = true;
  int n_poses = 0;                        // IMUpose.size() of the last propagation (0 after Reset)
  double* d_in = nullptr;                 // [state26 | P | v_imu samples]
  double* h_in = nullptr;                 // pinned staging of d_in
  ImuRecord* d_rec = nullptr;
  ImuRecord* h_rec = nullptr;             // pinned read-back
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

extern "C" void flb_imu_default_config(flb_imu_config* c) {
  if (!c) return;
  *c = flb_imu_config{};
  for (int i = 0; i < 3; ++i) {
    c->Lidar_T_wrt_IMU[i] = 0.0;
    c->Lidar_R_wrt_IMU[4 * i] = 1.0;
    c->cov_gyr_scale[i] = 0.1;
    c->cov_acc_scale[i] = 0.1;
    c->cov_bias_gyr[i] = 0.0001;
    c->cov_bias_acc[i] = 0.0001;
  }
}

static int imu_check_config(const flb_imu_config* c) {
  struct F { const char* name; const double* v; int n; bool cov; };
  const F fs[] = {{"Lidar_T_wrt_IMU", c->Lidar_T_wrt_IMU, 3, false}, {"Lidar_R_wrt_IMU", c->Lidar_R_wrt_IMU, 9, false},
                  {"cov_gyr_scale", c->cov_gyr_scale, 3, true}, {"cov_acc_scale", c->cov_acc_scale, 3, true},
                  {"cov_bias_gyr", c->cov_bias_gyr, 3, true}, {"cov_bias_acc", c->cov_bias_acc, 3, true}};
  for (const F& f : fs)
    for (int i = 0; i < f.n; ++i) {
      if (!std::isfinite(f.v[i])) return set_err("flb_imu_config.%s[%d] is not finite", f.name, i);
      if (f.cov && f.v[i] < 0) return set_err("flb_imu_config.%s[%d] is negative", f.name, i);
    }
  const double* R = c->Lidar_R_wrt_IMU;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double d = R[3 * i] * R[3 * j] + R[3 * i + 1] * R[3 * j + 1] + R[3 * i + 2] * R[3 * j + 2] - (i == j ? 1.0 : 0.0);
      if (!(std::fabs(d) < 1e-6)) return set_err("flb_imu_config.Lidar_R_wrt_IMU is not a rotation (R R^T != I)");
    }
  return 0;
}

extern "C" void flb_imu_destroy(flb_imu* imu) {
  if (!imu) return;
  flb_map* m = imu->map;
  if (m) {
    Q(cudaSetDevice(m->cfg.device));
    Q(cudaStreamSynchronize(m->stream));
  }
  if (imu->d_in) Q(cudaFree(imu->d_in));
  if (imu->d_rec) Q(cudaFree(imu->d_rec));
  if (imu->h_in) Q(cudaFreeHost(imu->h_in));
  if (imu->h_rec) Q(cudaFreeHost(imu->h_rec));
  if (imu->ev0) Q(cudaEventDestroy(imu->ev0));
  if (imu->ev1) Q(cudaEventDestroy(imu->ev1));
  delete imu;
  if (m) map_release(m);
}

extern "C" int flb_imu_create(flb_frontend* fe, const flb_imu_config* cfg, flb_imu** out) {
  if (!fe || !cfg || !out) return set_err("flb_imu_create: null argument");
  *out = nullptr;
  if (imu_check_config(cfg)) return 1;
  CU(cudaSetDevice(fe->ses->map->cfg.device));
  flb_imu* imu = new (std::nothrow) flb_imu();
  if (!imu) return set_err("out of host memory");
  imu->cfg = *cfg;
  cudaError_t e = cudaMalloc((void**)&imu->d_in, sizeof(double) * IMU_STAGE_DOUBLES);
  if (e == cudaSuccess) e = cudaMalloc((void**)&imu->d_rec, sizeof(ImuRecord));
  if (e == cudaSuccess) e = cudaMallocHost((void**)&imu->h_in, sizeof(double) * IMU_STAGE_DOUBLES);
  if (e == cudaSuccess) e = cudaMallocHost((void**)&imu->h_rec, sizeof(ImuRecord));
  if (e == cudaSuccess) e = cudaEventCreate(&imu->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&imu->ev1);
  if (e != cudaSuccess) {
    cudaGetLastError();
    flb_imu_destroy(imu);
    return set_err("flb_imu_create: %s", cudaGetErrorString(e));
  }
  imu->fe = fe;
  imu->map = fe->ses->map;
  imu->map->refs++;
  *out = imu;
  return 0;
}

static void imu_reset(flb_imu* imu) {   // ImuProcess::Reset (:90-102)
  imu->mean_acc[0] = 0; imu->mean_acc[1] = 0; imu->mean_acc[2] = -1.0;
  for (int i = 0; i < 3; ++i) { imu->mean_gyr[i] = 0; imu->angvel_last[i] = 0; }
  imu->need_init = true;
  imu->init_iter_num = 1;
  for (double& v : imu->last_imu) v = 0;
  imu->n_poses = 0;
}

extern "C" int flb_imu_reset(flb_imu* imu) {
  if (!imu) return set_err("null IMU processor");
  imu_reset(imu);
  return 0;
}

// Eigen's Quaternion from a rotation matrix (QuaternionBase::operator=(MatrixBase), the trace / largest-diagonal branches)
static void quat_from_matrix(const double* m, double* q /* x,y,z,w */) {
  const double t = m[0] + m[4] + m[8];
  if (t > 0) {
    double s = std::sqrt(t + 1.0);
    q[3] = 0.5 * s;
    s = 0.5 / s;
    q[0] = (m[7] - m[5]) * s;
    q[1] = (m[2] - m[6]) * s;
    q[2] = (m[3] - m[1]) * s;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[3 * i + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double s = std::sqrt(m[3 * i + i] - m[3 * j + j] - m[3 * k + k] + 1.0);
    q[i] = 0.5 * s;
    s = 0.5 / s;
    q[3] = (m[3 * k + j] - m[3 * j + k]) * s;
    q[j] = (m[3 * j + i] + m[3 * i + j]) * s;
    q[k] = (m[3 * k + i] + m[3 * i + k]) * s;
  }
}

static double imu_norm3(const double* v) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

// IMU_init (:174-233) and the rest of Process's initialisation branch (:405-427)
static void imu_init(flb_imu* imu, const double* imu7, int n_imu, double* x, double* P) {
  int N = imu->init_iter_num;
  if (imu->first_frame) {
    imu_reset(imu);
    N = 1;
    imu->first_frame = false;
    for (int i = 0; i < 3; ++i) { imu->mean_acc[i] = imu7[1 + i]; imu->mean_gyr[i] = imu7[4 + i]; }
  }
  for (int s = 0; s < n_imu; ++s) {
    const double* r = imu7 + (size_t)s * IMU_SAMPLE_DOUBLES;
    for (int i = 0; i < 3; ++i) {
      const double ca = r[1 + i], cg = r[4 + i];
      imu->mean_acc[i] += (ca - imu->mean_acc[i]) / N;
      imu->mean_gyr[i] += (cg - imu->mean_gyr[i]) / N;
      const double da = ca - imu->mean_acc[i], dg = cg - imu->mean_gyr[i];
      imu->cov_acc[i] = imu->cov_acc[i] * (N - 1.0) / N + da * da * (N - 1.0) / (N * N);
      imu->cov_gyr[i] = imu->cov_gyr[i] * (N - 1.0) / N + dg * dg * (N - 1.0) / (N * N);
    }
    N++;
  }
  // grav = S2(-mean_acc / |mean_acc| * G_m_s2): the S2 constructor normalises, then scales to 98090 / 10000
  const double na = imu_norm3(imu->mean_acc);
  double g[3];
  for (int i = 0; i < 3; ++i) g[i] = -imu->mean_acc[i] / na * IMU_G_M_S2;
  const double ng = imu_norm3(g);
  for (int i = 0; i < 3; ++i) x[23 + i] = g[i] / ng * (98090.0 / 10000.0);
  for (int i = 0; i < 3; ++i) { x[17 + i] = imu->mean_gyr[i]; x[11 + i] = imu->cfg.Lidar_T_wrt_IMU[i]; }
  quat_from_matrix(imu->cfg.Lidar_R_wrt_IMU, x + 7);
  for (int e = 0; e < NDOF * NDOF; ++e) P[e] = 0.0;
  static const double diag[NDOF] = {1, 1, 1, 1, 1, 1, 1e-5, 1e-5, 1e-5, 1e-5, 1e-5, 1e-5, 1, 1, 1,
                                    1e-4, 1e-4, 1e-4, 1e-3, 1e-3, 1e-3, 1e-5, 1e-5};
  for (int i = 0; i < NDOF; ++i) P[i * NDOF + i] = diag[i];
  imu->init_iter_num = N;
  for (int k = 0; k < IMU_SAMPLE_DOUBLES; ++k) imu->last_imu[k] = imu7[(size_t)(n_imu - 1) * IMU_SAMPLE_DOUBLES + k];
  if (imu->init_iter_num > IMU_MAX_INI_COUNT) {
    // cov_acc *= pow(G_m_s2 / |mean_acc|, 2) (:417) is overwritten by the next line of the reference: not restated
    imu->need_init = false;
    for (int i = 0; i < 3; ++i) { imu->cov_acc[i] = imu->cfg.cov_acc_scale[i]; imu->cov_gyr[i] = imu->cfg.cov_gyr_scale[i]; }
  }
}

extern "C" int flb_imu_process(flb_imu* imu, const double* imu7, int n_imu, double lidar_beg_time, double lidar_end_time,
                               double* state26, double* P, float leaf, flb_imu_result* out) {
  if (!imu) return set_err("null IMU processor");
  if (!state26 || !P) return set_err("flb_imu_process: null state26 or P");
  if (n_imu < 0 || n_imu > MAX_IMU_POSES - 1) return set_err("n_imu = %d outside [0, %d]", n_imu, MAX_IMU_POSES - 1);
  if (n_imu > 0 && !imu7) return set_err("flb_imu_process: null IMU samples");
  for (int k = 0; k < n_imu * IMU_SAMPLE_DOUBLES; ++k)
    if (!std::isfinite(imu7[k])) return set_err("IMU sample %d has a non-finite value", k / IMU_SAMPLE_DOUBLES);
  if (!std::isfinite(lidar_beg_time) || !std::isfinite(lidar_end_time)) return set_err("non-finite lidar time");
  if (!std::isfinite(leaf)) return set_err("leaf size is not finite");
  for (int k = 0; k < 26; ++k) if (!std::isfinite(state26[k])) return set_err("state26[%d] is not finite", k);
  for (int k = 0; k < NDOF * NDOF; ++k) if (!std::isfinite(P[k])) return set_err("P[%d] is not finite", k);
  flb_frontend* f = imu->fe;
  flb_session* s = f->ses;
  flb_map* m = s->map;
  if (leaf > 0.f && s->pending_n >= 0) return set_err("flb_imu_process: a prefetched scan is pending on this session");
  flb_imu_result r{};
  r.n_down = -1;
  if (out) *out = r;
  if (n_imu == 0) return 0;                                 // FLB_IMU_EMPTY (:398-401)
  if (imu->need_init) {
    imu_init(imu, imu7, n_imu, state26, P);
    r.status = FLB_IMU_INIT;
    if (out) *out = r;
    return 0;
  }
  CU(cudaSetDevice(m->cfg.device));
  cudaStream_t st = m->stream;
  const int ns = n_imu + 1;
  double* h = imu->h_in;
  memcpy(h, state26, sizeof(double) * 26);
  memcpy(h + 26, P, sizeof(double) * NDOF * NDOF);
  memcpy(h + 26 + NDOF * NDOF, imu->last_imu, sizeof(double) * IMU_SAMPLE_DOUBLES);
  memcpy(h + 26 + NDOF * NDOF + IMU_SAMPLE_DOUBLES, imu7, sizeof(double) * IMU_SAMPLE_DOUBLES * (size_t)n_imu);
  ImuParams p{};
  p.n_samples = ns;
  p.acc_norm = imu_norm3(imu->mean_acc);
  for (int i = 0; i < 12; ++i) p.q_init[i] = imu->Qd[i];
  for (int i = 0; i < 3; ++i) {
    p.q_cov[i] = imu->cov_gyr[i]; p.q_cov[3 + i] = imu->cov_acc[i];
    p.q_cov[6 + i] = imu->cfg.cov_bias_gyr[i]; p.q_cov[9 + i] = imu->cfg.cov_bias_acc[i];
    p.angvel_last[i] = imu->angvel_last[i]; p.acc_s_last[i] = imu->acc_s_last[i];
  }
  p.last_lidar_end_time = imu->last_lidar_end_time;
  p.pcl_beg = lidar_beg_time;
  p.pcl_end = lidar_end_time;
  CU(cudaEventRecord(imu->ev0, st));
  CU(cudaMemcpyAsync(imu->d_in, h, sizeof(double) * (26 + NDOF * NDOF + IMU_SAMPLE_DOUBLES * (size_t)ns), cudaMemcpyHostToDevice, st));
  k_imu_propagate<<<1, IMU_THREADS, sizeof(double) * IMU_SAMPLE_DOUBLES * (size_t)ns, st>>>(p, imu->d_in, f->d_poses, imu->d_rec);
  m->launches++;
  CU(cudaGetLastError());
  if (f->n_raw > 0) {
    if (fe_undistort_enqueue(f, ns, UndistortEnd{}, imu->d_rec->x, &imu->d_rec->n_poses)) return 1;
  } else {
    f->sorted = true;
  }
  if (leaf > 0.f && vg_enqueue(m, f->vg, fe_cloud(f), fe_curv(f), f->n_raw, leaf, s->body, f->down_curv, s->cap, st)) return 1;
  CU(cudaMemcpyAsync(imu->h_rec, imu->d_rec, sizeof(ImuRecord), cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(imu->ev1, st));
  CU(cudaStreamSynchronize(st));
  const ImuRecord& rec = *imu->h_rec;
  memcpy(state26, rec.x, sizeof(double) * 26);
  memcpy(P, rec.P, sizeof(double) * NDOF * NDOF);
  for (int i = 0; i < 3; ++i) { imu->angvel_last[i] = rec.angvel_last[i]; imu->acc_s_last[i] = rec.acc_s_last[i]; }
  imu->n_poses = rec.n_poses;
  if (rec.n_poses > 1) memcpy(imu->Qd, p.q_cov, sizeof(p.q_cov));   // Q keeps the blocks the last segment assigned
  memcpy(imu->last_imu, imu7 + (size_t)(n_imu - 1) * IMU_SAMPLE_DOUBLES, sizeof(double) * IMU_SAMPLE_DOUBLES);
  imu->last_lidar_end_time = lidar_end_time;
  r.status = FLB_IMU_PROPAGATED;
  r.n_poses = rec.n_poses;
  r.n_predicts = rec.n_poses;                               // n_poses - 1 segments + the final predict
  CU(cudaEventElapsedTime(&r.gpu_ms, imu->ev0, imu->ev1));
  if (leaf > 0.f) {
    const int n = f->n_raw;
    int nd = (int)f->vg.h_mm.p[7];
    if (f->vg.h_mm.p[6]) {   // PCL's int32 overflow guard: output = input (as flb_frontend_voxel_filter)
      if (n > s->cap) return set_err("voxel filter overflow guard: unfiltered scan of %d points exceeds max_scan_points=%d", n, s->cap);
      CU(cudaMemcpyAsync(s->body, fe_cloud(f), sizeof(float4) * (size_t)n, cudaMemcpyDeviceToDevice, st));
      CU(cudaMemcpyAsync(f->down_curv, fe_curv(f), sizeof(float) * (size_t)n, cudaMemcpyDeviceToDevice, st));
      nd = n;
    }
    if (nd > s->cap) return set_err("filtered scan of %d points exceeds max_scan_points=%d", nd, s->cap);
    f->n_down = nd;
    r.n_down = nd;
    if (scan_reset(s, nd)) return 1;
  }
  if (out) *out = r;
  return 0;
}

extern "C" int flb_imu_download_poses(flb_imu* imu, double* out22, int cap, int* n) {
  if (!imu) return set_err("null IMU processor");
  if (n) *n = imu->n_poses;
  const int c = std::min(imu->n_poses, cap);
  if (c <= 0 || !out22) return 0;
  flb_map* m = imu->fe->ses->map;
  CU(cudaSetDevice(m->cfg.device));
  CU(cudaMemcpyAsync(out22, imu->fe->d_poses, sizeof(double) * IMU_POSE_DOUBLES * (size_t)c, cudaMemcpyDeviceToHost, m->stream));
  CU(cudaStreamSynchronize(m->stream));
  return 0;
}

extern "C" int flb_imu_info(const flb_imu* imu, flb_imu_state* o) {
  if (!imu || !o) return set_err("flb_imu_info: null argument");
  for (int i = 0; i < 3; ++i) {
    o->mean_acc[i] = imu->mean_acc[i]; o->mean_gyr[i] = imu->mean_gyr[i]; o->cov_acc[i] = imu->cov_acc[i];
    o->cov_gyr[i] = imu->cov_gyr[i]; o->angvel_last[i] = imu->angvel_last[i]; o->acc_s_last[i] = imu->acc_s_last[i];
  }
  o->last_lidar_end_time = imu->last_lidar_end_time;
  for (int k = 0; k < IMU_SAMPLE_DOUBLES; ++k) o->last_imu[k] = imu->last_imu[k];
  o->init_iter_num = imu->init_iter_num;
  o->imu_need_init = imu->need_init ? 1 : 0;
  o->b_first_frame = imu->first_frame ? 1 : 0;
  o->n_poses = imu->n_poses;
  return 0;
}

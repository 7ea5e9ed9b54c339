/*
 * fastlio_b200.h — C ABI of the H100-native FAST-LIO2 per-scan hot path.
 *
 * This is the drop-in boundary for the path named in BASELINE.json:north_star.  Each entry point states the
 * reference interface it replaces (paths relative to the reference repo Yixin-F/better_fastlio2):
 *
 *   map object       KD_TREE<PointType> ikdtree            include/ikd-Tree/ikd_Tree.h:225-249, src/laserMapping.cpp:116
 *   measurement pass h_share_model(state_ikfom&, dyn_share_datastruct<double>&)      src/laserMapping.cpp:1876-2004
 *   filter update    esekf::update_iterated_dyn_share_modified(R, solve_time)
 *                                                          include/IKFoM_toolkit/esekfom/esekfom.hpp:1620-1938
 *   map insert       map_incremental()                     src/laserMapping.cpp:1440-1496
 *   map delete       lasermap_fov_segment()                src/laserMapping.cpp:1136-1200
 *
 * Conventions
 *   - Plain pointers and sizes only; no C++/torch types.  All functions return 0 on success, non-zero on error
 *     (never throw); flb_last_error() returns a thread-local message.  The reference has no error codes on this
 *     path (SURVEY.md §8b) — the C++ facades in include/fastlio_b200/ map errors to valid=false / ROS_ERROR.
 *   - Points are float xyz with a caller-given byte stride (12 for packed xyz, 16 for float4, 48 for
 *     pcl::PointXYZINormal as used by PointType, common_lib.h:161).  Input buffers are borrowed for the call.
 *   - All *host* pointers unless the name says "_dev".  Calls on one handle must be serialised by the caller (the
 *     reference issues all map/search calls from the main thread); different handles are independent.
 *   - There is NO CPU fallback: every compute entry point fails loudly if no CUDA device is usable.
 *
 * State layout "state26" (doubles), mirrors state_ikfom (include/use-ikfom.hpp:21-30):
 *   [0:3) pos | [3:7) rot quaternion (x,y,z,w = Eigen coeffs order) | [7:11) offset_R_L_I (x,y,z,w) |
 *   [11:14) offset_T_L_I | [14:17) vel | [17:20) bg | [20:23) ba | [23:26) grav (S2, |g| = 9.809)
 * Covariance: 23x23 doubles, row-major, error-state order pos,rot,offR,offT,vel,bg,ba,grav(2).
 */
#ifndef FASTLIO_B200_H_
#define FASTLIO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FLB_NUM_MATCH_POINTS 5 /* NUM_MATCH_POINTS, include/common_lib.h:149 */
#define FLB_STATE_DIM 26
#define FLB_STATE_DOF 23

typedef struct flb_map flb_map;         /* device hashed-voxel map; replaces KD_TREE<PointType> */
typedef struct flb_session flb_session; /* per-scan measurement context; replaces h_share_model's file-scope globals */

/* ------------------------------------------------------------------------------------------------ errors / device */
const char* flb_last_error(void);
int flb_device_count(void);          /* number of CUDA devices visible (0 => every compute call fails) */
const char* flb_version(void);

/* ------------------------------------------------------------------------------------------------ map (KD_TREE API) */
typedef struct flb_map_config {
  float voxel_size;        /* downsample_size / filter_size_map_min (KD_TREE ctor box_length, ikd_Tree.h:226) */
  int max_points;          /* capacity in points (valid + overflow chains); 0 -> 8M */
  int max_blocks;          /* capacity in 4x4x4-voxel blocks; 0 -> max_points/4.  Device memory ~1.5 KB per block, of
                              which 76 B are the coarse level (one coarse cell per block at most: sparse content never
                              fills it) */
  int device;              /* CUDA device ordinal */
} flb_map_config;

int flb_map_create(const flb_map_config* cfg, flb_map** out);     /* KD_TREE::KD_TREE, ikd_Tree.cpp:9-17 */
void flb_map_destroy(flb_map* m);                                 /* KD_TREE::~KD_TREE, ikd_Tree.cpp:19-27 */
int flb_map_set_downsample_param(flb_map* m, float voxel_size);   /* set_downsample_param, ikd_Tree.cpp:39-42
                                                                     (only legal while the map is empty) */
int flb_map_has_root(const flb_map* m);                           /* Root_Node != nullptr test, laserMapping.cpp:2328 */

/* Build (ikd_Tree.cpp:352-364): replace contents by the cloud, inserted verbatim (no per-voxel dedupe). */
int flb_map_build(flb_map* m, const float* xyz, int n, int stride_bytes);
/* reconstruct (ikd_Tree.cpp:1393-1405): delete everything then Build. */
int flb_map_reconstruct(flb_map* m, const float* xyz, int n, int stride_bytes);
/* Add_Points (ikd_Tree.cpp:413-489). downsample_on!=0: per-voxel winner = closest to the voxel centre (sequential
 * semantics of the reference reproduced for the resulting map).  *n_added = number of voxels whose content changed
 * (the reference returns the number of sequential add operations, which its caller overwrites without reading,
 * laserMapping.cpp:1492-1494; the two differ only when several new points fall into one voxel). */
int flb_map_add_points(flb_map* m, const float* xyz, int n, int stride_bytes, int downsample_on, int* n_added);
/* PointType-aware variants.  The reference tree stores whole pcl::PointXYZINormal records (ikd_Tree.h:64-86) and hands them
 * back from Nearest_Search / flatten (featsFromMap for publishing and saving, laserMapping.cpp:2361-2367); FAST-LIO map
 * points carry x, y, z, intensity (normals and curvature are zero, laserMapping.cpp:1101-1110).  These entry points read the
 * intensity at off_intensity bytes into each record (< 0: none -> 0) and keep it with the map point; the plain xyz entry
 * points above store intensity 0, except that 16-byte records are always taken as (x, y, z, intensity). */
int flb_map_build_pt(flb_map* m, const void* pts, int n, int stride_bytes, int off_intensity);
int flb_map_reconstruct_pt(flb_map* m, const void* pts, int n, int stride_bytes, int off_intensity);
int flb_map_add_points_pt(flb_map* m, const void* pts, int n, int stride_bytes, int off_intensity, int downsample_on, int* n_added);
/* Delete_Point_Boxes (ikd_Tree.cpp:535-556): boxes = nb x {min xyz, max xyz} (BoxPointType, ikd_Tree.h:32-35),
 * half-open test min <= p < max (ikd_Tree.cpp:670); *n_deleted = number of points removed. */
int flb_map_delete_boxes(flb_map* m, const float* boxes6, int nb, int* n_deleted);
/* Delete_Points (ikd_Tree.cpp:513-533): remove points equal to the given ones within 1e-6 per axis (same_point). */
int flb_map_delete_points(flb_map* m, const float* xyz, int n, int stride_bytes, int* n_deleted);
/* Nearest_Search (ikd_Tree.cpp:366-397), batched over nq queries: exact k-NN (k <= 5 on the fast path, <= 20
 * otherwise) among valid points with float squared distances, ascending; max_dist <= 0 means unbounded (the
 * reference default INFINITY), otherwise a neighbour is kept when d2 <= max_dist * max_dist in double, as the
 * reference compares.  out_xyz[nq*k*3], out_d2[nq*k] (unfilled = NaN / INF), out_cnt[nq]. */
int flb_map_nearest_search(flb_map* m, const float* q_xyz, int nq, int stride_bytes, int k, float max_dist,
                           float* out_xyz, float* out_d2, int* out_cnt);
/* Box_Search (ikd_Tree.cpp:399-404) / Radius_Search (:406-411): points in a half-open box / within radius.
 * Writes up to cap points; *n_found is the total. */
int flb_map_box_search(flb_map* m, const float* box6, float* out_xyz, int cap, int* n_found);
int flb_map_radius_search(flb_map* m, const float* center_xyz, float radius, float* out_xyz, int cap, int* n_found);
/* the same searches returning (x, y, z, intensity) records: out_xyzi[nq*k*4] resp. out_xyzi[cap*4] */
int flb_map_nearest_search_xyzi(flb_map* m, const float* q_xyz, int nq, int stride_bytes, int k, float max_dist,
                                float* out_xyzi, float* out_d2, int* out_cnt);
int flb_map_box_search_xyzi(flb_map* m, const float* box6, float* out_xyzi, int cap, int* n_found);
int flb_map_radius_search_xyzi(flb_map* m, const float* center_xyz, float radius, float* out_xyzi, int cap, int* n_found);
int flb_map_validnum(flb_map* m);  /* validnum(), ikd_Tree.cpp:128-145 ; -1 on error */
int flb_map_size(flb_map* m);      /* size(), ikd_Tree.cpp:78-96 (== validnum here: no lazy tombstones) */
/* flatten (ikd_Tree.cpp:1325-1352): all valid points, arbitrary order. Writes up to cap; *n = total valid. */
int flb_map_flatten(flb_map* m, float* out_xyz, int cap, int* n);
int flb_map_flatten_xyzi(flb_map* m, float* out_xyzi, int cap, int* n);   /* (x, y, z, intensity) records */
/* tree_range (ikd_Tree.h:245): bounding box of valid points {min xyz, max xyz}. */
int flb_map_range(flb_map* m, float* box6);

typedef struct flb_map_stats {
  int valid_points, blocks_in_use, block_capacity, overflow_in_use, overflow_capacity;
  int hash_capacity, hash_tombstones, coarse_cells, rehash_count;
  size_t device_bytes;
} flb_map_stats;
int flb_map_get_stats(flb_map* m, flb_map_stats* out);

/* Optional per-kernel-class timing with CUDA events on the map's stream (used by bench.py for the roofline figure;
 * no reference counterpart — the reference's own timers are omp_get_wtime marks, laserMapping.cpp:2253-2402). */
enum { FLB_K_TRANSFORM = 0, FLB_K_KNN, FLB_K_RESIDUAL, FLB_K_REDUCE, FLB_K_CLASSIFY, FLB_K_INSERT, FLB_K_DELETE, FLB_K_COUNT = 8 };
typedef struct flb_profile {
  double ms[FLB_K_COUNT];      /* accumulated device time per class */
  int launches[FLB_K_COUNT];   /* kernels launched per class */
  int regions[FLB_K_COUNT];    /* timed regions per class (e.g. one per k-NN pass) */
  long long knn_phase[4];      /* queries resolved by search phase A (5^3 voxel stencil) / B0 (3^3 blocks) /
                                  B (3^3 coarse cells) / C (exhaustive coarse scan) */
  long long knn_head_candidates; /* stencil kernel: occupied stencil voxels visited (one 16-B load each) */
  long long knn_chain_nodes;     /* stencil kernel: overflow-chain nodes visited (voxels holding > 1 point) */
  long long knn_chain_max;       /* largest number of chain nodes visited by a single query */
} flb_profile;
int flb_map_profile_enable(flb_map* m, int on);
int flb_map_profile_read(flb_map* m, flb_profile* out, int reset);

/* ------------------------------------------------------------------------------------------------ session (per scan) */
typedef struct flb_session_config {
  int max_scan_points;      /* capacity N of feats_down_body (the reference caps at 100000, laserMapping.cpp:52) */
  int extrinsic_est_en;     /* mapping/extrinsic_est_en, laserMapping.cpp:44 */
  int max_iterations;       /* NUM_MAX_ITERATIONS (ikdtree/max_iteration), laserMapping.cpp:2064; 0..7, else flb_session_create fails */
  double laser_point_cov;   /* LASER_POINT_COV, laserMapping.cpp:14 (0.001) */
  double filter_size_map_min; /* ikdtree/filter_size_map_min as the DOUBLE the caller holds, laserMapping.cpp:56 */
  double limit[FLB_STATE_DOF]; /* epsi, laserMapping.cpp:2148-2149 (0.001 each) */
} flb_session_config;

void flb_session_default_config(flb_session_config* cfg);
int flb_session_create(flb_map* m, const flb_session_config* cfg, flb_session** out);
void flb_session_destroy(flb_session* s);

/* feats_down_body (laserMapping.cpp:2322-2325): upload the voxel-downsampled, undistorted scan (LiDAR frame).
 * Resets the per-scan caches (Nearest_Points, point_selected_surf := true, laserMapping.cpp:2131). */
int flb_scan_upload(flb_session* s, const float* body_xyz, int n, int stride_bytes);
/* same for PointType records: the intensity at off_intensity (< 0: none) travels with the point into the map, as
 * pointBodyToWorld copies it (laserMapping.cpp:1101-1110).  16-byte records are (x, y, z, intensity). */
int flb_scan_upload_pt(flb_session* s, const void* body_pts, int n, int stride_bytes, int off_intensity);
/* Asynchronous variant for streaming callers: starts the host->device copy of the NEXT scan on a copy stream into a
 * second buffer and returns immediately, so the transfer overlaps the processing of the current scan.  The scan
 * becomes current at the next flb_scan_step / flb_esikf_update called with body == NULL (which waits for the copy).
 * body_xyz must stay valid (pinned memory recommended) until then; stride 12 or 16 only. */
int flb_scan_prefetch(flb_session* s, const float* body_xyz, int n, int stride_bytes);
/* Same, when the scan already lives in device memory as n float4 (x, y, z, intensity) on the session's device.  The scan is
 * read IN PLACE (no copy; its address travels with the staged inputs of the step): the buffer must stay valid and unmodified
 * until the last call working on this scan (flb_scan_step[_finish], flb_esikf_update, flb_map_incremental, flb_pass...) returned. */
int flb_scan_set_device(flb_session* s, const void* body_xyz4_dev, int n);

typedef struct flb_pass_result {
  int valid;               /* ekfom_data.valid (false when effct_feat_num < 1, laserMapping.cpp:1956-1961) */
  int effct_feat_num;      /* M */
  double total_residual;   /* sum |pd2|, laserMapping.cpp:1951 */
  double HTH[144];         /* h_x^T h_x, 12x12 row-major (esekfom.hpp:1790) */
  double HTh[12];          /* h_x^T h */
} flb_pass_result;

/* One h_share_model call (laserMapping.cpp:1876-2004) for the iterate `state26`; search != 0 == ekfom_data.converge
 * (re-run the 5-NN), else the cached Nearest_Points / point_selected_surf are reused.  Returns the reduced normal
 * equations (boundary B3 of SURVEY.md §8b). */
int flb_pass(flb_session* s, const double* state26, int search, flb_pass_result* out);
/* Exact rows of the last flb_pass (boundary B1): h_x as M x 12 COLUMN-major doubles (Eigen::MatrixXd layout,
 * esekfom.hpp:82) with leading dimension ld >= M, and h[M] (= -pd2, laserMapping.cpp:2001). */
int flb_pass_rows(flb_session* s, double* h_x_colmajor, int ld, double* h, int capacity_rows, int* M);

typedef struct flb_update_stats {
  int passes, search_passes, effct_feat_num, converged_count;
  double total_residual;
  float gpu_ms;            /* device time of all kernels of this update (CUDA events; inside flb_scan_step: %globaltimer span from
                              the sequence's first kernel to just behind its last update kernel) */
} flb_update_stats;

/* update_iterated_dyn_share_modified (esekfom.hpp:1620-1938) with the built-in measurement model: state26 / P23x23
 * hold the propagated state in and the posterior out. */
int flb_esikf_update(flb_session* s, double* state26, double* P, flb_update_stats* stats);

/* Update engine: 1 (default) = device-driven — all passes of the iterated update are enqueued up front and the
 * 23-DOF algebra runs in a device kernel (no host round trip inside a scan); 0 = host-driven — the reference's
 * structure, one synchronisation per pass with the algebra in C++ on the host.  Both give the same result to ~1e-15;
 * the device engine falls back to the host one for the under-determined M < 23 branch (esekfom.hpp:1720-1750). */
int flb_session_set_update_engine(flb_session* s, int device_driven);

/* map_incremental (laserMapping.cpp:1440-1496) with the posterior state: classify every scan point with the cached
 * neighbours, then Add_Points(PointToAdd,true) and Add_Points(PointNoNeedDownsample,false). */
int flb_map_incremental(flb_session* s, const double* state26, int flg_EKF_inited, int* n_to_add, int* n_no_downsample);

/* Debug / parity: the per-scan caches. Any pointer may be NULL. nbr_xyz[N*5*3], nbr_d2[N*5], nbr_cnt[N],
 * selected[N] (point_selected_surf), normvec[N*4] (nx,ny,nz,pd2), world_xyz[N*3] (feats_down_world). */
int flb_neighbors_download(flb_session* s, float* nbr_xyz, float* nbr_d2, int* nbr_cnt, unsigned char* selected,
                           float* normvec, float* world_xyz);

/* ------------------------------------------------------------------------------------------------ fov segment (host) */
typedef struct flb_fov_state {
  float local_map_min[3], local_map_max[3]; /* LocalMap_Points, laserMapping.cpp:1132 */
  int initialized;                          /* Localmap_Initialized, :1133 */
  double cube_len;                          /* mapping/cube_len */
  float det_range;                          /* mapping/det_range (DET_RANGE) */
  double pos_lid[3];                        /* pos_lid, laserMapping.cpp:2383 — LiDAR position of the PREVIOUS
                                               posterior (zero before the first update, as the reference's
                                               zero-initialised global); maintained by flb_scan_step */
} flb_fov_state;
/* lasermap_fov_segment (laserMapping.cpp:1136-1200): moves the local-map cube and deletes the slabs that left it.
 * pos_lid = LiDAR position in world. *n_boxes (<=3) / *n_deleted = kdtree_delete_counter. */
int flb_fov_segment(flb_map* m, flb_fov_state* fov, const double* pos_lid, float* boxes_out18, int* n_boxes,
                    int* n_deleted);

/* ------------------------------------------------------------------------------------------------ whole per-scan step */
typedef struct flb_scan_result {
  flb_update_stats update;
  int n_to_add, n_no_downsample, n_deleted, map_valid;
  float gpu_ms_total;      /* update + insert kernels (+ the on-stream upload and the box deletes when `body` is passed: CUDA
                              events then; otherwise the device-side span of the step's sequence) */
  int kernel_launches;     /* number of kernels launched by this step */
} flb_scan_result;
/* The timed region of SURVEY.md §8d: lasermap_fov_segment -> update_iterated_dyn_share_modified -> map_incremental
 * (laserMapping.cpp:2320, :2380, :2401) for one scan.  body may be NULL if the scan was already set with
 * flb_scan_upload / flb_scan_set_device.  fov may be NULL to skip the fov segment. */
int flb_scan_step(flb_session* s, flb_fov_state* fov, const float* body_xyz, int n, int stride_bytes, double* state26,
                  double* P, int flg_EKF_inited, flb_scan_result* out);

/* The same step split at its single synchronisation point, for streaming callers:
 *   flb_scan_step_begin(...);  flb_scan_prefetch(next scan);  flb_scan_step_finish(...);
 * overlaps the upload of the next scan with the kernels of this one.
 * Replay / batch callers whose next prior does not depend on this posterior may keep TWO steps in flight
 *   begin(k); prefetch(k+1); loop { begin(k+1); finish(k); prefetch(k+2); ... }
 * so that the device never waits for the host between scans (finish always collects the OLDEST step; a third begin is
 * refused).  Results are identical to alternating calls.  Constraints of the two-deep mode: the device-driven engine only; the
 * fov segment of step k+1 sees the lidar position of step k-1; a scan with fewer than 23 effective rows (the explicit-row
 * branch, esekfom.hpp:1720-1750, handled on the host) makes flb_scan_step_finish fail if a younger step is already queued.
 * A live filter (prior k+1 = IMU propagation of posterior k) alternates begin / finish and is unaffected. */
int flb_scan_step_begin(flb_session* s, flb_fov_state* fov, const float* body_xyz, int n, int stride_bytes,
                        const double* state26, const double* P, int flg_EKF_inited);
int flb_scan_step_finish(flb_session* s, flb_fov_state* fov, double* state26, double* P, flb_scan_result* out);

/* ------------------------------------------------------------------------------------------------ front-end rows
 * The callers / data formats either side of the per-scan path (SURVEY.md §8f), so that a raw scan never leaves the
 * GPU between the driver callback and the update:
 *   meas.lidar --UndistortPcl--> feats_undistort --downSizeFilterSurf.filter--> feats_down_body --> flb_scan_step
 * A front end belongs to one session and shares its stream; calls are serialised by the caller like all others.
 * Points are the reference's PointType (pcl::PointXYZINormal, common_lib.h:161): 48-byte stride, x@0 y@4 z@8,
 * intensity@32, curvature@36 (= time offset in ms, preprocess.cpp) — stride and offsets are parameters. */
typedef struct flb_frontend flb_frontend;
#define FLB_IMU_POSE_DOUBLES 22 /* Pose6D (msg/Pose6D.msg, set_pose6d common_lib.h:446-460):
                                   offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9] row-major */
#define FLB_MAX_IMU_POSES 256

int flb_frontend_create(flb_session* s, int max_raw_points, flb_frontend** out);
void flb_frontend_destroy(flb_frontend* f);
/* meas.lidar (IMU_Processing.hpp:242 "pcl_out = *(meas.lidar)"): upload the raw scan. off_intensity / off_curvature are
 * byte offsets of those float fields inside a point, or -1 when absent (treated as 0).  The buffer holds n whole records
 * (n * stride_bytes bytes are copied), as a std::vector<PointType> / pcl::PointCloud does. */
int flb_frontend_upload(flb_frontend* f, const void* pts, int n, int stride_bytes, int off_intensity, int off_curvature);
/* ImuProcess::UndistortPcl, the per-point part (IMU_Processing.hpp:243 sort by time, :334-386 backward compensation).
 * imu_poses = n_poses x 22 doubles = the IMUpose vector built by a host-side forward propagation (:260-322, kf.predict;
 * flb_imu_process below runs it on the device instead); state26_end = imu_state after the last predict (:329).  Result: feats_undistort in time order
 * (ties keep upload order; the reference's std::sort leaves them unspecified). */
int flb_frontend_undistort(flb_frontend* f, const double* imu_poses, int n_poses, const double* state26_end);
/* downSizeFilterSurf.setInputCloud(feats_undistort); downSizeFilterSurf.filter(*feats_down_body)
 * (laserMapping.cpp:2322-2323, leaf = mappingSurfLeafSize :2135): pcl::VoxelGrid centroid filter (PCL 1.10 semantics:
 * float leaf index relative to the cloud minimum, output ordered by leaf index, centroid of x,y,z,intensity,curvature;
 * PCL's int32 overflow guard returns the input unchanged).  The result becomes the session's current scan
 * (as flb_scan_upload would); *n_out = feats_down_size.  Sums run in time order inside a leaf (PCL: unspecified). */
int flb_frontend_voxel_filter(flb_frontend* f, float leaf_size, int* n_out);
/* The three calls above in one (one synchronisation): raw scan in, feats_down_body left on the device as the session's
 * current scan.  imu_poses == NULL or n_poses == 0 skips the undistortion (no IMU / already compensated). */
int flb_frontend_process(flb_frontend* f, const void* pts, int n, int stride_bytes, int off_intensity, int off_curvature,
                         const double* imu_poses, int n_poses, const double* state26_end, float leaf_size, int* n_out);
/* Read back feats_undistort (x,y,z,intensity per point; curvature; perm[j] = upload index of sorted point j) and
 * feats_down_body.  Any output pointer may be NULL; at most cap points are written, *n = the cloud size. */
int flb_frontend_download_undistorted(flb_frontend* f, float* out_xyzi, float* out_curvature, int* out_perm, int cap, int* n);
int flb_frontend_download_down(flb_frontend* f, float* out_xyzi, float* out_curvature, int cap, int* n);
/* publish_frame_world / map saving (laserMapping.cpp:1502-1540): RGBpointBodyToWorld (:1101-1110) of every point of
 * feats_down_body (which = 0, dense_pub_en false) or feats_undistort (which = 1) with the posterior state. */
int flb_frontend_points_to_world(flb_frontend* f, int which, const double* state26, float* out_xyzi, int cap, int* n);

/* Camera colouring of the published scan, publish_frame_world_color (laserMapping.cpp:310-392).
 * flb_frontend_camera_config is paramSetting (:279-289): cam_ex = 16 row-major doubles (externalMat, 4x4), cam_in = 12
 * (internalMatProject, 3x4), as read at :2045-2046; width x height bounds the image (the reference's Wmax x Hmax =
 * 1280 x 720, :232-233).  M = cam_in * cam_ex is formed once, in double.  Configuring zero-fills the device image (the
 * reference's zero-initialised image_color).  Non-finite parameters and non-positive sizes are rejected. */
int flb_frontend_camera_config(flb_frontend* f, const double cam_ex[16], const double cam_in[12], int width, int height);
/* imageCallback (:250-276) after cv_bridge::toCvShare(msg, "bgr8"): copies the top-left height x width window of a
 * bgr8 image of any row step (step_bytes >= 3 * cols) to the device.  An image smaller than the configured size is
 * rejected (the reference reads past it). */
int flb_frontend_camera_image(flb_frontend* f, const unsigned char* bgr8, int rows, int cols, int step_bytes);
/* The two loops of publish_frame_world_color on feats_down_body (which = 0) or feats_undistort (which = 1): a point is
 * kept iff its pixel (u, v) = trunc(M*(x,y,z,1) / c2) lies in the image and its lidar-frame x > 0; kept points stay in
 * cloud order with x,y,z in the world frame (as flb_frontend_points_to_world), the source intensity, and the colour as
 * one 32-bit word with the bytes b, g, r, a = 255 (PCL_ADD_RGB).  At most cap records are written; *n = the kept count.
 * DESIGN.md §9 states the contract and its deviations. */
int flb_frontend_points_colorize(flb_frontend* f, int which, const double* state26, float* out_xyzi, unsigned* out_bgra, int cap,
                                 int* n);
/* publish_frame_body (laserMapping.cpp:1543-1558): RGBpointBodyLidarToIMU (:1113-1122), offR * p + offT in double, of
 * every point of feats_undistort, intensity carried.  At most cap points are written; *n = the cloud size. */
int flb_frontend_points_to_imu(flb_frontend* f, const double* state26, float* out_xyzi, int cap, int* n);

/* Preprocess::process (src/preprocess.cpp) with feature extraction off (feature_extract_enable, laserMapping.cpp:2040):
 * driver records -> the PointType cloud that becomes meas.lidar, on the device.  Parameters as read at
 * laserMapping.cpp:2034-2041 (preprocess.h:8-14 for the enums):
 *   lidar_type 1 LIVOX   CustomMsg     livox_handler, feature-off branch (preprocess.cpp:178-204)
 *              2 VELO16  PointCloud2   velodyne_handler (:302-340, :417-473); per-point time synthesised from the
 *                                      azimuth, ring by ring, when the last record's time is not > 0
 *              3 OUST64  PointCloud2   oust64_handler, feature-off branch (:271-297)
 *   time_unit  0 SEC, 1 MS, 2 US, 3 NS (time_unit_scale 1e3f, 1, 1e-3f, 1e-6f; preprocess.cpp:65-82)
 * Record fields (byte offsets inside one record of `stride` bytes, -1 = absent, read as 0 like pcl::fromROSMsg does for
 * a field with no match; x, y, z are required).  Field types are fixed per sensor:
 *   LIVOX   off_time = offset_time u32 (ns), off_intensity = reflectivity u8, off_tag u8, off_line u8, x y z f32
 *   VELO16  x y z intensity f32, off_time = time f32, off_ring = ring u16            (preprocess.h:94-107)
 *   OUST64  x y z intensity f32, off_time = t u32                                      (preprocess.h:109-128)
 * Offsets need no alignment (packed PointCloud2 layouts such as point_step 22 are read as they are). */
typedef struct {
  int lidar_type;        /* 1 LIVOX, 2 VELO16, 3 OUST64 */
  int n_scans;           /* preprocess/scan_line */
  int scan_rate;         /* preprocess/scan_rate (Hz) */
  int point_filter_num;  /* point_filter_num, >= 1 */
  int time_unit;         /* preprocess/timestamp_unit */
  double blind;          /* preprocess/blind (m) */
} flb_preprocess_config;

typedef struct {
  int stride;            /* bytes per record (PointCloud2 point_step, sizeof(CustomPoint)) */
  int off_x, off_y, off_z, off_intensity, off_time, off_ring, off_tag, off_line;
} flb_raw_layout;

/* Decode, decimate, blind-cut and time-stamp n driver records in one upload and one synchronisation; the kept points
 * (input order, normals zero) become the front end's current raw scan exactly as flb_frontend_upload would leave it, so
 * flb_frontend_undistort / _voxel_filter / _download_undistorted follow unchanged.  *n_out = pl_surf.size() and
 * *last_curvature = pl_surf.points.back().curvature (0 for an empty result): what sync_packages needs for
 * lidar_end_time (laserMapping.cpp:1374-1405).  Either output pointer may be NULL.  Arguments are validated before any
 * device work; a Velodyne ring >= n_scans (undefined behaviour in the reference) fails the call and leaves an empty
 * scan. */
int flb_frontend_preprocess(flb_frontend* f, const flb_preprocess_config* cfg, const flb_raw_layout* layout, const void* records,
                            int n, int* n_out, float* last_curvature);

/* Stand-alone pcl::VoxelGrid centroid filter on a host cloud (the reference's other VoxelGrid call sites, e.g.
 * laserMapping.cpp:640-643, :1780-1789), run on the map's device/stream.  out_xyzi = x,y,z,intensity per point. */
int flb_voxel_grid_filter(flb_map* m, const void* pts, int n, int stride_bytes, int off_intensity, float leaf_size,
                          float* out_xyzi, int cap, int* n_out);
/* recontructIKdTree, the data-parallel part (laserMapping.cpp:632-664): for the selected key frames k (clouds[k] with
 * sizes[k] points in the key frame's own frame, poses6[k] = x,y,z,roll,pitch,yaw of cloudKeyPoses6D) do
 * subMap += transformPointCloud(cloud_k, pose_k) (common_lib.h:711-734), VoxelGrid(leaf), ikdtree.reconstruct(result).
 * The filtered sub-map (featsFromMap, :664) is returned in out_xyzi (up to cap points); *n_points = its size.  The
 * key-frame selection itself (pose radius search, :621-635) is back-end bookkeeping and stays with the caller. */
int flb_map_reconstruct_keyframes(flb_map* m, const void* const* clouds, const int* sizes, int n_keyframes, int stride_bytes,
                                  int off_intensity, const float* poses6, float leaf_size, float* out_xyzi, int cap,
                                  int* n_points);

/* ------------------------------------------------------------------------------------------------ key-frame store
 * surfCloudKeyFrames (laserMapping.cpp:756-758) kept on the device: each key frame is the whole undistorted scan
 * (feats_undistort) in its own body frame, stored as x,y,z,intensity + curvature (20 bytes per point) in a fixed-capacity,
 * append-only arena sized at creation.  Poses are not stored (iSAM2 rewrites them, correctPoses :780-795): every reader
 * takes them at call time.  A store is created on a map, uses its device and stream and keeps it alive until destroyed.
 * The library takes no lock: calls on a store are serialised by the caller with every other call on that map, from all
 * threads (a loop-closure thread and the main loop hold one common mutex around their calls, INTEGRATION.md §3, §5).
 * Every call validates all its arguments before any device work; a failed call leaves the store unchanged. */
typedef struct flb_keyframes flb_keyframes;
#define FLB_KF_POSE6 0  /* transforms = n_ids x {x, y, z, roll, pitch, yaw}: pcl::getTransformation, as transformPointCloud
                           with a PointTypePose (common_lib.h:711-734) */
#define FLB_KF_AFFINE 1 /* transforms = n_ids x row-major 3x4 float affine (e.g. keyTrans.inverse() * keyNearTrans,
                           laserMapping.cpp:873-875); an affine equal to the identity copies the stored records verbatim,
                           curvature included (*nearKeyframes += *surfCloudKeyFrames[key], :869).  The test is on the
                           values: any entry whose affine is exactly the identity is copied, not computed */

int flb_keyframes_create(flb_map* m, long long max_points, int max_keyframes, flb_keyframes** out);
void flb_keyframes_destroy(flb_keyframes* kf);
/* pcl::copyPointCloud(*feats_undistort, *thisSurfKeyFrame); surfCloudKeyFrames.push_back(...)  (laserMapping.cpp:756-758):
 * appends the front end's current scan (time-sorted and compensated after flb_frontend_undistort, else in upload order) as
 * the next key frame, device to device on the map stream with no synchronisation.  *index = the new key frame's id.
 * Fails when the front end's session is on another map or either capacity would be exceeded. */
int flb_keyframes_append_frontend(flb_keyframes* kf, flb_frontend* fe, int* index);
/* The same from n host records (restoring a session, tests): offsets as flb_frontend_upload. */
int flb_keyframes_append(flb_keyframes* kf, const void* pts, int n, int stride_bytes, int off_intensity, int off_curvature,
                         int* index);
/* Key frame `id` as stored: x,y,z,intensity per point and curvature (either pointer may be NULL); at most cap points are
 * written, *n = its size (copyPointCloud(*surfCloudKeyFrames[i]) of the per-key-frame saver, laserMapping.cpp:2504). */
int flb_keyframes_download(flb_keyframes* kf, int id, float* out_xyzi, float* out_curvature, int cap, int* n);
/* Number of key frames, stored points and device bytes held by the store, and the device bytes of the readers' scratch
 * its map currently holds (any pointer may be NULL).  No device work. */
int flb_keyframes_info(const flb_keyframes* kf, int* n_keyframes, long long* n_points, long long* device_bytes,
                       long long* map_scratch_bytes);
/* Size of key frame `id`, or -1 (with flb_last_error) when it does not exist. */
int flb_keyframes_size(const flb_keyframes* kf, int id);
/* flb_map_reconstruct_keyframes with the clouds taken from the store: for j < n_ids, subMap += transformPointCloud(
 * key frame ids[j], poses6[j]) in that order, VoxelGrid(leaf), ikdtree.reconstruct(result); featsFromMap out.  The store
 * must have been created on m.  The selection (radius search over the key poses, :621-635) stays with the caller. */
int flb_map_reconstruct_from_keyframes(flb_map* m, const flb_keyframes* kf, const int* ids, int n_ids, const float* poses6,
                                       float leaf_size, float* out_xyzi, int cap, int* n_points);
/* Map assembly from the store, ids in order, each key frame with its own transform (transform_kind FLB_KF_POSE6 or
 * FLB_KF_AFFINE); transformed points get curvature 0 as transformPointCloud writes them.  leaf_size > 0: pcl::VoxelGrid
 * centroid filter with curvature carried (publishGlobalMap :1866-1869, SurfMap.pcd / filterGlobalMap.pcd :1780-1789;
 * PCL's int32 overflow guard returns the assembled cloud unchanged); leaf_size == 0: the dense concatenation
 * (GlobalMap.pcd :1796, loop sub-maps :856-883).  At most cap points are written, *n_out = the full size (size the buffer
 * from flb_keyframes_info / flb_keyframes_size beforehand). */
int flb_keyframes_assemble(flb_keyframes* kf, const int* ids, int n_ids, int transform_kind, const float* transforms,
                           float leaf_size, float* out_xyzi, float* out_curvature, int cap, int* n_out);
/* The readers above keep their scratch with the map, grown to the largest selection so far and only for what a call
 * uses (a dense assembly needs no filter buffers): a save map of the whole run can leave gigabytes behind.  This frees
 * all of it (waits for the map's stream); the next reader allocates again. */
int flb_map_release_keyframe_scratch(flb_map* m);

/* ------------------------------------------------------------------------------------------------ Scan Context
 * SCManager::makeScancontext (include/sc-relo/Scancontext.cpp:195-251) of key-frame clouds in the store, computed where
 * they are: each point is transformed exactly as flb_keyframes_assemble writes it, binned into one of 20 rings x 60
 * sectors out to 80 m and max-reduced; only the descriptors come back.  Semantics are the reference's, types included:
 * pt.z = (float)(z + lidar_height) in double; range = sqrtf(x*x + y*y) without FMA; the angle of xy2theta with a float
 * quotient, double atan and degrees, rounded to float (x = -0, y > 0 gives -90 degrees, x = ±0, y = 0 NaN); a point is
 * skipped when range > 80 (a NaN range is kept); ring / sector = clamp(ceil(...), 1, 20 / 60) in double, a NaN landing
 * in index 1; a bin keeps the largest pt.z above -1000, a bin no point beat is 0.  Each descriptor is 20 x 60 doubles,
 * row-major (ring, sector), every value exactly a float or 0.  The device's double atan is within 2 ulp of glibc's: a
 * point whose angle lies within one float ulp of a 6-degree boundary can land in the neighbouring sector (DESIGN.md §5).
 * Every argument is checked before any device work; one synchronisation per call; the store is not modified.  The chunk
 * table and the descriptor keys are map-side key-frame scratch (flb_keyframes_info, flb_map_release_keyframe_scratch). */
#define FLB_SC_RINGS 20     /* PC_NUM_RING, Scancontext.h:86 (const in the reference) */
#define FLB_SC_SECTORS 60   /* PC_NUM_SECTOR, :87; PC_MAX_RADIUS 80 m, :88 */
/* makeScancontext(loop sub-map of the selection) (performLoopClosure, laserMapping.cpp:932-933): ids in order, transforms
 * as flb_keyframes_assemble (FLB_KF_POSE6 / FLB_KF_AFFINE, the identity copies), empty key frames dropped; out_desc = 20 x
 * 60 doubles row-major.  n_ids == 0 (or only empty key frames): all zeros. */
int flb_keyframes_scan_context(flb_keyframes* kf, const int* ids, int n_ids, int transform_kind, const float* transforms,
                               double lidar_height, double* out_desc);
/* makeScancontext(*surfCloudKeyFrames[ids[j]]) for every j, the stored records as they are (the saver, :2504-2505):
 * out_descs = n_ids x 20 x 60 doubles; an empty key frame gives all zeros. */
int flb_keyframes_scan_contexts(flb_keyframes* kf, const int* ids, int n_ids, double lidar_height, double* out_descs);

/* ------------------------------------------------------------------------------------------------ loop registration
 * performLoopClosure's ICP (laserMapping.cpp:946-974): pcl::IterativeClosestPoint<PointType, PointType> (PCL 1.10) with an
 * identity guess, between the two dense loop sub-maps of the store, computed where they are; no cloud is downloaded.
 * Source = the dense assembly of (src_ids, src_transforms), then transformPointCloud(.., pose6 src_pre_pose6) when it is
 * not NULL (the Scan Context yaw `com`, :954-962); target = the dense assembly of (tgt_ids, tgt_transforms); both as
 * flb_keyframes_assemble writes them.  A point's index is its position in the assembled cloud.  Each iteration pairs every
 * finite source point with its exact nearest finite target point (float d² = (dx*dx + dy*dy) + dz*dz; equal d²: the lower
 * target index), keeps the pairs with d² <= max_correspondence_distance² (in double), stops with NO_CORRESPONDENCES below 3
 * pairs, fits R, t by Umeyama (SVD of the cross-covariance, reflection-corrected; sums in double, fixed order), applies
 * the float increment to the source and to the final transformation and runs the DefaultConvergenceCriteria tests.
 * fitness_score is getFitnessScore(): the mean nearest d² of the original source moved once by the final transformation.
 * DESIGN.md §9 states the contract and its deviations from PCL.  Every argument is checked before any device work; one
 * synchronisation per iteration; the store and the map are not modified.  The sub-maps, the target index and the
 * reduction buffers are map-side key-frame scratch (flb_keyframes_info, flb_map_release_keyframe_scratch). */
#define FLB_ICP_NOT_CONVERGED 0      /* CONVERGENCE_CRITERIA_NOT_CONVERGED (also: empty source or target) */
#define FLB_ICP_ITERATIONS 1         /* nr_iterations >= max_iterations */
#define FLB_ICP_TRANSFORM 2          /* the increment is within transformation_epsilon */
#define FLB_ICP_ABS_MSE 3            /* |mse - previous mse| < 1e-12 */
#define FLB_ICP_REL_MSE 4            /* |mse - previous mse| / previous mse < euclidean_fitness_epsilon */
#define FLB_ICP_NO_CORRESPONDENCES 5 /* fewer than 3 pairs: not converged, the transformation so far is kept */
typedef struct flb_icp_config {
  double max_correspondence_distance;  /* setMaxCorrespondenceDistance (200, laserMapping.cpp:948) */
  int max_iterations;                  /* setMaximumIterations (100, :949) */
  double transformation_epsilon;       /* setTransformationEpsilon (1e-6, :950) */
  double euclidean_fitness_epsilon;    /* setEuclideanFitnessEpsilon (1e-6, :951) */
} flb_icp_config;
typedef struct flb_icp_result {
  float final_transformation[16];      /* getFinalTransformation(), row-major 4x4 */
  int converged;                       /* hasConverged() */
  int iterations, state;               /* nr_iterations_; FLB_ICP_* */
  int n_source, n_target, n_correspondences;   /* assembled sizes; pairs of the last iteration */
  double fitness_score;                /* getFitnessScore(); DBL_MAX when no point counts */
} flb_icp_result;
/* Registers the source selection onto the target selection.  Empty source or target (after dropping non-finite target
 * points): not converged, 0 iterations, identity, fitness DBL_MAX.  out_corr_index / out_corr_d2 (optional, n_source
 * entries each) receive the last iteration's nearest target index and its d² for every source point, before the distance
 * cut (-1 and +inf for a non-finite source point or when nothing was registered). */
int flb_keyframes_icp(flb_keyframes* kf, const int* src_ids, int n_src, int src_kind, const float* src_transforms,
                      const float* src_pre_pose6, const int* tgt_ids, int n_tgt, int tgt_kind, const float* tgt_transforms,
                      const flb_icp_config* cfg, flb_icp_result* out, int* out_corr_index, float* out_corr_d2);

/* ------------------------------------------------------------------------------------------------ inter-session registration
 * IncreMapping::run's inter-session loops (multi-session Incremental_mapping.cpp: addSCloops :651-696 with
 * doICPVirtualRelative :462-522, addRSloops :787-837 with doICPGlobalRelative :525-583), every pair of a round in one
 * call.  Pair p's source is src_ids[src_offsets[p] .. src_offsets[p+1]), each key frame moved by its own src_poses6 row
 * (FLB_KF_POSE6: transformPointCloud(.., &PointTypePose), a zero pose computed, not copied, as
 * loopFindNearKeyframesLocalCoord :119-139 does), concatenated as flb_keyframes_assemble writes it and, for
 * leaf_size > 0, VoxelGrid-filtered exactly as that call filters (PCL's int32 overflow guard included); leaf_size == 0
 * keeps the dense concatenation.  The target is built the same way from tgt_offsets / tgt_ids / tgt_poses6.  Each pair is
 * then registered as flb_keyframes_icp registers it (identity guess, no pre-pose): out[p] is that call's result on the
 * same clouds, bit for bit, with n_source / n_target the sizes after filtering.  An empty source, or a target without a
 * finite point, gives flb_keyframes_icp's empty result.  The pairs run in lockstep: each iteration is one exact 1-NN pass
 * over every active pair, one copy and one synchronisation; a pair that stops (converged or NO_CORRESPONDENCES) leaves
 * the lockstep and the others go on.  Pairs are packed in order into rounds whose summed grid cells stay within 2^27 (at
 * least one pair per round); a pair's result depends only on its own selections, never on its round or the other pairs.
 * Every argument is checked before any device work and an error names the pair and the field; n_pairs == 0 does
 * nothing.  The store and the map are not modified; the packed clouds and indices are map-side key-frame scratch
 * (flb_keyframes_info, flb_map_release_keyframe_scratch).  DESIGN.md §9 "Inter-session registration". */
typedef struct flb_icp_batch_stats {
  int rounds;            /* rounds the call split the batch into (pairs registered together in lockstep) */
  int setup_syncs;       /* host synchronisations spent on assembly, filters and index builds (one per filtered
                            selection, one per target box) */
  int iteration_syncs;   /* host synchronisations of the lockstep iterations and the fitness passes: per round, the most
                            passes any of its pairs ran (its iterations, plus one if it stopped with NO_CORRESPONDENCES),
                            plus one for the fitness pass */
} flb_icp_batch_stats;
int flb_keyframes_icp_batch(flb_keyframes* kf, int n_pairs, const int* src_offsets, const int* src_ids, const float* src_poses6,
                            const int* tgt_offsets, const int* tgt_ids, const float* tgt_poses6, float leaf_size,
                            const flb_icp_config* cfg, flb_icp_result* out /* n_pairs */, flb_icp_batch_stats* stats /* may be NULL */);

/* ------------------------------------------------------------------------------------------------ relocalisation registration
 * The online relocaliser's registration (pose_estimator::run, reg[0].run(curCloud, nearCloud), pose_estimator.cpp:180-269,
 * :566-596): FRICP<3>::point_to_point as Registeration::run (include/FRICP-toolkit/registeration.h:36-175) calls it, for
 * the four point-to-point modes.  Source = a host cloud (records of src_stride bytes, x, y, z floats first, intensity at
 * src_off_intensity or < 0 for none), moved by transformPointCloud(.., pose6 src_pose6) when that is not NULL (initPose,
 * :185).  Target = for every tgt_ids[j] the stored key frame moved by pose6 tgt_pre_pose6 (pose_ext; NULL: skipped) and
 * then by pose6 tgt_poses6[j] (cloudKeyPoses6D), each stage rounding like transformPointCloud, concatenated in order
 * (:189-194).  A point's index is its position in its cloud.  Non-finite points are dropped from both clouds; the clouds
 * are scaled by max(|source extent|, |target extent|) and de-meaned in double; each iteration matches every source point
 * to its exact nearest target point (double d², equal d²: the lower target index); Welsch weights, the weighted Kabsch
 * step, Anderson acceleration on the SE(3) log and the ν schedule follow the reference.  DESIGN.md §9 states the contract
 * and its deviations.  Every argument is checked before any device work; one synchronisation per iteration (two when
 * Anderson rejects); the store and the map are not modified.  The clouds, the target index and the reduction buffers are
 * map-side key-frame scratch (flb_keyframes_info, flb_map_release_keyframe_scratch). */
#define FLB_FRICP_ICP 0                /* regMode 0: no robust function, no Anderson acceleration */
#define FLB_FRICP_FAST 2               /* regMode 2: Anderson acceleration */
#define FLB_FRICP_ROBUST 3             /* regMode 3: Welsch */
#define FLB_FRICP_FAST_ROBUST 4        /* regMode 4: Welsch and Anderson acceleration (config/online_relo.yaml) */
#define FLB_FRICP_OK 0                 /* registered */
#define FLB_FRICP_FEW_TARGET 1         /* fewer than 2 finite target points: identity, nothing registered */
#define FLB_FRICP_NO_SOURCE 2          /* no finite source point: identity, nothing registered */
typedef struct flb_fricp_config {
  int mode;                            /* FLB_FRICP_*: regMode 0, 2, 3 or 4; any other mode is rejected */
  int max_icp;                         /* ICP::Parameters::max_icp (100): iterations per ν stage */
  double stop;                         /* stop (1e-5): a stage ends when |T - T_prev|_F < stop (normalised units) */
  int anderson_m;                      /* anderson_m (5), 1..5 */
  double nu_begin_k, nu_end_k, nu_alpha; /* 3, 1/(3√3), 1/2 */
} flb_fricp_config;
typedef struct flb_fricp_result {
  double res_trans[16];                /* Registeration::run's res_trans, row-major 4x4, translation in the caller's units */
  int status;                          /* FLB_FRICP_OK / _FEW_TARGET / _NO_SOURCE */
  int stages, iterations, rejections;  /* ν stages, ICP iterations over all stages, Anderson rejections */
  double scale, mu_source[3], mu_target[3];   /* the normalisation: p_n = p / scale - mu */
  double nu_begin, nu_end;             /* the Welsch scale's first and last value (0 without a robust function) */
  double energy;                       /* convergence energy at the final ν */
  int n_source, n_target;              /* source points; assembled target points */
  int n_source_finite, n_target_finite;
  int log_n;                           /* rows written to out_log */
} flb_fricp_result;
/* The reference's defaults (ICP::Parameters, ICP.h:518-566) with mode FLB_FRICP_FAST_ROBUST. */
void flb_fricp_default_config(flb_fricp_config* cfg);
/* Registers the source onto the target.  out_corr_index / out_resid (optional, n_src entries each) receive the last pass's
 * matched target index and its residual |T x - q| in normalised units (-1 and +inf for a non-finite source point or when
 * nothing was registered).  out_log (optional, log_cap rows of 5 doubles): per iteration the stage, the energy at the
 * start of the iteration, the last accepted energy before it, |T - T_prev|_F and 1 (accepted or no Anderson) / 0
 * (Anderson rejected). */
int flb_keyframes_fricp(flb_keyframes* kf, const void* src_points, int n_src, int src_stride, int src_off_intensity,
                        const float* src_pose6, const int* tgt_ids, int n_tgt, const float* tgt_pre_pose6, const float* tgt_poses6,
                        const flb_fricp_config* cfg, flb_fricp_result* out, int* out_corr_index, double* out_resid,
                        double* out_log, int log_cap);

/* ------------------------------------------------------------------------------------------------ relocalisation Sparse ICP
 * The relocaliser's regMode 7 (Sparse ICP, SICP::point_to_point, include/FRICP-toolkit/ICP.h:275-380, with Registeration's
 * SICP::Parameters, registeration.h:67-69, :143-146).  Source, target, the dropping of non-finite points and the
 * normalisation are flb_keyframes_fricp's.  Each ICP iteration matches every source point X_i to its exact nearest target
 * point Q_i (double d², equal d²: the lower target index), then runs the ADMM loop: Z = (X - Q) + C/μ shrunk by the ℓp
 * operator, the unweighted Kabsch step onto U = (Q + Z) - C/μ, X and T moved, C += μ ((X - Q) - Z), μ *= alpha while
 * μ < max_mu, until max |P| and Σ|ΔX|²/n are both below stop or max_outer passes.  Z and C persist across ICP iterations;
 * μ restarts from mu.  The ICP loop ends after max_icp iterations or when max |X - X_prev| < stop.  DESIGN.md §9 states
 * the contract and its deviations.  The whole ADMM loop runs on the device: one synchronisation per ICP iteration.  Every
 * argument is checked before any device work; the store and the map are not modified.  The ADMM state is map-side
 * key-frame scratch (flb_keyframes_info, flb_map_release_keyframe_scratch).  Statuses are FLB_FRICP_*; FEW_TARGET means
 * no finite target point. */
typedef struct flb_sicp_config {
  double p;                            /* the ℓp exponent (0.4), in (0, 1] */
  double mu, alpha, max_mu;            /* the penalty's start (10), growth factor (1.2, >= 1) and cap (1e5) */
  int max_icp, max_outer;              /* ICP iterations (100); ADMM iterations per ICP iteration (100) */
  double stop;                         /* stopping threshold (1e-5, normalised units) */
} flb_sicp_config;
typedef struct flb_sicp_result {
  double res_trans[16];                /* Registeration::run's res_trans, row-major 4x4, translation in the caller's units */
  int status;                          /* FLB_FRICP_OK / _FEW_TARGET / _NO_SOURCE */
  int iterations, admm_iterations;     /* ICP iterations; ADMM iterations over all of them */
  double scale, mu_source[3], mu_target[3];   /* the normalisation: p_n = p / scale - mu */
  int n_source, n_target;              /* source points; assembled target points */
  int n_source_finite, n_target_finite;
  double primal, dual, stop, mu_exit;  /* the last ICP iteration's max |P|, Σ|ΔX|²/n, max |X - X_prev| and μ at its exit */
  int syncs;                           /* host synchronisations the call made */
  int admm_blocks;                     /* blocks of 256 threads the ADMM kernel ran on (all resident) */
  int log_n;                           /* rows written to out_log */
} flb_sicp_result;
/* Registeration's SICP::Parameters: p 0.4, mu 10, alpha 1.2, max_mu 1e5, max_icp 100, max_outer 100, stop 1e-5. */
void flb_sicp_default_config(flb_sicp_config* cfg);
/* Registers the source onto the target.  out_corr_index / out_resid (optional, n_src entries each) receive the last ICP
 * iteration's matched target index and the residual |X - Q| of that match in normalised units, before its ADMM loop (-1
 * and +inf for a non-finite source point or when nothing was matched).  out_log (optional, log_cap rows of 5 doubles): per
 * ICP iteration the ADMM iterations, primal, dual, stop and μ at its exit. */
int flb_keyframes_sicp(flb_keyframes* kf, const void* src_points, int n_src, int src_stride, int src_off_intensity,
                       const float* src_pose6, const int* tgt_ids, int n_tgt, const float* tgt_pre_pose6, const float* tgt_poses6,
                       const flb_sicp_config* cfg, flb_sicp_result* out, int* out_corr_index, double* out_resid,
                       double* out_log, int log_cap);

/* ------------------------------------------------------------------------------------------------ relocalisation AA-ICP
 * The relocaliser's regMode 1 (AA-ICP, AAICP::point_to_point_aaicp, include/FRICP-toolkit/ICP.h:841-1033, with
 * Registeration's ICP::Parameters: no robust function, no initial transform).  Source, target, the dropping of non-finite
 * points and the normalisation are flb_keyframes_fricp's.  Each iteration matches every moved source point X = final X0
 * to its exact nearest target point Q (double d², equal d²: the lower target index), takes the unweighted Kabsch step on
 * (X, Q) into T, and mixes the 6-vectors (eulerAngles(0, 1, 2), t) of the transforms by Anderson acceleration over the
 * whole history, restarting it when the energy Σ|X - Q|² rises by more than error_overflow_threshold relative.  The loop
 * ends after max_icp iterations or when |final - final_prev|_F < stop after the first.  DESIGN.md §9 states the contract
 * and its deviations.  One synchronisation per iteration; the Euler, QR and Anderson work runs on the host.  Every
 * argument is checked before any device work; the store and the map are not modified.  The scratch is
 * flb_keyframes_fricp's map-side key-frame scratch.  Statuses are FLB_FRICP_*; FEW_TARGET means no finite target point. */
typedef struct flb_aaicp_config {
  int max_icp;                         /* ICP::Parameters::max_icp (100), >= 0 */
  double stop;                         /* stop (1e-5, normalised units), finite and >= 0 */
  double error_overflow_threshold;     /* error_overflow_threshold_ (0.05), finite: the relative energy rise that resets */
} flb_aaicp_config;
typedef struct flb_aaicp_result {
  double res_trans[16];                /* Registeration::run's res_trans, row-major 4x4, translation in the caller's units */
  int status;                          /* FLB_FRICP_OK / _FEW_TARGET / _NO_SOURCE */
  int iterations;                      /* par.convergence_iter: the loop index at exit (passes run - 1 when the stop test
                                          ended the loop, max_icp otherwise) */
  int accepted, resets;                /* Anderson steps taken; times the first heuristic reset the history */
  int history;                         /* columns of the Anderson history u at exit */
  double energy;                       /* convergence_energy: Σ |final X0 - Q|² over the last pass's matches */
  double scale, mu_source[3], mu_target[3];   /* the normalisation: p_n = p / scale - mu */
  int n_source, n_target;              /* source points; assembled target points */
  int n_source_finite, n_target_finite;
  int syncs;                           /* host synchronisations the call made */
  int log_n;                           /* rows written to out_log */
} flb_aaicp_result;
/* Registeration's ICP::Parameters as AA-ICP reads them: max_icp 100, stop 1e-5, error_overflow_threshold 0.05. */
void flb_aaicp_default_config(flb_aaicp_config* cfg);
/* Registers the source onto the target.  out_corr_index / out_resid (optional, n_src entries each) receive the last
 * pass's matched target index and |X - Q| in normalised units (-1 and +inf for a non-finite source point or when no pass
 * ran).  out_log (optional, log_cap rows of 6 doubles): per iteration the energy, the previous energy before the first
 * heuristic's test, the outcome (-1 the first iteration, 1 Anderson step accepted, 0 reset), the number of α in u_next,
 * |final - final_prev|_F and the smallest margin of the alphas_cond tests made (+inf when none was made). */
int flb_keyframes_aaicp(flb_keyframes* kf, const void* src_points, int n_src, int src_stride, int src_off_intensity,
                        const float* src_pose6, const int* tgt_ids, int n_tgt, const float* tgt_pre_pose6, const float* tgt_poses6,
                        const flb_aaicp_config* cfg, flb_aaicp_result* out, int* out_corr_index, double* out_resid,
                        double* out_log, int log_cap);

/* ------------------------------------------------------------------------------------------------ IMU propagation
 * ImuProcess::Process (src/IMU_Processing.hpp:393-434) on a front end: IMU_init (:174-233, with the MAX_INI_COUNT logic
 * of :405-427) on the host, the forward propagation of UndistortPcl (:241-331, kf.predict esekfom.hpp:280-384) in one
 * device kernel that writes IMUpose and the end state where the undistortion reads them, then the undistortion and
 * (optionally) the voxel filter of the front end's current raw scan.  DESIGN.md §10 states the contract. */
typedef struct flb_imu flb_imu;

typedef struct flb_imu_config {
  double Lidar_T_wrt_IMU[3];  /* set_extrinsic (laserMapping.cpp:2142-2143) */
  double Lidar_R_wrt_IMU[9];  /* row-major rotation */
  double cov_gyr_scale[3];    /* set_gyr_cov: cov_gyr after initialisation */
  double cov_acc_scale[3];    /* set_acc_cov: cov_acc after initialisation */
  double cov_bias_gyr[3];     /* set_gyr_bias_cov */
  double cov_bias_acc[3];     /* set_acc_bias_cov */
} flb_imu_config;

/* status of flb_imu_process */
#define FLB_IMU_EMPTY 0       /* meas.imu empty: nothing done (:398-401) */
#define FLB_IMU_INIT 1        /* IMU_init ran; state26 / P written; the scan was not touched (:405-427) */
#define FLB_IMU_PROPAGATED 2  /* propagated and undistorted (:430) */

typedef struct flb_imu_result {
  int status;
  int n_poses;        /* IMUpose.size() (1 + the segments that were not skipped) */
  int n_predicts;     /* kf.predict calls: n_poses - 1 + 1 */
  int n_down;         /* feats_down_size when leaf > 0, else -1 */
  float gpu_ms;       /* device time of the call from the staging upload to the read-back (0 unless status 2) */
} flb_imu_result;

typedef struct flb_imu_state {  /* the persistent members of ImuProcess */
  double mean_acc[3], mean_gyr[3], cov_acc[3], cov_gyr[3];
  double last_lidar_end_time; /* last_lidar_end_time_ (0 before the first propagation) */
  double angvel_last[3], acc_s_last[3];
  double last_imu[7];         /* last_imu_: stamp, acc, gyro (zero before the first sample) */
  int init_iter_num, imu_need_init, b_first_frame, n_poses;
} flb_imu_state;

/* laserMapping.cpp's defaults (:51, :2142-2146): gyr / acc 0.1, biases 1e-4, identity extrinsic. */
void flb_imu_default_config(flb_imu_config* cfg);
/* Every field must be finite; errors name the field.  The propagation uses the front end's stream and pose buffer. */
int flb_imu_create(flb_frontend* fe, const flb_imu_config* cfg, flb_imu** out);
void flb_imu_destroy(flb_imu* imu);
/* ImuProcess::Reset (:90-102): b_first_frame_ is left as it is. */
int flb_imu_reset(flb_imu* imu);
/* p_imu->Process(Measures, kf, feats_undistort) (laserMapping.cpp:2256).  imu7 = the n_imu samples of meas.imu in order
 * (stamp, ax, ay, az, gx, gy, gz), 0 <= n_imu <= FLB_MAX_IMU_POSES - 1; state26 / P (23x23 row-major) come in as
 * kf.get_x() / kf.get_P() and go out as the prior.  The scan is the front end's current raw scan (flb_frontend_upload or
 * flb_frontend_preprocess); leaf > 0 then runs the voxel filter into feats_down_body as flb_frontend_voxel_filter does.
 * A propagation (status 2) ends in exactly one synchronisation, which returns the prior, P and the filtered count.
 * Non-finite samples, times or state and n_imu out of range are rejected with nothing changed. */
int flb_imu_process(flb_imu* imu, const double* imu7, int n_imu, double lidar_beg_time, double lidar_end_time, double* state26,
                    double* P, float leaf, flb_imu_result* out);
/* IMUpose of the last propagation (n x 22 doubles, FLB_IMU_POSE_DOUBLES layout); at most cap records, *n = its size. */
int flb_imu_download_poses(flb_imu* imu, double* out22, int cap, int* n);
int flb_imu_info(const flb_imu* imu, flb_imu_state* out);

/* Stream access for callers that overlap work (returns a cudaStream_t as void*). */
void* flb_session_stream(flb_session* s);
int flb_session_sync(flb_session* s);

#ifdef __cplusplus
}
#endif
#endif /* FASTLIO_B200_H_ */

"""ctypes view of the C ABI in include/fastlio_b200.h (libfastlio_b200.so, hand-written sm_90a CUDA).

This is plumbing for tests / bench only: the product is the shared library and the C++ facades under
include/fastlio_b200/.  Class and method names mirror the reference interface they stand in for
(KD_TREE: include/ikd-Tree/ikd_Tree.h:225-249; esekf update + h_share_model: esekfom.hpp:1620, laserMapping.cpp:1876).

There is NO CPU fallback: if the CUDA library is missing or no device is visible, calls raise FlbError.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# FLB_LIB selects another build of the SAME library (debug/trace or A/B kernel variants); there is still no CPU fallback
LIB_PATH = os.environ.get("FLB_LIB") or os.path.join(_HERE, "libfastlio_b200.so")

NACC_DOF = 23


class FlbError(RuntimeError):
    pass


class MapConfig(C.Structure):
    _fields_ = [("voxel_size", C.c_float), ("max_points", C.c_int), ("max_blocks", C.c_int), ("device", C.c_int)]


class MapStats(C.Structure):
    _fields_ = [("valid_points", C.c_int), ("blocks_in_use", C.c_int), ("block_capacity", C.c_int),
                ("overflow_in_use", C.c_int), ("overflow_capacity", C.c_int), ("hash_capacity", C.c_int),
                ("hash_tombstones", C.c_int), ("coarse_cells", C.c_int), ("rehash_count", C.c_int),
                ("device_bytes", C.c_size_t)]


class SessionConfig(C.Structure):
    _fields_ = [("max_scan_points", C.c_int), ("extrinsic_est_en", C.c_int), ("max_iterations", C.c_int),
                ("laser_point_cov", C.c_double), ("filter_size_map_min", C.c_double), ("limit", C.c_double * 23)]


class PassResult(C.Structure):
    _fields_ = [("valid", C.c_int), ("effct_feat_num", C.c_int), ("total_residual", C.c_double),
                ("HTH", C.c_double * 144), ("HTh", C.c_double * 12)]


class UpdateStats(C.Structure):
    _fields_ = [("passes", C.c_int), ("search_passes", C.c_int), ("effct_feat_num", C.c_int),
                ("converged_count", C.c_int), ("total_residual", C.c_double), ("gpu_ms", C.c_float)]


class FovState(C.Structure):
    _fields_ = [("local_map_min", C.c_float * 3), ("local_map_max", C.c_float * 3), ("initialized", C.c_int),
                ("cube_len", C.c_double), ("det_range", C.c_float), ("pos_lid", C.c_double * 3)]


class ScanResult(C.Structure):
    _fields_ = [("update", UpdateStats), ("n_to_add", C.c_int), ("n_no_downsample", C.c_int), ("n_deleted", C.c_int),
                ("map_valid", C.c_int), ("gpu_ms_total", C.c_float), ("kernel_launches", C.c_int)]


class Profile(C.Structure):
    _fields_ = [("ms", C.c_double * 8), ("launches", C.c_int * 8), ("regions", C.c_int * 8), ("knn_phase", C.c_longlong * 4),
                ("knn_head_candidates", C.c_longlong), ("knn_chain_nodes", C.c_longlong), ("knn_chain_max", C.c_longlong)]


class PreprocessConfig(C.Structure):
    _fields_ = [("lidar_type", C.c_int), ("n_scans", C.c_int), ("scan_rate", C.c_int), ("point_filter_num", C.c_int),
                ("time_unit", C.c_int), ("blind", C.c_double)]


class RawLayout(C.Structure):
    _fields_ = [("stride", C.c_int), ("off_x", C.c_int), ("off_y", C.c_int), ("off_z", C.c_int), ("off_intensity", C.c_int),
                ("off_time", C.c_int), ("off_ring", C.c_int), ("off_tag", C.c_int), ("off_line", C.c_int)]


class IcpConfig(C.Structure):
    _fields_ = [("max_correspondence_distance", C.c_double), ("max_iterations", C.c_int),
                ("transformation_epsilon", C.c_double), ("euclidean_fitness_epsilon", C.c_double)]


class FricpConfig(C.Structure):
    _fields_ = [("mode", C.c_int), ("max_icp", C.c_int), ("stop", C.c_double), ("anderson_m", C.c_int),
                ("nu_begin_k", C.c_double), ("nu_end_k", C.c_double), ("nu_alpha", C.c_double)]


class FricpResult(C.Structure):
    _fields_ = [("res_trans", C.c_double * 16), ("status", C.c_int), ("stages", C.c_int), ("iterations", C.c_int),
                ("rejections", C.c_int), ("scale", C.c_double), ("mu_source", C.c_double * 3), ("mu_target", C.c_double * 3),
                ("nu_begin", C.c_double), ("nu_end", C.c_double), ("energy", C.c_double), ("n_source", C.c_int),
                ("n_target", C.c_int), ("n_source_finite", C.c_int), ("n_target_finite", C.c_int), ("log_n", C.c_int)]


FRICP_STATUS = ["OK", "FEW_TARGET", "NO_SOURCE"]


class SicpConfig(C.Structure):
    _fields_ = [("p", C.c_double), ("mu", C.c_double), ("alpha", C.c_double), ("max_mu", C.c_double), ("max_icp", C.c_int),
                ("max_outer", C.c_int), ("stop", C.c_double)]


class SicpResult(C.Structure):
    _fields_ = [("res_trans", C.c_double * 16), ("status", C.c_int), ("iterations", C.c_int), ("admm_iterations", C.c_int),
                ("scale", C.c_double), ("mu_source", C.c_double * 3), ("mu_target", C.c_double * 3), ("n_source", C.c_int),
                ("n_target", C.c_int), ("n_source_finite", C.c_int), ("n_target_finite", C.c_int), ("primal", C.c_double),
                ("dual", C.c_double), ("stop", C.c_double), ("mu_exit", C.c_double), ("syncs", C.c_int), ("admm_blocks", C.c_int),
                ("log_n", C.c_int)]


class AaicpConfig(C.Structure):
    _fields_ = [("max_icp", C.c_int), ("stop", C.c_double), ("error_overflow_threshold", C.c_double)]


class AaicpResult(C.Structure):
    _fields_ = [("res_trans", C.c_double * 16), ("status", C.c_int), ("iterations", C.c_int), ("accepted", C.c_int),
                ("resets", C.c_int), ("history", C.c_int), ("energy", C.c_double), ("scale", C.c_double),
                ("mu_source", C.c_double * 3), ("mu_target", C.c_double * 3), ("n_source", C.c_int), ("n_target", C.c_int),
                ("n_source_finite", C.c_int), ("n_target_finite", C.c_int), ("syncs", C.c_int), ("log_n", C.c_int)]


class IcpResult(C.Structure):
    _fields_ = [("final_transformation", C.c_float * 16), ("converged", C.c_int), ("iterations", C.c_int), ("state", C.c_int),
                ("n_source", C.c_int), ("n_target", C.c_int), ("n_correspondences", C.c_int), ("fitness_score", C.c_double)]


class ImuConfig(C.Structure):
    _fields_ = [("Lidar_T_wrt_IMU", C.c_double * 3), ("Lidar_R_wrt_IMU", C.c_double * 9), ("cov_gyr_scale", C.c_double * 3),
                ("cov_acc_scale", C.c_double * 3), ("cov_bias_gyr", C.c_double * 3), ("cov_bias_acc", C.c_double * 3)]


class ImuResult(C.Structure):
    _fields_ = [("status", C.c_int), ("n_poses", C.c_int), ("n_predicts", C.c_int), ("n_down", C.c_int), ("gpu_ms", C.c_float)]


class ImuState(C.Structure):
    _fields_ = [("mean_acc", C.c_double * 3), ("mean_gyr", C.c_double * 3), ("cov_acc", C.c_double * 3), ("cov_gyr", C.c_double * 3),
                ("last_lidar_end_time", C.c_double), ("angvel_last", C.c_double * 3), ("acc_s_last", C.c_double * 3),
                ("last_imu", C.c_double * 7), ("init_iter_num", C.c_int), ("imu_need_init", C.c_int), ("b_first_frame", C.c_int),
                ("n_poses", C.c_int)]


IMU_EMPTY, IMU_INIT, IMU_PROPAGATED = 0, 1, 2


class IcpBatchStats(C.Structure):
    _fields_ = [("rounds", C.c_int), ("setup_syncs", C.c_int), ("iteration_syncs", C.c_int)]


K_CLASSES = ["transform", "knn", "residual", "reduce", "classify", "insert", "delete"]

_lib = None

# every symbol include/fastlio_b200.h declares
EXPORTS = [
    "flb_last_error", "flb_device_count", "flb_version", "flb_map_create", "flb_map_destroy",
    "flb_map_set_downsample_param", "flb_map_has_root", "flb_map_build", "flb_map_reconstruct", "flb_map_add_points",
    "flb_map_delete_boxes", "flb_map_delete_points", "flb_map_nearest_search", "flb_map_box_search",
    "flb_map_radius_search", "flb_map_validnum", "flb_map_size", "flb_map_flatten", "flb_map_range",
    "flb_map_get_stats", "flb_session_default_config", "flb_session_create", "flb_session_destroy", "flb_scan_upload",
    "flb_scan_set_device", "flb_pass", "flb_pass_rows", "flb_esikf_update", "flb_map_incremental",
    "flb_neighbors_download", "flb_fov_segment", "flb_scan_step", "flb_session_stream", "flb_session_sync",
    "flb_map_profile_enable", "flb_map_profile_read", "flb_session_set_update_engine", "flb_scan_prefetch", "flb_scan_step_begin", "flb_scan_step_finish",
    "flb_frontend_create", "flb_frontend_destroy", "flb_frontend_upload", "flb_frontend_undistort",
    "flb_frontend_voxel_filter", "flb_frontend_process", "flb_frontend_download_undistorted", "flb_frontend_download_down",
    "flb_frontend_points_to_world", "flb_voxel_grid_filter", "flb_map_reconstruct_keyframes",
    "flb_map_build_pt", "flb_map_reconstruct_pt", "flb_map_add_points_pt", "flb_map_nearest_search_xyzi",
    "flb_map_box_search_xyzi", "flb_map_radius_search_xyzi", "flb_map_flatten_xyzi", "flb_scan_upload_pt",
    "flb_frontend_preprocess",
    "flb_keyframes_create", "flb_keyframes_destroy", "flb_keyframes_append_frontend", "flb_keyframes_append",
    "flb_keyframes_download", "flb_keyframes_info", "flb_keyframes_size", "flb_map_reconstruct_from_keyframes",
    "flb_keyframes_assemble", "flb_map_release_keyframe_scratch",
    "flb_keyframes_scan_context", "flb_keyframes_scan_contexts", "flb_keyframes_icp",
    "flb_keyframes_icp_batch",
    "flb_fricp_default_config", "flb_keyframes_fricp", "flb_sicp_default_config", "flb_keyframes_sicp",
    "flb_aaicp_default_config", "flb_keyframes_aaicp",
    "flb_frontend_camera_config", "flb_frontend_camera_image", "flb_frontend_points_colorize", "flb_frontend_points_to_imu",
    "flb_imu_default_config", "flb_imu_create", "flb_imu_destroy", "flb_imu_reset", "flb_imu_process",
    "flb_imu_download_poses", "flb_imu_info",
]


def lib():
    """Load the CUDA library. Fails loudly when it has not been built (python __graft_entry__.py build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FlbError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        vp, ip, fp, dp = C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.c_void_p
        L.flb_last_error.restype = C.c_char_p
        L.flb_version.restype = C.c_char_p
        L.flb_map_create.argtypes = [C.POINTER(MapConfig), C.POINTER(vp)]
        L.flb_map_destroy.argtypes = [vp]
        L.flb_map_destroy.restype = None
        L.flb_map_set_downsample_param.argtypes = [vp, C.c_float]
        L.flb_map_has_root.argtypes = [vp]
        L.flb_map_build.argtypes = [vp, fp, C.c_int, C.c_int]
        L.flb_map_reconstruct.argtypes = [vp, fp, C.c_int, C.c_int]
        L.flb_map_add_points.argtypes = [vp, fp, C.c_int, C.c_int, C.c_int, ip]
        L.flb_map_build_pt.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
        L.flb_map_reconstruct_pt.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
        L.flb_map_add_points_pt.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, ip]
        L.flb_map_nearest_search_xyzi.argtypes = [vp, fp, C.c_int, C.c_int, C.c_int, C.c_float, fp, fp, vp]
        L.flb_map_box_search_xyzi.argtypes = [vp, fp, fp, C.c_int, ip]
        L.flb_map_radius_search_xyzi.argtypes = [vp, fp, C.c_float, fp, C.c_int, ip]
        L.flb_map_flatten_xyzi.argtypes = [vp, fp, C.c_int, ip]
        L.flb_scan_upload_pt.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
        L.flb_map_delete_boxes.argtypes = [vp, fp, C.c_int, ip]
        L.flb_map_delete_points.argtypes = [vp, fp, C.c_int, C.c_int, ip]
        L.flb_map_nearest_search.argtypes = [vp, fp, C.c_int, C.c_int, C.c_int, C.c_float, fp, fp, vp]
        L.flb_map_box_search.argtypes = [vp, fp, fp, C.c_int, ip]
        L.flb_map_radius_search.argtypes = [vp, fp, C.c_float, fp, C.c_int, ip]
        L.flb_map_validnum.argtypes = [vp]
        L.flb_map_size.argtypes = [vp]
        L.flb_map_flatten.argtypes = [vp, fp, C.c_int, ip]
        L.flb_map_range.argtypes = [vp, fp]
        L.flb_map_get_stats.argtypes = [vp, C.POINTER(MapStats)]
        L.flb_session_default_config.argtypes = [C.POINTER(SessionConfig)]
        L.flb_session_default_config.restype = None
        L.flb_session_create.argtypes = [vp, C.POINTER(SessionConfig), C.POINTER(vp)]
        L.flb_session_destroy.argtypes = [vp]
        L.flb_session_destroy.restype = None
        L.flb_scan_upload.argtypes = [vp, fp, C.c_int, C.c_int]
        L.flb_scan_set_device.argtypes = [vp, vp, C.c_int]
        L.flb_scan_prefetch.argtypes = [vp, fp, C.c_int, C.c_int]
        L.flb_pass.argtypes = [vp, dp, C.c_int, C.POINTER(PassResult)]
        L.flb_pass_rows.argtypes = [vp, dp, C.c_int, dp, C.c_int, ip]
        L.flb_esikf_update.argtypes = [vp, dp, dp, C.POINTER(UpdateStats)]
        L.flb_map_incremental.argtypes = [vp, dp, C.c_int, ip, ip]
        L.flb_neighbors_download.argtypes = [vp, fp, fp, vp, vp, fp, fp]
        L.flb_fov_segment.argtypes = [vp, C.POINTER(FovState), dp, fp, ip, ip]
        L.flb_scan_step.argtypes = [vp, C.POINTER(FovState), fp, C.c_int, C.c_int, dp, dp, C.c_int, C.POINTER(ScanResult)]
        L.flb_scan_step_begin.argtypes = [vp, C.POINTER(FovState), fp, C.c_int, C.c_int, dp, dp, C.c_int]
        L.flb_scan_step_finish.argtypes = [vp, C.POINTER(FovState), dp, dp, C.POINTER(ScanResult)]
        L.flb_session_stream.argtypes = [vp]
        L.flb_session_stream.restype = vp
        L.flb_session_sync.argtypes = [vp]
        L.flb_session_set_update_engine.argtypes = [vp, C.c_int]
        L.flb_map_profile_enable.argtypes = [vp, C.c_int]
        L.flb_map_profile_read.argtypes = [vp, C.POINTER(Profile), C.c_int]
        L.flb_frontend_create.argtypes = [vp, C.c_int, C.POINTER(vp)]
        L.flb_frontend_destroy.argtypes = [vp]
        L.flb_frontend_destroy.restype = None
        L.flb_frontend_upload.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]
        L.flb_frontend_undistort.argtypes = [vp, dp, C.c_int, dp]
        L.flb_frontend_voxel_filter.argtypes = [vp, C.c_float, ip]
        L.flb_frontend_process.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, dp, C.c_int, dp, C.c_float, ip]
        L.flb_frontend_download_undistorted.argtypes = [vp, fp, fp, vp, C.c_int, ip]
        L.flb_frontend_download_down.argtypes = [vp, fp, fp, C.c_int, ip]
        L.flb_frontend_points_to_world.argtypes = [vp, C.c_int, dp, fp, C.c_int, ip]
        L.flb_frontend_camera_config.argtypes = [vp, dp, dp, C.c_int, C.c_int]
        L.flb_frontend_camera_image.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
        L.flb_frontend_points_colorize.argtypes = [vp, C.c_int, dp, fp, vp, C.c_int, ip]
        L.flb_frontend_points_to_imu.argtypes = [vp, dp, fp, C.c_int, ip]
        L.flb_voxel_grid_filter.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_float, fp, C.c_int, ip]
        L.flb_frontend_preprocess.argtypes = [vp, C.POINTER(PreprocessConfig), C.POINTER(RawLayout), vp, C.c_int, ip,
                                              C.POINTER(C.c_float)]
        L.flb_map_reconstruct_keyframes.argtypes = [vp, C.POINTER(vp), ip, C.c_int, C.c_int, C.c_int, fp, C.c_float, fp,
                                                    C.c_int, ip]
        llp = C.POINTER(C.c_longlong)
        L.flb_keyframes_create.argtypes = [vp, C.c_longlong, C.c_int, C.POINTER(vp)]
        L.flb_keyframes_destroy.argtypes = [vp]
        L.flb_keyframes_destroy.restype = None
        L.flb_keyframes_append_frontend.argtypes = [vp, vp, ip]
        L.flb_keyframes_append.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, ip]
        L.flb_keyframes_download.argtypes = [vp, C.c_int, fp, fp, C.c_int, ip]
        L.flb_keyframes_info.argtypes = [vp, ip, llp, llp, llp]
        L.flb_map_release_keyframe_scratch.argtypes = [vp]
        L.flb_keyframes_size.argtypes = [vp, C.c_int]
        L.flb_map_reconstruct_from_keyframes.argtypes = [vp, vp, vp, C.c_int, fp, C.c_float, fp, C.c_int, ip]
        L.flb_keyframes_assemble.argtypes = [vp, vp, C.c_int, C.c_int, fp, C.c_float, fp, fp, C.c_int, ip]
        L.flb_keyframes_scan_context.argtypes = [vp, vp, C.c_int, C.c_int, fp, C.c_double, dp]
        L.flb_keyframes_scan_contexts.argtypes = [vp, vp, C.c_int, C.c_double, dp]
        L.flb_keyframes_icp.argtypes = [vp, vp, C.c_int, C.c_int, fp, fp, vp, C.c_int, C.c_int, fp, C.POINTER(IcpConfig),
                                        C.POINTER(IcpResult), vp, fp]
        L.flb_keyframes_icp_batch.argtypes = [vp, C.c_int, vp, vp, fp, vp, vp, fp, C.c_float, C.POINTER(IcpConfig),
                                              C.POINTER(IcpResult), C.POINTER(IcpBatchStats)]
        L.flb_fricp_default_config.argtypes = [C.POINTER(FricpConfig)]
        L.flb_fricp_default_config.restype = None
        L.flb_keyframes_fricp.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, fp, vp, C.c_int, fp, fp, C.POINTER(FricpConfig),
                                          C.POINTER(FricpResult), vp, dp, dp, C.c_int]
        L.flb_sicp_default_config.argtypes = [C.POINTER(SicpConfig)]
        L.flb_sicp_default_config.restype = None
        L.flb_keyframes_sicp.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, fp, vp, C.c_int, fp, fp, C.POINTER(SicpConfig),
                                         C.POINTER(SicpResult), vp, dp, dp, C.c_int]
        L.flb_aaicp_default_config.argtypes = [C.POINTER(AaicpConfig)]
        L.flb_aaicp_default_config.restype = None
        L.flb_keyframes_aaicp.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, fp, vp, C.c_int, fp, fp, C.POINTER(AaicpConfig),
                                          C.POINTER(AaicpResult), vp, dp, dp, C.c_int]
        L.flb_imu_default_config.argtypes = [C.POINTER(ImuConfig)]
        L.flb_imu_default_config.restype = None
        L.flb_imu_create.argtypes = [vp, C.POINTER(ImuConfig), C.POINTER(vp)]
        L.flb_imu_destroy.argtypes = [vp]
        L.flb_imu_destroy.restype = None
        L.flb_imu_reset.argtypes = [vp]
        L.flb_imu_process.argtypes = [vp, dp, C.c_int, C.c_double, C.c_double, dp, dp, C.c_float, C.POINTER(ImuResult)]
        L.flb_imu_download_poses.argtypes = [vp, dp, C.c_int, ip]
        L.flb_imu_info.argtypes = [vp, C.POINTER(ImuState)]
        _lib = L
    return _lib


def _chk(rc):
    if rc != 0:
        raise FlbError(lib().flb_last_error().decode())


def _xyz(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] not in (3, 4):
        raise ValueError("points must be (n,3) or (n,4) float32")
    return a


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class KDTree:
    """Device hashed-voxel map behind the KD_TREE<PointType> API of the reference (ikd_Tree.h:225-249)."""

    def __init__(self, voxel_size=0.2, max_points=1 << 20, max_blocks=0, device=0):
        self.h = C.c_void_p()
        cfg = MapConfig(float(voxel_size), int(max_points), int(max_blocks), int(device))
        _chk(lib().flb_map_create(C.byref(cfg), C.byref(self.h)))
        self.voxel_size = float(voxel_size)
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            lib().flb_map_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_downsample_param(self, v):
        _chk(lib().flb_map_set_downsample_param(self.h, float(v)))

    @property
    def Root_Node(self):
        return True if lib().flb_map_has_root(self.h) else None

    def Build(self, pts):
        pts = _xyz(pts)
        _chk(lib().flb_map_build(self.h, _p(pts), len(pts), pts.strides[0]))

    def reconstruct(self, pts):
        pts = _xyz(pts)
        _chk(lib().flb_map_reconstruct(self.h, _p(pts), len(pts), pts.strides[0]))

    def Add_Points(self, pts, downsample_on):
        pts = _xyz(pts)
        n = C.c_int(0)
        _chk(lib().flb_map_add_points(self.h, _p(pts), len(pts), pts.strides[0], 1 if downsample_on else 0, C.byref(n)))
        return n.value

    # PointType-aware variants: (n, 4) arrays of x, y, z, intensity (ikd_Tree.h:64-86 keeps whole records)
    def Build_xyzi(self, pts4):
        a = np.ascontiguousarray(pts4, np.float32).reshape(-1, 4)
        _chk(lib().flb_map_build_pt(self.h, _p(a), len(a), 16, 12))

    def Add_Points_xyzi(self, pts4, downsample_on):
        a = np.ascontiguousarray(pts4, np.float32).reshape(-1, 4)
        n = C.c_int(0)
        _chk(lib().flb_map_add_points_pt(self.h, _p(a), len(a), 16, 12, 1 if downsample_on else 0, C.byref(n)))
        return n.value

    def Build_pointtype(self, points48):
        a = np.ascontiguousarray(points48, np.float32).reshape(-1, 12)
        _chk(lib().flb_map_build_pt(self.h, _p(a), len(a), POINT_STRIDE, OFF_INTENSITY))

    def Nearest_Search_xyzi(self, q, k=5, max_dist=0.0):
        q = _xyz(q)
        n = len(q)
        out = np.empty((n, k, 4), np.float32)
        d2 = np.empty((n, k), np.float32)
        cnt = np.empty(n, np.int32)
        _chk(lib().flb_map_nearest_search_xyzi(self.h, _p(q), n, q.strides[0], k, float(max_dist), _p(out), _p(d2), _p(cnt)))
        return out, d2, cnt

    def flatten_xyzi(self):
        n = C.c_int(0)
        _chk(lib().flb_map_flatten_xyzi(self.h, None, 0, C.byref(n)))
        out = np.empty((max(n.value, 1), 4), np.float32)
        n2 = C.c_int(0)
        _chk(lib().flb_map_flatten_xyzi(self.h, _p(out), n.value, C.byref(n2)))
        return out[:min(n.value, n2.value)].copy()

    def Box_Search_xyzi(self, box6, cap=1 << 20):
        b = np.ascontiguousarray(box6, np.float32).reshape(6)
        out = np.empty((cap, 4), np.float32)
        n = C.c_int(0)
        _chk(lib().flb_map_box_search_xyzi(self.h, _p(b), _p(out), cap, C.byref(n)))
        return out[:min(n.value, cap)].copy()

    def Delete_Point_Boxes(self, boxes):
        b = np.ascontiguousarray(boxes, np.float32).reshape(-1, 6)
        n = C.c_int(0)
        _chk(lib().flb_map_delete_boxes(self.h, _p(b), len(b), C.byref(n)))
        return n.value

    def Delete_Points(self, pts):
        pts = _xyz(pts)
        n = C.c_int(0)
        _chk(lib().flb_map_delete_points(self.h, _p(pts), len(pts), pts.strides[0], C.byref(n)))
        return n.value

    def Nearest_Search(self, q, k=5, max_dist=0.0):
        q = _xyz(q)
        n = len(q)
        xyz = np.empty((n, k, 3), np.float32)
        d2 = np.empty((n, k), np.float32)
        cnt = np.empty(n, np.int32)
        _chk(lib().flb_map_nearest_search(self.h, _p(q), n, q.strides[0], k, float(max_dist), _p(xyz), _p(d2), _p(cnt)))
        return xyz, d2, cnt

    def Box_Search(self, box6, cap=1 << 20):
        b = np.ascontiguousarray(box6, np.float32).reshape(6)
        out = np.empty((cap, 3), np.float32)
        n = C.c_int(0)
        _chk(lib().flb_map_box_search(self.h, _p(b), _p(out), cap, C.byref(n)))
        return out[:min(n.value, cap)].copy()

    def Radius_Search(self, center, radius, cap=1 << 20):
        c = np.ascontiguousarray(center, np.float32).reshape(3)
        out = np.empty((cap, 3), np.float32)
        n = C.c_int(0)
        _chk(lib().flb_map_radius_search(self.h, _p(c), float(radius), _p(out), cap, C.byref(n)))
        return out[:min(n.value, cap)].copy()

    def validnum(self):
        v = lib().flb_map_validnum(self.h)
        if v < 0:
            raise FlbError(lib().flb_last_error().decode())
        return v

    def size(self):
        return self.validnum()

    def flatten(self):
        n = C.c_int(0)
        _chk(lib().flb_map_flatten(self.h, None, 0, C.byref(n)))
        out = np.empty((max(n.value, 1), 3), np.float32)
        n2 = C.c_int(0)
        _chk(lib().flb_map_flatten(self.h, _p(out), n.value, C.byref(n2)))
        return out[:min(n.value, n2.value)].copy()

    def tree_range(self):
        b = np.zeros(6, np.float32)
        _chk(lib().flb_map_range(self.h, _p(b)))
        return b

    def profile_enable(self, on=True):
        _chk(lib().flb_map_profile_enable(self.h, 1 if on else 0))

    def profile_read(self, reset=True):
        p = Profile()
        _chk(lib().flb_map_profile_read(self.h, C.byref(p), 1 if reset else 0))
        out = {}
        for i, k in enumerate(K_CLASSES):
            out[k] = {"ms": p.ms[i], "launches": p.launches[i], "regions": p.regions[i]}
        out["knn_phase"] = [int(p.knn_phase[i]) for i in range(4)]
        out["knn_head_candidates"] = int(p.knn_head_candidates)
        out["knn_chain_nodes"] = int(p.knn_chain_nodes)
        out["knn_chain_max"] = int(p.knn_chain_max)
        return out

    def stats(self):
        s = MapStats()
        _chk(lib().flb_map_get_stats(self.h, C.byref(s)))
        return {f[0]: getattr(s, f[0]) for f in MapStats._fields_}


class Session:
    """Per-scan measurement context: h_share_model + update_iterated_dyn_share_modified + map_incremental."""

    def __init__(self, tree, max_scan_points=131072, extrinsic_est_en=False, max_iterations=4, laser_point_cov=0.001,
                 filter_size_map_min=None, limit=None):
        self.tree = tree
        cfg = SessionConfig()
        lib().flb_session_default_config(C.byref(cfg))
        cfg.max_scan_points = int(max_scan_points)
        cfg.extrinsic_est_en = 1 if extrinsic_est_en else 0
        cfg.max_iterations = int(max_iterations)
        cfg.laser_point_cov = float(laser_point_cov)
        cfg.filter_size_map_min = float(filter_size_map_min if filter_size_map_min is not None else tree.voxel_size)
        if limit is not None:
            for i in range(23):
                cfg.limit[i] = float(limit[i])
        self.cfg = cfg
        self.h = C.c_void_p()
        _chk(lib().flb_session_create(tree.h, C.byref(cfg), C.byref(self.h)))
        self.n = 0

    def close(self):
        if getattr(self, "h", None):
            lib().flb_session_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def scan_upload(self, body):
        body = _xyz(body)
        _chk(lib().flb_scan_upload(self.h, _p(body), len(body), body.strides[0]))
        self.n = len(body)

    def scan_upload_xyzi(self, body4):
        """feats_down_body with intensity: (n, 4) float32 x, y, z, intensity (travels into the map, laserMapping.cpp:1101-1110)."""
        a = np.ascontiguousarray(body4, np.float32).reshape(-1, 4)
        self.n = len(a)
        _chk(lib().flb_scan_upload_pt(self.h, _p(a), len(a), 16, 12))

    def scan_prefetch_ptr(self, ptr, n, stride):
        """Start the async upload of the NEXT scan (raw host pointer, pinned recommended)."""
        _chk(lib().flb_scan_prefetch(self.h, C.c_void_p(ptr), int(n), int(stride)))
        self._pending_n = int(n)

    def scan_set_device(self, dev_ptr, n):
        _chk(lib().flb_scan_set_device(self.h, C.c_void_p(dev_ptr), int(n)))
        self.n = int(n)

    def h_share_model(self, state26, converge=True):
        st = np.ascontiguousarray(state26, np.float64)
        r = PassResult()
        _chk(lib().flb_pass(self.h, _p(st), 1 if converge else 0, C.byref(r)))
        return {"valid": bool(r.valid), "effct_feat_num": r.effct_feat_num, "total_residual": r.total_residual,
                "HTH": np.array(r.HTH[:]).reshape(12, 12), "HTh": np.array(r.HTh[:])}

    def pass_rows(self):
        cap = max(self.n, 1)
        hx = np.zeros((12, cap), np.float64)  # column-major M x 12 with ld = cap
        h = np.zeros(cap, np.float64)
        M = C.c_int(0)
        _chk(lib().flb_pass_rows(self.h, _p(hx), cap, _p(h), cap, C.byref(M)))
        return hx[:, :M.value].T.copy(), h[:M.value].copy()

    def update_iterated_dyn_share_modified(self, state26, P):
        st = np.array(state26, np.float64).copy()
        Pm = np.ascontiguousarray(np.array(P, np.float64).reshape(23, 23)).copy()
        us = UpdateStats()
        _chk(lib().flb_esikf_update(self.h, _p(st), _p(Pm), C.byref(us)))
        return st, Pm, {f[0]: getattr(us, f[0]) for f in UpdateStats._fields_}

    def map_incremental(self, state26, flg_EKF_inited=True):
        st = np.ascontiguousarray(state26, np.float64)
        a, b = C.c_int(0), C.c_int(0)
        _chk(lib().flb_map_incremental(self.h, _p(st), 1 if flg_EKF_inited else 0, C.byref(a), C.byref(b)))
        return a.value, b.value

    def neighbors(self):
        n = self.n
        nbr = np.empty((n, 5, 3), np.float32)
        d2 = np.empty((n, 5), np.float32)
        cnt = np.empty(n, np.int32)
        sel = np.empty(n, np.uint8)
        nv = np.empty((n, 4), np.float32)
        world = np.empty((n, 3), np.float32)
        _chk(lib().flb_neighbors_download(self.h, _p(nbr), _p(d2), _p(cnt), _p(sel), _p(nv), _p(world)))
        return {"nbr": nbr, "d2": d2, "cnt": cnt, "sel": sel, "normvec": nv, "world": world}

    def scan_step(self, fov, body, state26, P, flg_EKF_inited=True):
        st = np.array(state26, np.float64).copy()
        Pm = np.ascontiguousarray(np.array(P, np.float64).reshape(23, 23)).copy()
        r = ScanResult()
        if body is not None:
            body = _xyz(body)
            self.n = len(body)
            _chk(lib().flb_scan_step(self.h, C.byref(fov) if fov is not None else None, _p(body), len(body),
                                     body.strides[0], _p(st), _p(Pm), 1 if flg_EKF_inited else 0, C.byref(r)))
        else:
            _chk(lib().flb_scan_step(self.h, C.byref(fov) if fov is not None else None, None, 0, 0, _p(st), _p(Pm),
                                     1 if flg_EKF_inited else 0, C.byref(r)))
        return st, Pm, r

    def scan_step_ptr(self, fov, ptr, n, stride, state26, P, flg_EKF_inited=True):
        """flb_scan_step on a raw host pointer (e.g. pinned memory owned by the caller); state26/P updated in place."""
        r = ScanResult()
        if ptr:
            self.n = int(n)
        elif getattr(self, "_pending_n", None) is not None:
            self.n, self._pending_n = self._pending_n, None
        _chk(lib().flb_scan_step(self.h, C.byref(fov) if fov is not None else None, C.c_void_p(ptr) if ptr else None,
                                 int(n), int(stride), _p(state26), _p(P), 1 if flg_EKF_inited else 0, C.byref(r)))
        return r

    def set_update_engine(self, device_driven=True):
        _chk(lib().flb_session_set_update_engine(self.h, 1 if device_driven else 0))

    def scan_step_begin(self, fov, state26, P, flg_EKF_inited=True):
        """Enqueue the step for the scan made current by scan_upload / scan_set_device / scan_prefetch_ptr."""
        if getattr(self, "_pending_n", None) is not None:
            self.n, self._pending_n = self._pending_n, None
        _chk(lib().flb_scan_step_begin(self.h, C.byref(fov) if fov is not None else None, None, 0, 0, _p(state26), _p(P),
                                       1 if flg_EKF_inited else 0))

    def scan_step_finish(self, fov, state26, P):
        r = ScanResult()
        _chk(lib().flb_scan_step_finish(self.h, C.byref(fov) if fov is not None else None, _p(state26), _p(P), C.byref(r)))
        return r

    def stream_ptr(self):
        return lib().flb_session_stream(self.h)

    def sync(self):
        _chk(lib().flb_session_sync(self.h))


POINT_STRIDE = 48      # pcl::PointXYZINormal (PointType, common_lib.h:161)
OFF_INTENSITY = 32
OFF_CURVATURE = 36


def pack_pointtype(xyz, intensity=None, curvature=None):
    """Host buffer of n reference PointType records (48 B: x,y,z,_, nx,ny,nz,_, intensity,curvature,_,_)."""
    xyz = np.asarray(xyz, np.float32)
    buf = np.zeros((len(xyz), 12), np.float32)
    buf[:, 0:3] = xyz[:, :3]
    if intensity is not None:
        buf[:, 8] = intensity
    if curvature is not None:
        buf[:, 9] = curvature
    return buf


class FrontEnd:
    """Device front end of one session: meas.lidar -> UndistortPcl -> VoxelGrid -> feats_down_body (SURVEY.md §8f)."""

    def __init__(self, session, max_raw_points=262144):
        self.session = session
        self.cap = int(max_raw_points)
        self.h = C.c_void_p()
        _chk(lib().flb_frontend_create(session.h, self.cap, C.byref(self.h)))

    def close(self):
        if getattr(self, "h", None):
            lib().flb_frontend_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def upload(self, points48):
        """points48: (n,12) float32 PointType records (see pack_pointtype)."""
        b = np.ascontiguousarray(points48, np.float32)
        assert b.ndim == 2 and b.shape[1] == 12
        _chk(lib().flb_frontend_upload(self.h, _p(b), len(b), POINT_STRIDE, OFF_INTENSITY, OFF_CURVATURE))
        self.n_raw = len(b)

    def upload_ptr(self, ptr, n, stride=POINT_STRIDE, off_i=OFF_INTENSITY, off_c=OFF_CURVATURE):
        _chk(lib().flb_frontend_upload(self.h, C.c_void_p(ptr), int(n), stride, off_i, off_c))
        self.n_raw = int(n)

    def undistort(self, imu_poses, state26_end):
        poses = np.ascontiguousarray(imu_poses, np.float64).reshape(-1, 22)
        st = np.ascontiguousarray(state26_end, np.float64)
        _chk(lib().flb_frontend_undistort(self.h, _p(poses), len(poses), _p(st)))

    def voxel_filter(self, leaf):
        n = C.c_int(0)
        _chk(lib().flb_frontend_voxel_filter(self.h, float(leaf), C.byref(n)))
        self.session.n = n.value
        return n.value

    def process_ptr(self, ptr, n, imu_poses, state26_end, leaf, stride=POINT_STRIDE, off_i=OFF_INTENSITY, off_c=OFF_CURVATURE):
        """flb_frontend_process on a raw host pointer; imu_poses must already be a C-contiguous (k,22) float64 array."""
        cnt = C.c_int(0)
        _chk(lib().flb_frontend_process(self.h, C.c_void_p(ptr), int(n), stride, off_i, off_c, _p(imu_poses), len(imu_poses),
                                        _p(state26_end), float(leaf), C.byref(cnt)))
        self.n_raw = int(n)
        self.session.n = cnt.value
        return cnt.value

    def preprocess(self, records, cfg, layout=None):
        """Preprocess::process on the device: driver records (numpy structured array in message order) -> the front
        end's raw scan.  cfg: PreprocessConfig or preprocess_config() kwargs; layout: RawLayout, or raw_layout() name
        overrides (default: fields found by name).  Returns (pl_surf size, last point's curvature)."""
        rec, c, lay = _preprocess_args(records, cfg, layout)
        self.n_raw = 0   # a failed call leaves an empty scan
        n, last = C.c_int(0), C.c_float(0)
        _chk(lib().flb_frontend_preprocess(self.h, C.byref(c), C.byref(lay), _p(rec) if len(rec) else None, len(rec), C.byref(n),
                                           C.byref(last)))
        self.n_raw = n.value
        return n.value, np.float32(last.value)

    def download_undistorted(self):
        n = self.n_raw
        xyzi = np.empty((max(n, 1), 4), np.float32)
        cur = np.empty(max(n, 1), np.float32)
        perm = np.empty(max(n, 1), np.int32)
        cnt = C.c_int(0)
        _chk(lib().flb_frontend_download_undistorted(self.h, _p(xyzi), _p(cur), _p(perm), n, C.byref(cnt)))
        return xyzi[:n], cur[:n], perm[:n]

    def download_down(self):
        cnt = C.c_int(0)
        _chk(lib().flb_frontend_download_down(self.h, None, None, 0, C.byref(cnt)))
        n = cnt.value
        xyzi = np.empty((max(n, 1), 4), np.float32)
        cur = np.empty(max(n, 1), np.float32)
        _chk(lib().flb_frontend_download_down(self.h, _p(xyzi), _p(cur), n, C.byref(cnt)))
        return xyzi[:n], cur[:n]

    def points_to_world(self, which, state26):
        st = np.ascontiguousarray(state26, np.float64)
        cnt = C.c_int(0)
        out = np.empty((self.cap, 4), np.float32)
        _chk(lib().flb_frontend_points_to_world(self.h, int(which), _p(st), _p(out), self.cap, C.byref(cnt)))
        return out[:cnt.value].copy()

    def set_camera(self, cam_ex, cam_in, width=1280, height=720):
        """paramSetting: cam_ex 16 and cam_in 12 row-major doubles; width x height bounds the image (Wmax x Hmax)."""
        ex = np.ascontiguousarray(cam_ex, np.float64).reshape(-1)
        ki = np.ascontiguousarray(cam_in, np.float64).reshape(-1)
        if ex.size != 16 or ki.size != 12:
            raise ValueError("cam_ex must hold 16 and cam_in 12 values")
        _chk(lib().flb_frontend_camera_config(self.h, _p(ex), _p(ki), int(width), int(height)))

    def upload_image(self, img):
        """imageCallback: img is a (rows, cols, 3) uint8 bgr8 array; rows may be padded (a row stride above 3 * cols)."""
        a = np.asarray(img)
        if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
            raise ValueError("image must be a (rows, cols, 3) uint8 array")
        if a.strides[1:] != (3, 1) or a.strides[0] < 3 * a.shape[1]:
            a = np.ascontiguousarray(a)
        _chk(lib().flb_frontend_camera_image(self.h, C.c_void_p(a.ctypes.data), a.shape[0], a.shape[1], a.strides[0]))

    def colorize(self, which, state26, cap=None):
        """publish_frame_world_color: returns (xyzi (k,4) float32 in the world frame, bgra (k,) uint32 with the bytes
        b, g, r, a, kept count); k = min(kept count, cap)."""
        st = np.ascontiguousarray(state26, np.float64)
        cap = self.cap if cap is None else int(cap)
        xyzi = np.empty((max(cap, 1), 4), np.float32)
        bgra = np.empty(max(cap, 1), np.uint32)
        cnt = C.c_int(0)
        _chk(lib().flb_frontend_points_colorize(self.h, int(which), _p(st), _p(xyzi), _p(bgra), cap, C.byref(cnt)))
        k = min(cnt.value, cap)
        return xyzi[:k].copy(), bgra[:k].copy(), cnt.value

    def to_imu(self, state26):
        """publish_frame_body: feats_undistort in the IMU frame (x, y, z, intensity)."""
        st = np.ascontiguousarray(state26, np.float64)
        cnt = C.c_int(0)
        out = np.empty((self.cap, 4), np.float32)
        _chk(lib().flb_frontend_points_to_imu(self.h, _p(st), _p(out), self.cap, C.byref(cnt)))
        return out[:cnt.value].copy()


def imu_config(**kw):
    """flb_imu_config with laserMapping.cpp's defaults; keyword arguments override fields (sequences of 3 or 9 values)."""
    c = ImuConfig()
    lib().flb_imu_default_config(C.byref(c))
    for k, v in kw.items():
        arr = getattr(c, k)
        v = np.asarray(v, np.float64).reshape(-1)
        if len(v) != len(arr):
            raise ValueError(f"{k} takes {len(arr)} values")
        for i, x in enumerate(v):
            arr[i] = float(x)
    return c


class Imu:
    """ImuProcess on a front end (IMU_Processing.hpp): IMU_init on the host, the forward propagation, the undistortion
    and the voxel filter of the front end's current raw scan on the device."""

    def __init__(self, frontend, cfg=None, **kw):
        self.frontend = frontend
        self.h = C.c_void_p()
        c = cfg if cfg is not None else imu_config(**kw)
        _chk(lib().flb_imu_create(frontend.h, C.byref(c), C.byref(self.h)))

    def close(self):
        if getattr(self, "h", None):
            lib().flb_imu_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        _chk(lib().flb_imu_reset(self.h))

    def process(self, imu7, lidar_beg_time, lidar_end_time, state26, P, leaf=0.0):
        """Process(meas, kf, feats_undistort): imu7 (n,7) = stamp, acc, gyro of meas.imu.  Returns (state26, P, result) with
        the prior; the inputs are not modified."""
        a = np.ascontiguousarray(np.asarray(imu7, np.float64).reshape(-1, 7))
        x = np.array(state26, np.float64, copy=True).reshape(26)
        Pm = np.array(P, np.float64, copy=True).reshape(23, 23)
        r = ImuResult()
        _chk(lib().flb_imu_process(self.h, _p(a) if len(a) else None, len(a), float(lidar_beg_time), float(lidar_end_time), _p(x),
                                   _p(Pm), float(leaf), C.byref(r)))
        if r.n_down >= 0:
            self.frontend.session.n = r.n_down
        return x, Pm, r

    def poses(self):
        n = C.c_int(0)
        _chk(lib().flb_imu_download_poses(self.h, None, 0, C.byref(n)))
        out = np.zeros((max(n.value, 1), 22))
        _chk(lib().flb_imu_download_poses(self.h, _p(out), n.value, C.byref(n)))
        return out[:n.value]

    def info(self):
        s = ImuState()
        _chk(lib().flb_imu_info(self.h, C.byref(s)))
        d = {k: (np.array(getattr(s, k)) if isinstance(getattr(s, k), C.Array) else getattr(s, k)) for k, _ in ImuState._fields_}
        return d


# Preprocess parameters (preprocess.h:8-14, laserMapping.cpp:2034-2041)
LIVOX, VELO16, OUST64 = 1, 2, 3
SEC, MS, US, NS = 0, 1, 2, 3
# record field -> names matched in a structured dtype, first match wins (pcl::fromROSMsg matches fields by name)
_FIELD_NAMES = {"x": ("x",), "y": ("y",), "z": ("z",), "intensity": ("intensity", "reflectivity"),
                "time": ("time", "t", "offset_time"), "ring": ("ring",), "tag": ("tag",), "line": ("line",)}


def preprocess_config(lidar_type, n_scans=16, scan_rate=10, point_filter_num=1, time_unit=MS, blind=0.01):
    return PreprocessConfig(int(lidar_type), int(n_scans), int(scan_rate), int(point_filter_num), int(time_unit), float(blind))


def raw_layout(dtype, **names):
    """flb_raw_layout of a numpy structured dtype: offsets of the fields found by name; names= overrides a lookup
    (a field name, or None for "absent")."""
    dtype = np.dtype(dtype)
    lay = RawLayout(dtype.itemsize, *([-1] * 8))
    for key, cands in _FIELD_NAMES.items():
        if key in names:
            cands = () if names[key] is None else (names[key],)
        for c in cands:
            if dtype.names and c in dtype.names:
                setattr(lay, "off_" + key, dtype.fields[c][1])
                break
    return lay


def _preprocess_args(records, cfg, layout):
    rec = np.ascontiguousarray(records)
    c = cfg if isinstance(cfg, PreprocessConfig) else preprocess_config(**cfg)
    lay = layout if isinstance(layout, RawLayout) else raw_layout(rec.dtype, **(layout or {}))
    return rec, c, lay


def voxel_grid_filter(tree, points48, leaf):
    """pcl::VoxelGrid centroid filter of a host cloud of PointType records -> (m,4) x,y,z,intensity."""
    b = np.ascontiguousarray(points48, np.float32)
    out = np.empty((max(len(b), 1), 4), np.float32)
    n = C.c_int(0)
    _chk(lib().flb_voxel_grid_filter(tree.h, _p(b), len(b), POINT_STRIDE, OFF_INTENSITY, float(leaf), _p(out), len(out), C.byref(n)))
    return out[:n.value].copy()


def reconstruct_keyframes(tree, clouds48, poses6, leaf):
    """recontructIKdTree's data-parallel part: transform + concatenate + VoxelGrid + reconstruct. Returns featsFromMap."""
    clouds = [np.ascontiguousarray(c, np.float32) for c in clouds48]
    k = len(clouds)
    ptrs = (C.c_void_p * max(k, 1))(*[c.ctypes.data for c in clouds])
    sizes = (C.c_int * max(k, 1))(*[len(c) for c in clouds])
    p6 = np.ascontiguousarray(poses6, np.float32).reshape(-1, 6)
    total = sum(len(c) for c in clouds)
    out = np.empty((max(total, 1), 4), np.float32)
    n = C.c_int(0)
    _chk(lib().flb_map_reconstruct_keyframes(tree.h, ptrs, sizes, k, POINT_STRIDE, OFF_INTENSITY, _p(p6), float(leaf), _p(out),
                                             len(out), C.byref(n)))
    return out[:n.value].copy()


KF_POSE6, KF_AFFINE = 0, 1   # FLB_KF_POSE6 / FLB_KF_AFFINE
# FLB_ICP_* convergence states
ICP_STATES = ["NOT_CONVERGED", "ITERATIONS", "TRANSFORM", "ABS_MSE", "REL_MSE", "NO_CORRESPONDENCES"]
SC_RINGS, SC_SECTORS = 20, 60  # FLB_SC_RINGS / FLB_SC_SECTORS


class KeyFrameStore:
    """surfCloudKeyFrames on the device (laserMapping.cpp:756-758): body-frame key-frame clouds, x,y,z,intensity +
    curvature, in a fixed-capacity append-only arena on the map's device; every reader takes the poses at call time."""

    def __init__(self, tree, max_points, max_keyframes):
        self.tree = tree
        self.h = C.c_void_p()
        _chk(lib().flb_keyframes_create(tree.h, int(max_points), int(max_keyframes), C.byref(self.h)))

    def close(self):
        if getattr(self, "h", None):
            lib().flb_keyframes_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def append_frontend(self, fe):
        """The front end's current feats_undistort becomes the next key frame (device to device). Returns its id."""
        k = C.c_int(-1)
        _chk(lib().flb_keyframes_append_frontend(self.h, fe.h, C.byref(k)))
        return k.value

    def append(self, points48):
        """(n,12) float32 PointType records (see pack_pointtype). Returns the new key frame's id."""
        b = np.ascontiguousarray(points48, np.float32).reshape(-1, 12)
        k = C.c_int(-1)
        _chk(lib().flb_keyframes_append(self.h, _p(b) if len(b) else None, len(b), POINT_STRIDE, OFF_INTENSITY, OFF_CURVATURE,
                                        C.byref(k)))
        return k.value

    def size(self, k):
        v = lib().flb_keyframes_size(self.h, int(k))
        if v < 0:
            raise FlbError(lib().flb_last_error().decode())
        return v

    def info(self):
        nk, npts, nb, ns = C.c_int(0), C.c_longlong(0), C.c_longlong(0), C.c_longlong(0)
        _chk(lib().flb_keyframes_info(self.h, C.byref(nk), C.byref(npts), C.byref(nb), C.byref(ns)))
        return {"n_keyframes": nk.value, "n_points": npts.value, "device_bytes": nb.value, "map_scratch_bytes": ns.value}

    def release_scratch(self):
        """Free the readers' scratch the map keeps (e.g. after a save map); the next reader allocates again."""
        _chk(lib().flb_map_release_keyframe_scratch(self.tree.h))

    def download(self, k):
        """Key frame k as stored: ((n,4) x,y,z,intensity, (n,) curvature)."""
        n = self.size(k)
        xyzi = np.empty((max(n, 1), 4), np.float32)
        cur = np.empty(max(n, 1), np.float32)
        cnt = C.c_int(0)
        _chk(lib().flb_keyframes_download(self.h, int(k), _p(xyzi), _p(cur), n, C.byref(cnt)))
        return xyzi[:n].copy(), cur[:n].copy()

    def _selection_size(self, ids):
        return sum(self.size(int(i)) for i in ids) if len(ids) else 0

    def reconstruct(self, ids, poses6, leaf, cap=None):
        """recontructIKdTree from the store: transform ids[j] by poses6[j], concatenate, VoxelGrid(leaf), rebuild the map.
        Returns featsFromMap ((m,4) x,y,z,intensity)."""
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        p6 = np.ascontiguousarray(poses6, np.float32).reshape(-1, 6)
        if len(p6) != len(ids):
            raise ValueError("one pose per selected key frame")
        cap = self._selection_size(ids) if cap is None else int(cap)
        out = np.empty((max(cap, 1), 4), np.float32)
        n = C.c_int(0)
        _chk(lib().flb_map_reconstruct_from_keyframes(self.tree.h, self.h, _p(ids) if len(ids) else None, len(ids),
                                                      _p(p6) if len(ids) else None, float(leaf), _p(out), cap, C.byref(n)))
        return out[:min(n.value, cap)].copy()

    def assemble(self, ids, poses6=None, affines=None, leaf=0.0, cap=None, return_size=False):
        """Concatenate ids in order, each transformed by its pose6 (x,y,z,roll,pitch,yaw) or its row-major 3x4 affine;
        leaf > 0 filters with pcl::VoxelGrid (curvature carried).  Returns ((m,4) x,y,z,intensity, (m,) curvature)
        [, full size when return_size]."""
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        kind, tr = self._transforms(ids, poses6, affines)
        cap = self._selection_size(ids) if cap is None else int(cap)
        xyzi = np.empty((max(cap, 1), 4), np.float32)
        cur = np.empty(max(cap, 1), np.float32)
        n = C.c_int(0)
        _chk(lib().flb_keyframes_assemble(self.h, _p(ids) if len(ids) else None, len(ids), kind, _p(tr) if len(ids) else None,
                                          float(leaf), _p(xyzi), _p(cur), cap, C.byref(n)))
        m = min(n.value, cap)
        res = (xyzi[:m].copy(), cur[:m].copy())
        return res + (n.value,) if return_size else res

    @staticmethod
    def _transforms(ids, poses6, affines):
        if (poses6 is None) == (affines is None):
            raise ValueError("pass exactly one of poses6 / affines")
        kind = KF_POSE6 if poses6 is not None else KF_AFFINE
        tr = np.ascontiguousarray(poses6 if poses6 is not None else affines, np.float32).reshape(-1)
        if len(tr) != len(ids) * (6 if kind == KF_POSE6 else 12):
            raise ValueError("one transform per selected key frame")
        return kind, tr

    def scan_context(self, ids, poses6=None, affines=None, lidar_height=1.5):
        """SCManager::makeScancontext of the dense assembly of ids (transforms as assemble), computed on the device:
        (20, 60) float64, row-major (ring, sector); 0 where no point is."""
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        kind, tr = self._transforms(ids, poses6, affines)
        out = np.empty((SC_RINGS, SC_SECTORS), np.float64)
        _chk(lib().flb_keyframes_scan_context(self.h, _p(ids) if len(ids) else None, len(ids), kind, _p(tr) if len(ids) else None,
                                              float(lidar_height), _p(out)))
        return out

    def scan_contexts(self, ids, lidar_height=1.5):
        """makeScancontext of every key frame ids[j] as stored (the key-frame saver): (k, 20, 60) float64."""
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        out = np.empty((len(ids), SC_RINGS, SC_SECTORS), np.float64)
        _chk(lib().flb_keyframes_scan_contexts(self.h, _p(ids) if len(ids) else None, len(ids), float(lidar_height),
                                               _p(out) if len(ids) else None))
        return out

    @staticmethod
    def _icp_dict(r):
        return {"final_transformation": np.array(r.final_transformation[:], np.float32).reshape(4, 4), "converged": bool(r.converged),
                "iterations": r.iterations, "state": r.state, "state_name": ICP_STATES[r.state], "n_source": r.n_source,
                "n_target": r.n_target, "n_correspondences": r.n_correspondences, "fitness_score": r.fitness_score}

    def icp(self, src_ids, tgt_ids, src_poses6=None, src_affines=None, tgt_poses6=None, tgt_affines=None, pre_pose6=None,
            max_correspondence_distance=200.0, max_iterations=100, transformation_epsilon=1e-6, euclidean_fitness_epsilon=1e-6,
            correspondences=False):
        """performLoopClosure's ICP on the device: the dense assembly of src_ids (then moved by pre_pose6, when given) onto
        the dense assembly of tgt_ids.  Returns a dict (final_transformation (4,4) float32, converged, iterations, state,
        state_name, n_source, n_target, n_correspondences, fitness_score) and, with correspondences=True, also the last
        iteration's nearest target index (-1: none) and d² of every source point."""
        src_ids = np.ascontiguousarray(src_ids, np.int32).reshape(-1)
        tgt_ids = np.ascontiguousarray(tgt_ids, np.int32).reshape(-1)
        sk, st = self._transforms(src_ids, src_poses6, src_affines)
        tk, tt = self._transforms(tgt_ids, tgt_poses6, tgt_affines)
        pre = None if pre_pose6 is None else np.ascontiguousarray(pre_pose6, np.float32).reshape(6)
        cfg = IcpConfig(float(max_correspondence_distance), int(max_iterations), float(transformation_epsilon),
                        float(euclidean_fitness_epsilon))
        r = IcpResult()
        idx = d2 = None
        if correspondences:
            n = self._selection_size(src_ids)
            idx = np.empty(max(n, 1), np.int32)
            d2 = np.empty(max(n, 1), np.float32)
        _chk(lib().flb_keyframes_icp(self.h, _p(src_ids) if len(src_ids) else None, len(src_ids), sk, _p(st) if len(src_ids) else None,
                                     _p(pre), _p(tgt_ids) if len(tgt_ids) else None, len(tgt_ids), tk,
                                     _p(tt) if len(tgt_ids) else None, C.byref(cfg), C.byref(r), _p(idx), _p(d2)))
        res = self._icp_dict(r)
        if correspondences:
            return res, idx[:r.n_source].copy(), d2[:r.n_source].copy()
        return res

    def icp_batch(self, pairs, leaf=0.2, max_correspondence_distance=30.0, max_iterations=10, transformation_epsilon=1e-6,
                  euclidean_fitness_epsilon=1e-6):
        """The multi-session mapper's inter-session registrations in one call: pairs is a list of (src_ids, src_poses6,
        tgt_ids, tgt_poses6), each selection assembled with its key frames' poses6 and, for leaf > 0, VoxelGrid-filtered
        (as assemble(ids, poses6, leaf=leaf)), then registered as icp() registers it.  Returns (a list of icp()'s dicts,
        one per pair, with n_source / n_target the filtered sizes, and a dict of rounds, setup_syncs, iteration_syncs)."""
        sides = ([], [], [], [])
        for src_ids, src_p6, tgt_ids, tgt_p6 in pairs:
            for j, (ids, p6) in enumerate(((src_ids, src_p6), (tgt_ids, tgt_p6))):
                ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
                p6 = np.ascontiguousarray(p6, np.float32).reshape(-1)
                if len(p6) != 6 * len(ids):
                    raise ValueError("one pose6 per selected key frame")
                sides[2 * j].append(ids)
                sides[2 * j + 1].append(p6)
        n = len(pairs)
        offs = [np.zeros(n + 1, np.int32), np.zeros(n + 1, np.int32)]
        cat = []
        for j in range(2):
            offs[j][1:] = np.cumsum([len(a) for a in sides[2 * j]]) if n else []
            cat.append(np.concatenate(sides[2 * j]) if n else np.zeros(0, np.int32))
            cat.append(np.concatenate(sides[2 * j + 1]) if n else np.zeros(0, np.float32))
        cfg = IcpConfig(float(max_correspondence_distance), int(max_iterations), float(transformation_epsilon),
                        float(euclidean_fitness_epsilon))
        res = (IcpResult * max(n, 1))()
        st = IcpBatchStats()
        _chk(lib().flb_keyframes_icp_batch(self.h, n, _p(offs[0]), _p(cat[0]) if len(cat[0]) else None,
                                           _p(cat[1]) if len(cat[0]) else None, _p(offs[1]), _p(cat[2]) if len(cat[2]) else None,
                                           _p(cat[3]) if len(cat[2]) else None, float(leaf), C.byref(cfg), res, C.byref(st)))
        stats = {"rounds": st.rounds, "setup_syncs": st.setup_syncs, "iteration_syncs": st.iteration_syncs}
        return [self._icp_dict(r) for r in res[:n]], stats

    def fricp(self, src_points, tgt_ids, tgt_poses6, tgt_pre_pose6=None, src_pose6=None, mode=4, max_icp=100, stop=1e-5,
              anderson_m=5, nu_begin_k=3.0, nu_end_k=1.0 / (3.0 * np.sqrt(3.0)), nu_alpha=0.5, correspondences=False, log=False,
              log_cap=4096):
        """The relocaliser's registration on the device (Registeration(mode).run(curCloud, nearCloud)): the host source
        ((n,3) / (n,4) float32 x,y,z[,intensity], or (n,12) PointType records), moved by src_pose6 (initPose) when given,
        onto the key frames tgt_ids each moved by tgt_pre_pose6 (pose_ext) when given and then by its tgt_poses6 row.
        Returns a dict (res_trans (4,4) float64, status, status_name, stages, iterations, rejections, scale, mu_source,
        mu_target, nu_begin, nu_end, energy, n_source, n_target, n_source_finite, n_target_finite) and, in this order when
        asked for, the last pass's matched target index (-1: none) and residual of every source point, and the
        per-iteration log ((k, 5): stage, energy, previous accepted energy, |T - T_prev|_F, accepted)."""
        def cfg():
            return FricpConfig(int(mode), int(max_icp), float(stop), int(anderson_m), float(nu_begin_k), float(nu_end_k),
                               float(nu_alpha))
        return self._reloc("flb_keyframes_fricp", cfg, FricpResult(), lambda r: {
            "res_trans": np.array(r.res_trans[:], np.float64).reshape(4, 4), "status": r.status,
            "status_name": FRICP_STATUS[r.status], "stages": r.stages, "iterations": r.iterations, "rejections": r.rejections,
            "scale": r.scale, "mu_source": np.array(r.mu_source[:]), "mu_target": np.array(r.mu_target[:]),
            "nu_begin": r.nu_begin, "nu_end": r.nu_end, "energy": r.energy, "n_source": r.n_source, "n_target": r.n_target,
            "n_source_finite": r.n_source_finite, "n_target_finite": r.n_target_finite},
            src_points, tgt_ids, tgt_poses6, tgt_pre_pose6, src_pose6, correspondences, log, log_cap, 5)

    @staticmethod
    def _source(src_points):
        pts = np.ascontiguousarray(src_points, np.float32)
        if pts.ndim != 2 or pts.shape[1] not in (3, 4, 12):
            raise ValueError("src_points must be (n,3), (n,4) or (n,12) float32")
        off_i = -1 if pts.shape[1] == 3 else (12 if pts.shape[1] == 4 else OFF_INTENSITY)
        return pts, 4 * pts.shape[1], off_i

    def _reloc(self, fn, make_cfg, r, as_dict, src_points, tgt_ids, tgt_poses6, tgt_pre_pose6, src_pose6, correspondences, log,
               log_cap, log_width):
        """fricp / sicp / aaicp through the C entry point named fn with the config make_cfg() (built once the clouds are
        checked) into the result struct r: as_dict(r) and, in this order when asked for, the matched target index and
        residual of every source point and the log (log_width columns)."""
        pts, stride, off_i = self._source(src_points)
        n = len(pts)
        ids = np.ascontiguousarray(tgt_ids, np.int32).reshape(-1)
        p6 = np.ascontiguousarray(tgt_poses6, np.float32).reshape(-1, 6)
        if len(p6) != len(ids):
            raise ValueError("one pose per target key frame")
        pre = None if tgt_pre_pose6 is None else np.ascontiguousarray(tgt_pre_pose6, np.float32).reshape(6)
        sp = None if src_pose6 is None else np.ascontiguousarray(src_pose6, np.float32).reshape(6)
        cfg = make_cfg()
        idx = resid = lg = None
        if correspondences:
            idx = np.empty(max(n, 1), np.int32)
            resid = np.empty(max(n, 1), np.float64)
        if log:
            lg = np.zeros((max(int(log_cap), 1), log_width), np.float64)
        _chk(getattr(lib(), fn)(self.h, _p(pts) if n else None, n, stride, off_i, _p(sp), _p(ids) if len(ids) else None, len(ids),
                                _p(pre), _p(p6) if len(ids) else None, C.byref(cfg), C.byref(r), _p(idx), _p(resid), _p(lg),
                                int(log_cap) if log else 0))
        res = as_dict(r)
        out = (res,)
        if correspondences:
            out += (idx[:n].copy(), resid[:n].copy())
        if log:
            out += (lg[:r.log_n].copy(),)
        return out if len(out) > 1 else res

    def sicp(self, src_points, tgt_ids, tgt_poses6, tgt_pre_pose6=None, src_pose6=None, p=0.4, mu=10.0, alpha=1.2, max_mu=1e5,
             max_icp=100, max_outer=100, stop=1e-5, correspondences=False, log=False, log_cap=4096):
        """The relocaliser's Sparse ICP (regMode 7) on the device, with the clouds of fricp(): the host source, moved by
        src_pose6 when given, onto the key frames tgt_ids each moved by tgt_pre_pose6 when given and then by its tgt_poses6
        row.  Returns a dict (res_trans (4,4) float64, status, status_name, iterations, admm_iterations, scale, mu_source,
        mu_target, n_source, n_target, n_source_finite, n_target_finite, primal, dual, stop, mu_exit, syncs, admm_blocks) and, in this
        order when asked for, the last ICP iteration's matched target index (-1: none) and residual of every source point,
        and the per-ICP-iteration log ((k, 5): ADMM iterations, primal, dual, stop, μ at exit)."""
        def cfg():
            return SicpConfig(float(p), float(mu), float(alpha), float(max_mu), int(max_icp), int(max_outer), float(stop))
        return self._reloc("flb_keyframes_sicp", cfg, SicpResult(), lambda r: {
            "res_trans": np.array(r.res_trans[:], np.float64).reshape(4, 4), "status": r.status,
            "status_name": FRICP_STATUS[r.status], "iterations": r.iterations, "admm_iterations": r.admm_iterations,
            "scale": r.scale, "mu_source": np.array(r.mu_source[:]), "mu_target": np.array(r.mu_target[:]),
            "n_source": r.n_source, "n_target": r.n_target, "n_source_finite": r.n_source_finite,
            "n_target_finite": r.n_target_finite, "primal": r.primal, "dual": r.dual, "stop": r.stop, "mu_exit": r.mu_exit,
            "syncs": r.syncs, "admm_blocks": r.admm_blocks},
            src_points, tgt_ids, tgt_poses6, tgt_pre_pose6, src_pose6, correspondences, log, log_cap, 5)

    def aaicp(self, src_points, tgt_ids, tgt_poses6, tgt_pre_pose6=None, src_pose6=None, max_icp=100, stop=1e-5,
              error_overflow_threshold=0.05, correspondences=False, log=False, log_cap=4096):
        """The relocaliser's AA-ICP (regMode 1) on the device, with the clouds of fricp(): the host source, moved by
        src_pose6 when given, onto the key frames tgt_ids each moved by tgt_pre_pose6 when given and then by its tgt_poses6
        row.  Returns a dict (res_trans (4,4) float64, status, status_name, iterations, accepted, resets, history, energy,
        scale, mu_source, mu_target, n_source, n_target, n_source_finite, n_target_finite, syncs) and, in this order when
        asked for, the last pass's matched target index (-1: none) and residual of every source point, and the
        per-iteration log ((k, 6): energy, previous energy, outcome (-1 first, 1 accepted, 0 reset), α count,
        |final - final_prev|_F, smallest alphas_cond margin)."""
        def cfg():
            return AaicpConfig(int(max_icp), float(stop), float(error_overflow_threshold))
        return self._reloc("flb_keyframes_aaicp", cfg, AaicpResult(), lambda r: {
            "res_trans": np.array(r.res_trans[:], np.float64).reshape(4, 4), "status": r.status,
            "status_name": FRICP_STATUS[r.status], "iterations": r.iterations, "accepted": r.accepted, "resets": r.resets,
            "history": r.history, "energy": r.energy, "scale": r.scale, "mu_source": np.array(r.mu_source[:]),
            "mu_target": np.array(r.mu_target[:]), "n_source": r.n_source, "n_target": r.n_target,
            "n_source_finite": r.n_source_finite, "n_target_finite": r.n_target_finite, "syncs": r.syncs},
            src_points, tgt_ids, tgt_poses6, tgt_pre_pose6, src_pose6, correspondences, log, log_cap, 6)


def make_fov(cube_len=200.0, det_range=100.0):
    f = FovState()
    f.cube_len = float(cube_len)
    f.det_range = float(det_range)
    f.initialized = 0
    return f


def fov_segment(tree, fov, pos_lid):
    boxes = np.zeros(18, np.float32)
    nb, nd = C.c_int(0), C.c_int(0)
    p = np.ascontiguousarray(pos_lid, np.float64)
    _chk(lib().flb_fov_segment(tree.h, C.byref(fov), _p(p), _p(boxes), C.byref(nb), C.byref(nd)))
    return boxes.reshape(3, 6)[:nb.value].copy(), nd.value


def device_count():
    return lib().flb_device_count()

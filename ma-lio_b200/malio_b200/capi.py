"""ctypes binding of include/malio_b200.h (libmalio_b200.so, built in-tree by ma-lio_b200/csrc/Makefile).

The library is the product; this module only marshals numpy arrays through the C-ABI.  There is no CPU
fallback: if the shared library is missing, or no CUDA device is usable, the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

MAX_LIDAR = 3
K = 5
MAX_DOF = 17 + 6 * MAX_LIDAR
MAX_COV = 512   # MALIO_MAX_COV
NCCL_UNIQUE_ID_BYTES = 128

OK = 0
ERR_INVALID_ARG, ERR_CUDA, ERR_NCCL, ERR_NO_EFFECTIVE_POINTS, ERR_STATE, ERR_TREE_TOO_DEEP, ERR_CAPACITY = range(1, 8)

LINK_HAS_LEFT = 0x80000000
LINK_HAS_RIGHT = 0x40000000
LINK_POINT_DELETED = 0x20000000
LINK_INDEX_MASK = 0x0FFFFFFF
MAP_SKIP, MAP_ADD, MAP_ADD_NO_DOWNSAMPLE, MAP_DROP = 0, 1, 2, 3
WORLD_DOWNSAMPLED, WORLD_DENSE = 0, 1

# numpy views of the C structs
MAP_NODE = np.dtype([("xyz", "<f4", 3), ("link", "<u4"), ("lbox", "<f4", 6), ("rbox", "<f4", 6)])
MAP_POINT = np.dtype([("xyz", "<f4", 3), ("link", "<u4")])
POSE = np.dtype([("q", "<f8", 4), ("t", "<f8", 3), ("T", "<f8", (4, 4)), ("cov", "<f8", (6, 6))])   # malio_pose
SCAN_PT = np.dtype([("xyz", "<f4", 3), ("lidar", "<u2"), ("table_idx", "<u2")])
POSE_ENTRY = np.dtype([("T", "<f8", (4, 4)), ("cov", "<f8", (6, 6))])
RIGID = np.dtype([("q", "<f8", 4), ("t", "<f8", 3)])
LIVOX_PT = np.dtype([("xyz", "<f4", 3), ("reflectivity", "u1"), ("tag", "u1"), ("line", "u1"), ("pad", "u1"), ("offset_time", "<u4")])
OUSTER_PT = np.dtype([("xyz", "<f4", 3), ("intensity", "<f4"), ("ring", "<u2"), ("pad", "<u2"), ("t", "<u4")])
RAW_PT = np.dtype([("xyz", "<f4", 3), ("curvature", "<f4")])   # malio_raw_pt
IDX_UNTOUCHED = -(1 << 31)
assert MAP_NODE.itemsize == 64 and SCAN_PT.itemsize == 16 and POSE_ENTRY.itemsize == 416 and RIGID.itemsize == 56


class Rigid(C.Structure):
    _fields_ = [("q", C.c_double * 4), ("t", C.c_double * 3)]


class UndistortArgs(C.Structure):
    _fields_ = [("beg_time", C.c_double), ("extrinsic", Rigid), ("lt_imu_frame", Rigid), ("ctrl_t", C.c_void_p),
                ("ctrl_T", C.c_void_p), ("n_ctrl", C.c_uint32), ("imu_cov_t", C.c_void_p), ("n_cov", C.c_uint32),
                ("cov_pointer", C.c_int32)]


class ScanUncArgs(C.Structure):
    _fields_ = [("imu_cov", C.c_void_p), ("n_cov", C.c_uint32), ("extrinsic", C.c_void_p), ("uncertainty", C.c_void_p)]


class PassState(C.Structure):
    _fields_ = [("rot", C.c_double * 4), ("pos", C.c_double * 3), ("ext", Rigid * MAX_LIDAR)]


class Params(C.Structure):
    _fields_ = [("n_lidar", C.c_int32), ("extrinsic_est_en", C.c_int32), ("plane_th", C.c_float),
                ("knn_max_sqdist", C.c_float), ("cov_threshold", C.c_double), ("point_cov_max", C.c_double),
                ("point_cov_min", C.c_double), ("plane_cov_max", C.c_double), ("plane_cov_min", C.c_double),
                ("localize_cov_max", C.c_double), ("localize_cov_min", C.c_double),
                ("localize_thresh_max", C.c_double), ("localize_thresh_min", C.c_double),
                ("range_min", C.c_double), ("range_max", C.c_double)]


class Config(C.Structure):
    _fields_ = [("params", Params), ("device", C.c_int32), ("sort_queries", C.c_int32),
                ("max_points", C.c_uint32), ("max_map_nodes", C.c_uint32), ("knn_cell_size", C.c_float)]


class PassStats(C.Structure):
    _fields_ = [("n_points", C.c_uint32), ("n_eff", C.c_uint32), ("valid", C.c_int32), ("searched", C.c_int32),
                ("u_min", C.c_double), ("u_max", C.c_double), ("tau_min", C.c_double), ("tau_max", C.c_double),
                ("sigma", C.c_double * 3), ("loc_weight", C.c_double), ("ms_sort", C.c_float), ("ms_knn", C.c_float),
                ("ms_plane", C.c_float), ("ms_reduce", C.c_float), ("ms_total", C.c_float)]


class State(C.Structure):
    _fields_ = [("pos", C.c_double * 3), ("rot", C.c_double * 4), ("ext", Rigid * MAX_LIDAR),
                ("vel", C.c_double * 3), ("bg", C.c_double * 3), ("ba", C.c_double * 3), ("grav", C.c_double * 3)]

    def copy(self) -> "State":
        s = State()
        C.memmove(C.byref(s), C.byref(self), C.sizeof(State))
        return s

    def pass_state(self) -> PassState:
        ps = PassState()
        ps.rot[:] = self.rot[:]
        ps.pos[:] = self.pos[:]
        for l in range(MAX_LIDAR):
            ps.ext[l].q[:] = self.ext[l].q[:]
            ps.ext[l].t[:] = self.ext[l].t[:]
        return ps


class Counters(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("knn_launches", C.c_uint64), ("knn_queries", C.c_uint64),
                ("knn_ms", C.c_double), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("knn_fallback_queries", C.c_uint64), ("knn_ring2_queries", C.c_uint64),
                ("knn_candidates", C.c_uint64), ("pass_launches", C.c_uint64), ("pass_points", C.c_uint64),
                ("pass_fit_launches", C.c_uint64), ("pass_ms", C.c_double), ("knn_tie_queries", C.c_uint64),
                ("map_slots", C.c_uint64), ("map_live", C.c_uint64), ("map_compactions", C.c_uint64),
                ("exchange_min_wait_ms", C.c_double), ("exchange_sum_wait_ms", C.c_double), ("exchange_passes", C.c_uint64)]


class WindowReport(C.Structure):
    """malio_window_report: what one malio_prior_map_window call did."""
    _fields_ = [("initialized", C.c_int32), ("moved", C.c_int32), ("cube", C.c_float * 6), ("n_boxes", C.c_uint32),
                ("boxes", C.c_float * 18), ("n_killed", C.c_uint32), ("n_entered", C.c_uint32), ("n_live", C.c_uint32)]


class ExtendReport(C.Structure):
    """malio_extend_report: what one malio_prior_map_extend call added to the session."""
    _fields_ = [("n_candidates", C.c_uint32), ("n_admitted", C.c_uint32), ("n_inserted", C.c_uint32), ("n_session", C.c_uint64)]


class RelocArgs(C.Structure):
    """malio_reloc_args: candidate yaws yaw_lo + k * yaw_step (k < n_yaw) and the lattice (res, half_xy, half_z)."""
    _fields_ = [("yaw_lo", C.c_double), ("yaw_step", C.c_double), ("n_yaw", C.c_uint32), ("res", C.c_double),
                ("half_xy", C.c_uint32), ("half_z", C.c_uint32)]


class RelocReport(C.Structure):
    """malio_reloc_report: the best candidate of one malio_relocalize call and what the search did."""
    _fields_ = [("rot", C.c_double * 4), ("pos", C.c_double * 3), ("yaw_index", C.c_int32), ("offset", C.c_int32 * 3),
                ("score", C.c_uint32), ("n_points", C.c_uint32), ("n_candidates", C.c_uint64), ("nodes_bounded", C.c_uint64),
                ("leaves_scored", C.c_uint64), ("device_bytes", C.c_uint64)]


PLACE_MAX_BINS, PLACE_MAX_K1, PLACE_MAX_K2 = 4096, 1024, 32   # MALIO_PLACE_MAX_*


class PlaceArgs(C.Structure):
    """malio_place_args: column edge, lattice step, stencil radius, bins, the sensor's height and the level steps."""
    _fields_ = [("cell", C.c_double), ("step", C.c_double), ("r_max", C.c_double), ("n_ring", C.c_uint32), ("n_sector", C.c_uint32),
                ("sensor_height", C.c_double), ("z_lo", C.c_double), ("dz", C.c_double), ("fov_up", C.c_double),
                ("block_level", C.c_uint32)]


class PlaceDbReport(C.Structure):
    """malio_place_db_report: what one malio_place_db_build made."""
    _fields_ = [("n_positions", C.c_uint64), ("grid_nx", C.c_uint32), ("grid_ny", C.c_uint32), ("n_stencil", C.c_uint32),
                ("bytes_per_position", C.c_uint32), ("device_bytes", C.c_uint64), ("scratch_bytes", C.c_uint64)]


class GlobalArgs(C.Structure):
    """malio_global_args: stage-1 / stage-2 survivors and the verification's yaw step and lattice."""
    _fields_ = [("k1", C.c_uint32), ("k2", C.c_uint32), ("yaw_step", C.c_double), ("res", C.c_double), ("half_xy", C.c_uint32),
                ("half_z", C.c_uint32)]


class GlobalCandidate(C.Structure):
    """malio_global_candidate: one stage-2 survivor, its guess and its verification."""
    _fields_ = [("position", C.c_uint32), ("shift", C.c_uint32), ("d1", C.c_uint32), ("d2", C.c_uint32), ("col", C.c_int32 * 2),
                ("z_s", C.c_double), ("guess_rot", C.c_double * 4), ("guess_pos", C.c_double * 3), ("rot", C.c_double * 4),
                ("pos", C.c_double * 3), ("score", C.c_uint32), ("n_points", C.c_uint32)]


class GlobalReport(C.Structure):
    """malio_global_report: the best verified pose of one malio_relocalize_global call and every stage's list."""
    _fields_ = [("rot", C.c_double * 4), ("pos", C.c_double * 3), ("score", C.c_uint32), ("n_points", C.c_uint32),
                ("best_rank", C.c_uint32), ("n_candidates", C.c_uint32), ("n_stage1", C.c_uint32), ("verify", RelocArgs),
                ("cand", GlobalCandidate * PLACE_MAX_K2), ("stage1", C.c_uint32 * PLACE_MAX_K1), ("stage1_d1", C.c_uint32 * PLACE_MAX_K1),
                ("query", C.c_uint8 * PLACE_MAX_BINS), ("ms_rank", C.c_double), ("ms_verify", C.c_double), ("device_bytes", C.c_uint64)]


class CarveArgs(C.Structure):
    """malio_carve_args: how far a ray of malio_world_voxel_accumulate_carve is followed (m) and the margin before its end (m)."""
    _fields_ = [("max_range", C.c_float), ("end_margin", C.c_float)]


class CarveKeep(C.Structure):
    """malio_carve_keep: a voxel is dropped when miss >= min_miss and miss > max_miss_per_hit * hit."""
    _fields_ = [("min_miss", C.c_uint32), ("max_miss_per_hit", C.c_float)]


STORE_BLOCK_POINTS = 1 << 24   # MALIO_STORE_BLOCK_POINTS


class StoredScan(C.Structure):
    """malio_stored_scan: a stored scan's record: the caller's time stamp, the state it was stored with, the temporal compensation
    of LiDAR l >= 1 at l - 1, the slot tags and the points per slot (0 beyond L)."""
    _fields_ = [("time", C.c_double), ("state", PassState), ("temporal_comp", Rigid * (MAX_LIDAR - 1)),
                ("slot_tag", C.c_float * MAX_LIDAR), ("n_points", C.c_uint32 * MAX_LIDAR)]


GRID_POINTS, GRID_VOXEL_MAP, GRID_PRIOR = 0, 1, 2            # MALIO_GRID_* sources
GRID_FREE, GRID_OCCUPIED, GRID_UNKNOWN = 0, 100, 255         # nav_msgs/OccupancyGrid values
GRID_MAX_BYTES = 16 << 30
GRID_MAX_BOUND = 1 << 24


class GridArgs(C.Structure):
    """malio_grid_args: cell edge, the region (first cell, cells along x and y), the ground half-width in cells, the obstacle
    band above the ground (m) and the band points that make a cell occupied."""
    _fields_ = [("res", C.c_float), ("i0", C.c_int32), ("j0", C.c_int32), ("nx", C.c_uint32), ("ny", C.c_uint32),
                ("ground_halfwidth", C.c_uint32), ("h_lo", C.c_float), ("h_hi", C.c_float), ("min_obstacle_points", C.c_uint32)]


class GridReport(C.Structure):
    """malio_grid_report: points used / non-finite / outside the padded region, cells per class, peak scratch bytes."""
    _fields_ = [("n_used", C.c_uint64), ("n_nonfinite", C.c_uint64), ("n_outside", C.c_uint64), ("n_occupied", C.c_uint64),
                ("n_free", C.c_uint64), ("n_unknown", C.c_uint64), ("device_bytes", C.c_uint64)]


MATCH_MAX_LEVELS = 4                 # MALIO_MATCH_MAX_LEVELS
MATCH_JACOBI_SWEEPS = 8              # MALIO_MATCH_JACOBI_SWEEPS
MATCH_KEY_RANGE = 1 << 20            # MALIO_MATCH_KEY_RANGE
MATCH_MAX_BYTES = 16 << 30           # MALIO_MATCH_MAX_BYTES
POSE_GRAPH_MAX_LOOPS = 256           # MALIO_POSE_GRAPH_MAX_LOOPS


class MatchArgs(C.Structure):
    """malio_match_args: the submap (stored scans [target_first, target_first + target_count)), the levels' leaves and gates
    (coarse to fine), Gauss-Newton steps and end tests per level, the plane test and the residual sigma."""
    _fields_ = [("target_first", C.c_uint64), ("target_count", C.c_uint64), ("n_levels", C.c_uint32),
                ("leaf", C.c_float * MATCH_MAX_LEVELS), ("gate", C.c_float * MATCH_MAX_LEVELS), ("max_iter", C.c_uint32),
                ("eps_rot", C.c_double), ("eps_pos", C.c_double), ("min_points", C.c_uint32), ("planarity", C.c_double),
                ("sigma", C.c_double)]


class MatchReport(C.Structure):
    """malio_match_report: the estimate, the loop edge T_anchor^-1 T_est and its 6 x 6 information, the fit's quality, steps
    per level, the submap's size and the call's peak scratch bytes."""
    _fields_ = [("rot", C.c_double * 4), ("pos", C.c_double * 3), ("rel_rot", C.c_double * 4), ("rel_pos", C.c_double * 3),
                ("info", C.c_double * 36), ("rms", C.c_double), ("fitness", C.c_double), ("eig_min", C.c_double),
                ("n_points", C.c_uint32), ("n_inliers", C.c_uint32), ("iterations", C.c_uint32 * MATCH_MAX_LEVELS),
                ("converged", C.c_int32), ("target_points", C.c_uint64), ("target_voxels", C.c_uint64 * MATCH_MAX_LEVELS),
                ("device_bytes", C.c_uint64)]


class PoseEdge(C.Structure):
    """malio_pose_edge: a loop edge a -> b, Z = (rot, pos) = T_a^-1 T_b, and its information (order [dtheta, dt])."""
    _fields_ = [("a", C.c_uint64), ("b", C.c_uint64), ("rot", C.c_double * 4), ("pos", C.c_double * 3), ("info", C.c_double * 36)]


class PoseGraphArgs(C.Structure):
    _fields_ = [("sigma_rot", C.c_double), ("sigma_pos", C.c_double), ("max_iter", C.c_uint32), ("eps_rot", C.c_double),
                ("eps_pos", C.c_double)]


class PoseGraphReport(C.Structure):
    _fields_ = [("iterations", C.c_uint32), ("converged", C.c_int32), ("chi2_odo", C.c_double), ("chi2_loop", C.c_double),
                ("chi2_loop_before", C.c_double), ("ms", C.c_double)]


class UpdateReport(C.Structure):
    _fields_ = [("passes", C.c_int32), ("searches", C.c_int32), ("converged_count", C.c_int32),
                ("last_status", C.c_int32), ("n_eff_last", C.c_uint32), ("ms_device_total", C.c_float),
                ("ms_host_solve", C.c_float), ("dx_last", C.c_double * MAX_DOF)]


_LIB_NAME = "libmalio_b200.so"
_lib = None

EXPORTS = [
    "malio_default_params", "malio_create", "malio_destroy", "malio_last_error", "malio_version",
    "malio_get_nccl_unique_id", "malio_comm_init", "malio_upload_map", "malio_upload_scan", "malio_measure",
    "malio_download_rows", "malio_download_aux", "malio_knn", "malio_ieskf_update", "malio_build_static_snapshot",
    "malio_rearm_scan", "malio_get_counters", "malio_set_timing", "malio_upload_map_compact", "malio_download_map_nodes", "malio_map_incremental",
    "malio_map_build", "malio_map_add_points", "malio_map_delete_boxes", "malio_map_sync_voxels", "malio_map_commit", "malio_map_info",
    "malio_map_download", "malio_read_livox_bin", "malio_read_ouster_bin", "malio_preprocess_livox", "malio_preprocess_ouster",
    "malio_undistort", "malio_bspline_get_pose", "malio_voxel_grid", "malio_upload_scan_device", "malio_scan_uncertainty",
    "malio_pose_initial", "malio_compound_pose_with_cov", "malio_compound_inv_pose_with_cov", "malio_build_pose_unc",
    "malio_world_register", "malio_world_accumulate", "malio_world_save_pcd", "malio_write_pcd_binary",
    "malio_knn_device", "malio_map_build_device", "malio_map_add_points_device",
    "malio_upload_scan_from_device", "malio_download_aux_device", "malio_map_incremental_device", "malio_world_register_device",
    "malio_undistort_device", "malio_voxel_grid_device", "malio_scan_uncertainty_resident", "malio_upload_scan_resident",
    "malio_world_voxel_accumulate", "malio_world_voxel_download_device", "malio_world_voxel_save_pcd", "malio_world_voxel_info",
    "malio_prior_map_load", "malio_prior_map_load_device", "malio_prior_map_window", "malio_prior_map_info", "malio_prior_map_clear",
    "malio_read_pcd", "malio_relocalize",
    "malio_world_voxel_accumulate_carve", "malio_world_voxel_evidence_device", "malio_world_voxel_download_kept_device",
    "malio_world_voxel_save_pcd_kept",
    "malio_place_db_build", "malio_place_db_info", "malio_place_db_download", "malio_relocalize_global",
    "malio_world_voxel_seed", "malio_world_voxel_seed_device", "malio_world_voxel_changes_device",
    "malio_world_voxel_save_changes_pcd",
    "malio_prior_map_extend", "malio_prior_map_session_download",
    "malio_grid_build_device", "malio_grid_build", "malio_grid_extent_device", "malio_write_grid_pgm",
    "malio_scan_store_add", "malio_scan_store_put", "malio_scan_store_get", "malio_scan_store_register_device",
    "malio_scan_store_info", "malio_scan_store_clear", "malio_world_voxel_rebuild",
    "malio_scan_store_match", "malio_pose_graph_optimize",
]


def lib_path() -> str:
    # MALIO_LIB_PATH: another build of the same library (kernel-parameter experiments); the product default is in-tree
    return os.environ.get("MALIO_LIB_PATH") or os.path.join(os.path.dirname(os.path.abspath(__file__)), _LIB_NAME)


def load() -> C.CDLL:
    """Load the product library; raises if it has not been built (no silent fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise RuntimeError(f"{path} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           f"or `make -C ma-lio_b200/csrc`")
    lib = C.CDLL(path)
    vp, u32, i32 = C.c_void_p, C.c_uint32, C.c_int
    lib.malio_default_params.argtypes = [C.POINTER(Params), i32]
    lib.malio_default_params.restype = None
    lib.malio_create.argtypes = [C.POINTER(vp), C.POINTER(Config)]
    lib.malio_destroy.argtypes = [vp]
    lib.malio_destroy.restype = None
    lib.malio_last_error.argtypes = [vp]
    lib.malio_last_error.restype = C.c_char_p
    lib.malio_version.restype = C.c_char_p
    lib.malio_get_nccl_unique_id.argtypes = [vp]
    lib.malio_comm_init.argtypes = [vp, vp, i32, i32]
    lib.malio_upload_map.argtypes = [vp, vp, vp, u32, u32]
    lib.malio_upload_map_compact.argtypes = [vp, vp, vp, u32, u32, vp]
    lib.malio_download_map_nodes.argtypes = [vp, vp, u32]
    lib.malio_map_incremental.argtypes = [vp, vp, C.c_double, i32, vp, vp]
    lib.malio_pose_initial.restype = None
    lib.malio_pose_initial.argtypes = [vp, vp, vp, vp]
    lib.malio_compound_pose_with_cov.restype = None
    lib.malio_compound_pose_with_cov.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.malio_compound_inv_pose_with_cov.restype = None
    lib.malio_compound_inv_pose_with_cov.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.malio_build_pose_unc.argtypes = [i32, vp, vp, vp, vp, vp, vp]
    lib.malio_upload_scan.argtypes = [vp, vp, u32, vp, vp, vp]
    lib.malio_map_build.argtypes = [vp, vp, vp, vp, u32]
    lib.malio_map_add_points.argtypes = [vp, vp, vp, vp, u32]
    lib.malio_map_delete_boxes.argtypes = [vp, vp, u32, C.POINTER(u32)]
    lib.malio_map_sync_voxels.argtypes = [vp, vp, u32, vp, vp, vp, u32, C.POINTER(u32)]
    lib.malio_map_commit.argtypes = [vp]
    lib.malio_map_info.argtypes = [vp, C.POINTER(u32), C.POINTER(u32)]
    lib.malio_map_download.argtypes = [vp, vp, vp, vp, vp, u32, C.POINTER(u32)]
    lib.malio_read_livox_bin.argtypes = [C.c_char_p, vp, u32, C.POINTER(u32), i32]
    lib.malio_read_ouster_bin.argtypes = [C.c_char_p, vp, u32, C.POINTER(u32), i32]
    lib.malio_preprocess_livox.argtypes = [vp, u32, i32, i32, C.c_double, vp, vp, u32, C.POINTER(u32)]
    lib.malio_preprocess_ouster.argtypes = [vp, u32, i32, C.c_double, C.c_float, vp, vp, u32, C.POINTER(u32)]
    lib.malio_undistort.argtypes = [vp, i32, vp, u32, C.POINTER(UndistortArgs), vp, vp, vp, vp, C.POINTER(u32), vp]
    lib.malio_bspline_get_pose.argtypes = [vp, vp, u32, C.c_double, vp, vp]
    lib.malio_voxel_grid.argtypes = [vp, i32, vp, u32, C.c_float, vp, u32, C.POINTER(u32)]
    lib.malio_upload_scan_device.argtypes = [vp, vp, vp, vp, C.POINTER(u32)]
    lib.malio_scan_uncertainty.argtypes = [vp, C.POINTER(ScanUncArgs), vp, u32, vp, vp, vp, vp]
    lib.malio_world_register.argtypes = [vp, C.POINTER(PassState), i32, vp, vp, u32, C.POINTER(u32)]
    lib.malio_world_accumulate.argtypes = [vp, C.POINTER(PassState), vp, C.POINTER(C.c_uint64)]
    lib.malio_world_save_pcd.argtypes = [vp, C.c_char_p, i32]
    lib.malio_world_voxel_accumulate.argtypes = [vp, vp, vp, C.c_float, vp]
    lib.malio_world_voxel_download_device.argtypes = [vp, vp, C.c_uint64, vp, vp]
    lib.malio_world_voxel_save_pcd.argtypes = [vp, C.c_char_p, i32]
    lib.malio_world_voxel_info.argtypes = [vp, vp, vp, vp]
    lib.malio_world_voxel_accumulate_carve.argtypes = [vp, vp, vp, C.c_float, vp, vp]
    lib.malio_world_voxel_evidence_device.argtypes = [vp, vp, C.c_uint64, vp, vp]
    lib.malio_world_voxel_download_kept_device.argtypes = [vp, vp, vp, C.c_uint64, vp, vp]
    lib.malio_world_voxel_save_pcd_kept.argtypes = [vp, C.c_char_p, vp, i32]
    lib.malio_world_voxel_seed.argtypes = [vp, vp, C.c_uint64, C.c_float, u32, vp]
    lib.malio_world_voxel_seed_device.argtypes = [vp, vp, C.c_uint64, C.c_float, u32, vp, vp]
    lib.malio_world_voxel_changes_device.argtypes = [vp, vp, vp, C.c_uint64, vp, vp, C.c_uint64, vp, vp]
    lib.malio_world_voxel_save_changes_pcd.argtypes = [vp, vp, C.c_char_p, C.c_char_p, vp, vp]
    lib.malio_scan_store_add.argtypes = [vp, vp, vp, C.c_double, vp]
    lib.malio_scan_store_put.argtypes = [vp, vp, vp, vp]
    lib.malio_scan_store_get.argtypes = [vp, C.c_uint64, vp, vp, C.c_uint64, vp]
    lib.malio_scan_store_register_device.argtypes = [vp, C.c_uint64, vp, vp, C.c_uint64, vp, vp]
    lib.malio_scan_store_info.argtypes = [vp, vp, vp, vp]
    lib.malio_scan_store_clear.argtypes = [vp]
    lib.malio_world_voxel_rebuild.argtypes = [vp, C.c_uint64, C.c_uint64, vp, C.c_float, vp, vp]
    lib.malio_scan_store_match.argtypes = [vp, C.c_uint64, C.c_uint64, vp, vp, vp]
    lib.malio_pose_graph_optimize.argtypes = [vp, C.c_uint64, vp, u32, vp, vp, vp, vp]
    lib.malio_write_pcd_binary.argtypes = [C.c_char_p, vp, C.c_uint64]
    lib.malio_read_pcd.argtypes = [C.c_char_p, vp, C.c_uint64, vp]
    lib.malio_prior_map_load.argtypes = [vp, vp, vp, vp, u32]
    lib.malio_prior_map_load_device.argtypes = [vp, vp, vp, vp, u32, vp]
    lib.malio_prior_map_window.argtypes = [vp, vp, C.c_double, C.c_float, vp]
    lib.malio_prior_map_info.argtypes = [vp, vp, vp, vp]
    lib.malio_prior_map_clear.argtypes = [vp]
    lib.malio_prior_map_extend.argtypes = [vp, vp, C.c_double, vp]
    lib.malio_prior_map_session_download.argtypes = [vp, vp, C.c_uint64, vp]
    lib.malio_relocalize.argtypes = [vp, vp, vp, vp]
    lib.malio_place_db_build.argtypes = [vp, vp, vp]
    lib.malio_place_db_info.argtypes = [vp, vp, vp]
    lib.malio_place_db_download.argtypes = [vp, vp, vp, vp, vp, C.c_uint64, vp]
    lib.malio_relocalize_global.argtypes = [vp, vp, vp, vp]
    lib.malio_grid_build_device.argtypes = [vp, i32, vp, C.c_uint64, vp, vp, vp, vp, vp, vp]
    lib.malio_grid_build.argtypes = [vp, vp, C.c_uint64, vp, vp, vp, vp]
    lib.malio_grid_extent_device.argtypes = [vp, i32, vp, C.c_uint64, vp, C.c_float, vp, vp]
    lib.malio_write_grid_pgm.argtypes = [C.c_char_p, C.c_char_p, vp, u32, u32, C.c_float, C.c_int32, C.c_int32]
    lib.malio_measure.argtypes = [vp, C.POINTER(PassState), i32, vp, vp, C.POINTER(PassStats)]
    lib.malio_download_rows.argtypes = [vp, vp, vp, u32, C.POINTER(u32)]
    lib.malio_download_aux.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.malio_knn.argtypes = [vp, vp, u32, vp, vp, C.POINTER(C.c_float)]
    # device pointers and a cudaStream_t (torch: tensor.data_ptr(), torch.cuda.Stream.cuda_stream)
    lib.malio_knn_device.argtypes = [vp, vp, u32, vp, vp, vp]
    lib.malio_map_build_device.argtypes = [vp, vp, vp, vp, u32, vp]
    lib.malio_map_add_points_device.argtypes = [vp, vp, vp, vp, u32, vp]
    lib.malio_upload_scan_from_device.argtypes = [vp, vp, u32, vp, vp, vp, vp]
    lib.malio_download_aux_device.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.malio_map_incremental_device.argtypes = [vp, vp, C.c_double, i32, vp, vp, vp]
    lib.malio_world_register_device.argtypes = [vp, vp, i32, vp, vp, u32, vp, vp]
    lib.malio_undistort_device.argtypes = [vp, i32, vp, u32, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.malio_voxel_grid_device.argtypes = [vp, i32, vp, u32, C.c_float, vp, u32, vp, vp]
    lib.malio_scan_uncertainty_resident.argtypes = [vp, vp, vp, vp]
    lib.malio_upload_scan_resident.argtypes = [vp, vp]
    lib.malio_ieskf_update.argtypes = [vp, C.POINTER(State), vp, i32, C.c_double, C.POINTER(UpdateReport)]
    lib.malio_build_static_snapshot.argtypes = [vp, u32, vp, vp, C.POINTER(u32)]
    lib.malio_rearm_scan.argtypes = [vp]
    lib.malio_get_counters.argtypes = [vp, C.POINTER(Counters)]
    lib.malio_set_timing.argtypes = [vp, i32]
    _lib = lib
    return lib


def ptr(a):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


class MalioError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"malio status {status}: {msg}")
        self.status = status


def default_params(n_lidar: int) -> Params:
    """The reference defaults (City.yaml / mapping_city.launch) — the same values malio_default_params() fills in; kept in
    Python as well so that input generators (synth.py) work without mapping the CUDA library (bench.py --impl reference).
    tests/test_oracle_cpu.py checks the two agree."""
    p = Params()
    p.n_lidar = n_lidar
    p.extrinsic_est_en = 1
    p.plane_th = 0.4
    p.knn_max_sqdist = 5.0
    p.cov_threshold = 0.5
    p.point_cov_max, p.point_cov_min = 0.00125, 0.00075
    p.plane_cov_max, p.plane_cov_min = 1.0, 0.8
    p.localize_cov_max, p.localize_cov_min = 2.0, 0.3
    p.localize_thresh_max, p.localize_thresh_min = 0.7, 0.2
    p.range_min, p.range_max = 0.0, 1.0
    return p


def default_params_from_library(n_lidar: int) -> Params:
    p = Params()
    load().malio_default_params(C.byref(p), n_lidar)
    return p

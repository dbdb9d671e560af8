"""Python host-side binding of the C ABI (include/superodom_b200.h) via ctypes.

Used by the parity tests and bench.py; the reference's own host language is C++, whose binding is the header-only
shim include/superodom_b200/LidarSlam.hpp.  No torch types cross this boundary: numpy arrays for host buffers,
raw device pointers (ints) for the *_device entry points.  There is no CPU fallback: `Context()` raises if the
shared library is missing or no sm_90 device is present.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SO_LIB_PATH") or os.path.join(_HERE, "libsuperodom_b200.so")      # SO_LIB_PATH: A/B builds (scripts/)
MAX_ICP_ITERS = 32

EXPORTS = [
    "so_create", "so_destroy", "so_last_error", "so_device_available", "so_set_stream",
    "so_map_set_resolution", "so_map_set_origin", "so_map_get_origin", "so_map_shift", "so_map_set_points",
    "so_map_set_edge_points", "so_map_add_surf", "so_map_add_edge", "so_map_add_scan", "so_map_add_registered_scan", "so_map_add_registered_edges", "so_map_add_scan_edge", "so_map_counts_5x5", "so_map_download", "so_map_size",
    "so_map_archive", "so_map_archive_info", "so_map_download_all",
    "so_free_space_defaults", "so_map_clear_free_space", "so_map_clear_free_space_registered", "so_map_clear_free_space_keyframes",
    "so_scan_prefilter", "so_scan_deskew", "so_scan_extract_uniform", "so_scan_extract_edges", "so_register", "so_register_prefiltered", "so_register_injected", "so_set_pose_sink", "so_register_batch", "so_register_batch_edges", "so_register_batch_device",
    "so_register_undistort", "so_register_undistort_edges", "so_register_prefiltered_undistort", "so_register_batch_undistort", "so_undistort_points", "so_register_optimized", "so_register_optimized_edges", "so_register_prefiltered_optimized", "so_register_batch_optimized", "so_evaluate_optimized", "so_evaluate_optimized_edges", "so_correspond", "so_correspond_seeded", "so_ordered_scans", "so_correspond_edge", "so_evaluate", "so_covariance",
    "so_register_degeneracy", "so_register_batch_degeneracy", "so_degeneracy_analysis", "so_solve", "so_solve_optimized",
    "so_knn", "so_knn_device", "so_sampling_indices", "so_localize_global", "so_localize_scores", "so_localize_global_size", "so_localize_global_bnb", "so_localize_bnb_keys", "so_localize_bnb_bounds", "so_map_bounds", "so_map_bounds_all", "so_kernel_launches", "so_bytes_copied", "so_build_flags", "so_profile_enable", "so_profile_get",
    "so_knn_graph", "so_knn_graph_stats",
    "so_keyframe_reserve", "so_keyframe_add_registered", "so_keyframe_import", "so_keyframe_info", "so_keyframe_poses", "so_keyframe_download", "so_map_from_keyframes",
    "so_register_keyframes", "so_register_keyframes_degeneracy",
    "so_loop_opts_defaults", "so_loop_candidates", "so_loop_candidates_range", "so_keyframe_descriptors",
    "so_loop_prior", "so_loop_verify_opts_defaults", "so_loop_verify", "so_loop_verify_degeneracy", "so_loop_edge_information",
    "so_pose_graph_opts_defaults", "so_pose_graph_check", "so_pose_graph_solve", "so_pose_graph_check_constant", "so_pose_graph_solve_constant",
]


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_map_points", C.c_uint32), ("max_scan_points", C.c_uint32),
                ("max_batch", C.c_uint32), ("line_res", C.c_float), ("plane_res", C.c_float)]


class IcpOpts(C.Structure):
    _fields_ = [("max_icp_iters", C.c_int32), ("max_surface_features", C.c_int32), ("lm_max_iterations", C.c_int32),
                ("yaw_ratio", C.c_float), ("skip_map_checks", C.c_int32), ("use_pose_prior", C.c_int32),
                ("visual_confidence_factor", C.c_float), ("prior_uncertainty", C.c_float * 3)]


class IcpResult(C.Structure):
    _fields_ = [("pose", C.c_double * 7), ("pose_opt", C.c_double * 7), ("status", C.c_int32), ("n_iterations", C.c_int32),
                ("iter_n_surf", C.c_int32 * MAX_ICP_ITERS), ("iter_n_edge", C.c_int32 * MAX_ICP_ITERS),
                ("iter_dtrans", C.c_double * MAX_ICP_ITERS), ("iter_drot", C.c_double * MAX_ICP_ITERS),
                ("iter_lm_steps", C.c_int32 * MAX_ICP_ITERS), ("iter_lm_successful", C.c_int32 * MAX_ICP_ITERS),
                ("iter_lm_termination", C.c_int32 * MAX_ICP_ITERS), ("iter_cost", C.c_double * MAX_ICP_ITERS),
                ("hist_obs", C.c_int32 * 9), ("hist_reject_plane", C.c_int32 * 7), ("hist_reject_line", C.c_int32 * 7),
                ("cov", C.c_double * 36),
                ("pos_err", C.c_double), ("pos_dir", C.c_double * 3), ("pos_inv_cond", C.c_double),
                ("ori_err_deg", C.c_double), ("ori_dir", C.c_double * 3), ("ori_inv_cond", C.c_double),
                ("total_translation", C.c_double), ("total_rotation", C.c_double),
                ("translation_from_last", C.c_double), ("rotation_from_last", C.c_double),
                ("map_surf_5x5", C.c_int32), ("map_edge_5x5", C.c_int32), ("scan_surf_num", C.c_int32), ("scan_edge_num", C.c_int32),
                ("pos_in_localmap", C.c_int32 * 3), ("prediction_source", C.c_int32),
                ("time_ms", C.c_double), ("time_total_ms", C.c_double), ("knn_searched", C.c_int32), ("knn_verified", C.c_int32)]


class Undistort(C.Structure):
    """so_undistort: within-scan motion compensation of one scan (mode 0 NONE, 1 APPROXIMATED)."""
    _fields_ = [("mode", C.c_int32), ("rotation", C.c_int32), ("prev_pose", C.c_double * 7), ("dt", C.c_double)]


def undistort(prev_pose7, dt: float, rotation: bool = True, mode: int = 1) -> Undistort:
    return Undistort(int(mode), int(rotation), (C.c_double * 7)(*[float(v) for v in prev_pose7]), float(dt))


class Motion(C.Structure):
    """so_motion: the motion prior of so_register_optimized* (D0 over dt seconds, information per accepted correspondence)."""
    _fields_ = [("dt", C.c_double), ("motion_prior", C.c_double * 7), ("motion_info", C.c_double * 6)]


class MotionResult(C.Structure):
    """so_motion_result: icp.pose_opt = T (the pose at time 0), motion = D, pose_end = T * D (the pose at time dt)."""
    _fields_ = [("icp", IcpResult), ("motion", C.c_double * 7), ("pose_end", C.c_double * 7)]


# motion_info per accepted correspondence that the accuracy sweep of scripts/bench_undistort.py chose (DESIGN.md §4); the C++ shim's
# LidarSLAM::OptimizedMotionInformation defaults to the same value
DEFAULT_MOTION_INFO = 0.0


def motion(dt: float, prior7=(0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0), info=(DEFAULT_MOTION_INFO,) * 6) -> Motion:
    return Motion(float(dt), (C.c_double * 7)(*[float(v) for v in prior7]), (C.c_double * 6)(*[float(v) for v in info]))


class Degeneracy(C.Structure):
    """so_degeneracy: thresholds on sqrt(i_k / i_max) of the translation / rotation information (each in [0, 1)); constrain = 1 keeps
    the solve off the flagged directions, 0 only reports them."""
    _fields_ = [("pos_threshold", C.c_double), ("ori_threshold", C.c_double), ("constrain", C.c_int32), ("pad_", C.c_int32)]


def degeneracy(pos_threshold: float, ori_threshold: float, constrain: bool = True) -> Degeneracy:
    return Degeneracy(float(pos_threshold), float(ori_threshold), int(constrain), 0)


class DegeneracyResult(C.Structure):
    """so_degeneracy_result: the registration, flagged directions per ICP iteration, and the last iteration's eigenpairs of I_t and
    I_theta (ascending; axes[3k:3k+3] = eigenvector k) with their flags (bit k: eigenvector k flagged)."""
    _fields_ = [("icp", IcpResult), ("iter_n_flag_pos", C.c_int32 * MAX_ICP_ITERS), ("iter_n_flag_ori", C.c_int32 * MAX_ICP_ITERS),
                ("pos_info", C.c_double * 3), ("pos_axes", C.c_double * 9), ("ori_info", C.c_double * 3), ("ori_axes", C.c_double * 9),
                ("flags_pos", C.c_int32), ("flags_ori", C.c_int32)]


class GlobalOpts(C.Structure):
    """so_global_opts: zero fields take the defaults (res 0.25 m, yaw_step 2 deg, max_range 40 m, score_points 1024, dilate 1,
    k 16, nms_xy 1 m, nms_yaw 10 deg).  whole_map 1: search and refine over the window plus the block archive."""
    _fields_ = [("half_x", C.c_double), ("half_y", C.c_double), ("half_z", C.c_double), ("yaw_half", C.c_double),
                ("res", C.c_double), ("yaw_step", C.c_double), ("max_range", C.c_double), ("score_points", C.c_int32),
                ("dilate", C.c_int32), ("k", C.c_int32), ("whole_map", C.c_int32), ("nms_xy", C.c_double), ("nms_yaw", C.c_double)]


class GlobalCandidate(C.Structure):
    _fields_ = [("prior", C.c_double * 7), ("score", C.c_int32), ("n_success", C.c_int32), ("cost", C.c_double),
                ("pose", C.c_double * 7), ("status", C.c_int32), ("pad_", C.c_int32)]


class GlobalResult(C.Structure):
    _fields_ = [("pose", C.c_double * 7), ("status", C.c_int32), ("winner", C.c_int32), ("n_candidates", C.c_int32),
                ("best_score", C.c_int32), ("n_hypotheses", C.c_uint64), ("n_score_points", C.c_int32), ("n_windows", C.c_int32),
                ("time_raster_ms", C.c_double), ("time_dilate_ms", C.c_double), ("time_score_ms", C.c_double),
                ("time_sort_ms", C.c_double), ("time_refine_ms", C.c_double), ("time_total_ms", C.c_double), ("icp", IcpResult)]


def global_opts(half_x=0.0, half_y=0.0, half_z=0.0, yaw_half=0.0, res=0.0, yaw_step=0.0, max_range=0.0, score_points=0, dilate=0,
                k=0, nms_xy=0.0, nms_yaw=0.0, whole_map=False) -> GlobalOpts:
    """whole_map: True / False, or an int passed through as given (the library accepts 0 and 1)."""
    return GlobalOpts(half_x, half_y, half_z, yaw_half, res, yaw_step, max_range, score_points, dilate, k, int(whole_map), nms_xy, nms_yaw)


BNB_LEVELS = 32


class BnbStats(C.Structure):
    """so_bnb_stats: where the branch-and-bound search spent its work (per level: bounds computed and nodes discarded)."""
    _fields_ = [("lmax", C.c_int32), ("kstar_score", C.c_int32), ("root_nodes", C.c_uint64),
                ("scored", C.c_uint64 * BNB_LEVELS), ("discarded", C.c_uint64 * BNB_LEVELS), ("leaves_scored", C.c_uint64),
                ("steps", C.c_uint64), ("pyramid_bytes", C.c_uint64), ("time_build_ms", C.c_double), ("time_search_ms", C.c_double)]


def whole_map_opts(map_lo, map_hi, center_pose7, **kw) -> GlobalOpts:
    """global_opts whose x/y region around the centre covers the map's bounding box (Context.map_bounds): half_x / half_y are the
    largest distance from the centre to the box along each axis.  The centre then supplies only z, roll/pitch and the yaw origin;
    the remaining options (yaw_half, res, ...) are passed through."""
    hx = max(float(map_hi[0]) - float(center_pose7[0]), float(center_pose7[0]) - float(map_lo[0]), 0.0)
    hy = max(float(map_hi[1]) - float(center_pose7[1]), float(center_pose7[1]) - float(map_lo[1]), 0.0)
    return global_opts(half_x=hx, half_y=hy, **kw)


class FreeSpace(C.Structure):
    """so_free_space: range-image geometry (degrees) and decision constants of free-space clearing."""
    _fields_ = [("az_res_deg", C.c_float), ("el_res_deg", C.c_float), ("el_min_deg", C.c_float), ("el_max_deg", C.c_float),
                ("dilate", C.c_int32), ("margin", C.c_float), ("margin_rel", C.c_float), ("min_range", C.c_float), ("max_range", C.c_float)]


class FreeSpaceResult(C.Structure):
    _fields_ = [("n_image_points", C.c_uint64), ("n_pixels_hit", C.c_uint64), ("n_candidates", C.c_uint64), ("n_removed", C.c_uint64),
                ("n_after", C.c_uint64 * 2)]


class FreeSpaceKeyframesResult(C.Structure):
    _fields_ = [("n_keyframes", C.c_uint64), ("n_image_points", C.c_uint64), ("n_pixels_hit", C.c_uint64), ("n_candidates", C.c_uint64),
                ("n_removed", C.c_uint64), ("n_after", C.c_uint64 * 2), ("n_tiles", C.c_uint64), ("time_ms", C.c_double)]


def free_space(**kw) -> FreeSpace:
    """so_free_space_defaults, then the given fields (e.g. el_res_deg=2.0, el_min_deg=-16, el_max_deg=16 for a VLP-16)."""
    o = FreeSpace()
    load_library().so_free_space_defaults(C.byref(o))
    for k, v in kw.items():
        if not hasattr(o, k):
            raise TypeError(f"so_free_space has no field {k}")
        setattr(o, k, v)
    return o


class LoopOpts(C.Structure):
    """so_loop_opts: Scan Context geometry (rings, sectors, max_range m, height_offset m) and the search's exclude_recent."""
    _fields_ = [("rings", C.c_int32), ("sectors", C.c_int32), ("max_range", C.c_double), ("height_offset", C.c_double),
                ("exclude_recent", C.c_int32), ("pad_", C.c_int32)]


class LoopStats(C.Structure):
    _fields_ = [("n_described", C.c_uint64), ("time_describe_ms", C.c_double), ("time_search_ms", C.c_double)]


# so_loop_candidate
LOOP_CANDIDATE_DTYPE = np.dtype([("query", "<i4"), ("id", "<i4"), ("distance", "<f8"), ("shift", "<i4"), ("n_pairs", "<i4"),
                                 ("yaw", "<f8")], align=True)


def loop_opts(**kw) -> LoopOpts:
    """so_loop_opts_defaults, then the given fields."""
    o = LoopOpts()
    load_library().so_loop_opts_defaults(C.byref(o))
    for k, v in kw.items():
        if not hasattr(o, k) or k == "pad_":
            raise TypeError(f"so_loop_opts has no field {k}")
        setattr(o, k, v)
    return o


class LoopVerifyOpts(C.Structure):
    """so_loop_verify_opts: the submap (half_window, the eligible id range, exclude_recent), the alignment (icp), the overlap radius
    (inlier_dist m), the range-image options of the conflict tests (image) and the decision thresholds."""
    _fields_ = [("half_window", C.c_int32), ("id_begin", C.c_int32), ("id_end", C.c_int32), ("exclude_recent", C.c_int32),
                ("icp", IcpOpts), ("inlier_dist", C.c_double), ("image", FreeSpace), ("min_overlap", C.c_double),
                ("max_conflict", C.c_double)]


class LoopVerifyResult(C.Structure):
    _fields_ = [("query", C.c_int32), ("id", C.c_int32), ("skipped", C.c_int32), ("accepted", C.c_int32), ("reg", IcpResult),
                ("rel7", C.c_double * 7), ("n_submap_keyframes", C.c_int32), ("pad_", C.c_int32), ("n_submap_points", C.c_uint64),
                ("n_query_points", C.c_uint64), ("n_inliers", C.c_uint64), ("overlap", C.c_double), ("rmse", C.c_double),
                ("n_cand_query", C.c_uint64), ("n_conflict_query", C.c_uint64), ("n_cand_map", C.c_uint64), ("n_conflict_map", C.c_uint64),
                ("conflict_query", C.c_double), ("conflict_map", C.c_double), ("time_ms", C.c_double)]


def loop_verify_opts(image: FreeSpace | dict | None = None, icp: dict | None = None, **kw) -> LoopVerifyOpts:
    """so_loop_verify_opts_defaults, then the given fields; image: a FreeSpace or the fields of one over its defaults; icp: fields of
    so_icp_opts over the defaults (max_icp_iters 20, max_surface_features 0, lm_max_iterations 4)."""
    o = LoopVerifyOpts()
    load_library().so_loop_verify_opts_defaults(C.byref(o))
    if image is not None:
        o.image = image if isinstance(image, FreeSpace) else free_space(**image)
    for k, v in (icp or {}).items():
        if not hasattr(o.icp, k):
            raise TypeError(f"so_icp_opts has no field {k}")
        setattr(o.icp, k, v)
    for k, v in kw.items():
        if not hasattr(o, k) or k in ("icp", "image"):
            raise TypeError(f"so_loop_verify_opts has no field {k}")
        setattr(o, k, v)
    return o


def loop_prior(cand7, query7, yaw: float) -> np.ndarray:
    """Host-only so_loop_prior: the alignment prior of a loop candidate from the candidate's and the query's poses and its yaw."""
    a = np.ascontiguousarray(cand7, dtype=np.float64)
    b = np.ascontiguousarray(query7, dtype=np.float64)
    out = np.zeros(7, np.float64)
    load_library().so_loop_prior(_p(a), _p(b), float(yaw), _p(out))
    return out


def loop_edge_information(reg_pose, deg: DegeneracyResult, S) -> np.ndarray:
    """Host-only so_loop_edge_information: the square-root information S [6, 6] (or its diagonal, 6 values) of a loop edge with the
    directions deg flags (a loop_verify_degeneracy result) left out -> [6, 6].  Raises SuperOdomError (.code SO_ERR_ARG) as the C call
    fails."""
    L = load_library()
    p = np.ascontiguousarray(reg_pose, dtype=np.float64)
    s = np.asarray(S, np.float64)
    s = np.ascontiguousarray(np.diag(s) if s.shape == (6,) else s.reshape(6, 6))
    if p.shape != (7,):
        raise ValueError(f"reg_pose: a pose7, got shape {p.shape}")
    out = np.zeros((6, 6), np.float64)
    rc = L.so_loop_edge_information(_p(p), C.byref(deg), _p(s), _p(out))
    if rc < 0:
        err = SuperOdomError(f"so_loop_edge_information failed ({rc}): " + L.so_last_error().decode())
        err.code = rc
        raise err
    return out


# so_pose_edge, so_pose_graph_opts, so_pose_graph_result
POSE_EDGE_DTYPE = np.dtype([("i", "<i4"), ("j", "<i4"), ("z", "<f8", 7), ("sqrt_info", "<f8", 36), ("cauchy", "<f8")], align=True)


class PoseGraphOpts(C.Structure):
    _fields_ = [("fixed", C.c_int32), ("max_iterations", C.c_int32)]


class PoseGraphResult(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("successful", C.c_int32), ("unsuccessful", C.c_int32), ("termination", C.c_int32),
                ("pcg_iterations", C.c_uint64), ("initial_cost", C.c_double), ("final_cost", C.c_double), ("gmax", C.c_double),
                ("radius", C.c_double), ("time_ms", C.c_double)]


def pose_edges(edges) -> np.ndarray:
    """Edges as a POSE_EDGE_DTYPE array: given as one, or as tuples (i, j, z7, sqrt_info, cauchy=0), sqrt_info a 6x6 matrix or the
    diagonal of one (6 values)."""
    if isinstance(edges, np.ndarray) and edges.dtype == POSE_EDGE_DTYPE:
        return np.ascontiguousarray(edges)
    out = np.zeros(len(edges), POSE_EDGE_DTYPE)
    for k, e in enumerate(edges):
        s = np.asarray(e[3], np.float64)
        out[k]["i"], out[k]["j"], out[k]["z"] = int(e[0]), int(e[1]), np.asarray(e[2], np.float64)
        out[k]["sqrt_info"] = (np.diag(s) if s.shape == (6,) else s.reshape(6, 6)).ravel()
        out[k]["cauchy"] = float(e[4]) if len(e) > 4 else 0.0
    return out


def pose_graph_check(n_nodes: int, edges, fixed: int = 0, max_iterations: int = 50):
    """Host-only so_pose_graph_check: raises SuperOdomError with .code = SO_ERR_ARG (-1) and the cause for a graph the solve refuses."""
    L = load_library()
    e = pose_edges(edges)
    o = PoseGraphOpts(int(fixed), int(max_iterations))
    rc = L.so_pose_graph_check(int(n_nodes), _p(e) if len(e) else None, len(e), C.byref(o))
    if rc < 0:
        err = SuperOdomError(f"so_pose_graph_check failed ({rc}): " + L.so_last_error().decode())
        err.code = rc
        raise err


def pose_graph_check_constant(n_nodes: int, edges, constant, max_iterations: int = 50):
    """Host-only so_pose_graph_check_constant: as pose_graph_check, with the nodes where constant (a mask of n_nodes) is set held
    constant in place of one fixed node."""
    L = load_library()
    e = pose_edges(edges)
    m = np.ascontiguousarray(constant, dtype=np.uint8)
    if m.shape != (int(n_nodes),):
        raise ValueError(f"constant: a mask of {n_nodes} nodes, got shape {m.shape}")
    o = PoseGraphOpts(0, int(max_iterations))
    rc = L.so_pose_graph_check_constant(int(n_nodes), _p(e) if len(e) else None, len(e), _p(m), C.byref(o))
    if rc < 0:
        err = SuperOdomError(f"so_pose_graph_check_constant failed ({rc}): " + L.so_last_error().decode())
        err.code = rc
        raise err


class EdgeOpts(C.Structure):
    """so_edge_opts: zero fields take the defaults (min_range 0, edge_threshold 0.1, voxel_leaf 0 = no filter, max_per_sector 20)."""
    _fields_ = [("min_range", C.c_float), ("edge_threshold", C.c_float), ("voxel_leaf", C.c_float), ("max_per_sector", C.c_int32)]


CORR_DTYPE = np.dtype([("n", "<f8", 3), ("d", "<f8"), ("w", "<f8"), ("nn", "<u4", 5), ("nn_d2", "<f4", 5),
                       ("status", "u1"), ("obs", "u1", 3), ("pad_", "u1", 4)], align=True)

EDGE_CORR_DTYPE = np.dtype([("a", "<f8", 3), ("b", "<f8", 3), ("w", "<f8"), ("nn", "<u4", 10), ("selected_mask", "<u4"),
                            ("status", "u1"), ("n_selected", "u1"), ("pad_", "u1", 2)], align=True)

# so_solve's rows, problems and results
SOLVE_ROW_DTYPE = np.dtype([("p", "<f4", 3), ("pad_", "<f4"), ("n", "<f8", 3), ("d", "<f8"), ("w", "<f8")], align=True)
SOLVE_PROBLEM_DTYPE = np.dtype([("n_rows", "<u4"), ("lm_max_iterations", "<i4"), ("pose", "<f8", 7), ("use_pose_prior", "<i4"),
                                ("visual_confidence_factor", "<f4"), ("prior_uncertainty", "<f4", 3), ("pad_", "<i4"), ("x0", "<f8", 7)],
                               align=True)
SOLVE_RESULT_DTYPE = np.dtype([("pose", "<f8", 7), ("initial_cost", "<f8"), ("final_cost", "<f8"), ("lm_iterations", "<i4"),
                               ("successful", "<i4"), ("unsuccessful", "<i4"), ("termination", "<i4"), ("radius", "<f8"),
                               ("decrease_factor", "<f8"), ("gmax", "<f8"), ("n_flag_pos", "<i4"), ("n_flag_ori", "<i4"),
                               ("status", "<i4"), ("pad_", "<i4")], align=True)
# so_solve_optimized's problems and results (rows: SOLVE_ROW_DTYPE, with one float32 time per row)
SOLVE_OPTIMIZED_PROBLEM_DTYPE = np.dtype([("n_rows", "<u4"), ("lm_max_iterations", "<i4"), ("pose", "<f8", 7), ("motion", "<f8", 7),
                                          ("dt", "<f8"), ("motion_prior", "<f8", 7), ("motion_info", "<f8", 6)], align=True)
SOLVE_OPTIMIZED_RESULT_DTYPE = np.dtype([("solve", SOLVE_RESULT_DTYPE), ("motion", "<f8", 7), ("cov", "<f8", 36)], align=True)

_lib = None


def load_library():
    """dlopen the in-tree shared library and declare signatures.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} missing: run `python -m superodom_b200.build` (no CPU fallback exists)")
    L = C.CDLL(LIB_PATH)
    L.so_create.restype = C.c_void_p
    L.so_create.argtypes = [C.POINTER(Config)]
    L.so_destroy.argtypes = [C.c_void_p]
    L.so_last_error.restype = C.c_char_p
    L.so_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    L.so_map_set_resolution.argtypes = [C.c_void_p, C.c_float, C.c_float]
    L.so_map_set_origin.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_map_get_origin.argtypes = [C.c_void_p, C.c_void_p]
    L.so_map_shift.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_map_set_points.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]
    L.so_map_add_surf.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]
    L.so_map_add_scan.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p]
    L.so_map_add_registered_scan.argtypes = [C.c_void_p, C.c_void_p]
    L.so_map_add_registered_edges.argtypes = [C.c_void_p, C.c_void_p]
    L.so_map_add_scan_edge.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p]
    L.so_map_set_edge_points.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]
    L.so_map_add_edge.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]
    L.so_correspond_edge.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_map_counts_5x5.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_map_download.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_map_size.restype = C.c_size_t
    L.so_map_size.argtypes = [C.c_void_p]
    L.so_map_archive.argtypes = [C.c_void_p, C.c_size_t]
    L.so_map_archive_info.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_map_download_all.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_free_space_defaults.restype = None
    L.so_free_space_defaults.argtypes = [C.c_void_p]
    L.so_map_clear_free_space.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p,
                                          C.c_void_p]
    L.so_map_clear_free_space_registered.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_map_clear_free_space_keyframes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p,
                                                    C.c_void_p]
    L.so_scan_prefilter.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.so_scan_deskew.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_double, C.c_void_p, C.c_void_p, C.c_size_t,
                                 C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_scan_extract_uniform.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_float, C.c_int,
                                          C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_scan_extract_edges.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p,
                                        C.c_size_t, C.c_void_p]
    L.so_register.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                              C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_prefiltered.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_injected.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    L.so_register_undistort.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p]
    L.so_register_undistort_edges.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_prefiltered_undistort.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_batch_undistort.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_undistort_points.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p,
                                      C.c_void_p]
    L.so_register_optimized.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p]
    L.so_register_optimized_edges.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_evaluate_optimized_edges.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                              C.c_void_p, C.c_void_p, C.c_double, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_prefiltered_optimized.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_batch_optimized.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_evaluate_optimized.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p,
                                        C.c_double, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_set_pose_sink.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]
    L.so_register_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                    C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_batch_edges.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                          C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_correspond.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_int32,
                                C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_correspond_seeded.argtypes = list(L.so_correspond.argtypes) + [C.c_void_p]
    L.so_ordered_scans.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.so_evaluate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    L.so_register_degeneracy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_batch_degeneracy.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t,
                                               C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_degeneracy_analysis.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.so_solve_optimized.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    L.so_knn_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    L.so_sampling_indices.argtypes = [C.c_uint32, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_localize_global.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_localize_scores.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_size_t, C.c_void_p, C.c_void_p]
    L.so_localize_global_size.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_localize_global_bnb.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.so_localize_bnb_keys.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_size_t, C.c_void_p, C.c_void_p]
    L.so_localize_bnb_bounds.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_map_bounds.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_map_bounds_all.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_kernel_launches.restype = C.c_uint64
    L.so_kernel_launches.argtypes = [C.c_void_p, C.c_int]
    L.so_bytes_copied.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    L.so_profile_enable.argtypes = [C.c_void_p, C.c_int]
    L.so_profile_get.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    L.so_knn_graph.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.so_knn_graph_stats.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.so_keyframe_reserve.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t]
    L.so_keyframe_add_registered.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_keyframe_import.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p,
                                     C.c_void_p]
    L.so_keyframe_info.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_keyframe_poses.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_keyframe_download.argtypes = [C.c_void_p, C.c_int32, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_map_from_keyframes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int]
    L.so_register_keyframes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_register_keyframes_degeneracy.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p]
    L.so_loop_opts_defaults.restype = None
    L.so_loop_opts_defaults.argtypes = [C.c_void_p]
    L.so_loop_candidates.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    L.so_loop_candidates_range.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                           C.c_void_p]
    L.so_keyframe_descriptors.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.so_loop_prior.restype = None
    L.so_loop_prior.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    L.so_loop_verify_opts_defaults.restype = None
    L.so_loop_verify_opts_defaults.argtypes = [C.c_void_p]
    L.so_loop_verify.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.so_loop_verify_degeneracy.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_loop_edge_information.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_pose_graph_opts_defaults.restype = None
    L.so_pose_graph_opts_defaults.argtypes = [C.c_void_p]
    L.so_pose_graph_check.argtypes = [C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.so_pose_graph_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p]
    L.so_pose_graph_check_constant.argtypes = [C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.so_pose_graph_solve_constant.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p]
    _lib = L
    return L


def build_flags() -> int:
    return int(load_library().so_build_flags())


def sampling_indices(n: int, max_surface_features: int) -> np.ndarray:
    """Indices a registration capped at max_surface_features processes (calculateSamplingRate + shouldProcessPoint,
    LidarSlam.cpp:346-359).  Host-only."""
    L = load_library()
    out = np.empty(n, np.uint32)
    cnt = C.c_size_t(0)
    if L.so_sampling_indices(n, max_surface_features, out.ctypes.data_as(C.c_void_p), n, C.byref(cnt)) != 0:
        raise SuperOdomError("so_sampling_indices failed")
    return out[:cnt.value].copy()


def localize_global_size(opts: GlobalOpts | None = None, **kw):
    """Host-only: (dims (NX, NY, NZ, NYAW), hypothesis count, bitmap bytes) of a global localization search; raises SuperOdomError
    with .code = SO_ERR_ARG (-1) / SO_ERR_CAPACITY (-3) on invalid or too large searches."""
    L = load_library()
    o = opts if opts is not None else global_opts(**kw)
    dims = np.zeros(4, np.int32)
    nh, nb = C.c_uint64(), C.c_uint64()
    rc = L.so_localize_global_size(C.byref(o), _p(dims), C.byref(nh), C.byref(nb))
    if rc < 0:
        e = SuperOdomError(f"so_localize_global_size failed ({rc}): " + L.so_last_error().decode())
        e.code = rc
        raise e
    return tuple(int(v) for v in dims), nh.value, nb.value


def device_available() -> bool:
    return bool(load_library().so_device_available())


class SuperOdomError(RuntimeError):
    pass


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Context:
    """One registration context == one LidarSLAM + LocalMap instance on one GPU."""

    def __init__(self, device: int = 0, max_map_points: int = 4 << 20, max_scan_points: int = 262144, max_batch: int = 1,
                 plane_res: float = 0.4, line_res: float = 0.2):
        self.L = load_library()
        cfg = Config(device, max_map_points, max_scan_points, max_batch, line_res, plane_res)
        h = self.L.so_create(C.byref(cfg))
        if not h:
            raise SuperOdomError("so_create failed: " + self.L.so_last_error().decode())
        self.h = C.c_void_p(h)
        self.max_batch = max_batch

    def close(self):
        if getattr(self, "h", None):
            self.L.so_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc, what):
        if rc < 0:
            raise SuperOdomError(f"{what} failed ({rc}): " + self.L.so_last_error().decode())
        return rc

    # ---- stream / instrumentation
    def set_stream(self, cuda_stream_ptr: int | None):
        self._chk(self.L.so_set_stream(self.h, C.c_void_p(cuda_stream_ptr or 0)), "so_set_stream")

    def kernel_launches(self, reset: bool = False) -> int:
        return int(self.L.so_kernel_launches(self.h, int(reset)))

    def bytes_copied(self, reset: bool = False):
        a, b = C.c_uint64(), C.c_uint64()
        self._chk(self.L.so_bytes_copied(self.h, C.byref(a), C.byref(b), int(reset)), "so_bytes_copied")
        return a.value, b.value

    def profile_enable(self, on: bool):
        self._chk(self.L.so_profile_enable(self.h, int(on)), "so_profile_enable")

    def profile_get(self, cls: int, reset: bool = False):
        ms = C.c_double()
        n = C.c_uint64()
        self._chk(self.L.so_profile_get(self.h, cls, C.byref(ms), C.byref(n), int(reset)), "so_profile_get")
        return ms.value, n.value

    def knn_graph(self):
        """The surf store's neighbour graph (built when none is valid): (point ids [n] in search order, neighbour ids [n, k],
        radius [n]) -- see so_knn_graph."""
        k = C.c_uint32()
        n = C.c_size_t()
        self._chk(self.L.so_knn_graph(self.h, None, None, None, 0, C.byref(k), C.byref(n)), "so_knn_graph")
        ids = np.zeros(n.value, np.uint32)
        nbr = np.zeros((n.value, k.value), np.uint32)
        rad = np.zeros(n.value, np.float32)
        if n.value:
            self._chk(self.L.so_knn_graph(self.h, _p(ids), _p(nbr), _p(rad), n.value, C.byref(k), C.byref(n)), "so_knn_graph")
        return ids, nbr, rad

    def knn_graph_stats(self, on: bool = True) -> np.ndarray:
        """[MAX_ICP_ITERS, 2] counts since the last call (queries searched, queries the neighbour graph answered) per ICP
        iteration; on: reset and keep counting, else stop."""
        out = np.zeros(2 * MAX_ICP_ITERS, np.uint64)
        self._chk(self.L.so_knn_graph_stats(self.h, int(on), _p(out)), "so_knn_graph_stats")
        return out.reshape(MAX_ICP_ITERS, 2)

    # ---- map
    def map_set_resolution(self, line_res: float, plane_res: float):
        self._chk(self.L.so_map_set_resolution(self.h, line_res, plane_res), "so_map_set_resolution")

    def map_set_points(self, xyzi: np.ndarray):
        a = np.ascontiguousarray(xyzi, dtype=np.float32)
        assert a.ndim == 2 and a.shape[1] >= 3
        stride = a.shape[1] * 4
        ioff = 12 if a.shape[1] >= 4 else stride
        self._chk(self.L.so_map_set_points(self.h, _p(a), a.shape[0], stride, ioff), "so_map_set_points")

    def map_set_edge_points(self, xyzi: np.ndarray):
        a = np.ascontiguousarray(xyzi, dtype=np.float32)
        stride = a.shape[1] * 4
        self._chk(self.L.so_map_set_edge_points(self.h, _p(a), a.shape[0], stride, 12 if a.shape[1] >= 4 else stride), "so_map_set_edge_points")

    def map_add_edge(self, xyzi: np.ndarray):
        a = np.ascontiguousarray(xyzi, dtype=np.float32)
        stride = a.shape[1] * 4
        self._chk(self.L.so_map_add_edge(self.h, _p(a), a.shape[0], stride, 12 if a.shape[1] >= 4 else stride), "so_map_add_edge")

    def map_add_scan_edge(self, scan_xyzi: np.ndarray, pose7):
        a = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        stride = a.shape[1] * 4
        self._chk(self.L.so_map_add_scan_edge(self.h, _p(a), a.shape[0], stride, 12 if a.shape[1] >= 4 else stride, _p(pose)), "so_map_add_scan_edge")

    def map_add_surf(self, xyzi: np.ndarray):
        a = np.ascontiguousarray(xyzi, dtype=np.float32)
        stride = a.shape[1] * 4
        self._chk(self.L.so_map_add_surf(self.h, _p(a), a.shape[0], stride, 12 if a.shape[1] >= 4 else stride), "so_map_add_surf")

    def map_add_scan(self, scan_xyzi: np.ndarray, pose7):
        a = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        stride = a.shape[1] * 4
        self._chk(self.L.so_map_add_scan(self.h, _p(a), a.shape[0], stride, 12 if a.shape[1] >= 4 else stride, _p(pose)), "so_map_add_scan")

    def map_add_registered_scan(self, pose7):
        """Insert the surf scan last passed to register() (still on the device) at pose7."""
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        self._chk(self.L.so_map_add_registered_scan(self.h, _p(pose)), "so_map_add_registered_scan")

    def map_add_registered_edges(self, pose7):
        """Insert the edge cloud last passed to register() / register_undistort_edges() (still on the device) at pose7."""
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        self._chk(self.L.so_map_add_registered_edges(self.h, _p(pose)), "so_map_add_registered_edges")

    def map_set_origin(self, t):
        t = np.ascontiguousarray(t, dtype=np.float64)
        o = np.zeros(3, np.int32)
        self._chk(self.L.so_map_set_origin(self.h, _p(t), _p(o)), "so_map_set_origin")
        return o

    def map_origin(self):
        o = np.zeros(3, np.int32)
        self._chk(self.L.so_map_get_origin(self.h, _p(o)), "so_map_get_origin")
        return o

    def map_shift(self, t):
        t = np.ascontiguousarray(t, dtype=np.float64)
        o = np.zeros(3, np.int32)
        self._chk(self.L.so_map_shift(self.h, _p(t), _p(o)), "so_map_shift")
        return o

    def map_counts_5x5(self, ijk, with_edge: bool = False):
        ijk = np.ascontiguousarray(ijk, dtype=np.int32)
        ne, ns = C.c_int32(), C.c_int32()
        self._chk(self.L.so_map_counts_5x5(self.h, _p(ijk), C.byref(ne), C.byref(ns)), "so_map_counts_5x5")
        return (ne.value, ns.value) if with_edge else ns.value

    def map_size(self) -> int:
        return int(self.L.so_map_size(self.h))

    def map_download(self, mode: int = 0, ijk=None) -> np.ndarray:
        n = C.c_size_t()
        cap = self.map_size()
        out = np.zeros((max(cap, 1), 4), np.float32)
        ij = np.ascontiguousarray(ijk if ijk is not None else [0, 0, 0], dtype=np.int32)
        self._chk(self.L.so_map_download(self.h, mode, _p(ij), _p(out), cap, C.byref(n)), "so_map_download")
        if n.value > cap:                  # a pending origin change restored archived blocks: the window grew in this call
            cap = n.value
            out = np.zeros((cap, 4), np.float32)
            self._chk(self.L.so_map_download(self.h, mode, _p(ij), _p(out), cap, C.byref(n)), "so_map_download")
        return out[: n.value]

    # ---- block archive (the map beyond the 21 x 21 x 11 window; off by default)
    def map_archive(self, cap_points: int):
        """Turn the block archive on with room for cap_points points per store, resize it (contents kept), or 0: off and freed."""
        self._chk(self.L.so_map_archive(self.h, int(cap_points)), "so_map_archive")

    def map_archive_info(self, store: int = 0):
        """-> (points, blocks, capacity) of the archive of store 0 (surf) or 1 (edge)."""
        p, b, c = C.c_size_t(), C.c_size_t(), C.c_size_t()
        self._chk(self.L.so_map_archive_info(self.h, store, C.byref(p), C.byref(b), C.byref(c)), "so_map_archive_info")
        return p.value, b.value, c.value

    def map_download_all(self, store: int = 0) -> np.ndarray:
        """Window plus archive of store 0 (surf) or 1 (edge), ordered by world block (z, y, x), then by the order within the block."""
        n = C.c_size_t()
        cap = self.map_size() + self.map_archive_info(store)[0]       # the whole map, unless a pending origin change drops points
        out = np.zeros((max(cap, 1), 4), np.float32)
        self._chk(self.L.so_map_download_all(self.h, store, _p(out), cap, C.byref(n)), "so_map_download_all")
        if n.value > cap:
            cap = n.value
            out = np.zeros((cap, 4), np.float32)
            self._chk(self.L.so_map_download_all(self.h, store, _p(out), cap, C.byref(n)), "so_map_download_all")
        return out[: n.value]

    # ---- keyframes (off until keyframe_reserve): registered scans kept on the device, the map rebuilt from them
    def keyframe_reserve(self, cap_points: int, cap_frames: int):
        """Room for cap_points points in each of the surf and edge pools and for cap_frames keyframes; 0, 0 frees the store."""
        self._chk(self.L.so_keyframe_reserve(self.h, int(cap_points), int(cap_frames)), "so_keyframe_reserve")

    def keyframe_add_registered(self, pose7) -> int:
        """Keep the scan (and edge cloud) of the last single-scan register*() as a keyframe at pose7 -> its id."""
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        i = C.c_int32()
        self._chk(self.L.so_keyframe_add_registered(self.h, _p(pose), C.byref(i)), "so_keyframe_add_registered")
        return i.value

    def keyframe_import(self, surf_xyzi: np.ndarray, pose7, edge_xyzi: np.ndarray | None = None) -> int:
        """Append a keyframe from sensor-frame, already compensated clouds [n, 4] (x, y, z, intensity) at pose7 -> its id.  The clouds
        are kept verbatim: keyframe_download(id, store) returns them bit for bit."""
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        a = np.ascontiguousarray(surf_xyzi, dtype=np.float32).reshape(-1, 4)
        e = np.ascontiguousarray(edge_xyzi if edge_xyzi is not None else np.zeros((0, 4)), dtype=np.float32).reshape(-1, 4)
        i = C.c_int32()
        self._chk(self.L.so_keyframe_import(self.h, _p(a) if len(a) else None, len(a), _p(e) if len(e) else None, len(e), 16, 12, _p(pose),
                                            C.byref(i)), "so_keyframe_import")
        return i.value

    def keyframe_info(self):
        """-> (keyframes, surf pool points, edge pool points)"""
        f, p, e = C.c_size_t(), C.c_size_t(), C.c_size_t()
        self._chk(self.L.so_keyframe_info(self.h, C.byref(f), C.byref(p), C.byref(e)), "so_keyframe_info")
        return f.value, p.value, e.value

    def keyframe_poses(self) -> np.ndarray:
        n = C.c_size_t()
        self._chk(self.L.so_keyframe_poses(self.h, None, 0, C.byref(n)), "so_keyframe_poses")
        out = np.zeros((n.value, 7), np.float64)
        if n.value:
            self._chk(self.L.so_keyframe_poses(self.h, _p(out), n.value, C.byref(n)), "so_keyframe_poses")
        return out

    def keyframe_download(self, kf_id: int, store: int = 0, pose7=None) -> np.ndarray:
        """Keyframe kf_id of store 0 (surf) or 1 (edge): sensor frame, or at pose7 as the rebuild transforms it."""
        pose = np.ascontiguousarray(pose7, dtype=np.float64) if pose7 is not None else None
        n = C.c_size_t()
        self._chk(self.L.so_keyframe_download(self.h, int(kf_id), int(store), _p(pose) if pose is not None else None, None, 0, C.byref(n)),
                  "so_keyframe_download")
        out = np.zeros((max(n.value, 1), 4), np.float32)
        self._chk(self.L.so_keyframe_download(self.h, int(kf_id), int(store), _p(pose) if pose is not None else None, _p(out), n.value,
                                              C.byref(n)), "so_keyframe_download")
        return out[: n.value]

    def map_from_keyframes(self, src: "Context", ids, poses, stores: int = 3):
        """Replace the selected stores (1 surf, 2 edge, 3 both) with the map of src's keyframes ids at poses [n, 7]."""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        poses = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
        assert len(ids) == len(poses)
        self._chk(self.L.so_map_from_keyframes(self.h, src.h, _p(ids), len(ids), _p(poses), int(stores)), "so_map_from_keyframes")

    def register_keyframes(self, src: "Context", ids, priors, max_icp_iters: int, max_surface_features: int = 0, **kw):
        """src's keyframes ids registered against this context's map from priors [n, 7] -> [IcpResult]"""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        priors = np.ascontiguousarray(priors, dtype=np.float64).reshape(-1, 7)
        assert len(ids) == len(priors)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        res = (IcpResult * len(ids))()
        self._chk(self.L.so_register_keyframes(self.h, src.h, _p(ids), len(ids), _p(priors), C.byref(o), res), "so_register_keyframes")
        return list(res)

    def register_keyframes_degeneracy(self, src: "Context", ids, priors, ds, max_icp_iters: int, max_surface_features: int = 0, **kw):
        """register_keyframes with the degeneracy-aware solve; ds: one Degeneracy per keyframe, or one for all -> [DegeneracyResult]"""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        priors = np.ascontiguousarray(priors, dtype=np.float64).reshape(-1, 7)
        assert len(ids) == len(priors)
        ds = [ds] * len(ids) if isinstance(ds, Degeneracy) else list(ds)
        assert len(ds) == len(ids)
        da = (Degeneracy * max(len(ids), 1))(*ds)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        res = (DegeneracyResult * max(len(ids), 1))()
        self._chk(self.L.so_register_keyframes_degeneracy(self.h, src.h, _p(ids), len(ids), _p(priors), da, C.byref(o), res),
                  "so_register_keyframes_degeneracy")
        return list(res)[: len(ids)]

    # ---- loop detection over the keyframes (Scan Context; descriptors cached per keyframe, computed by these calls)
    def loop_candidates(self, queries, k: int, opts: LoopOpts | None = None, stats: bool = False, ids=None, **kw):
        """For each query keyframe its k best eligible keyframes -> structured array [n, k] of LOOP_CANDIDATE_DTYPE (distance
        ascending, then id; id -1 in unused slots); with stats=True also {n_described, time_describe_ms, time_search_ms}.  kw: fields
        of so_loop_opts over the defaults.  ids=(begin, end): the eligible keyframes are those of [begin, end) but the query
        (so_loop_candidates_range; exclude_recent is not used), else those below query - exclude_recent."""
        q = np.ascontiguousarray(np.atleast_1d(queries), dtype=np.int32)
        o = opts if opts is not None else loop_opts(**kw)
        out = np.zeros((len(q), max(int(k), 1)), LOOP_CANDIDATE_DTYPE)
        st = LoopStats()
        if ids is None:
            self._chk(self.L.so_loop_candidates(self.h, _p(q), len(q), C.byref(o), int(k), _p(out), C.byref(st)), "so_loop_candidates")
        else:
            b, e = (int(v) for v in ids)
            self._chk(self.L.so_loop_candidates_range(self.h, _p(q), len(q), C.byref(o), b, e, int(k), _p(out), C.byref(st)),
                      "so_loop_candidates_range")
        if stats:
            return out, dict(n_described=st.n_described, time_describe_ms=st.time_describe_ms, time_search_ms=st.time_search_ms)
        return out

    def keyframe_descriptors(self, ids, opts: LoopOpts | None = None, **kw) -> np.ndarray:
        """The Scan Context images of keyframes ids as the search sees them -> float32 [n, rings, sectors]."""
        i = np.ascontiguousarray(np.atleast_1d(ids), dtype=np.int32)
        o = opts if opts is not None else loop_opts(**kw)
        out = np.zeros((len(i), max(o.rings, 1), max(o.sectors, 1)), np.float32)
        self._chk(self.L.so_keyframe_descriptors(self.h, _p(i), len(i), C.byref(o), _p(out)), "so_keyframe_descriptors")
        return out

    # ---- loop verification (so_loop_verify)
    def loop_prior(self, cand) -> np.ndarray:
        """so_loop_prior of a candidate (a LOOP_CANDIDATE_DTYPE row) from this context's current keyframe poses."""
        poses = self.keyframe_poses()
        return loop_prior(poses[int(cand["id"])], poses[int(cand["query"])], float(cand["yaw"]))

    def loop_verify(self, scratch: "Context", candidates, opts: LoopVerifyOpts | None = None, **kw) -> list:
        """Verify loop candidates (LOOP_CANDIDATE_DTYPE, any shape; as loop_candidates returns them) of this context's keyframes
        through the scratch context, whose map is overwritten -> [LoopVerifyResult] in the candidates' order.  kw: see
        loop_verify_opts."""
        c = np.ascontiguousarray(np.asarray(candidates, LOOP_CANDIDATE_DTYPE).reshape(-1))
        o = opts if opts is not None else loop_verify_opts(**kw)
        res = (LoopVerifyResult * max(len(c), 1))()
        self._chk(self.L.so_loop_verify(self.h, scratch.h, _p(c) if len(c) else None, len(c), C.byref(o), res), "so_loop_verify")
        return list(res)[: len(c)]

    def loop_verify_degeneracy(self, scratch: "Context", candidates, d: Degeneracy, opts: LoopVerifyOpts | None = None, **kw):
        """loop_verify with the degeneracy-aware alignment (so_loop_verify_degeneracy; d: a Degeneracy, see degeneracy()) ->
        ([LoopVerifyResult], [DegeneracyResult]); loop_edge_information(r.reg.pose, deg, S) gives the edge's square-root information."""
        c = np.ascontiguousarray(np.asarray(candidates, LOOP_CANDIDATE_DTYPE).reshape(-1))
        o = opts if opts is not None else loop_verify_opts(**kw)
        res = (LoopVerifyResult * max(len(c), 1))()
        deg = (DegeneracyResult * max(len(c), 1))()
        self._chk(self.L.so_loop_verify_degeneracy(self.h, scratch.h, _p(c) if len(c) else None, len(c), C.byref(o), C.byref(d), res, deg),
                  "so_loop_verify_degeneracy")
        return list(res)[: len(c)], list(deg)[: len(c)]

    # ---- pose graph (so_pose_graph_solve)
    def pose_graph_solve(self, init, edges, fixed: int = 0, max_iterations: int = 50, weights: bool = False, constant=None):
        """The keyframe pose graph from init [n, 7] -> (poses [n, 7], result dict) and, with weights=True, each edge's final rho'.
        edges: see pose_edges().  constant: a mask of n nodes held constant (so_pose_graph_solve_constant), in place of `fixed`."""
        x = np.ascontiguousarray(init, dtype=np.float64).reshape(-1, 7)
        e = pose_edges(edges)
        out = np.zeros_like(x)
        w = np.zeros(max(len(e), 1), np.float64) if weights else None
        o = PoseGraphOpts(int(fixed), int(max_iterations))
        r = PoseGraphResult()
        if constant is None:
            self._chk(self.L.so_pose_graph_solve(self.h, _p(x), len(x), _p(e) if len(e) else None, len(e), C.byref(o), _p(out),
                                                 _p(w) if w is not None else None, C.byref(r)), "so_pose_graph_solve")
        else:
            m = np.ascontiguousarray(constant, dtype=np.uint8)
            if m.shape != (len(x),):
                raise ValueError(f"constant: a mask of {len(x)} nodes, got shape {m.shape}")
            self._chk(self.L.so_pose_graph_solve_constant(self.h, _p(x), len(x), _p(e) if len(e) else None, len(e), _p(m), C.byref(o),
                                                          _p(out), _p(w) if w is not None else None, C.byref(r)),
                      "so_pose_graph_solve_constant")
        res = {k: getattr(r, k) for k, _ in PoseGraphResult._fields_}
        return (out, res, w[:len(e)]) if weights else (out, res)

    # ---- free-space clearing (off unless called)
    @staticmethod
    def _free_result(r: FreeSpaceResult) -> dict:
        return dict(n_image_points=r.n_image_points, n_pixels_hit=r.n_pixels_hit, n_candidates=r.n_candidates, n_removed=r.n_removed,
                    n_after=(r.n_after[0], r.n_after[1]))

    def map_clear_free_space(self, scan_xyzi: np.ndarray, pose7, opts: FreeSpace | None = None, stores: int = 1) -> dict:
        """Remove the window map points that the sensor-frame scan (at pose7) saw clearly past; stores: 1 surf, 2 edge, 3 both."""
        a = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = opts if opts is not None else free_space()
        r = FreeSpaceResult()
        stride = a.shape[1] * 4
        self._chk(self.L.so_map_clear_free_space(self.h, int(stores), _p(a), a.shape[0], stride, 12 if a.shape[1] >= 4 else stride, _p(pose),
                                                 C.byref(o), C.byref(r)), "so_map_clear_free_space")
        return self._free_result(r)

    def map_clear_free_space_registered(self, pose7, opts: FreeSpace | None = None, stores: int = 1) -> dict:
        """The same against the scan last passed to a single-scan register*(), as map_add_registered_scan(pose7) would insert it."""
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = opts if opts is not None else free_space()
        r = FreeSpaceResult()
        self._chk(self.L.so_map_clear_free_space_registered(self.h, int(stores), _p(pose), C.byref(o), C.byref(r)),
                  "so_map_clear_free_space_registered")
        return self._free_result(r)

    def map_clear_free_space_keyframes(self, src: "Context", ids, poses, opts: FreeSpace | None = None, stores: int = 1) -> dict:
        """Clear this context's map against the surf clouds of src's keyframes ids at poses [n, 7], all at once: the map each
        map_clear_free_space of a keyframe in turn leaves (src may be this context, e.g. after map_from_keyframes)."""
        ids = np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)
        poses = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
        if len(ids) != len(poses):
            raise ValueError(f"map_clear_free_space_keyframes: {len(ids)} ids but {len(poses)} poses")
        o = opts if opts is not None else free_space()
        r = FreeSpaceKeyframesResult()
        self._chk(self.L.so_map_clear_free_space_keyframes(self.h, src.h, _p(ids) if len(ids) else None, len(ids),
                                                           _p(poses) if len(ids) else None, int(stores), C.byref(o), C.byref(r)),
                  "so_map_clear_free_space_keyframes")
        return dict(n_keyframes=r.n_keyframes, n_image_points=r.n_image_points, n_pixels_hit=r.n_pixels_hit, n_candidates=r.n_candidates,
                    n_removed=r.n_removed, n_after=(r.n_after[0], r.n_after[1]), n_tiles=r.n_tiles, time_ms=r.time_ms)

    # ---- scan pre-filter
    def scan_prefilter(self, scan_xyzi: np.ndarray, line_res: float, plane_res: float, auto_voxel_size: bool = True, download: bool = True):
        """-> (filtered float32 [m,4], line_res, plane_res, average_distance); download=False leaves the filtered cloud on the device
        (for register_prefiltered) and returns its point count in place of the array."""
        a = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        lr, pr = C.c_float(line_res), C.c_float(plane_res)
        out = np.empty((max(len(a), 1), 4), np.float32) if download else None
        n = C.c_size_t()
        avg = C.c_double(0.0)
        stride = a.shape[1] * 4
        self._chk(self.L.so_scan_prefilter(self.h, _p(a), a.shape[0], stride, 12 if a.shape[1] >= 4 else stride, int(auto_voxel_size),
                                           C.byref(lr), C.byref(pr), _p(out) if download else None, len(out) if download else 0, C.byref(n), C.byref(avg)),
                  "so_scan_prefilter")
        return (out[: n.value] if download else int(n.value)), lr.value, pr.value, avg.value

    def scan_deskew(self, points: np.ndarray, time_col: int, lidar_start_time: float, sample_times, sample_poses, imu_only: bool = False, T_i_l=None):
        """points: float32 [n, C] with x,y,z first and the per-point time in column time_col; rewritten IN PLACE.
        -> (start_pose7, n_past_end)"""
        assert points.dtype == np.float32 and points.flags.c_contiguous and points.ndim == 2
        st = np.ascontiguousarray(sample_times, np.float64)
        sp = np.ascontiguousarray(sample_poses, np.float64).reshape(-1, 7)
        til = np.ascontiguousarray(T_i_l if T_i_l is not None else [0, 0, 0, 0, 0, 0, 1], np.float64)
        out = np.zeros(7, np.float64)
        past = C.c_size_t(0)
        self._chk(self.L.so_scan_deskew(self.h, _p(points), points.shape[0], points.shape[1] * 4, time_col * 4, float(lidar_start_time), _p(st), _p(sp),
                                        len(st), int(imu_only), _p(til), _p(out), C.byref(past)), "so_scan_deskew")
        return out, past.value

    def scan_extract_uniform(self, points: np.ndarray, time_col: int, skip_num: int, block_range: float, int_abs: bool = False):
        """-> float32 [m, 4] {x, y, z, intensity = time} (featureExtraction::uniformFeatureExtraction)"""
        a = np.ascontiguousarray(points, dtype=np.float32)
        out = np.zeros((max(len(a), 1), 4), np.float32)
        n = C.c_size_t()
        self._chk(self.L.so_scan_extract_uniform(self.h, _p(a), a.shape[0], a.shape[1] * 4, time_col * 4, int(skip_num), float(block_range), int(int_abs),
                                                 _p(out), len(out), C.byref(n)), "so_scan_extract_uniform")
        return out[: n.value]

    def scan_extract_edges(self, records: np.ndarray, time_offset: int = 20, ring_offset: int = 24, min_range: float = 0.0,
                           edge_threshold: float = 0.0, voxel_leaf: float = 0.0, max_per_sector: int = 0) -> np.ndarray:
        """LOAM edge features of a raw scan -> float32 [m, 4] {x, y, z, intensity = time}, ordered by (ring, position), or by voxel
        with voxel_leaf > 0.  records: one row per point (point_os::PointcloudXYZITR: float32 [n, 8], time at byte 20, uint16 ring
        at byte 24); zero options take the defaults of so_edge_opts."""
        a = np.ascontiguousarray(records)
        n = a.shape[0] if a.ndim else 0
        stride = a.nbytes // n if n else max(a.itemsize * (a.shape[1] if a.ndim == 2 else 1), 1)
        o = EdgeOpts(float(min_range), float(edge_threshold), float(voxel_leaf), int(max_per_sector))
        out = np.zeros((max(n, 1), 4), np.float32)
        m = C.c_size_t()
        self._chk(self.L.so_scan_extract_edges(self.h, _p(a), n, stride, int(time_offset), int(ring_offset), C.byref(o), _p(out), len(out),
                                               C.byref(m)), "so_scan_extract_edges")
        return out[: m.value]

    # ---- registration
    @staticmethod
    def _opts(max_icp_iters, max_surface_features=0, lm_max_iterations=4, yaw_ratio=0.0, skip_map_checks=False, pose_prior=None):
        """pose_prior = (visual_confidence_factor, (ux, uy, uz)) enables the SE3AbsolutatePoseFactor rows."""
        o = IcpOpts(max_icp_iters, max_surface_features, lm_max_iterations, yaw_ratio, int(skip_map_checks), 0, 0.0, (C.c_float * 3)(0, 0, 0))
        if pose_prior is not None:
            o.use_pose_prior = 1
            o.visual_confidence_factor = float(pose_prior[0])
            o.prior_uncertainty = (C.c_float * 3)(*[float(v) for v in pose_prior[1]])
        return o

    def register(self, scan_xyzi: np.ndarray, pose7, max_icp_iters: int, max_surface_features: int = 0, edge_xyzi=None, **kw) -> IcpResult:
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        r = IcpResult()
        stride = s.shape[1] * 4
        e, ne = None, 0
        if edge_xyzi is not None and len(edge_xyzi):
            ea = np.ascontiguousarray(edge_xyzi, dtype=np.float32)
            assert ea.shape[1] == s.shape[1]
            e, ne = _p(ea), ea.shape[0]
        self._chk(self.L.so_register(self.h, _p(s), s.shape[0], e, ne, stride, 12 if s.shape[1] >= 4 else stride,
                                     _p(pose), C.byref(o), C.byref(r)), "so_register")
        return r

    def set_pose_sink(self, d_rows_ptr: int | None, cap_rows: int = 0, first_row: int = 0):
        """Device buffer [cap_rows, 8] float64 that every following registration call appends {pose_opt[7], status + 256 n_iter} rows to."""
        self._chk(self.L.so_set_pose_sink(self.h, C.c_void_p(d_rows_ptr or 0), cap_rows, first_row), "so_set_pose_sink")

    def register_injected(self, scan_xyzi: np.ndarray, pose7, max_icp_iters: int, nn_ids: np.ndarray, max_surface_features: int = 0, **kw) -> IcpResult:
        """so_register with caller-supplied neighbour sets: nn_ids [iters, n, 5] (int64 with -1 = none, or uint32 with 0xFFFFFFFF)."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        ids = np.asarray(nn_ids)
        assert ids.ndim == 3 and ids.shape[1:] == (s.shape[0], 5)
        if ids.dtype != np.uint32:
            ids = np.where(ids < 0, 0xFFFFFFFF, ids).astype(np.uint32)
        ids = np.ascontiguousarray(ids)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        r = IcpResult()
        stride = s.shape[1] * 4
        self._chk(self.L.so_register_injected(self.h, _p(s), s.shape[0], stride, 12 if s.shape[1] >= 4 else stride, _p(pose), C.byref(o),
                                              _p(ids), ids.shape[0], C.byref(r)), "so_register_injected")
        return r

    def correspond_edge(self, edge_xyzi: np.ndarray, pose7):
        e = np.ascontiguousarray(edge_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        corr = np.zeros(e.shape[0], EDGE_CORR_DTYPE)
        hr = np.zeros(7, np.int32)
        stride = e.shape[1] * 4
        self._chk(self.L.so_correspond_edge(self.h, _p(e), e.shape[0], stride, 12 if e.shape[1] >= 4 else stride, _p(pose), _p(corr), _p(hr)),
                  "so_correspond_edge")
        return corr, hr

    def register_prefiltered(self, pose7, max_icp_iters: int, max_surface_features: int = 0, **kw) -> IcpResult:
        """so_register of the cloud the last scan_prefilter call left on the device."""
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        res = IcpResult()
        rc = self.L.so_register_prefiltered(self.h, _p(pose), C.byref(o), C.byref(res))
        if rc < 0:
            self._chk(rc, "so_register_prefiltered")
        return res

    # ---- within-scan motion compensation (u: an Undistort, see undistort()); time_col: the column holding each point's time
    def register_undistort(self, scan_xyzi: np.ndarray, pose7, u: Undistort, max_icp_iters: int, max_surface_features: int = 0,
                           time_col: int = 3, **kw) -> IcpResult:
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        r = IcpResult()
        stride = s.shape[1] * 4
        rc = self.L.so_register_undistort(self.h, _p(s), s.shape[0], stride, 12 if s.shape[1] >= 4 else stride, time_col * 4, _p(pose),
                                          C.byref(u), C.byref(o), C.byref(r))
        self._chk(rc, "so_register_undistort")
        return r

    def register_undistort_edges(self, scan_xyzi: np.ndarray, edge_xyzi, pose7, u: Undistort, max_icp_iters: int,
                                 max_surface_features: int = 0, time_col: int = 3, **kw) -> IcpResult:
        """register_undistort with an edge cloud (same columns as the scan, its time in the same column) for the line branch."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        r = IcpResult()
        stride = s.shape[1] * 4
        e, ne = None, 0
        if edge_xyzi is not None and len(edge_xyzi):
            ea = np.ascontiguousarray(edge_xyzi, dtype=np.float32)
            assert ea.shape[1] == s.shape[1]
            e, ne = _p(ea), ea.shape[0]
        rc = self.L.so_register_undistort_edges(self.h, _p(s), s.shape[0], e, ne, stride, 12 if s.shape[1] >= 4 else stride, time_col * 4,
                                                _p(pose), C.byref(u), C.byref(o), C.byref(r))
        self._chk(rc, "so_register_undistort_edges")
        return r

    def register_prefiltered_undistort(self, pose7, u: Undistort, max_icp_iters: int, max_surface_features: int = 0, **kw) -> IcpResult:
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        r = IcpResult()
        self._chk(self.L.so_register_prefiltered_undistort(self.h, _p(pose), C.byref(u), C.byref(o), C.byref(r)), "so_register_prefiltered_undistort")
        return r

    def register_batch_undistort(self, scans_xyzi: np.ndarray, n_points, poses, us, max_icp_iters: int, max_surface_features: int = 0,
                                 time_col: int = 3, **kw):
        """us: one Undistort per scan."""
        n_points = np.ascontiguousarray(n_points, dtype=np.uint32)
        poses = np.ascontiguousarray(poses, dtype=np.float64)
        ns = len(n_points)
        ua = (Undistort * ns)(*us)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        res = (IcpResult * ns)()
        a = np.ascontiguousarray(scans_xyzi, dtype=np.float32)
        stride = a.shape[1] * 4
        self._chk(self.L.so_register_batch_undistort(self.h, _p(a), _p(n_points), ns, stride, 12, time_col * 4, _p(poses), ua, C.byref(o), res),
                  "so_register_batch_undistort")
        return res

    def undistort_points(self, xyzi: np.ndarray, pose7, u: Undistort, time_col: int = 3) -> np.ndarray:
        """pInit of every point at T_cur = pose7 -> float32 [n, 4] {x, y, z, intensity}."""
        a = np.ascontiguousarray(xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        out = np.zeros((max(len(a), 1), 4), np.float32)
        stride = a.shape[1] * 4
        self._chk(self.L.so_undistort_points(self.h, _p(a), a.shape[0], stride, 12 if a.shape[1] >= 4 else stride, time_col * 4, _p(pose),
                                             C.byref(u), _p(out)), "so_undistort_points")
        return out[: len(a)]

    # ---- within-scan motion estimated by the registration (m: a Motion, see motion()); time_col: the column holding each point's time
    def register_optimized(self, scan_xyzi: np.ndarray, pose7, m: Motion, max_icp_iters: int, max_surface_features: int = 0,
                           time_col: int = 3, **kw) -> MotionResult:
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        r = MotionResult()
        stride = s.shape[1] * 4
        rc = self.L.so_register_optimized(self.h, _p(s), s.shape[0], stride, 12 if s.shape[1] >= 4 else stride, time_col * 4, _p(pose),
                                          C.byref(m), C.byref(o), C.byref(r))
        self._chk(rc, "so_register_optimized")
        return r

    def register_prefiltered_optimized(self, pose7, m: Motion, max_icp_iters: int, max_surface_features: int = 0, **kw) -> MotionResult:
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        r = MotionResult()
        self._chk(self.L.so_register_prefiltered_optimized(self.h, _p(pose), C.byref(m), C.byref(o), C.byref(r)), "so_register_prefiltered_optimized")
        return r

    def register_batch_optimized(self, scans_xyzi: np.ndarray, n_points, poses, ms, max_icp_iters: int, max_surface_features: int = 0,
                                 time_col: int = 3, **kw):
        """ms: one Motion per scan."""
        n_points = np.ascontiguousarray(n_points, dtype=np.uint32)
        poses = np.ascontiguousarray(poses, dtype=np.float64)
        ns = len(n_points)
        ma = (Motion * ns)(*ms)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        res = (MotionResult * ns)()
        a = np.ascontiguousarray(scans_xyzi, dtype=np.float32)
        stride = a.shape[1] * 4
        self._chk(self.L.so_register_batch_optimized(self.h, _p(a), _p(n_points), ns, stride, 12, time_col * 4, _p(poses), ma, C.byref(o), res),
                  "so_register_batch_optimized")
        return res

    def evaluate_optimized(self, xyzi: np.ndarray, pose7, motion7, dt: float, max_surface_features: int = 0, time_col: int = 3):
        """Plane rows' (H [12, 12], g [12], cost) at (T = pose7, D = motion7) over the correspondences at T of float(u(D))."""
        a = np.ascontiguousarray(xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        mot = np.ascontiguousarray(motion7, dtype=np.float64)
        H = np.zeros((12, 12))
        g = np.zeros(12)
        cost = C.c_double()
        stride = a.shape[1] * 4
        self._chk(self.L.so_evaluate_optimized(self.h, _p(a), a.shape[0], stride, 12 if a.shape[1] >= 4 else stride, time_col * 4, _p(pose),
                                               _p(mot), float(dt), int(max_surface_features), _p(H), _p(g), C.byref(cost)),
                  "so_evaluate_optimized")
        return H, g, cost.value

    def register_optimized_edges(self, scan_xyzi: np.ndarray, edge_xyzi, pose7, m: Motion, max_icp_iters: int, max_surface_features: int = 0,
                                 time_col: int = 3, **kw) -> MotionResult:
        """register_optimized with an edge cloud (same columns as the scan, its time in the same column) for the line branch."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        r = MotionResult()
        stride = s.shape[1] * 4
        e, ne = self._edge_arg(edge_xyzi, s)
        rc = self.L.so_register_optimized_edges(self.h, _p(s), s.shape[0], e, ne, stride, 12 if s.shape[1] >= 4 else stride, time_col * 4,
                                                _p(pose), C.byref(m), C.byref(o), C.byref(r))
        self._chk(rc, "so_register_optimized_edges")
        return r

    def evaluate_optimized_edges(self, xyzi: np.ndarray, edge_xyzi, pose7, motion7, dt: float, max_surface_features: int = 0, time_col: int = 3):
        """evaluate_optimized with the edge cloud's line rows added."""
        a = np.ascontiguousarray(xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        mot = np.ascontiguousarray(motion7, dtype=np.float64)
        H = np.zeros((12, 12))
        g = np.zeros(12)
        cost = C.c_double()
        stride = a.shape[1] * 4
        e, ne = self._edge_arg(edge_xyzi, a)
        self._chk(self.L.so_evaluate_optimized_edges(self.h, _p(a), a.shape[0], e, ne, stride, 12 if a.shape[1] >= 4 else stride, time_col * 4,
                                                     _p(pose), _p(mot), float(dt), int(max_surface_features), _p(H), _p(g), C.byref(cost)),
                  "so_evaluate_optimized_edges")
        return H, g, cost.value

    @staticmethod
    def _edge_arg(edge_xyzi, s):
        """(pointer, count) of an optional edge cloud laid out like s; the array is kept alive by the caller's reference"""
        if edge_xyzi is None or not len(edge_xyzi):
            return None, 0
        assert edge_xyzi.dtype == np.float32 and edge_xyzi.flags.c_contiguous and edge_xyzi.shape[1] == s.shape[1]
        return _p(edge_xyzi), edge_xyzi.shape[0]

    def register_batch(self, scans_xyzi: np.ndarray, n_points, poses, max_icp_iters: int, max_surface_features: int = 0, **kw):
        """scans_xyzi: float32 [sum(n_points), 4] host array (pinned or pageable)."""
        n_points = np.ascontiguousarray(n_points, dtype=np.uint32)
        poses = np.ascontiguousarray(poses, dtype=np.float64)
        ns = len(n_points)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        res = (IcpResult * ns)()
        assert scans_xyzi.dtype == np.float32 and scans_xyzi.flags.c_contiguous
        stride = scans_xyzi.shape[1] * 4
        self._chk(self.L.so_register_batch(self.h, _p(scans_xyzi), _p(n_points), ns, stride, 12, _p(poses), C.byref(o), res),
                  "so_register_batch")
        return res

    def register_batch_edges(self, scans_xyzi: np.ndarray, n_points, edges_xyzi: np.ndarray, n_edge, poses, max_icp_iters: int,
                             max_surface_features: int = 0, **kw):
        """register_batch with one edge cloud per scan: edges_xyzi float32 [sum(n_edge), 4], clouds back to back."""
        n_points = np.ascontiguousarray(n_points, dtype=np.uint32)
        n_edge = np.ascontiguousarray(n_edge, dtype=np.uint32)
        poses = np.ascontiguousarray(poses, dtype=np.float64)
        ns = len(n_points)
        assert len(n_edge) == ns
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        res = (IcpResult * ns)()
        scans_xyzi = np.ascontiguousarray(scans_xyzi, dtype=np.float32)
        edges_xyzi = np.ascontiguousarray(edges_xyzi, dtype=np.float32).reshape(-1, 4)
        self._chk(self.L.so_register_batch_edges(self.h, _p(scans_xyzi), _p(n_points), _p(edges_xyzi) if len(edges_xyzi) else None, _p(n_edge), ns,
                                                 16, 12, _p(poses), C.byref(o), res), "so_register_batch_edges")
        return res

    def register_batch_device(self, d_scans_ptr: int, n_points, poses, max_icp_iters: int, max_surface_features: int = 0, **kw):
        n_points = np.ascontiguousarray(n_points, dtype=np.uint32)
        poses = np.ascontiguousarray(poses, dtype=np.float64)
        ns = len(n_points)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        res = (IcpResult * ns)()
        self._chk(self.L.so_register_batch_device(self.h, C.c_void_p(d_scans_ptr), _p(n_points), ns, _p(poses), C.byref(o), res),
                  "so_register_batch_device")
        return res

    def ordered_scans(self, n: int) -> np.ndarray:
        """Test hook: the first n points of the cell-ordered scan buffer the last batch registration left (n x 4 float32;
        column 3 holds the point's index inside its scan as a uint32 bit pattern)."""
        out = np.empty((n, 4), np.float32)
        self._chk(self.L.so_ordered_scans(self.h, _p(out), n), "so_ordered_scans")
        return out

    def correspond(self, scan_xyzi: np.ndarray, pose7, max_surface_features: int = 0, seed_pose=None):
        """Correspondences at pose7 -> (corr, hist_obs, hist_rej).  seed_pose: run them as ICP iteration 1 of a registration that
        started at seed_pose, searching with the bound iteration 0's neighbours give (so_correspond_seeded)."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        corr = np.zeros(s.shape[0], CORR_DTYPE)
        ho = np.zeros(9, np.int32)
        hr = np.zeros(7, np.int32)
        stride = s.shape[1] * 4
        args = (self.h, _p(s), s.shape[0], stride, 12 if s.shape[1] >= 4 else stride, _p(pose), max_surface_features, _p(corr), _p(ho), _p(hr))
        if seed_pose is None:
            self._chk(self.L.so_correspond(*args), "so_correspond")
        else:
            prev = np.ascontiguousarray(seed_pose, dtype=np.float64)
            self._chk(self.L.so_correspond_seeded(*args, _p(prev)), "so_correspond_seeded")
        return corr, ho, hr

    def evaluate(self, pose7):
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        H = np.zeros((6, 6))
        g = np.zeros(6)
        cost = C.c_double()
        self._chk(self.L.so_evaluate(self.h, _p(pose), _p(H), _p(g), C.byref(cost)), "so_evaluate")
        return H, g, cost.value

    def covariance(self, H) -> IcpResult:
        """The covariance step that ends a registration, on a symmetric H [6, 6] or [12, 12]: cov and the error fields of the result."""
        a = np.ascontiguousarray(H, dtype=np.float64)
        assert a.ndim == 2 and a.shape[0] == a.shape[1] and a.shape[0] in (6, 12)
        r = IcpResult()
        self._chk(self.L.so_covariance(self.h, _p(a), a.shape[0], C.byref(r)), "so_covariance")
        return r

    # ---- degeneracy-aware registration (d: a Degeneracy, see degeneracy())
    def register_degeneracy(self, scan_xyzi: np.ndarray, pose7, d: Degeneracy, max_icp_iters: int, max_surface_features: int = 0,
                            edge_xyzi=None, **kw) -> DegeneracyResult:
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        r = DegeneracyResult()
        stride = s.shape[1] * 4
        ea = None if edge_xyzi is None or not len(edge_xyzi) else np.ascontiguousarray(edge_xyzi, dtype=np.float32)
        e, ne = self._edge_arg(ea, s)
        rc = self.L.so_register_degeneracy(self.h, _p(s), s.shape[0], e, ne, stride, 12 if s.shape[1] >= 4 else stride, _p(pose),
                                           C.byref(d), C.byref(o), C.byref(r))
        self._chk(rc, "so_register_degeneracy")
        return r

    def register_batch_degeneracy(self, scans_xyzi: np.ndarray, n_points, poses, ds, max_icp_iters: int, max_surface_features: int = 0,
                                  edges_xyzi=None, n_edge=None, **kw):
        """ds: one Degeneracy per scan; edges_xyzi / n_edge (optional): one edge cloud per scan, back to back."""
        n_points = np.ascontiguousarray(n_points, dtype=np.uint32)
        poses = np.ascontiguousarray(poses, dtype=np.float64)
        ns = len(n_points)
        da = (Degeneracy * ns)(*ds)
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        res = (DegeneracyResult * ns)()
        a = np.ascontiguousarray(scans_xyzi, dtype=np.float32)
        e, ne = None, None
        if n_edge is not None:
            ne = np.ascontiguousarray(n_edge, dtype=np.uint32)
            assert len(ne) == ns
            ea = np.ascontiguousarray(edges_xyzi, dtype=np.float32).reshape(-1, a.shape[1])
            e = _p(ea) if len(ea) else None
        self._chk(self.L.so_register_batch_degeneracy(self.h, _p(a), _p(n_points), e, None if ne is None else _p(ne), ns, a.shape[1] * 4, 12,
                                                      _p(poses), da, C.byref(o), res), "so_register_batch_degeneracy")
        return res

    def degeneracy_analysis(self, H, d: Degeneracy) -> DegeneracyResult:
        """The analysis a degeneracy-aware solve begins with, on a symmetric H [6, 6]: eigenpairs and flags of I_t and I_theta."""
        a = np.ascontiguousarray(H, dtype=np.float64)
        assert a.shape == (6, 6)
        r = DegeneracyResult()
        self._chk(self.L.so_degeneracy_analysis(self.h, _p(a), C.byref(d), C.byref(r)), "so_degeneracy_analysis")
        return r

    def solve(self, rows: np.ndarray, problems: np.ndarray, ds=None) -> np.ndarray:
        """One ICP iteration's solve per problem on given correspondences (so_solve): rows [sum n_rows] of SOLVE_ROW_DTYPE, problem
        b's after problem b - 1's; problems [B] of SOLVE_PROBLEM_DTYPE; ds: None or one Degeneracy per problem.
        -> [B] of SOLVE_RESULT_DTYPE."""
        rows = np.ascontiguousarray(rows, dtype=SOLVE_ROW_DTYPE)
        problems = np.ascontiguousarray(problems, dtype=SOLVE_PROBLEM_DTYPE)
        assert int(problems["n_rows"].sum()) == len(rows)
        out = np.zeros(len(problems), SOLVE_RESULT_DTYPE)
        da = None if ds is None else (Degeneracy * len(problems))(*ds)
        self._chk(self.L.so_solve(self.h, _p(rows) if len(rows) else None, _p(problems), len(problems), da, _p(out)), "so_solve")
        return out

    def solve_optimized(self, rows: np.ndarray, times: np.ndarray, problems: np.ndarray) -> np.ndarray:
        """The two-block solve of so_register_optimized per problem on given correspondences (so_solve_optimized): rows [sum n_rows] of
        SOLVE_ROW_DTYPE and times [sum n_rows] float32, problem b's after problem b - 1's; problems [B] of
        SOLVE_OPTIMIZED_PROBLEM_DTYPE.  -> [B] of SOLVE_OPTIMIZED_RESULT_DTYPE."""
        rows = np.ascontiguousarray(rows, dtype=SOLVE_ROW_DTYPE)
        times = np.ascontiguousarray(times, dtype=np.float32)
        problems = np.ascontiguousarray(problems, dtype=SOLVE_OPTIMIZED_PROBLEM_DTYPE)
        assert int(problems["n_rows"].sum()) == len(rows) == len(times)
        out = np.zeros(len(problems), SOLVE_OPTIMIZED_RESULT_DTYPE)
        self._chk(self.L.so_solve_optimized(self.h, _p(rows) if len(rows) else None, _p(times) if len(times) else None, _p(problems),
                                            len(problems), _p(out)), "so_solve_optimized")
        return out

    # ---- global localization
    def localize_global(self, scan_xyzi: np.ndarray, center_pose7, max_icp_iters: int, opts: GlobalOpts | None = None,
                        max_surface_features: int = 0, **kw):
        """Global localization of a sensor-frame surf cloud around center_pose7 -> (pose [7], GlobalResult, [GlobalCandidate]).
        Soft statuses are in result.status; errors raise."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        c = np.ascontiguousarray(center_pose7, dtype=np.float64)
        g = opts if opts is not None else global_opts()
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        cands = (GlobalCandidate * 64)()
        r = GlobalResult()
        stride = s.shape[1] * 4
        self._chk(self.L.so_localize_global(self.h, _p(s) if len(s) else None, s.shape[0], stride, 12 if s.shape[1] >= 4 else stride, _p(c),
                                            C.byref(g), C.byref(o), cands, 64, C.byref(r)), "so_localize_global")
        return np.array(r.pose), r, [cands[i] for i in range(min(r.n_candidates, 64))]

    def localize_scores(self, scan_xyzi: np.ndarray, center_pose7, opts: GlobalOpts | None = None):
        """Score of every hypothesis -> (uint16 [NYAW, NZ, NY, NX], number of score points)."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        c = np.ascontiguousarray(center_pose7, dtype=np.float64)
        g = opts if opts is not None else global_opts()
        (nx, ny, nz, nyaw), nh, _ = localize_global_size(g)
        scores = np.zeros(max(nh, 1), np.uint16)
        dims = np.zeros(4, np.int32)
        npts = C.c_int32()
        stride = s.shape[1] * 4
        self._chk(self.L.so_localize_scores(self.h, _p(s) if len(s) else None, s.shape[0], stride, 12 if s.shape[1] >= 4 else stride, _p(c),
                                            C.byref(g), _p(scores), nh, _p(dims), C.byref(npts)), "so_localize_scores")
        assert tuple(dims) == (nx, ny, nz, nyaw)
        return scores[:nh].reshape(nyaw, nz, ny, nx), npts.value

    def localize_global_bnb(self, scan_xyzi: np.ndarray, center_pose7, max_icp_iters: int, opts: GlobalOpts | None = None,
                            max_surface_features: int = 0, **kw):
        """so_localize_global by branch-and-bound (same results, up to 2^32 hypotheses) -> (pose [7], GlobalResult,
        [GlobalCandidate], BnbStats)."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        c = np.ascontiguousarray(center_pose7, dtype=np.float64)
        g = opts if opts is not None else global_opts()
        o = self._opts(max_icp_iters, max_surface_features, **kw)
        cands = (GlobalCandidate * 64)()
        r = GlobalResult()
        st = BnbStats()
        stride = s.shape[1] * 4
        self._chk(self.L.so_localize_global_bnb(self.h, _p(s) if len(s) else None, s.shape[0], stride, 12 if s.shape[1] >= 4 else stride,
                                                _p(c), C.byref(g), C.byref(o), cands, 64, C.byref(r), C.byref(st)), "so_localize_global_bnb")
        return np.array(r.pose), r, [cands[i] for i in range(min(r.n_candidates, 64))], st

    def localize_bnb_keys(self, scan_xyzi: np.ndarray, center_pose7, opts: GlobalOpts | None = None):
        """The sorted key prefix the branch-and-bound finds -> (uint64 keys [min(n_hyp, 64 k)], BnbStats)."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        c = np.ascontiguousarray(center_pose7, dtype=np.float64)
        g = opts if opts is not None else global_opts()
        keys = np.zeros(64 * 64, np.uint64)
        n = C.c_size_t()
        st = BnbStats()
        stride = s.shape[1] * 4
        self._chk(self.L.so_localize_bnb_keys(self.h, _p(s) if len(s) else None, s.shape[0], stride, 12 if s.shape[1] >= 4 else stride,
                                              _p(c), C.byref(g), _p(keys), len(keys), C.byref(n), C.byref(st)), "so_localize_bnb_keys")
        return keys[:n.value].copy(), st

    def localize_bnb_bounds(self, scan_xyzi: np.ndarray, center_pose7, level: int, opts: GlobalOpts | None = None):
        """Bound U of every node of pyramid level `level` -> uint16 [NYAW, NZ, ceil(NY / 2^level), ceil(NX / 2^level)]."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        c = np.ascontiguousarray(center_pose7, dtype=np.float64)
        g = opts if opts is not None else global_opts()
        dims = np.zeros(4, np.int32)
        stride = s.shape[1] * 4
        args = (self.h, _p(s) if len(s) else None, s.shape[0], stride, 12 if s.shape[1] >= 4 else stride, _p(c), C.byref(g), level)
        rc = self.L.so_localize_bnb_bounds(*args, None, 0, _p(dims))          # host-only: the level's dims with a capacity error
        if rc != -3:
            self._chk(rc, "so_localize_bnb_bounds")
        nbx, nby, nz, nyaw = (int(v) for v in dims)
        n = nbx * nby * nz * nyaw
        out = np.zeros(max(n, 1), np.uint16)
        self._chk(self.L.so_localize_bnb_bounds(*args, _p(out), n, _p(dims)), "so_localize_bnb_bounds")
        assert tuple(dims) == (nbx, nby, nz, nyaw)
        return out[:n].reshape(nyaw, nz, nby, nbx)

    def map_bounds(self):
        """Bounding box of the surf map, reduced on the device -> (lo float32 [3], hi float32 [3], point count)."""
        lo, hi = np.zeros(3, np.float32), np.zeros(3, np.float32)
        n = C.c_size_t()
        self._chk(self.L.so_map_bounds(self.h, _p(lo), _p(hi), C.byref(n)), "so_map_bounds")
        return lo, hi, n.value

    def map_bounds_all(self):
        """map_bounds over the surf window plus the surf block archive (so_map_bounds_all) -> (lo, hi, point count)."""
        lo, hi = np.zeros(3, np.float32), np.zeros(3, np.float32)
        n = C.c_size_t()
        self._chk(self.L.so_map_bounds_all(self.h, _p(lo), _p(hi), C.byref(n)), "so_map_bounds_all")
        return lo, hi, n.value

    # ---- k-NN
    def knn(self, q_xyz: np.ndarray, k: int = 5, max_d2: float = 0.0):
        q = np.ascontiguousarray(q_xyz, dtype=np.float32)
        nq = q.shape[0]
        idx = np.empty((nq, k), np.uint32)
        d2 = np.empty((nq, k), np.float32)
        self._chk(self.L.so_knn(self.h, _p(q), nq, q.shape[1] * 4, k, C.c_float(max_d2), _p(idx), _p(d2)), "so_knn")
        return idx, d2

    def knn_device(self, d_q_ptr: int, nq: int, k: int, max_d2: float, d_idx_ptr: int, d_d2_ptr: int):
        self._chk(self.L.so_knn_device(self.h, C.c_void_p(d_q_ptr), nq, k, C.c_float(max_d2), C.c_void_p(d_idx_ptr),
                                       C.c_void_p(d_d2_ptr)), "so_knn_device")

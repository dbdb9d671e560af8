"""ctypes binding of the CPU oracle (oracle/so_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package never imports this module.

Prefers oracle/_ref/libso_oracle_ref.so (restatement + the reference's own octree header
compiled verbatim) and falls back to oracle/libso_oracle.so (restatement only).
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
MAX_ICP_ITERS = 32

STATUS_NAMES = ["SUCCESS", "NOT_ENOUGH_NEIGHBORS", "NEIGHBORS_TOO_FAR", "BAD_PCA_STRUCTURE",
                "INVALID_NUMERICAL", "MSE_TOO_LARGE", "UNKNOWN"]


class Opts(C.Structure):
    _fields_ = [("plane_res", C.c_float), ("max_icp_iters", C.c_int32), ("max_surface_features", C.c_int32),
                ("lm_max_iterations", C.c_int32), ("knn_mode", C.c_int32), ("n_threads", C.c_int32),
                ("yaw_ratio", C.c_float), ("skip_map_checks", C.c_int32), ("use_pose_prior", C.c_int32),
                ("visual_confidence_factor", C.c_float), ("prior_uncertainty", C.c_float * 3), ("line_res", C.c_float)]


class Result(C.Structure):
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
                ("pos_in_localmap", C.c_int32 * 3), ("pad_", C.c_int32),
                ("time_ms", C.c_double), ("time_knn_ms", C.c_double)]


CORR_DTYPE = np.dtype([("p", "<f8", 3), ("n", "<f8", 3), ("d", "<f8"), ("w", "<f8"), ("eigval", "<f8", 3),
                       ("mean_dist", "<f8"), ("nn", "<i8", 5), ("nn_d2", "<f4", 5), ("status", "<i4"), ("obs", "<i4", 3)],
                      align=True)


EDGE_CORR_DTYPE = np.dtype([("p", "<f8", 3), ("a", "<f8", 3), ("b", "<f8", 3), ("w", "<f8"), ("nn", "<i8", 10), ("sel", "<i4", 10),
                            ("n_sel", "<i4"), ("status", "<i4")], align=True)


def _source_id() -> str:
    """First 16 hex digits of so_oracle.cpp's SHA-256 (what the Makefile compiles into the library)."""
    with open(os.path.join(_HERE, "so_oracle.cpp"), "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()[:16]


def _built_from_source(path: str) -> bool:
    """path exists and was compiled from the so_oracle.cpp beside this file (file times cannot tell: a checkout or a copy
    sets them)."""
    if not os.path.exists(path):
        return False
    with open(path, "rb") as f:
        return b"so_oracle source id " + _source_id().encode() + b";" in f.read()


def build(force: bool = False) -> None:
    """Compile the oracle (plain lib always; _ref lib when /root/reference exists)."""
    lib = os.path.join(_HERE, "libso_oracle.so")
    sid = "SRC_ID=" + _source_id()
    if force or not _built_from_source(lib):
        subprocess.check_call(["make", "-B", "-C", _HERE, sid, "libso_oracle.so"], stdout=subprocess.DEVNULL)
    ref = os.path.join(_HERE, "_ref", "libso_oracle_ref.so")
    if os.path.isdir("/root/reference") and (force or not _built_from_source(ref)):
        subprocess.check_call(["make", "-C", _HERE, sid, "ref"], stdout=subprocess.DEVNULL)


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    ref = os.path.join(_HERE, "_ref", "libso_oracle_ref.so")
    plain = os.path.join(_HERE, "libso_oracle.so")
    # a _ref library compiled from another version of so_oracle.cpp (it is rebuilt only where the reference tree exists) is not used
    if not _built_from_source(ref) and not _built_from_source(plain):
        build()
    path = ref if _built_from_source(ref) else plain
    assert _built_from_source(path), f"{path} was not compiled from {os.path.join(_HERE, 'so_oracle.cpp')}"
    L = C.CDLL(path)
    L.orc_map_create.restype = C.c_void_p
    L.orc_map_destroy.argtypes = [C.c_void_p]
    L.orc_map_set_points.restype = C.c_int64
    L.orc_map_set_points.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int]
    L.orc_map_shift.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_map_get_origin.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_map_set_origin.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_map_counts_5x5.restype = C.c_int32
    L.orc_map_counts_5x5.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_correspond.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_float, C.c_int, C.c_int, C.c_int,
                                 C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_evaluate.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_solve.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_covariance.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_float, C.c_void_p]
    L.orc_solve_optimized.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                      C.c_double, C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_register.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_set_nn_trace.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    L.orc_register_full.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_map_set_edge_points.restype = C.c_int64
    L.orc_map_set_edge_points.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]
    L.orc_correspond_edge.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_sizeof_edge_corr.restype = C.c_size_t
    L.orc_sym_eig.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_deskew.restype = C.c_int64
    L.orc_deskew.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_double, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_extract_uniform.restype = C.c_int64
    L.orc_extract_uniform.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_size_t]
    L.orc_colpiv_qr_solve.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_pose_plus.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_yaw_round_trip.argtypes = [C.c_void_p, C.c_void_p, C.c_double]
    L.orc_lidar_uncertainty.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_sizeof_corr.restype = C.c_size_t
    L.orc_sizeof_result.restype = C.c_size_t
    assert L.orc_sizeof_corr() == CORR_DTYPE.itemsize, (L.orc_sizeof_corr(), CORR_DTYPE.itemsize)
    assert L.orc_sizeof_result() == C.sizeof(Result), (L.orc_sizeof_result(), C.sizeof(Result))
    assert L.orc_sizeof_edge_corr() == EDGE_CORR_DTYPE.itemsize, (L.orc_sizeof_edge_corr(), EDGE_CORR_DTYPE.itemsize)
    L._path = path
    _lib = L
    return L


def has_ref_octree() -> bool:
    return bool(lib().orc_has_ref_octree())


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class OracleMap:
    """LocalMap stand-in: block grid (21x21x11 of 50 m) + per-block surf cloud + k-NN index."""

    def __init__(self, xyzi: np.ndarray | None = None, ref_octree: bool | None = None):
        self.L = lib()
        self.h = C.c_void_p(self.L.orc_map_create())
        self.xyzi = None
        if xyzi is not None:
            self.set_points(xyzi, ref_octree)

    def __del__(self):
        try:
            if self.h:
                self.L.orc_map_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def set_points(self, xyzi: np.ndarray, ref_octree: bool | None = None) -> int:
        xyzi = np.ascontiguousarray(xyzi, dtype=np.float32)
        self.xyzi = xyzi
        if ref_octree is None:
            ref_octree = has_ref_octree()
        return int(self.L.orc_map_set_points(self.h, _p(xyzi), xyzi.shape[0], xyzi.shape[1], int(ref_octree)))

    def set_origin(self, o):
        """Set LocalMap::origin_ directly (call before set_points: binning uses it)."""
        o = np.ascontiguousarray(o, dtype=np.int32)
        self.L.orc_map_set_origin(self.h, _p(o))

    def set_edge_points(self, xyzi: np.ndarray) -> int:
        xyzi = np.ascontiguousarray(xyzi, dtype=np.float32)
        self.edge_xyzi = xyzi
        return int(self.L.orc_map_set_edge_points(self.h, _p(xyzi), xyzi.shape[0], xyzi.shape[1]))

    def correspond_edge(self, edge_scan_xyzi, pose7, line_res, knn_mode=0):
        s = np.ascontiguousarray(edge_scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        corr = np.zeros(s.shape[0], EDGE_CORR_DTYPE)
        hr = np.zeros(7, np.int32)
        self.L.orc_correspond_edge(self.h, _p(s), s.shape[0], s.shape[1], _p(pose), C.c_float(line_res), knn_mode, _p(corr), _p(hr))
        return corr, hr

    def origin(self):
        o = np.zeros(3, np.int32)
        self.L.orc_map_get_origin(self.h, _p(o))
        return o

    def shift(self, t):
        t = np.ascontiguousarray(t, dtype=np.float64)
        out = np.zeros(3, np.int32)
        self.L.orc_map_shift(self.h, _p(t), _p(out))
        return out

    def counts_5x5(self, ijk) -> int:
        ijk = np.ascontiguousarray(ijk, dtype=np.int32)
        return int(self.L.orc_map_counts_5x5(self.h, _p(ijk)))

    def knn(self, q_xyz: np.ndarray, k: int = 5, mode: int = 0):
        q = np.ascontiguousarray(q_xyz, dtype=np.float32)
        nq = q.shape[0]
        idx = np.empty((nq, k), np.int64)
        d2 = np.empty((nq, k), np.float32)
        found = np.empty(nq, np.uint8)
        rc = self.L.orc_knn(self.h, _p(q), nq, q.shape[1], k, mode, _p(idx), _p(d2), _p(found))
        assert rc == 0
        return idx, d2, found.astype(bool)

    def correspond(self, scan_xyzi, pose7, plane_res, max_surface_features=0, knn_mode=0, n_threads=1):
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        corr = np.zeros(s.shape[0], CORR_DTYPE)
        ho = np.zeros(9, np.int32)
        hr = np.zeros(7, np.int32)
        self.L.orc_correspond(self.h, _p(s), s.shape[0], s.shape[1], _p(pose), C.c_float(plane_res), max_surface_features,
                              knn_mode, n_threads, _p(corr), _p(ho), _p(hr))
        return corr, ho, hr

    def register(self, scan_xyzi, pose7, plane_res, max_icp_iters, max_surface_features=0, knn_mode=0, n_threads=1,
                 lm_max_iterations=4, yaw_ratio=0.0, skip_map_checks=False, pose_prior=None, edge_xyzi=None, line_res=0.1,
                 nn_trace: np.ndarray | None = None) -> Result:
        """pose_prior = (visual_confidence_factor, (ux, uy, uz)) enables the SE3AbsolutatePoseFactor rows.
        nn_trace: optional int64 [iters, n, 5] array that receives the neighbour ids of every ICP iteration (-1 = none)."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = Opts(plane_res, max_icp_iters, max_surface_features, lm_max_iterations, knn_mode, n_threads, yaw_ratio, int(skip_map_checks),
                 0, 0.0, (C.c_float * 3)(0, 0, 0), float(line_res))
        if pose_prior is not None:
            o.use_pose_prior = 1
            o.visual_confidence_factor = float(pose_prior[0])
            o.prior_uncertainty = (C.c_float * 3)(*[float(v) for v in pose_prior[1]])
        r = Result()
        if nn_trace is not None:
            assert nn_trace.dtype == np.int64 and nn_trace.flags.c_contiguous and nn_trace.shape[1:] == (s.shape[0], 5)
            nn_trace[:] = -1
            self.L.orc_set_nn_trace(_p(nn_trace), s.shape[0], nn_trace.shape[0])
        try:
            if edge_xyzi is not None and len(edge_xyzi):
                e = np.ascontiguousarray(edge_xyzi, dtype=np.float32)
                assert e.shape[1] == s.shape[1]
                self.L.orc_register_full(self.h, _p(s), s.shape[0], _p(e), e.shape[0], s.shape[1], _p(pose), C.byref(o), C.byref(r))
            else:
                self.L.orc_register(self.h, _p(s), s.shape[0], s.shape[1], _p(pose), C.byref(o), C.byref(r))
        finally:
            if nn_trace is not None:
                self.L.orc_set_nn_trace(None, 0, 0)
        return r


def evaluate(corr: np.ndarray, pose7, plane_res):
    L = lib()
    pose = np.ascontiguousarray(pose7, dtype=np.float64)
    H = np.zeros((6, 6))
    g = np.zeros(6)
    cost = C.c_double()
    nok = C.c_int64()
    L.orc_evaluate(_p(corr), corr.shape[0], _p(pose), C.c_float(plane_res), _p(H), _p(g), C.byref(cost), C.byref(nok))
    return H, g, cost.value, nok.value


def solve(corr: np.ndarray, pose7, plane_res, lm_max_iterations=4, pose_prior=None):
    """One ceres::Solve on the status-0 rows of corr from pose7.  pose_prior = (measurement pose7, visual_confidence_factor,
    (ux, uy, uz)) adds the SE3AbsolutatePoseFactor rows, their information from the number of those rows."""
    L = lib()
    pose = np.array(pose7, dtype=np.float64)
    summ = np.zeros(4, np.int32)
    costs = np.zeros(5)
    meas, vcf, unc = None, 0.0, None
    if pose_prior is not None:
        meas = np.ascontiguousarray(pose_prior[0], dtype=np.float64)
        vcf, unc = float(pose_prior[1]), np.ascontiguousarray(pose_prior[2], dtype=np.float32)
    L.orc_solve(_p(corr), corr.shape[0], _p(pose), C.c_float(plane_res), lm_max_iterations, None if meas is None else _p(meas),
                C.c_float(vcf), None if unc is None else _p(unc), _p(summ), _p(costs))
    return pose, dict(successful=int(summ[0]), unsuccessful=int(summ[1]), iterations=int(summ[2]), termination=int(summ[3]),
                      initial_cost=costs[0], final_cost=costs[1], radius=costs[2], decrease_factor=costs[3], gmax=costs[4])


def solve_optimized(P, tau, N, D, W, T7, motion7, dt, D0, info, plane_res, lm_max_iterations=4):
    """The two-block solve of so_register_optimized on given plane rows {p, tau, n, d, w} from (T7, motion7): the restatement's
    trust-region loop over 12 columns with the motion prior rows (measurement D0, multiplier sqrt(n * info_k)).
    -> (T, D, summary dict as solve's)."""
    L = lib()
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)         # noqa: E731
    P, N, D, W, D0, info = f64(P), f64(N), f64(D), f64(W), f64(D0), f64(info)
    tau = np.ascontiguousarray(tau, dtype=np.float32)
    T, M = np.array(T7, dtype=np.float64), np.array(motion7, dtype=np.float64)
    summ = np.zeros(4, np.int32)
    costs = np.zeros(5)
    L.orc_solve_optimized(_p(P), _p(tau), _p(N), _p(D), _p(W), len(P), _p(T), _p(M), float(dt), _p(D0), _p(info), C.c_float(plane_res),
                          lm_max_iterations, _p(summ), _p(costs))
    return T, M, dict(successful=int(summ[0]), unsuccessful=int(summ[1]), iterations=int(summ[2]), termination=int(summ[3]),
                      initial_cost=costs[0], final_cost=costs[1], radius=costs[2], decrease_factor=costs[3], gmax=costs[4])


def covariance(corr: np.ndarray, pose7, plane_res):
    L = lib()
    pose = np.ascontiguousarray(pose7, dtype=np.float64)
    cov = np.zeros((6, 6))
    rc = L.orc_covariance(_p(corr), corr.shape[0], _p(pose), C.c_float(plane_res), _p(cov))
    return cov if rc == 0 else None


def sym_eig(a: np.ndarray):
    a = np.ascontiguousarray(a, dtype=np.float64)
    n = a.shape[0]
    w = np.zeros(n)
    v = np.zeros((n, n))
    lib().orc_sym_eig(n, _p(a), _p(w), _p(v))
    return w, v


def colpiv_qr_solve(A: np.ndarray, b: np.ndarray):
    A = np.ascontiguousarray(A, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    x = np.zeros(3)
    lib().orc_colpiv_qr_solve(A.shape[0], _p(A), _p(b), _p(x))
    return x


def pose_plus(x, d):
    x = np.ascontiguousarray(x, dtype=np.float64)
    d = np.ascontiguousarray(d, dtype=np.float64)
    out = np.zeros(7)
    lib().orc_pose_plus(_p(x), _p(d), _p(out))
    return out


def yaw_round_trip(last, T, yaw_ratio=0.0):
    last = np.ascontiguousarray(last, dtype=np.float64)
    T = np.array(T, dtype=np.float64)
    lib().orc_yaw_round_trip(_p(last), _p(T), C.c_double(yaw_ratio))
    return T


def deskew(points, time_col, lidar_start_time, sample_times, sample_poses, imu_only=False, T_i_l=None):
    """featureExtraction::removePointDistortion (featureExtraction.cpp:222-314) on a copy of float32 [n, C] points.
    -> (deskewed copy, start_pose7, n_past_end)"""
    a = np.array(points, dtype=np.float32, order="C", copy=True)
    st = np.ascontiguousarray(sample_times, np.float64)
    sp = np.ascontiguousarray(sample_poses, np.float64).reshape(-1, 7)
    til = np.ascontiguousarray(T_i_l if T_i_l is not None else [0, 0, 0, 0, 0, 0, 1], np.float64)
    out = np.zeros(7)
    past = lib().orc_deskew(_p(a), a.shape[0], a.shape[1], time_col, float(lidar_start_time), _p(st), _p(sp), len(st), int(imu_only), _p(til), _p(out))
    return a, out, int(past)


def extract_uniform(points, time_col, skip_num, block_range, int_abs=False):
    """featureExtraction::uniformFeatureExtraction (featureExtraction.cpp:504-525) -> float32 [m, 4] {x,y,z,time}"""
    a = np.ascontiguousarray(points, dtype=np.float32)
    out = np.zeros((max(len(a), 1), 4), np.float32)
    m = lib().orc_extract_uniform(_p(a), a.shape[0], a.shape[1], time_col, int(skip_num), float(block_range), int(int_abs), _p(out), len(out))
    assert m >= 0
    return out[:m]


def lidar_uncertainty(hist9):
    h = np.ascontiguousarray(hist9, dtype=np.int32)
    u = np.zeros(6)
    lib().orc_lidar_uncertainty(_p(h), _p(u))
    return u


# ---------------------------------------------------------------------------------------------------------------
# numpy restatements of the map-insert path (integer / float32 element-wise work; SURVEY 8f row 1)
# ---------------------------------------------------------------------------------------------------------------
def transform_scan_numpy(scan_xyzi, pose7):
    """utils::TransformPoint (superodom_utils.h:116-127) for every point: double math, float32 store; intensity kept.
    Rotation = v + 2w(q x v) + 2 q x (q x v), the expression Eigen evaluates for quaternion * vector."""
    s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
    p = s[:, :3].astype(np.float64)
    x, y, z, w = [float(v) for v in pose7[3:]]
    ux = y * p[:, 2] - z * p[:, 1]
    uy = z * p[:, 0] - x * p[:, 2]
    uz = x * p[:, 1] - y * p[:, 0]
    ux = ux + ux
    uy = uy + uy
    uz = uz + uz
    ox = p[:, 0] + w * ux + (y * uz - z * uy)
    oy = p[:, 1] + w * uy + (z * ux - x * uz)
    oz = p[:, 2] + w * uz + (x * uy - y * ux)
    out = s.copy()
    out[:, 0] = (ox + float(pose7[0])).astype(np.float32)
    out[:, 1] = (oy + float(pose7[1])).astype(np.float32)
    out[:, 2] = (oz + float(pose7[2])).astype(np.float32)
    return out


def map_insert_numpy(old_xyzi, new_xyzi, leaf, origin=(10, 10, 5)):
    """LocalMap::addSurfPointCloud (LocalMap.h:591-645): bin the new world-frame points to blocks (off-grid dropped);
    every TOUCHED block is voxel-filtered as a whole (old block cloud followed by the new points; pcl::VoxelGrid
    semantics as in superodom_b200.synth.voxel_filter_blocks); untouched blocks are kept as they are.
    Returns the new map: untouched points in their old order, then the filtered blocks in (block, voxel) order."""
    from superodom_b200 import synth
    old = np.ascontiguousarray(old_xyzi, dtype=np.float32).reshape(-1, 4)
    new = np.ascontiguousarray(new_xyzi, dtype=np.float32).reshape(-1, 4)
    lin_old = synth.block_linear(synth.block_of(old[:, :3], origin))
    lin_new = synth.block_linear(synth.block_of(new[:, :3], origin))
    fin = np.isfinite(new[:, :3]).all(1)
    new, lin_new = new[(lin_new >= 0) & fin], lin_new[(lin_new >= 0) & fin]
    old, lin_old = old[lin_old >= 0], lin_old[lin_old >= 0]
    touched = np.zeros(21 * 21 * 11, dtype=bool)
    touched[lin_new] = True
    keep = old[~touched[lin_old]]
    work = np.concatenate([old[touched[lin_old]], new], 0)
    filt = synth.voxel_filter_blocks(work, leaf, origin) if len(work) else np.zeros((0, 4), np.float32)
    return np.concatenate([keep, filt], 0)


def adjust_voxel_size_numpy(scan_xyzi, line_res, plane_res, auto_voxel_size=True):
    """laserMapping::adjustVoxelSize (laserMapping.cpp:600-651) for the surf cloud: float32 sequential statistics, leaf
    selection, pcl::VoxelGrid(planeRes) over the whole cloud (oracle/voxel_grid_numpy.py, PCL's bounding-box index and its
    verbatim fall-back).  -> (filtered, line_res, plane_res, average_distance)."""
    from . import voxel_grid_numpy as vg
    s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
    avg = 0.0
    if auto_voxel_size and len(s):
        avg = vg.adjust_statistic(s)
        line_res, plane_res = vg.adjust_leaves(avg, line_res, plane_res)
    return vg.voxel_grid(s, plane_res), float(np.float32(line_res)), float(np.float32(plane_res)), avg


def cube_order(xyzi, origin=(10, 10, 5)):
    """Stable permutation that lists a cloud cube by cube in cube-index order -- the order LocalMap::getAllLocalMap emits
    (LocalMap.h:647-658) given per-cube clouds in their internal order."""
    from superodom_b200 import synth
    lin = synth.block_linear(synth.block_of(np.ascontiguousarray(xyzi, dtype=np.float32)[:, :3], origin))
    return np.argsort(lin, kind="stable")

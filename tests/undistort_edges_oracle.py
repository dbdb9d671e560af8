"""CPU oracle of within-scan motion compensation with an edge cloud: tests/cpp/undistort_edges_oracle.cpp (undistort_oracle.cpp, which
compiles the oracle's translation unit unchanged, plus orc_register_undistort_edges), compiled on first use into a temporary directory
with the oracle's own flags."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    out = os.path.join(tempfile.mkdtemp(prefix="so_und_edges_oracle_"), "libso_undistort_edges_oracle.so")
    subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-pthread", "-Wall",
                           "-Wno-unused-function", "-Wno-array-bounds", os.path.join(_HERE, "cpp", "undistort_edges_oracle.cpp"), "-o", out])
    L = C.CDLL(out)
    base = O.lib()                                              # the same entry points, declared once by the oracle's loader
    for name in ("orc_map_create", "orc_map_destroy", "orc_map_set_points", "orc_map_set_edge_points", "orc_map_set_origin",
                 "orc_map_get_origin", "orc_map_shift", "orc_map_counts_5x5", "orc_has_ref_octree", "orc_sizeof_result", "orc_register_full"):
        f, g = getattr(L, name), getattr(base, name)
        f.restype = g.restype
        if g.argtypes is not None:
            f.argtypes = g.argtypes
    L.orc_register_undistort_edges.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                               C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
    assert L.orc_sizeof_result() == C.sizeof(O.Result)
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class UndistortEdgesOracleMap(O.OracleMap):
    """OracleMap (surf and edge stores) whose library also carries the undistorted registration with an edge cloud."""

    def __init__(self, xyzi: np.ndarray | None = None, edge_xyzi: np.ndarray | None = None):
        self.L = lib()
        self.h = C.c_void_p(self.L.orc_map_create())
        if xyzi is not None:
            self.set_points(xyzi)
        if edge_xyzi is not None:
            self.set_edge_points(edge_xyzi)

    def set_points(self, xyzi: np.ndarray, ref_octree: bool | None = None) -> int:
        return super().set_points(xyzi, ref_octree=False)

    def register_undistort_edges(self, scan_xyzi, edge_xyzi, pose7, prev_pose7, dt, rotation, plane_res, max_icp_iters,
                                 max_surface_features=0, n_threads=1, skip_map_checks=False, line_res=0.1, time_col: int = 3) -> O.Result:
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        e = np.ascontiguousarray(edge_xyzi, dtype=np.float32).reshape(-1, s.shape[1])
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        prev = np.ascontiguousarray(prev_pose7, dtype=np.float64)
        o = O.Opts(plane_res, max_icp_iters, max_surface_features, 4, 0, n_threads, 0.0, int(skip_map_checks), 0, 0.0,
                   (C.c_float * 3)(0, 0, 0), float(line_res))
        r = O.Result()
        self.L.orc_register_undistort_edges(self.h, _p(s), s.shape[0], _p(e), e.shape[0], s.shape[1], time_col, _p(pose), _p(prev),
                                            float(dt), int(rotation), C.byref(o), C.byref(r))
        return r

    def register_full(self, scan_xyzi, edge_xyzi, pose7, plane_res, max_icp_iters, max_surface_features=0, n_threads=1, line_res=0.1):
        """orc_register_full (the oracle's plain registration with an edge cloud) from this library."""
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        e = np.ascontiguousarray(edge_xyzi, dtype=np.float32).reshape(-1, s.shape[1])
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        o = O.Opts(plane_res, max_icp_iters, max_surface_features, 4, 0, n_threads, 0.0, 0, 0, 0.0, (C.c_float * 3)(0, 0, 0), float(line_res))
        r = O.Result()
        self.L.orc_register_full(self.h, _p(s), s.shape[0], _p(e), e.shape[0], s.shape[1], _p(pose), C.byref(o), C.byref(r))
        return r

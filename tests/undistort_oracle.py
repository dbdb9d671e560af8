"""CPU oracle of within-scan motion compensation: tests/cpp/undistort_oracle.cpp (the oracle's translation unit, unchanged, plus
orc_register_undistort / orc_undistort_points), compiled on first use into a temporary directory with the oracle's own flags."""
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
    out = os.path.join(tempfile.mkdtemp(prefix="so_und_oracle_"), "libso_undistort_oracle.so")
    subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared", "-pthread", "-Wall",
                           "-Wno-unused-function", "-Wno-array-bounds", os.path.join(_HERE, "cpp", "undistort_oracle.cpp"), "-o", out])
    L = C.CDLL(out)
    base = O.lib()                                              # the same entry points, declared once by the oracle's loader
    for name in ("orc_map_create", "orc_map_destroy", "orc_map_set_points", "orc_map_set_origin", "orc_map_get_origin", "orc_map_shift",
                 "orc_map_counts_5x5", "orc_has_ref_octree", "orc_sizeof_result"):
        f, g = getattr(L, name), getattr(base, name)
        f.restype = g.restype
        if g.argtypes is not None:
            f.argtypes = g.argtypes
    L.orc_undistort_points.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p]
    L.orc_register_undistort.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_double, C.c_int,
                                         C.c_void_p, C.c_void_p]
    assert L.orc_sizeof_result() == C.sizeof(O.Result)
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def undistort_points(xyz_time: np.ndarray, pose7, prev_pose7, dt: float, rotation: bool = True, time_col: int = 3) -> np.ndarray:
    a = np.ascontiguousarray(xyz_time, dtype=np.float32)
    out = np.zeros((len(a), 3), np.float32)
    pose = np.ascontiguousarray(pose7, np.float64)
    prev = np.ascontiguousarray(prev_pose7, np.float64)
    lib().orc_undistort_points(_p(a), len(a), a.shape[1], time_col, _p(pose), _p(prev), float(dt), int(rotation), _p(out))
    return out


class UndistortOracleMap(O.OracleMap):
    """OracleMap whose library also carries the undistorted registration."""

    def __init__(self, xyzi: np.ndarray | None = None):
        self.L = lib()
        self.h = C.c_void_p(self.L.orc_map_create())
        if xyzi is not None:
            self.set_points(xyzi)

    def set_points(self, xyzi: np.ndarray, ref_octree: bool | None = None) -> int:
        return super().set_points(xyzi, ref_octree=False)

    def register_undistort(self, scan_xyzi, pose7, prev_pose7, dt, rotation, plane_res, max_icp_iters, max_surface_features=0,
                           n_threads=1, skip_map_checks=False, time_col: int = 3) -> O.Result:
        s = np.ascontiguousarray(scan_xyzi, dtype=np.float32)
        pose = np.ascontiguousarray(pose7, dtype=np.float64)
        prev = np.ascontiguousarray(prev_pose7, dtype=np.float64)
        o = O.Opts(plane_res, max_icp_iters, max_surface_features, 4, 0, n_threads, 0.0, int(skip_map_checks), 0, 0.0,
                   (C.c_float * 3)(0, 0, 0), 0.1)
        r = O.Result()
        self.L.orc_register_undistort(self.h, _p(s), s.shape[0], s.shape[1], time_col, _p(pose), _p(prev), float(dt), int(rotation),
                                      C.byref(o), C.byref(r))
        return r

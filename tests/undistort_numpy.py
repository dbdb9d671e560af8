"""numpy restatement of pInit (so_undistort.cu, mode APPROXIMATED) in the device's operation order.

Every product and sum is one IEEE double operation, as on the device (which rounds each one explicitly); Eigen's slerp, linear
branch included, with identity as its first argument.  Only acos / sin come from numpy instead of the device's FP64 library."""
from __future__ import annotations

import math

import numpy as np

EPS = 2.220446049250313e-16


def _qmul(a, b):
    return np.array([a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
                     a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2],
                     a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0],
                     a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]])


def _qrot(q, v):
    """q: [4] or [n, 4]; v: [3] or [n, 3] (so_internal.cuh qrot)."""
    q = np.asarray(q, np.float64)
    v = np.asarray(v, np.float64)
    qx, qy, qz, qw = (q[..., k] for k in range(4))
    vx, vy, vz = (v[..., k] for k in range(3))
    ux = qy * vz - qz * vy
    uy = qz * vx - qx * vz
    uz = qx * vy - qy * vx
    ux = ux + ux
    uy = uy + uy
    uz = uz + uz
    return np.stack([(vx + qw * ux) + (qy * uz - qz * uy),
                     (vy + qw * uy) + (qz * ux - qx * uz),
                     (vz + qw * uz) + (qx * uy - qy * ux)], -1)


def delta(prev_pose7, pose7):
    """(q_D, t_D) of D = T_prev^-1 * T_cur."""
    prev = np.asarray(prev_pose7, np.float64)
    cur = np.asarray(pose7, np.float64)
    qpc = np.array([-prev[3], -prev[4], -prev[5], prev[6]])
    q = _qmul(qpc, cur[3:])
    n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    q = q * (1.0 / math.sqrt(n2))
    t = _qrot(qpc, cur[:3] - prev[:3])
    return q, t


def undistort_points(xyz_time: np.ndarray, pose7, prev_pose7, dt: float, rotation: bool = True) -> np.ndarray:
    """xyz_time: [n, >= 4] float32 (x, y, z, time) -> pInit float32 [n, 3] at T_cur = pose7."""
    a = np.asarray(xyz_time, np.float32)
    qD, tD = delta(prev_pose7, pose7)
    tau = a[:, 3].astype(np.float64)
    with np.errstate(invalid="ignore"):
        alpha = np.where(np.isfinite(tau), tau / float(dt), 0.0)
    v = a[:, :3].astype(np.float64)
    if rotation:
        ad = abs(qD[3])
        if ad >= 1.0 - EPS:
            s0 = 1.0 - alpha
            s1 = alpha.copy()
        else:
            th = math.acos(ad)
            inv = 1.0 / math.sin(th)
            s0 = np.sin((1.0 - alpha) * th) * inv
            s1 = np.sin(alpha * th) * inv
        if qD[3] < 0.0:
            s1 = -s1
        qi = np.stack([s0 * 0.0 + s1 * qD[0], s0 * 0.0 + s1 * qD[1], s0 * 0.0 + s1 * qD[2], s0 + s1 * qD[3]], -1)
        o = _qrot(qi, v)
    else:
        o = v
    return (o + alpha[:, None] * tD[None, :]).astype(np.float32)

"""numpy restatement of the search stage of so_localize_global (score points, hypotheses, occupancy bitmap, dilation, scores).

Every floating-point expression is evaluated in the same order as the library (superodom_b200/csrc/so_global.cu for the host part,
so_reloc.cu for the device part, whose operations are explicitly rounded), and numpy never contracts a multiply-add, so the
scores are reproduced exactly, element for element.  Scalars go through Python's `math`, which calls the same libm as the host
library.  Shared by tests/test_global_localization.py and scripts/bench_reloc.py.
"""
from __future__ import annotations

import math

import numpy as np

DEFAULTS = dict(res=0.25, yaw_step=2.0 * math.pi / 180.0, max_range=40.0, score_points=1024, dilate=1, k=16, nms_xy=1.0,
                nms_yaw=10.0 * math.pi / 180.0)


def plan(half_x=0.0, half_y=0.0, half_z=0.0, yaw_half=0.0, **kw):
    """-> dict with the defaults applied and the grid: I, J, K, e, nx, ny, nz, nyaw, m_off, dpsi, n_hyp, bitmap dims."""
    o = dict(DEFAULTS)
    o.update({k: v for k, v in kw.items() if v})
    res = o["res"]
    I, J, K = math.floor(half_x / res), math.floor(half_y / res), math.floor(half_z / res)
    e = math.ceil(o["max_range"] / res)
    full = yaw_half >= math.pi
    if full:
        nyaw = max(1, math.floor(2.0 * math.pi / o["yaw_step"] + 0.5))
        m_off, dpsi = 0, 2.0 * math.pi / nyaw
    else:
        m_off = math.floor(yaw_half / o["yaw_step"])
        nyaw, dpsi = 2 * m_off + 1, o["yaw_step"]
    nx, ny, nz = 2 * I + 1, 2 * J + 1, 2 * K + 1
    bx, by, bz = nx + 2 * e, ny + 2 * e, nz + 2 * e
    return dict(o, I=I, J=J, K=K, e=e, nx=nx, ny=ny, nz=nz, nyaw=nyaw, m_off=m_off, dpsi=dpsi, n_hyp=nx * ny * nz * nyaw,
                bx=bx, by=by, bz=bz, bitmap_bytes=4 * ((bx + 31) // 32) * by * bz)


def score_points(scan_xyzi, score_points_cap, max_range):
    """Finite points within max_range (double squared range), then shouldProcessPoint capped at score_points_cap."""
    p = np.asarray(scan_xyzi, np.float32)
    p = p[np.isfinite(p[:, :3]).all(1)]
    x, y, z = (p[:, a].astype(np.float64) for a in range(3))
    p = p[~((x * x + y * y) + z * z > max_range * max_range)]
    n = len(p)
    if score_points_cap > 0 and n > score_points_cap:
        rate = 1.0 * score_points_cap / float(n)
        i = np.arange(n, dtype=np.float64)
        p = p[~(np.fmod(i * rate, 1.0) + 0.001 > rate)]
    return p


def _qmul(a, b):
    return [((a[3] * b[0] + a[0] * b[3]) + a[1] * b[2]) - a[2] * b[1],
            ((a[3] * b[1] + a[1] * b[3]) + a[2] * b[0]) - a[0] * b[2],
            ((a[3] * b[2] + a[2] * b[3]) + a[0] * b[1]) - a[1] * b[0],
            ((a[3] * b[3] - a[0] * b[0]) - a[1] * b[1]) - a[2] * b[2]]


def tf2_yaw(q):
    """tf2 Matrix3x3(q).getRPY yaw, in the library's operation order."""
    x, y, z, w = (float(v) for v in q)
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d
    xs, ys, zs = x * s, y * s, z * s
    wy, wz = w * ys, w * zs
    xy, xz, yy, zz = x * ys, x * zs, y * ys, z * zs
    m00, m10, m20 = 1.0 - (yy + zz), xy + wz, xz - wy
    if abs(m20) >= 1:
        return 0.0
    pitch = -math.asin(m20)
    return math.atan2(m10 / math.cos(pitch), m00 / math.cos(pitch))


def yaw_quaternions(P, center):
    """-> (yaw_c, [nyaw] yaws, [nyaw, 4] quaternions q_z(yaw_m) (x) q_rp)."""
    x, y, z, w = (float(v) for v in center[3:7])
    nrm = math.sqrt(((x * x + y * y) + z * z) + w * w)
    qc = [x / nrm, y / nrm, z / nrm, w / nrm]
    yaw_c = tf2_yaw(qc)
    h = -yaw_c * 0.5
    q_rp = _qmul([0.0, 0.0, math.sin(h), math.cos(h)], qc)
    yaws, qs = [], []
    for m in range(P["nyaw"]):
        psi = yaw_c + float(m - P["m_off"]) * P["dpsi"]
        hm = psi * 0.5
        yaws.append(psi)
        qs.append(_qmul([0.0, 0.0, math.sin(hm), math.cos(hm)], q_rp))
    return yaw_c, np.array(yaws), np.array(qs)


def _qrot(q, v):
    q0, q1, q2, q3 = (float(c) for c in q)
    ux = q1 * v[:, 2] - q2 * v[:, 1]
    uy = q2 * v[:, 0] - q0 * v[:, 2]
    uz = q0 * v[:, 1] - q1 * v[:, 0]
    ux = ux + ux
    uy = uy + uy
    uz = uz + uz
    return np.stack([(v[:, 0] + q3 * ux) + (q1 * uz - q2 * uy),
                     (v[:, 1] + q3 * uy) + (q2 * ux - q0 * uz),
                     (v[:, 2] + q3 * uz) + (q0 * uy - q1 * ux)], 1)


def bitmap(map_xyz, P, center):
    """Occupancy of the surf map in the search box, dilated by P['dilate'] voxels (cube): bool [bz, by, bx]."""
    res, e = P["res"], P["e"]
    lo = [float(center[a]) - float(s + e) * res for a, s in enumerate((P["I"], P["J"], P["K"]))]
    m = np.asarray(map_xyz, np.float32)[:, :3].astype(np.float64)
    f = np.floor((m - np.array(lo)) / res)
    dims = np.array([P["bx"], P["by"], P["bz"]])
    ok = ((f >= 0) & (f < dims)).all(1)
    w = f[ok].astype(np.int64)
    B = np.zeros((P["bz"], P["by"], P["bx"]), bool)
    B[w[:, 2], w[:, 1], w[:, 0]] = True
    d = P["dilate"]
    for ax in (2, 1, 0):                 # x, then y, then z (the order does not matter for a cube)
        src = B.copy()
        n = B.shape[ax]
        for s in range(1, d + 1):
            if s >= n:
                break
            hi = [slice(None)] * 3
            lo_ = [slice(None)] * 3
            hi[ax], lo_[ax] = slice(s, None), slice(None, n - s)
            B[tuple(hi)] |= src[tuple(lo_)]
            B[tuple(lo_)] |= src[tuple(hi)]
    return B


def localize_scores_numpy(scan_xyzi, center, map_xyz, half_x=0.0, half_y=0.0, half_z=0.0, yaw_half=0.0, **kw):
    """Steps 1-4 of so_localize_global -> (uint16 scores [nyaw, nz, ny, nx], number of score points)."""
    P = plan(half_x, half_y, half_z, yaw_half, **kw)
    pts = score_points(scan_xyzi, P["score_points"], P["max_range"])
    _, _, qs = yaw_quaternions(P, center)
    B = bitmap(map_xyz, P, center)
    pad = 2
    Bp = np.pad(B, pad)
    e, res = P["e"], P["res"]
    nx, ny, nz = P["nx"], P["ny"], P["nz"]
    v = pts[:, :3].astype(np.float64)
    out = np.zeros((P["nyaw"], nz, ny, nx), np.int64)
    for m, q in enumerate(qs):
        w = np.floor(_qrot(q, v) / res).astype(np.int64) + e + pad      # padded-bitmap index of shift (0, 0, 0)
        assert (w >= 0).all() and (w[:, 0] + nx <= Bp.shape[2]).all() and (w[:, 1] + ny <= Bp.shape[1]).all() and (w[:, 2] + nz <= Bp.shape[0]).all()
        acc = out[m]
        for p in range(len(w)):
            wx, wy, wz = w[p]
            acc += Bp[wz:wz + nz, wy:wy + ny, wx:wx + nx]
    return out.astype(np.uint16), len(pts)

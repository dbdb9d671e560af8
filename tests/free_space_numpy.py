"""Numpy restatement of so_map_clear_free_space (DESIGN.md §2, "Free-space clearing"), written apart from the device code.

A map point is removed when the scan saw clearly past it along its own line of sight:
  - range image of the scan (sensor frame, FP64 angles): column floor((az + pi) / az_res) with az in [-pi, pi), W = ceil(360 / az_res_deg)
    columns (the azimuth wraps); row floor((el - el_min) / el_res), points with el outside [el_min, el_max) left out; each pixel keeps
    the minimum float32 range of its points;
  - each map point: q = R^T (m - t) in FP64, range r_m and pixel; a candidate when min_range <= r_m <= max_range, its (2d+1)^2
    neighbourhood lies inside the elevation span and every pixel of it has a return; removed when the neighbourhood minimum exceeds
    r_m + max(margin, margin_rel * r_m).

`bounds` gives two sets the device's removal set must lie between, for the rounding differences of atan2 and of the rotation: scan
points within eps pixel of a pixel edge go into both pixels or into neither, and a map point ambiguous at a pixel edge, or within eps
metres of the threshold, is kept (lower set) or removed when any reading allows it (upper set).
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

DEG = math.pi / 180.0
UNKNOWN = np.float32(np.inf)


@dataclasses.dataclass
class Opts:
    """Mirror of so_free_space; the defaults are so_free_space_defaults' (DESIGN.md §2 records the study that set them)."""
    az_res_deg: float = 0.4
    el_res_deg: float = 0.4
    el_min_deg: float = -23.0
    el_max_deg: float = 23.0
    dilate: int = 2
    margin: float = 0.3
    margin_rel: float = 0.02
    min_range: float = 0.5
    max_range: float = 60.0


# sensor-specific image geometry used by the tests: el_res at least the beam spacing, every beam well inside a row
VLP16 = dict(az_res_deg=0.4, el_res_deg=2.0, el_min_deg=-16.0, el_max_deg=16.0)
OS1_128 = dict(az_res_deg=0.4, el_res_deg=0.4, el_min_deg=-23.0, el_max_deg=23.0)
SENSOR_IMAGE = {"vlp16": VLP16, "os1_128": OS1_128}


def opts_for(sensor: str, **kw) -> Opts:
    d = dict(SENSOR_IMAGE[sensor])
    d.update(kw)
    return Opts(**d)


def dims(o: Opts):
    W = int(math.ceil(360.0 / float(np.float32(o.az_res_deg))))
    H = int(math.ceil((float(np.float32(o.el_max_deg)) - float(np.float32(o.el_min_deg))) / float(np.float32(o.el_res_deg))))
    return W, H


def _geom(o: Opts):
    f = lambda v: float(np.float32(v))                     # the C struct holds floats
    return dict(az_res=f(o.az_res_deg) * DEG, el_res=f(o.el_res_deg) * DEG, el_min=f(o.el_min_deg) * DEG, el_max=f(o.el_max_deg) * DEG)


def _angles(p):
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    az = np.arctan2(y, x)
    az = np.where(az >= math.pi, az - 2 * math.pi, az)
    el = np.arctan2(z, np.hypot(x, y))
    return az, el


def _pixel_coords(az, el, g):
    """Continuous pixel coordinates (before floor) of the column and the row."""
    return (az + math.pi) / g["az_res"], (el - g["el_min"]) / g["el_res"]


def range_image(scan_xyz: np.ndarray, o: Opts, edge_eps: float = 0.0, mode: str = "both"):
    """-> (image [H, W] float32, UNKNOWN = no return, n_image_points, n_pixels_hit).  edge_eps > 0: a point within edge_eps pixel of a
    column or row edge goes into both candidate pixels (mode "both") or into neither ("neither")."""
    W, H = dims(o)
    g = _geom(o)
    p = np.asarray(scan_xyz, np.float64)[:, :3]
    p32 = np.asarray(scan_xyz, np.float32)[:, :3]
    fin = np.isfinite(p32).all(1)
    p, p32 = p[fin], p32[fin]
    r = np.sqrt((p * p).sum(1))
    ok = r > 0
    p, r = p[ok], r[ok]
    az, el = _angles(p)
    inside = (el >= g["el_min"]) & (el < g["el_max"])
    p, r, az, el = p[inside], r[inside], az[inside], el[inside]
    cu, ru = _pixel_coords(az, el, g)
    col = np.minimum(np.floor(cu).astype(np.int64), W - 1)
    row = np.floor(ru).astype(np.int64)
    keep = (row >= 0) & (row < H)
    img = np.full(H * W, UNKNOWN, np.float32)
    r32 = r.astype(np.float32)
    n_points = int(keep.sum())
    if edge_eps <= 0:
        np.minimum.at(img, row[keep] * W + col[keep] % W, r32[keep])
    else:
        fc, fr = cu - np.floor(cu), ru - np.floor(ru)
        amb_c = (fc < edge_eps) | (fc > 1 - edge_eps)
        amb_r = (fr < edge_eps) | (fr > 1 - edge_eps)
        if mode == "neither":
            k = keep & ~amb_c & ~amb_r
            np.minimum.at(img, row[k] * W + col[k] % W, r32[k])
        else:
            alt_c = np.where(fc < 0.5, col - 1, col + 1) % W
            alt_r = np.where(fr < 0.5, row - 1, row + 1)
            for cc, rr, m in ((col % W, row, keep), (alt_c, row, keep & amb_c), (col % W, alt_r, keep & amb_r),
                              (alt_c, alt_r, keep & amb_c & amb_r)):
                m = m & (rr >= 0) & (rr < H)
                np.minimum.at(img, rr[m] * W + cc[m], r32[m])
    return img.reshape(H, W), n_points, int(np.isfinite(img).sum())


def to_sensor(map_xyz: np.ndarray, pose7) -> np.ndarray:
    """q = R^T (m - t) in FP64, the quaternion normalised."""
    pose7 = np.asarray(pose7, np.float64)
    q = pose7[3:] / np.linalg.norm(pose7[3:])
    x, y, z, w = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return (np.asarray(map_xyz, np.float64)[:, :3] - pose7[:3]) @ R


def _neigh(img, row, col, d):
    """-> (every pixel of the neighbourhood has a return, its minimum with UNKNOWN as +inf, the rows lie inside the image)."""
    H, W = img.shape
    ok = (row - d >= 0) & (row + d < H)
    r, c = np.where(ok, row, d), col % W
    acc = np.full(len(row), UNKNOWN, np.float32)
    known = ok.copy()
    for dr in range(-d, d + 1):
        for dc in range(-d, d + 1):
            v = img[np.clip(r + dr, 0, H - 1), (c + dc) % W]
            known &= np.isfinite(v)
            acc = np.minimum(acc, v)
    return known, acc.astype(np.float64), ok


def removal_mask(map_xyz: np.ndarray, pose7, img: np.ndarray, o: Opts, edge_eps: float = 0.0, mode: str = "exact", img_min=None):
    """-> (removed [n] bool, candidate [n] bool).  Exact with edge_eps = 0.  With edge_eps > 0, `img` decides which pixels have a
    return and `img_min` (default img) gives the minima, the threshold moves by edge_eps, and a map point within edge_eps pixel of a
    pixel edge is read in every pixel it may fall in: mode "lower" removes it only when every reading does (threshold + edge_eps),
    "upper" when any reading does (threshold - edge_eps)."""
    H, W = img.shape
    img_min = img if img_min is None else img_min
    g = _geom(o)
    q = to_sensor(map_xyz, pose7)
    rm = np.sqrt((q * q).sum(1))
    az, el = _angles(q)
    cu, ru = _pixel_coords(az, el, g)
    in_rng = (rm >= float(np.float32(o.min_range))) & (rm <= float(np.float32(o.max_range)))
    shift = {"exact": 0.0, "lower": edge_eps, "upper": -edge_eps}[mode]
    thr = rm + np.maximum(float(np.float32(o.margin)), float(np.float32(o.margin_rel)) * rm) + shift
    d = int(o.dilate)

    def reading(col, row, in_span):
        known, _, ok = _neigh(img, row, col, d)
        _, mn, _ = _neigh(img_min, row, col, d)
        cand = in_span & ok & in_rng & known
        return cand, cand & (mn > thr)

    col0 = np.minimum(np.floor(cu).astype(np.int64), W - 1)
    row0 = np.clip(np.floor(ru), -1e6, 1e6).astype(np.int64)
    span0 = (el >= g["el_min"]) & (el < g["el_max"]) & (row0 >= 0) & (row0 < H)
    cand, rem = reading(col0, row0, span0)
    if mode == "exact":
        return rem, cand
    fc, fr = cu - np.floor(cu), ru - np.floor(ru)
    alt_c = np.where(fc < 0.5, col0 - 1, col0 + 1)
    alt_r = np.where(fr < 0.5, row0 - 1, row0 + 1)
    amb_c = (fc < edge_eps) | (fc > 1 - edge_eps)
    amb_r = (fr < edge_eps) | (fr > 1 - edge_eps)
    out = rem.copy()
    for cc, rr, m in ((alt_c, row0, amb_c), (col0, alt_r, amb_r), (alt_c, alt_r, amb_c & amb_r)):
        _, r2 = reading(cc, rr, (rr >= 0) & (rr < H))
        r2 = np.where(m, r2, rem)
        out = (out & r2) if mode == "lower" else (out | r2)
    return out, cand


def clear(map_xyz, scan_xyz, pose7, o: Opts):
    """-> (removed mask, stats dict) of one call on one store, exact (no edge sandwich)."""
    img, n_pts, n_hit = range_image(scan_xyz, o)
    rem, cand = removal_mask(map_xyz, pose7, img, o)
    return rem, dict(n_image_points=n_pts, n_pixels_hit=n_hit, n_candidates=int(cand.sum()), n_removed=int(rem.sum()))


def bounds(map_xyz, scan_xyz, pose7, o: Opts, eps: float = 1e-9):
    """-> (lower, upper) removal masks, the device's removal set lies between them.  A pixel's true point set lies between the
    image that puts every scan point within eps pixel of an edge into both candidate pixels ("both": more returns, smaller minima)
    and the one that puts it into neither.  A point is surely removed when the neighbourhood has returns even in "neither" and its
    minimum exceeds the threshold even in "both" (lower), and possibly removed when it has returns in "both" and its minimum in
    "neither" exceeds the threshold (upper)."""
    img_both, _, _ = range_image(scan_xyz, o, eps, "both")
    img_neither, _, _ = range_image(scan_xyz, o, eps, "neither")
    lo, _ = removal_mask(map_xyz, pose7, img_neither, o, eps, "lower", img_min=img_both)
    hi, _ = removal_mask(map_xyz, pose7, img_both, o, eps, "upper", img_min=img_neither)
    return lo, hi

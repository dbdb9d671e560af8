"""Numpy restatement of so_map_clear_free_space (DESIGN.md §2, "Free-space clearing"), written apart from the device code.

A map point is removed when the scan saw clearly past it along its own line of sight:
  - range image of the scan (sensor frame, FP64 angles): column floor((az + pi) / az_res) with az in [-pi, pi), W = ceil(360 / az_res_deg)
    columns (the azimuth wraps); row floor((el - el_min) / el_res), points with el outside [el_min, el_max) left out; each pixel keeps
    the minimum float32 range of its points and, apart from it, whether it has a return at all: a finite point whose float32 range
    overflows to +inf still makes its pixel known;
  - each map point: q = R^T (m - t) in FP64, range r_m and pixel; a candidate when min_range <= r_m <= max_range, its (2d+1)^2
    neighbourhood lies inside the elevation span and every pixel of it has a return; removed when the neighbourhood minimum exceeds
    r_m + max(margin, margin_rel * r_m).

`bounds` gives two sets the device's removal set must lie between, for the rounding differences of atan2 and of the rotation: scan
points within eps pixel of a pixel edge (the azimuth seam included, whose two sides are columns W - 1 and 0) or of el_max go into
every pixel they may fall in or into none, and a map point ambiguous at a pixel edge, or within eps metres of the threshold or of the
range gate, is kept (lower set) or removed when any reading allows it (upper set).
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

DEG = math.pi / 180.0
UNKNOWN = np.float32(np.inf)          # the minimum of a pixel without a return; whether a pixel has one is the separate `hit` mask


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


def _top(g):
    """Continuous row coordinate of el_max: H when the span is a whole number of rows, inside the partial top row otherwise."""
    return (g["el_max"] - g["el_min"]) / g["el_res"]


def _col_alt(cu, col, W, g, eps):
    """-> (ambiguous, the other column) of continuous column coordinates: within eps pixel of a column edge, or of the azimuth seam,
    where an azimuth that reads as pi on one side wraps to -pi (column 0) and (az + pi) / az_res >= W is clamped to column W - 1."""
    fc = cu - np.floor(cu)
    seam = (cu < eps) | (cu > 2 * math.pi / g["az_res"] - eps)
    alt = np.where(seam, np.where(col == 0, W - 1, 0), np.where(fc < 0.5, col - 1, col + 1) % W)
    return (fc < eps) | (fc > 1 - eps) | seam, alt


def range_image(scan_xyz: np.ndarray, o: Opts, edge_eps: float = 0.0, mode: str = "both"):
    """-> (image [H, W] float32 minima, UNKNOWN where no return; hit [H, W] bool, the pixel has a return; n_image_points,
    n_pixels_hit).  edge_eps > 0: a point within edge_eps pixel of a column or row edge, or of el_max, goes into every pixel it may fall
    in (mode "both") or into none ("neither")."""
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
    cu, ru = _pixel_coords(az, el, g)
    col = np.minimum(np.floor(cu).astype(np.int64), W - 1)
    row = np.floor(ru).astype(np.int64)
    keep = (el >= g["el_min"]) & (el < g["el_max"]) & (row >= 0) & (row < H)
    img = np.full(H * W, UNKNOWN, np.float32)
    hit = np.zeros(H * W, bool)
    with np.errstate(over="ignore"):
        r32 = r.astype(np.float32)                         # a range above the largest float rounds to +inf, as float(r) does

    def put(rr, cc, m):
        m = m & (rr >= 0) & (rr < H)
        np.minimum.at(img, rr[m] * W + cc[m], r32[m])
        hit[rr[m] * W + cc[m]] = True

    n_points = int(keep.sum())
    if edge_eps <= 0:
        put(row, col % W, keep)
    else:
        fr = ru - np.floor(ru)
        amb_c, alt_c = _col_alt(cu, col, W, g, edge_eps)
        amb_r = (fr < edge_eps) | (fr > 1 - edge_eps)      # el_min is a row edge; so is el_max unless the top row is partial
        near_top = np.abs(ru - _top(g)) < edge_eps
        if mode == "neither":
            put(row, col % W, keep & ~amb_c & ~amb_r & ~near_top)
        else:
            alt_r, top = np.where(fr < 0.5, row - 1, row + 1), np.minimum(row, H - 1)
            for cc, rr, m in ((col % W, row, keep), (alt_c, row, keep & amb_c), (col % W, alt_r, amb_r), (alt_c, alt_r, amb_c & amb_r),
                              (col % W, top, near_top), (alt_c, top, near_top & amb_c)):
                put(rr, cc, m)
    return img.reshape(H, W), hit.reshape(H, W), n_points, int(hit.sum())


def to_sensor(map_xyz: np.ndarray, pose7) -> np.ndarray:
    """q = R^T (m - t) in FP64, the quaternion normalised."""
    pose7 = np.asarray(pose7, np.float64)
    q = pose7[3:] / np.linalg.norm(pose7[3:])
    x, y, z, w = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return (np.asarray(map_xyz, np.float64)[:, :3] - pose7[:3]) @ R


def _neigh(img, hit, row, col, d):
    """-> (every pixel of the neighbourhood has a return, its minimum with UNKNOWN as +inf, the rows lie inside the image)."""
    H, W = img.shape
    ok = (row - d >= 0) & (row + d < H)
    r, c = np.where(ok, row, d), col % W
    acc = np.full(len(row), UNKNOWN, np.float32)
    known = ok.copy()
    for dr in range(-d, d + 1):
        for dc in range(-d, d + 1):
            rr, cc = np.clip(r + dr, 0, H - 1), (c + dc) % W
            known &= hit[rr, cc]
            acc = np.minimum(acc, img[rr, cc])
    return known, acc.astype(np.float64), ok


def removal_mask(map_xyz: np.ndarray, pose7, img: np.ndarray, hit: np.ndarray, o: Opts, edge_eps: float = 0.0, mode: str = "exact",
                 img_min=None):
    """-> (removed [n] bool, candidate [n] bool).  Exact with edge_eps = 0.  `hit` decides which pixels have a return and `img_min`
    (default img) gives the minima; with edge_eps > 0, the threshold moves by edge_eps, and a map point within edge_eps pixel of a
    pixel edge or of el_max is read in every pixel it may fall in: mode "lower" removes it only when every reading does (threshold
    + edge_eps, range gate narrowed by edge_eps), "upper" when any reading does (threshold - edge_eps, gate widened)."""
    H, W = img.shape
    img_min = img if img_min is None else img_min
    g = _geom(o)
    q = to_sensor(map_xyz, pose7)
    rm = np.sqrt((q * q).sum(1))
    az, el = _angles(q)
    cu, ru = _pixel_coords(az, el, g)
    shift = {"exact": 0.0, "lower": edge_eps, "upper": -edge_eps}[mode]
    in_rng = (rm >= float(np.float32(o.min_range)) + shift) & (rm <= float(np.float32(o.max_range)) - shift)
    thr = rm + np.maximum(float(np.float32(o.margin)), float(np.float32(o.margin_rel)) * rm) + shift
    d = int(o.dilate)

    def reading(col, row, in_span):
        known, _, ok = _neigh(img, hit, row, col, d)
        _, mn, _ = _neigh(img_min, hit, row, col, d)
        cand = in_span & ok & in_rng & known
        return cand, cand & (mn > thr)

    col0 = np.minimum(np.floor(cu).astype(np.int64), W - 1)
    row0 = np.clip(np.floor(ru), -1e6, 1e6).astype(np.int64)
    span0 = (el >= g["el_min"]) & (el < g["el_max"]) & (row0 >= 0) & (row0 < H)
    cand, rem = reading(col0, row0, span0)
    if mode == "exact":
        return rem, cand
    fr = ru - np.floor(ru)
    amb_c, alt_c = _col_alt(cu, col0, W, g, edge_eps)
    amb_r = (fr < edge_eps) | (fr > 1 - edge_eps)
    near_top = np.abs(ru - _top(g)) < edge_eps                 # may read as inside the (partial) top row or outside the span
    every = np.ones(len(rem), bool)
    rows = ((row0, span0, every), (np.where(fr < 0.5, row0 - 1, row0 + 1), None, amb_r), (np.minimum(row0, H - 1), None, near_top))
    out = rem.copy()
    for cc, mc in ((col0, every), (alt_c, amb_c)):
        for rr, in_span, mr in rows:
            if cc is col0 and rr is row0:
                continue
            _, r2 = reading(cc, rr, (rr >= 0) & (rr < H) if in_span is None else in_span)
            r2 = np.where(mc & mr, r2, rem)
            out = (out & r2) if mode == "lower" else (out | r2)
    if mode == "lower":
        out &= ~near_top
    return out, cand


def edge_points(xyz: np.ndarray, o: Opts, pose7=None, eps: float = 1e-9) -> np.ndarray:
    """-> mask of the points that may read two ways: within eps pixel of a column or row edge, of the azimuth seam or of el_max, at
    elevations from el_min to el_max; with pose7 they are map points (world frame), also ambiguous within eps metres of the range
    gate.  Where no point of either cloud is, and `bounds` agree, every counter of a call is decided exactly."""
    W, H = dims(o)
    g = _geom(o)
    p = np.asarray(xyz, np.float64)[:, :3]
    fin = np.isfinite(p).all(1)
    q = np.where(fin[:, None], p if pose7 is None else to_sensor(np.where(fin[:, None], p, 0.0), pose7), 1.0)
    cu, ru = _pixel_coords(*_angles(q), g)
    fr = ru - np.floor(ru)
    amb_c, _ = _col_alt(cu, np.minimum(np.floor(cu), W - 1).astype(np.int64), W, g, eps)
    out = (amb_c | (fr < eps) | (fr > 1 - eps) | (np.abs(ru - _top(g)) < eps)) & (ru > -eps) & (ru < _top(g) + eps)
    rm = np.sqrt((q * q).sum(1))
    if pose7 is not None:
        out |= (np.abs(rm - float(np.float32(o.min_range))) < eps) | (np.abs(rm - float(np.float32(o.max_range))) < eps)
    return out & fin & (rm > 0)


def clear(map_xyz, scan_xyz, pose7, o: Opts):
    """-> (removed mask, stats dict) of one call on one store, exact (no edge sandwich)."""
    img, hit, n_pts, n_hit = range_image(scan_xyz, o)
    rem, cand = removal_mask(map_xyz, pose7, img, hit, o)
    return rem, dict(n_image_points=n_pts, n_pixels_hit=n_hit, n_candidates=int(cand.sum()), n_removed=int(rem.sum()))


def bounds(map_xyz, scan_xyz, pose7, o: Opts, eps: float = 1e-9):
    """-> (lower, upper) removal masks, the device's removal set lies between them.  A pixel's true point set lies between the
    image that puts every scan point within eps pixel of an edge into both candidate pixels ("both": more returns, smaller minima)
    and the one that puts it into neither.  A point is surely removed when the neighbourhood has returns even in "neither" and its
    minimum exceeds the threshold even in "both" (lower), and possibly removed when it has returns in "both" and its minimum in
    "neither" exceeds the threshold (upper)."""
    img_both, hit_both, _, _ = range_image(scan_xyz, o, eps, "both")
    img_neither, hit_neither, _, _ = range_image(scan_xyz, o, eps, "neither")
    lo, _ = removal_mask(map_xyz, pose7, img_neither, hit_neither, o, eps, "lower", img_min=img_both)
    hi, _ = removal_mask(map_xyz, pose7, img_both, hit_both, o, eps, "upper", img_min=img_neither)
    return lo, hi

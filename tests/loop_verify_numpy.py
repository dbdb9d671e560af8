"""Numpy restatement of the scores of so_loop_verify (so_verify.cu), written apart from the device code.  Plain numpy and FP64; nothing
here calls the device.

Per candidate `id` of query keyframe `query`:
  - submap ids: the ids of [id - w, id + w] that are >= 0 and eligible (so_verify_rule.h: [0, query - exclude_recent) by default, or
    [id_begin, id_end) without the query);
  - overlap: each finite query point at reg.pose, its nearest surf point of its own 50 m block (LocalMap's block rule, synth.block_of /
    block_linear at the window's origin) with the distance rounded as exact_d2 (float32 differences, FP64 squares summed x, y, z,
    rounded to float32); an inlier when that d^2 <= float(inlier_dist^2).  The rounding is exact, so the inlier set and every d^2 are
    bit for bit;
  - sum: per 64-point CTA the halving tree of k_verify_overlap (non-inliers add 0), then k_verify_sum: per = ceil(grid / 256)
    contiguous runs each summed in order, then the 256 runs in order; rmse = sqrt(sum / n_inliers);
  - conflicts (free_space_numpy): the surf points against the query's range image at reg.pose, and the query points at reg.pose
    against every submap keyframe's image at its pose.  A point is a candidate when some image makes it one and a conflict when some
    image removes it: the device's in-order loop that stops at the first removal gives the same, since a removal needs a candidate;
  - decision: verify_accept's rule.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

import free_space_numpy as F

CTA = 64                  # kVerifyThreads
SUM_THREADS = 256         # kVerifySumThreads


# ------------------------------------------------------------------------------------------------------------- submap ids
def verify_range(query: int, id_begin: int, id_end: int, exclude_recent: int):
    if id_end < 0:
        return 0, max(query - exclude_recent, 0)
    return id_begin, id_end


def verify_eligible(rng, query: int, i: int) -> bool:
    return rng[0] <= i < rng[1] and i != query


def submap_ids(query: int, cand: int, half_window: int, id_begin: int = 0, id_end: int = -1, exclude_recent: int = 30):
    rng = verify_range(query, id_begin, id_end, exclude_recent)
    return [k for k in range(cand - half_window, cand + half_window + 1) if k >= 0 and verify_eligible(rng, query, k)]


# ------------------------------------------------------------------------------------------------------------- overlap
def exact_d2(q32: np.ndarray, m32: np.ndarray) -> np.ndarray:
    """exact_d2 (so_knn.cuh): float32 differences, FP64 squares summed in x, y, z order, rounded to float32."""
    d = (np.asarray(q32, np.float32) - np.asarray(m32, np.float32)).astype(np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]).astype(np.float32)


def nearest_in_block(q_xyz: np.ndarray, map_xyz: np.ndarray, origin, reach: float) -> np.ndarray:
    """-> float32 [n]: each query's smallest exact_d2 to a map point of its own block among those within `reach` metres, +inf when
    there is none (no block, an off-window or empty block, or nothing within reach).  A k-d tree per block proposes the candidates;
    the 16 nearest in FP64 within reach * (1 + 1e-5) always hold the point of smallest exact_d2 unless more than 15 others lie within
    float rounding of it, in which case they are coincident with it and give the same d^2."""
    from scipy.spatial import cKDTree
    from superodom_b200 import synth
    q = np.asarray(q_xyz, np.float32)[:, :3]
    m = np.asarray(map_xyz, np.float32)[:, :3]
    out = np.full(len(q), np.inf, np.float32)
    fin = np.isfinite(q).all(1)
    qb = np.full(len(q), -1, np.int64)
    qb[fin] = synth.block_linear(synth.block_of(q[fin], origin))
    mb = synth.block_linear(synth.block_of(m, origin)) if len(m) else np.zeros(0, np.int64)
    r = float(reach) * (1 + 1e-5) + 1e-6
    for b in np.unique(qb[qb >= 0]):
        mi = np.flatnonzero(mb == b)
        if not len(mi):
            continue
        qi = np.flatnonzero(qb == b)
        k = min(16, len(mi))
        _, nn = cKDTree(m[mi].astype(np.float64)).query(q[qi].astype(np.float64), k=k, distance_upper_bound=r)
        nn = nn.reshape(len(qi), k)
        ok = nn < len(mi)
        d2 = np.where(ok, exact_d2(q[qi, None, :], m[mi[np.where(ok, nn, 0)]]), np.float32(np.inf))
        out[qi] = d2.min(1)
    return out


def bound_of(inlier_dist: float) -> np.float32:
    """float(inlier_dist^2), as so_loop_verify passes it to the search."""
    return np.float32(np.float64(inlier_dist) * np.float64(inlier_dist))


# ------------------------------------------------------------------------------------------------------------- the fixed-order sum
def cta_partials(values: np.ndarray) -> np.ndarray:
    """k_verify_overlap's per-CTA sums: each run of 64 values (zero-padded) reduced by the halving tree s[t] += s[t + h]."""
    v = np.asarray(values, np.float64)
    grid = (len(v) + CTA - 1) // CTA
    s = np.zeros((grid, CTA), np.float64)
    s.reshape(-1)[: len(v)] = v
    h = CTA // 2
    while h:
        s[:, :h] = s[:, :h] + s[:, h:2 * h]
        h //= 2
    return s[:, 0].copy()


def verify_sum(partials) -> float:
    """k_verify_sum: per = ceil(n / 256) contiguous runs, each summed in order from 0.0, then the 256 runs in order."""
    p = [float(x) for x in partials]
    n = len(p)
    per = (n + SUM_THREADS - 1) // SUM_THREADS
    runs = []
    for t in range(SUM_THREADS):
        v = 0.0
        for k in range(t * per, min(n, t * per + per)):
            v += p[k]
        runs.append(v)
    tot = 0.0
    for v in runs:
        tot += v
    return tot


# ------------------------------------------------------------------------------------------------------------- conflicts
def image_opts(image) -> F.Opts:
    """free_space_numpy options from an so_free_space (ctypes) or a dict of its fields."""
    names = [f.name for f in dataclasses.fields(F.Opts)]
    get = (lambda k: image[k]) if isinstance(image, dict) else (lambda k: getattr(image, k))
    return F.Opts(**{k: (int(get(k)) if k == "dilate" else float(get(k))) for k in names})


def _test(points, pose7, scan_xyz, o: F.Opts, eps: float):
    """-> (cand_lo, cand_hi, rem_lo, rem_hi, rem_exact, cand_exact) of points against the image of scan_xyz (sensor frame) at pose7.
    Points within eps pixel of a pixel edge, or within eps metres of the range gate, are open in the lower / upper sets."""
    img, hit, _, _ = F.range_image(scan_xyz, o)
    rem, cand = F.removal_mask(points, pose7, img, hit, o)
    if eps <= 0:
        return cand, cand, rem, rem, rem, cand
    ib, hb, _, _ = F.range_image(scan_xyz, o, eps, "both")
    inn, hn, _, _ = F.range_image(scan_xyz, o, eps, "neither")
    lo, _ = F.removal_mask(points, pose7, inn, hn, o, eps, "lower", img_min=ib)
    hi, _ = F.removal_mask(points, pose7, ib, hb, o, eps, "upper", img_min=inn)
    amb = F.edge_points(points, o, pose7, eps)
    _, c_lo = F.removal_mask(points, pose7, inn, hn, o)
    _, c_hi = F.removal_mask(points, pose7, ib, hb, o)
    return c_lo & ~amb, c_hi | amb, lo, hi, rem, cand


def conflicts(points, scans, poses, o: F.Opts, eps: float = 1e-9):
    """points (world) against the images of scans[j] at poses[j]: a candidate of any image, removed by any image -> dict of the
    counts' lower and upper bounds and the exact (eps = 0) reading, and the number of points the bounds leave open."""
    pts = np.asarray(points, np.float32)[:, :3]
    pts = pts[np.isfinite(pts).all(1)]
    n = len(pts)
    acc = {k: np.zeros(n, bool) for k in ("c_lo", "c_hi", "r_lo", "r_hi", "r", "c")}
    for scan, pose in zip(scans, poses):
        if not n:
            break
        parts = _test(pts, pose, np.asarray(scan, np.float32)[:, :3], o, eps)
        for k, v in zip(("c_lo", "c_hi", "r_lo", "r_hi", "r", "c"), parts):
            acc[k] |= v
    return dict(cand=(int(acc["c_lo"].sum()), int(acc["c_hi"].sum())), conflict=(int(acc["r_lo"].sum()), int(acc["r_hi"].sum())),
                cand_exact=int(acc["c"].sum()), conflict_exact=int(acc["r"].sum()),
                open=int((acc["c_hi"] & ~acc["c_lo"]).sum() + (acc["r_hi"] & ~acc["r_lo"]).sum()))


def fraction(conflicts_: int, candidates: int) -> float:
    return conflicts_ / candidates if candidates else 0.0


def accept(status: int, overlap: float, conflict_query: float, conflict_map: float, min_overlap: float, max_conflict: float) -> bool:
    return status == 0 and overlap >= min_overlap and conflict_query <= max_conflict and conflict_map <= max_conflict


# ------------------------------------------------------------------------------------------------------------- one candidate
def scores(query_world, query_sensor, surf, origin, sub_scans, sub_poses, reg_pose, inlier_dist: float, image, reach: float | None = None,
           eps: float = 1e-9) -> dict:
    """Every score of one candidate.  query_world: the query keyframe at reg.pose as the device places it (so_keyframe_download with
    reg.pose); query_sensor: its sensor-frame cloud; surf, origin: the scratch context's surf store and window origin after the call;
    sub_scans / sub_poses: the submap keyframes' sensor-frame clouds and poses.  reach: the largest distance searched (default
    inlier_dist)."""
    o = image_opts(image)
    qw = np.asarray(query_world, np.float32)[:, :3]
    fin = np.isfinite(qw).all(1)
    bound = bound_of(inlier_dist)
    d2 = nearest_in_block(qw, surf, origin, math.sqrt(float(bound)) if reach is None else reach)
    hit = fin & (d2 <= bound)
    vals = np.where(hit, d2.astype(np.float64), 0.0)
    grid = (len(qw) + CTA - 1) // CTA
    total = verify_sum(cta_partials(vals)) if len(qw) else 0.0
    n_q, n_in = int(fin.sum()), int(hit.sum())
    cq = conflicts(qw, sub_scans, sub_poses, o, eps)
    cm = conflicts(surf, [query_sensor], [reg_pose], o, eps)
    return dict(n_query=n_q, n_inliers=n_in, d2=d2, inlier=hit, grid=grid, sum_d2=total,
                overlap=n_in / n_q if n_q else 0.0, rmse=math.sqrt(total / n_in) if n_in else 0.0, query=cq, map=cm)

"""Scenes and exact restatements for so_map_clear_free_space_keyframes at its edges (test_free_space_keyframes_edges*.py).

The restatements, written apart from the device code:
  - `restate`: the removal set of the batched call is the union over its entries of free_space_numpy.removal_mask's removals, per
    carved store, and n_candidates is the size of the union of the candidate masks (each point once), summed over the carved stores;
    the image counters are the per-entry sums.  Per entry only the map points within max_range + 1 m of the sensor (FP64 brute
    distance) are evaluated: a point farther than max_range is no candidate by the rule's range gate, whatever the cull does.
    Points that free_space_numpy.edge_points marks as ambiguous for some entry are held between `bounds` instead.
  - `cull_lists`: so_free_rule.h's block box and reach test, for the fixture-validity checks.
  - `tile_plan`: floor(kFreeTileBytes / (4 W H)) images a tile, kFreeTileBytes read from so_free_rule.h.

Builders return sensor-frame clouds [n, 4] float32 for keyframe_import, poses [7] (x, y, z, qx, qy, qz, qw) and world-frame map
points [m, 4] float32 whose intensity is the point's index, so a downloaded store names its points.
"""
from __future__ import annotations

import math
import os
import re

import numpy as np

import free_space_numpy as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLOCK, HALF = 50.0, 25.0
WINDOW = (21, 21, 11)
DEFAULT_ORIGIN = (10, 10, 5)
IDENTITY = np.array([0.0, 0, 0, 0, 0, 0, 1])
YAW_180 = np.array([0.0, 0, 0, 0, 0, 1, 0])          # R = diag(-1, -1, 1), exact from the quaternion

# 2 x 2 degree pixels over -20..20 degrees: 180 x 20 = 3 600 pixels, one tile holds thousands of images
COARSE = F.Opts(az_res_deg=2.0, el_res_deg=2.0, el_min_deg=-20.0, el_max_deg=20.0, dilate=1, margin=0.3, margin_rel=0.02,
                min_range=0.5, max_range=60.0)
# 4096 x 4096 pixels (2^24, the largest image): 64 MiB an image, 4 a tile
BIG = F.Opts(az_res_deg=0.087890625, el_res_deg=0.0087890625, el_min_deg=-18.0, el_max_deg=18.0, dilate=1, margin=0.3,
             margin_rel=0.02, min_range=0.5, max_range=60.0)
# block faces: one pixel (dilate 0), az = 0 (FACE_X: 45 columns of 8 deg) or az = +-90 deg (FACE_Y: 90 columns of 4 deg) and el = 0 at
# pixel centres
FACE_X = F.Opts(az_res_deg=8.0, el_res_deg=8.0, el_min_deg=-20.0, el_max_deg=20.0, dilate=0, margin=0.3, margin_rel=0.0,
                min_range=0.5, max_range=60.0)
FACE_Y = F.Opts(az_res_deg=4.0, el_res_deg=8.0, el_min_deg=-20.0, el_max_deg=20.0, dilate=0, margin=0.3, margin_rel=0.0,
                min_range=0.5, max_range=60.0)


# ------------------------------------------------------------------------------------------------------------ header constants
def tile_bytes() -> int:
    with open(os.path.join(ROOT, "superodom_b200", "csrc", "so_free_rule.h")) as f:
        m = re.search(r"constexpr size_t kFreeTileBytes = size_t\((\d+)\) << (\d+);", f.read())
    return int(m.group(1)) << int(m.group(2))


def tile_plan(n_entries: int, o: F.Opts):
    """-> (images per tile, number of tiles) of a call with n_entries entries (keyframes below 2^31 points a tile)."""
    W, H = F.dims(o)
    per = max(tile_bytes() // (4 * W * H), 1)
    return per, max(1, -(-n_entries // per))


# ------------------------------------------------------------------------------------------------------------ window blocks
def grid_coord(v, origin):
    """free_coord: int() of the quotient, one less for negative sums"""
    c = np.trunc(v / BLOCK).astype(np.int64)
    return c - (v < 0) + origin


def grid_block(xyz, origin=DEFAULT_ORIGIN) -> np.ndarray:
    """free_grid_block of float32 points: the window block, or -1"""
    p = np.asarray(xyz, np.float32)[:, :3].astype(np.float64)
    with np.errstate(invalid="ignore"):
        g = [grid_coord(p[:, a] + HALF, origin[a]) for a in range(3)]
    ok = np.isfinite(p).all(1)
    for a in range(3):
        ok &= (g[a] >= 0) & (g[a] < WINDOW[a])
    return np.where(ok, g[0] + WINDOW[0] * g[1] + WINDOW[0] * WINDOW[1] * g[2], -1)


def block_box(b, origin=DEFAULT_ORIGIN, pad=True):
    b = np.asarray(b, np.int64)
    g = np.stack([b % WINDOW[0], (b // WINDOW[0]) % WINDOW[1], b // (WINDOW[0] * WINDOW[1])], -1)
    lo = (g - np.asarray(origin)).astype(np.float64) * BLOCK - HALF
    hi = lo + BLOCK
    p = 1e-9 * (np.abs(lo) + np.abs(hi) + BLOCK) if pad else 0.0
    return lo - p, hi + p


def cull_lists(blocks, poses7, max_range, origin=DEFAULT_ORIGIN):
    """-> bool [len(blocks), len(poses7)]: entry j is in block b's list (free_block_in_reach of the padded box, 1e-9 slack)"""
    lo, hi = block_box(blocks, origin)
    t = np.asarray(poses7, np.float64).reshape(-1, 7)[:, :3]
    d = np.maximum(lo[:, None, :] - t[None], 0.0) + np.maximum(t[None] - hi[:, None, :], 0.0)
    return ~(np.sqrt((d * d).sum(-1)) > float(np.float32(max_range)) * (1.0 + 1e-9))


# ------------------------------------------------------------------------------------------------------------ the restatement
def restate(stores, clouds, poses, o: F.Opts, eps: float = 1e-9, exact_gate: bool = False):
    """The batched call of entries (clouds[e] at poses[e]) on the stores (list of two float32 [n, 4] or None for a store not
    carved) -> dict: removed / cand / lower / upper / ambiguous (per store masks), n_candidates, n_removed, n_image_points,
    n_pixels_hit, n_ambiguous_map, n_ambiguous_scan.  exact_gate: range-gate ties are exact by construction (an exact rotation) and
    are not counted as ambiguous."""
    out = dict(removed=[], cand=[], lower=[], upper=[], ambiguous=[])
    for s in stores:
        n = 0 if s is None else len(s)
        for k in ("removed", "cand", "lower", "upper", "ambiguous"):
            out[k].append(np.zeros(n, bool))
    n_img = n_hit = amb_scan = 0
    mr = float(np.float32(o.max_range)) + 1.0
    for cloud, pose in zip(clouds, poses):
        pose = np.asarray(pose, np.float64)
        img, hit, n_p, n_h = F.range_image(cloud, o)
        n_img += n_p
        n_hit += n_h
        a_scan = int(F.edge_points(cloud, o).sum()) if len(cloud) else 0
        amb_scan += a_scan
        for k, s in enumerate(stores):
            if s is None or len(s) == 0:
                continue
            d = np.asarray(s, np.float64)[:, :3] - pose[:3]
            sel = np.nonzero(np.sqrt((d * d).sum(1)) <= mr)[0]
            if len(sel) == 0:
                continue
            sub = s[sel]
            rem, cand = F.removal_mask(sub, pose, img, hit, o)
            amb = F.edge_points(F.to_sensor(sub, pose), o) if exact_gate else F.edge_points(sub, o, pose)
            lo = hi = rem
            if a_scan or amb.any():
                lo, hi = F.bounds(sub, cloud, pose, o, eps)
                amb = amb | (lo != hi) | (a_scan > 0)
            out["removed"][k][sel] |= rem
            out["cand"][k][sel] |= cand
            out["lower"][k][sel] |= lo
            out["upper"][k][sel] |= hi
            out["ambiguous"][k][sel] |= amb
    out["n_candidates"] = sum(int(c.sum()) for c in out["cand"])
    out["n_removed"] = sum(int(r.sum()) for r in out["removed"])
    out["n_image_points"], out["n_pixels_hit"] = n_img, n_hit
    out["n_ambiguous_map"] = sum(int(a.sum()) for a in out["ambiguous"])
    out["n_ambiguous_scan"] = amb_scan
    return out


# ------------------------------------------------------------------------------------------------------------ geometry helpers
def quat(roll, pitch, yaw):
    cr, sr, cp, sp, cy, sy = (math.cos(roll / 2), math.sin(roll / 2), math.cos(pitch / 2), math.sin(pitch / 2), math.cos(yaw / 2),
                              math.sin(yaw / 2))
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def rot(pose7):
    """free_pose's matrix, operation by operation"""
    q = [float(v) for v in np.asarray(pose7, np.float64)[3:]]
    nq = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    x, y, z, w = q[0] / nq, q[1] / nq, q[2] / nq, q[3] / nq
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def direction(az, el):
    """unit vectors of (az, el) in radians"""
    return np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], -1)


def pixel_dir(o: F.Opts, row, col, u=0.5, v=0.5):
    """directions into pixel (row, col) at fraction (u, v) of its width and height"""
    az = np.radians(-180.0 + (np.asarray(col) + u) * o.az_res_deg)
    el = np.radians(o.el_min_deg + (np.asarray(row) + v) * o.el_res_deg)
    return direction(az, el)


def xyzi(p, intensity=None) -> np.ndarray:
    p = np.asarray(p, np.float64).reshape(-1, 3)
    i = np.arange(len(p)) if intensity is None else intensity
    return np.c_[p, i].astype(np.float32)


def degenerate_returns():
    """returns that never reach an image: NaN and inf coordinates, the origin (r = 0), and points above and below the span"""
    pts = []
    for k in range(3):
        for v in (math.nan, math.inf, -math.inf):
            p = [1.0, 0.5, 0.25]
            p[k] = v
            pts.append(p)
    pts += [[0.0, 0.0, 0.0], [-0.0, -0.0, -0.0], [10.0, 0.0, 9.0], [-7.0, 3.0, -8.0], [0.0, 0.0, 25.0]]
    return np.array(pts)


# ------------------------------------------------------------------------------------------------------- case 1: spread keyframes
def spread_cloud(rng, o=COARSE, keep=0.85, r_lo=25.0, r_hi=90.0, extra=500):
    """A return inside most pixels (at 0.15..0.85 of the pixel, never near an edge), ranges uniform, plus `extra` returns in random
    directions (some outside the span)."""
    W, H = F.dims(o)
    rr, cc = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    m = rng.random(rr.size) < keep
    rr, cc = rr.reshape(-1)[m], cc.reshape(-1)[m]
    d = pixel_dir(o, rr, cc, rng.uniform(0.15, 0.85, len(rr)), rng.uniform(0.15, 0.85, len(rr)))
    p = d * rng.uniform(r_lo, r_hi, len(rr))[:, None]
    az, el = rng.uniform(-np.pi, np.pi, extra), np.radians(rng.uniform(-30.0, 30.0, extra))
    p = np.vstack([p, direction(az, el) * rng.uniform(3.0, 90.0, extra)[:, None]])
    return xyzi(p[rng.permutation(len(p))], np.ones(len(p)))


def spread_poses(rng, n_inside=290, n_outside=20, n_beyond=10):
    """Keyframes over most of the window and five z layers (yaw anywhere, roll and pitch up to ~0.3 rad, a few at 0.6), some just
    outside the window reaching its edge blocks, some beyond reach of every block; in random order."""
    out = []
    layers = np.array([-100.0, -40.0, 0.0, 35.0, 90.0])
    for _ in range(n_inside):
        out.append([rng.uniform(-490, 490), rng.uniform(-490, 490), rng.choice(layers) + rng.normal(0, 3.0)])
    for k in range(n_outside):                          # 5..50 m outside a face of the window (x, y in [-525, 525), z in [-275, 275))
        a, s = k % 3, 1 if k % 2 else -1
        p = [rng.uniform(-450, 450), rng.uniform(-450, 450), rng.uniform(-60, 60)]
        p[a] = s * ((525.0 if a < 2 else 275.0) + rng.uniform(5.0, 50.0))
        out.append(p)
    for k in range(n_beyond):                           # more than 60 m from every block
        a, s = k % 3, 1 if k % 2 else -1
        p = [rng.uniform(-300, 300), rng.uniform(-300, 300), rng.uniform(-60, 60)]
        p[a] = s * ((525.0 if a < 2 else 275.0) + rng.uniform(70.0, 300.0))
        out.append(p)
    poses = []
    for i, t in enumerate(out):
        big = rng.random() < 0.1
        rp = rng.normal(0, 0.6 if big else 0.12, 2).clip(-0.7, 0.7)
        poses.append(np.r_[t, quat(rp[0], rp[1], rng.uniform(-np.pi, np.pi))])
    poses = np.array(poses)
    return poses[rng.permutation(len(poses))]


def spread_map(rng, per_block=40, gz=range(2, 9), stride=1):
    """per_block uniform points in every window block of the z layers gz (and every stride-th block), world frame"""
    pts = []
    for k in gz:
        for j in range(0, WINDOW[1], stride):
            for i in range(0, WINDOW[0], stride):
                lo = (np.array([i, j, k]) - np.array(DEFAULT_ORIGIN)) * BLOCK - HALF
                pts.append(lo + rng.uniform(0.5, BLOCK - 0.5, (per_block, 3)))
    return np.vstack(pts)


def spread_case(seed=7, n_keyframes=320):
    rng = np.random.default_rng(seed)
    poses = spread_poses(rng, n_keyframes - 30)
    clouds = [spread_cloud(rng, keep=rng.uniform(0.7, 0.95)) for _ in range(len(poses))]
    surf = xyzi(spread_map(rng, 36))
    edge = xyzi(spread_map(rng, 14, stride=1), np.arange(14 * 21 * 21 * 7) + 10 ** 6)
    return dict(opts=COARSE, poses=poses, clouds=clouds, surf=surf, edge=edge)


SPREAD_SIZES = (1, 31, 32, 33, 127, 128, 129, 257, 320)


# ------------------------------------------------------------------------------------------------------- case 2: block faces
def _f32_step(v, toward):
    return float(np.nextafter(np.float32(v), np.float32(toward)))


def face_distances(max_range=60.0):
    """FP64 sensor ranges at the range gate: float(max_range) and one float32 and one FP64 step either side"""
    m = float(np.float32(max_range))
    return [_f32_step(m, 0), float(np.nextafter(m, 0.0)), m, float(np.nextafter(m, np.inf)), _f32_step(m, 1e9)]


def face_case(axis: int):
    """Map points on the x (axis 0) or y (axis 1) faces 25 + 50 k, k = -6..5 (both signs: the negative faces bucket by int() and
    c--, onto the block's upper face), each seen by one keyframe straight across the face at one of face_distances(), with one return
    behind it (the pixel at az 0 or +-90 deg, el 0).  Identity and 180 deg yaw poses: r_m is the FP64 difference itself.  Points lie
    10 m apart along the face, so no keyframe's pixel holds another's point."""
    o = FACE_X if axis == 0 else FACE_Y
    clouds, poses, pts, want = [], [], [], []
    dists = face_distances(o.max_range)
    n = 0
    for k in range(-6, 6):
        f = 25.0 + 50.0 * k
        upper = f + HALF < 0                          # the point buckets into the block below the face: the keyframe sits above it
        for j, dist in enumerate(dists):
            other = -270.0 + 10.0 * n                 # the point's place along the face
            n += 1
            m = np.zeros(3)
            m[axis], m[1 - axis], m[2] = f, other, 3.0 + 0.25 * j
            t = m.copy()
            t[axis] = f + dist if upper else f - dist
            if abs(t[axis] - m[axis]) != dist:          # an FP64 step of 60 m that the keyframe's coordinate cannot hold
                continue
            if axis == 0:
                pose = np.r_[t, YAW_180[3:] if upper else IDENTITY[3:]]   # the point at sensor +x
                d = np.array([1.0, 0.0, 0.0])
            else:
                pose = np.r_[t, IDENTITY[3:]]                              # the point at sensor -y or +y
                d = np.array([0.0, -1.0 if upper else 1.0, 0.0])
            clouds.append(xyzi(d * 100.0, np.ones(1)))
            poses.append(pose)
            pts.append(m)
            want.append(dist <= float(np.float32(o.max_range)))
    return dict(opts=o, clouds=clouds, poses=np.array(poses), surf=xyzi(pts), want=np.array(want))


def device_range(m, pose7):
    """r_m of free_decide restated operation by operation (no fused multiply-add): d = m - t, q_a = (d_x R_0a + d_y R_1a) + d_z R_2a,
    sqrt((q_x^2 + q_y^2) + q_z^2), R from free_pose's normalised quaternion"""
    R = rot(pose7)
    d = np.asarray(m, np.float32)[:, :3].astype(np.float64) - np.asarray(pose7, np.float64)[:3]
    q = [(d[:, 0] * R[0, a] + d[:, 1] * R[1, a]) + d[:, 2] * R[2, a] for a in range(3)]
    return np.sqrt((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2])


def face_near_case(rng, rows=30):
    """Points on x faces, each with a keyframe straight across at an FP64 distance a few steps above max_range (so the box is out
    of reach without the pad and the slack) under a small rotation: the rounding of the rotation puts some of them at r_m <= max_range,
    in range.  One return behind each point in a 3 x 3 patch of FACE_X pixels (dilate 1).  Points on one face lie 18 m apart, those
    of neighbouring faces 3.3 m apart in z, so no keyframe's patch holds another keyframe's point."""
    o = F.Opts(**{**FACE_X.__dict__, "dilate": 1})
    m_r = float(np.float32(o.max_range))
    clouds, poses, pts = [], [], []
    for i in range(12 * rows):
        k = i % 12 - 6
        f = 25.0 + 50.0 * k
        upper = f + HALF < 0
        m = np.array([f, -270.0 + 18.0 * (i // 12), -18.0 + 3.3 * (i % 12)])
        t = m.copy()
        t[0] = f + m_r if upper else f - m_r
        away = np.inf if upper else -np.inf
        for _ in range(int(rng.integers(1, 4))):        # one to three FP64 steps beyond max_range, as the difference rounds
            t[0] = float(np.nextafter(t[0], away))
            while not abs(f - t[0]) > m_r:
                t[0] = float(np.nextafter(t[0], away))
        yaw = (np.pi if upper else 0.0) + rng.normal(0, 0.02)
        pose = np.r_[t, quat(rng.normal(0, 0.02), rng.normal(0, 0.02), yaw)]
        q = (m - t) @ rot(pose)
        q /= np.linalg.norm(q)
        az, el = math.atan2(q[1], q[0]), math.asin(q[2])
        cloud = [direction(az + a * np.radians(o.az_res_deg), el + e * np.radians(o.el_res_deg)) * 100.0 for a in (-1, 0, 1)
                 for e in (-1, 0, 1)]
        clouds.append(xyzi(cloud, np.ones(9)))
        poses.append(pose)
        pts.append(m)
    return dict(opts=o, clouds=clouds, poses=np.array(poses), surf=xyzi(pts))


# ------------------------------------------------------------------------------------------------------- case 3: tile seams
def _interactions(o, entries, ids, poses, plan, n_points, rng, r_range=(12.0, 30.0)):
    """Map points placed against the entries of `plan`: a list of point kinds, each a list of (entry, "front" | "behind") -- the
    entry's cloud gets a 3 x 3 patch of returns around the point's pixel at r_m - 2 m (a candidate, kept) or r_m + 6 m (removed).
    Every point is placed at the centre of a fresh pixel of its first entry.  -> (world points [n, 3], kind per point, returns per id)"""
    W, H = F.dims(o)
    rets = {i: [] for i in set(ids)}
    pts, kind = [], []
    for kd, inter in enumerate(plan):
        placed = 0
        while placed < n_points:
            e0 = inter[0][0]
            row, col = int(rng.integers(H // 4, 3 * H // 4)), int(rng.integers(0, W))
            r = rng.uniform(*r_range)
            p0 = poses[e0]
            m = p0[:3] + rot(p0) @ (pixel_dir(o, row, col) * r)
            m = np.asarray(m, np.float32).astype(np.float64)
            patches = []
            for e, how in inter:
                q = (m - poses[e][:3]) @ rot(poses[e])
                rm = float(np.linalg.norm(q))
                az = math.atan2(q[1], q[0])
                el = math.atan2(q[2], math.hypot(q[0], q[1]))
                c = int(math.floor((az + math.pi) / math.radians(o.az_res_deg))) % W
                rw = int(math.floor((el - math.radians(o.el_min_deg)) / math.radians(o.el_res_deg)))
                patches.append((ids[e], rw, c, rm - 2.0 if how == "front" else rm + 6.0, rm))
            if not all(H // 8 <= rw < H - H // 8 and 8.0 <= rm <= 45.0 for _, rw, _, _, rm in patches):
                continue                                  # out of another entry's span or range: place it again
            for i, rw, c, rr, _ in patches:
                for dr in (-1, 0, 1):
                    for dc in (-1, 0, 1):
                        rets[i].append(pixel_dir(o, rw + dr, (c + dc) % W) * rr)
            placed += 1
            pts.append(m)
            kind.append(kd)
    return np.array(pts), np.array(kind), rets


# The tile-seam entries (BIG: 4 a tile): E* are empty keyframes; K1 closes tile 0 and opens tile 1 with another pose; tile 2 holds only
# empty keyframes
SEAM_LAYOUT = ["E0", "K0", "E1", "K1", "K1b", "K2", "K3", "E2", "E0", "E1", "E2", "E0", "K4"]
# point kinds, as (entry index, how) lists
SEAM_KINDS = {
    "candidate in tile 0, removed in tile 1": [(1, "front"), (5, "behind")],
    "candidate only in tile 3": [(12, "front")],
    "removed only in tile 3": [(12, "behind")],
    "removed in tile 0, candidate of tile 1": [(3, "behind"), (6, "front")],
    "candidate in tiles 0 and 1, kept": [(1, "front"), (6, "front")],
    "candidate under one pose, removed under the other (same id)": [(3, "front"), (4, "behind")],
    "removed in tile 1 by its last non-empty entry": [(6, "behind")],
}


def seam_case(seed=3, n_points=12, clutter=2500):
    """-> dict(opts, keyframes: {name: (cloud, import pose)}, names (entry -> keyframe name), poses [13, 7] (entry poses), surf,
    edge, kinds (per surf / edge point, index into SEAM_KINDS or -1 for clutter))"""
    rng = np.random.default_rng(seed)
    o = BIG
    base = {"K0": np.r_[3.0, -2.0, 0.25, IDENTITY[3:]], "K1": np.r_[-4.0, 6.0, -0.25, IDENTITY[3:]],
            "K2": np.r_[8.0, 5.0, 0.0, YAW_180[3:]], "K3": np.r_[-7.0, -9.0, 0.0, IDENTITY[3:]],
            "K4": np.r_[1.0, 12.0, 0.25, YAW_180[3:]]}
    names = list(SEAM_LAYOUT)
    entry_poses = []
    for nm in names:
        if nm == "K1b":
            entry_poses.append(np.r_[2.0, -6.0, 0.25, IDENTITY[3:]])
        elif nm.startswith("K"):
            entry_poses.append(base[nm])
        else:
            entry_poses.append(IDENTITY.copy())
    ids = [("K1" if nm == "K1b" else nm) for nm in names]
    kinds = list(SEAM_KINDS.values())
    sp, sk, rets = _interactions(o, names, ids, entry_poses, kinds, n_points, rng)
    ep, ek, rets_e = _interactions(o, names, ids, entry_poses, kinds, n_points // 2, rng)
    for k, v in rets_e.items():
        rets[k] += v
    keyframes = {}
    for nm in sorted(set(ids)):
        if nm.startswith("E"):
            keyframes[nm] = (np.zeros((0, 4), np.float32), IDENTITY.copy())
            continue
        designed = np.array(rets[nm]).reshape(-1, 3)
        az, el = rng.uniform(-np.pi, np.pi, clutter), np.radians(rng.uniform(-17.0, 17.0, clutter))
        far = direction(az, el) * rng.uniform(61.0, 90.0, clutter)[:, None]    # clutter beyond every designed point's reach
        deg = degenerate_returns()
        half = len(far) // 2
        # designed returns first, so the first point of each segment is one a wrong segment search would misplace
        cloud = np.vstack([designed, far[:half], deg[:7], far[half:], deg[7:]])
        keyframes[nm] = (xyzi(cloud, np.ones(len(cloud))), base.get(nm, IDENTITY))
    clutter_map = direction(rng.uniform(-np.pi, np.pi, 3000), np.radians(rng.uniform(-17.0, 17.0, 3000))) * rng.uniform(1.0, 58.0, 3000)[:, None]
    surf = np.vstack([sp, clutter_map[:2000]])
    edge = np.vstack([ep, clutter_map[2000:]])
    return dict(opts=o, keyframes=keyframes, names=names, ids=ids, poses=np.array(entry_poses),
                surf=xyzi(surf), edge=xyzi(edge, np.arange(len(edge)) + 10 ** 6),
                kinds=(np.r_[sk, -np.ones(2000, int)], np.r_[ek, -np.ones(1000, int)]))

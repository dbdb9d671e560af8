"""Seeded synthetic worlds, maps and LiDAR scans (SURVEY.md section 8d).

Shared by the oracle tests, the GPU parity tests and bench.py so that all of
them see identical bytes.  Nothing here touches the GPU or the oracle.

World: an analytic "warehouse" -- a closed room (ground z=-1.8 m, ceiling
z=+6 m, four outer walls) filled with axis-aligned boxes (shelving rows and
floor-to-ceiling pillars).  No face plane lies within 1 m of the world origin
(the reference plane fit ``A n = -1`` is undefined for planes through the
origin, LidarSlam.cpp:798-806).

Map: every face sampled on a lattice of pitch = leaf, jittered by
N(0, (0.02 m)^2) per axis (keeps the PCA gate lambda0 >= 1e-6 alive,
LidarSlam.cpp:772, and removes distance ties), then passed through the
per-block voxel-centroid filter of the reference insert path
(LocalMap.h:591-645; semantics of pcl::VoxelGrid restated in
``voxel_filter_blocks``).

Scans: ray-cast from a ground-truth pose, range noise N(0,(0.01 m)^2), returns
outside [0.2, 130] m dropped (featureExtraction.cpp:128-129 defaults).
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

BLOCK = 50.0          # LocalMap::voxelResulation (LocalMap.h:136)
HALF_BLOCK = 25.0     # LocalMap::halfVoxelResulation
GRID = (21, 21, 11)   # laserCloudWidth/Height/Depth (LocalMap.h:131-133)
ORIGIN0 = (10, 10, 5) # LocalMap() constructor origin (LocalMap.h:141-144)


# --------------------------------------------------------------------------
# scene
# --------------------------------------------------------------------------
@dataclasses.dataclass
class Scene:
    room: np.ndarray    # [6] xmin,xmax,ymin,ymax,zmin,zmax
    boxes: np.ndarray   # [nb,6] same layout

    def free(self, p: np.ndarray, margin: float = 0.6) -> bool:
        r = self.room
        if not (r[0] + margin < p[0] < r[1] - margin and r[2] + margin < p[1] < r[3] - margin
                and r[4] + 0.3 < p[2] < r[5] - 0.3):
            return False
        b = self.boxes
        inside = ((p[0] > b[:, 0] - margin) & (p[0] < b[:, 1] + margin) &
                  (p[1] > b[:, 2] - margin) & (p[1] < b[:, 3] + margin) &
                  (p[2] > b[:, 4] - margin) & (p[2] < b[:, 5] + margin))
        return not bool(inside.any())


def make_scene(half_extent: float, seed: int = 77, aisle: float = 5.0, half_extent_y: float | None = None,
               center=(0.0, 0.0)) -> Scene:
    """Room [-h,h] x [-hy,hy] x [-1.8,6] (then translated by `center`) with shelving rows every `aisle` metres and pillars."""
    sc = _make_scene_centered(float(half_extent), float(half_extent if half_extent_y is None else half_extent_y), seed, aisle)
    cx, cy = float(center[0]), float(center[1])
    if cx or cy:
        sh = np.array([cx, cx, cy, cy, 0.0, 0.0])
        sc = Scene(room=sc.room + sh, boxes=sc.boxes + sh)
    return sc


def _make_scene_centered(h: float, hy: float, seed: int, aisle: float) -> Scene:
    rng = np.random.default_rng(seed)
    room = np.array([-h, h, -hy, hy, -1.8, 6.0])
    boxes = []
    # shelving rows: long boxes parallel to x, broken into segments with gaps
    y = -hy + aisle
    row = 0
    while y < hy - aisle + 1e-9:
        if abs(y) >= 2.0:           # keep faces |y| >= 1 and the origin aisle free
            x = -h + 2.0
            while x < h - 2.0:
                seg = float(rng.uniform(4.0, 9.0))
                x1 = min(x + seg, h - 2.0)
                if x1 - x > 1.5 and not (x < 1.0 and x1 > -1.0):
                    top = float(rng.uniform(1.2, 4.5))      # box top z (>= 1 m from origin plane)
                    depth = float(rng.uniform(0.6, 1.4))
                    boxes.append([x, x1, y - depth / 2, y + depth / 2, -1.8, top])
                x = x1 + float(rng.uniform(1.5, 3.0))
        y += aisle
        row += 1
    # pillars (floor to ceiling) on a coarse lattice, jittered
    step = max(10.0, h / 4)
    for px in np.arange(-h + step / 2, h, step):
        for py in np.arange(-hy + step / 2 + 2.5, hy, step):
            cx = float(px + rng.uniform(-1, 1))
            cy = float(py + rng.uniform(-1, 1))
            if abs(cx) < 2.0 or abs(cy) < 2.0:
                continue
            s = float(rng.uniform(0.4, 0.8))
            boxes.append([cx - s, cx + s, cy - s, cy + s, -1.8, 6.0])
    boxes = np.array(boxes, dtype=np.float64).reshape(-1, 6)
    # enforce: no face plane within 1 m of the origin on any axis
    for ax in range(3):
        for side in (0, 1):
            c = boxes[:, 2 * ax + side]
            bad = np.abs(c) < 1.0
            c[bad] = np.where(c[bad] >= 0, 1.0 + 0.05 * ax, -1.0 - 0.05 * ax)
    keep = (boxes[:, 1] - boxes[:, 0] > 0.2) & (boxes[:, 3] - boxes[:, 2] > 0.2) & (boxes[:, 5] - boxes[:, 4] > 0.2)
    return Scene(room=room, boxes=boxes[keep])


def _face_samples(lo_u, hi_u, lo_v, hi_v, pitch):
    nu = max(1, int(math.floor((hi_u - lo_u) / pitch)))
    nv = max(1, int(math.floor((hi_v - lo_v) / pitch)))
    u = lo_u + (np.arange(nu) + 0.5) * pitch
    v = lo_v + (np.arange(nv) + 0.5) * pitch
    uu, vv = np.meshgrid(u, v, indexing="ij")
    return uu.ravel(), vv.ravel()


def _inside_any_numpy(pts, boxes, eps):
    ins_any = np.zeros(len(pts), dtype=bool)
    for b in boxes:
        ins_any |= ((pts[:, 0] > b[0] + eps) & (pts[:, 0] < b[1] - eps) & (pts[:, 1] > b[2] + eps) &
                    (pts[:, 1] < b[3] - eps) & (pts[:, 2] > b[4] + eps) & (pts[:, 2] < b[5] - eps))
    return ins_any


try:
    import numba as _nb0

    @_nb0.njit(parallel=True, cache=True)
    def _inside_any(pts, boxes, eps):
        n = pts.shape[0]
        out = np.zeros(n, np.bool_)
        for i in _nb0.prange(n):
            x = pts[i, 0]
            y = pts[i, 1]
            z = pts[i, 2]
            for b in range(boxes.shape[0]):
                if (x > boxes[b, 0] + eps and x < boxes[b, 1] - eps and y > boxes[b, 2] + eps and y < boxes[b, 3] - eps
                        and z > boxes[b, 4] + eps and z < boxes[b, 5] - eps):
                    out[i] = True
                    break
        return out
except Exception:                                             # pragma: no cover
    _inside_any = _inside_any_numpy


def sample_surfaces(scene: Scene, pitch: float, seed: int = 1234, noise: float = 0.02) -> np.ndarray:
    """Raw (unfiltered) surface samples, float32 [M,3]."""
    rng = np.random.default_rng(seed)
    chunks = []

    def add_box_faces(b, inward):
        x0, x1, y0, y1, z0, z1 = b
        for zc in (z0, z1):
            u, v = _face_samples(x0, x1, y0, y1, pitch)
            chunks.append(np.stack([u, v, np.full_like(u, zc)], 1))
        for xc in (x0, x1):
            u, v = _face_samples(y0, y1, z0, z1, pitch)
            chunks.append(np.stack([np.full_like(u, xc), u, v], 1))
        for yc in (y0, y1):
            u, v = _face_samples(x0, x1, z0, z1, pitch)
            chunks.append(np.stack([u, np.full_like(u, yc), v], 1))

    add_box_faces(scene.room, True)
    for b in scene.boxes:
        add_box_faces(b, False)
    pts = np.concatenate(chunks, 0)
    # drop samples strictly inside another box (hidden)
    pts = pts[~_inside_any(pts, np.ascontiguousarray(scene.boxes), 1e-6)]
    pts = pts + rng.normal(0.0, noise, size=pts.shape)
    return pts.astype(np.float32)


def sample_edges(scene: Scene, pitch: float, seed: int = 4321, noise: float = 0.01) -> np.ndarray:
    """Points along the 12 edges of every box (the line features a curvature-based extractor would emit), float32 [M,3]."""
    rng = np.random.default_rng(seed)
    chunks = []
    for b in scene.boxes:
        x0, x1, y0, y1, z0, z1 = b
        for (ax, lo, hi, others) in ((0, x0, x1, [(y, z) for y in (y0, y1) for z in (z0, z1)]),
                                     (1, y0, y1, [(x, z) for x in (x0, x1) for z in (z0, z1)]),
                                     (2, z0, z1, [(x, y) for x in (x0, x1) for y in (y0, y1)])):
            n = max(2, int((hi - lo) / pitch))
            t = lo + (np.arange(n) + 0.5) * (hi - lo) / n
            for (u, v) in others:
                p = np.zeros((n, 3))
                p[:, ax] = t
                oth = [a for a in range(3) if a != ax]
                p[:, oth[0]] = u
                p[:, oth[1]] = v
                chunks.append(p)
    pts = np.concatenate(chunks, 0) + rng.normal(0.0, noise, size=(sum(len(c) for c in chunks), 3))
    return pts.astype(np.float32)


def make_edge_map(scene: Scene, line_res: float) -> np.ndarray:
    raw = sample_edges(scene, line_res)
    xyzi = np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1)
    return voxel_filter_blocks(xyzi, line_res)


def make_edge_scan(edge_map_xyzi: np.ndarray, pose7: np.ndarray, seed: int, max_range: float = 30.0, keep_every: int = 3,
                   noise: float = 0.01) -> np.ndarray:
    """Edge points as the sensor would see them: nearby edge-map points, perturbed, expressed in the SENSOR frame."""
    rng = np.random.default_rng(seed)
    P = edge_map_xyzi[:, :3].astype(np.float64)
    d = np.linalg.norm(P - pose7[:3], axis=1)
    P = P[d < max_range][::keep_every]
    P = P + rng.normal(0.0, noise, size=P.shape)
    R = quat_to_R(pose7[3:])
    local = (P - pose7[:3]) @ R                      # R^T (p - t)
    return np.concatenate([local, np.ones((len(local), 1))], 1).astype(np.float32)


# --------------------------------------------------------------------------
# block binning + voxel-centroid filter (restates LocalMap.h:591-645 + pcl::VoxelGrid)
# --------------------------------------------------------------------------
def block_of(xyz: np.ndarray, origin=ORIGIN0) -> np.ndarray:
    """LocalMap.h:594-605: int((x+25)/50)+origin, minus one when x+25<0 (double arithmetic
    on float coordinates).  Returns int32 [n,3] grid indices (may be off-grid)."""
    v = xyz.astype(np.float64) + HALF_BLOCK
    c = np.trunc(v / BLOCK).astype(np.int64) + np.asarray(origin, dtype=np.int64)
    c -= (v < 0).astype(np.int64)
    return c.astype(np.int32)


def block_linear(c: np.ndarray) -> np.ndarray:
    """cubeInd = i + 21*j + 21*21*k, -1 when off-grid (LocalMap.h:607-609)."""
    ok = ((c[:, 0] >= 0) & (c[:, 0] < GRID[0]) & (c[:, 1] >= 0) & (c[:, 1] < GRID[1]) &
          (c[:, 2] >= 0) & (c[:, 2] < GRID[2]))
    lin = c[:, 0].astype(np.int64) + GRID[0] * c[:, 1].astype(np.int64) + GRID[0] * GRID[1] * c[:, 2].astype(np.int64)
    return np.where(ok, lin, -1)


def voxel_filter_blocks(xyzi: np.ndarray, leaf: float, origin=ORIGIN0) -> np.ndarray:
    """Per-block voxel-centroid filter.

    pcl::VoxelGrid semantics (PCL 1.12 voxel_grid.hpp, third-party, not in /root/reference):
    voxel = floor(coord * (1.0f/leaf)) per axis in float32; one output point per occupied
    voxel = centroid of all fields, accumulated in float32 and divided by float(count);
    output ordered by block, then by voxel index (k, j, i ascending).  PCL leaves the
    in-voxel accumulation order unspecified (std::sort on the voxel index only); this
    restatement fixes it to ascending input order.
    xyzi: float32 [n,4] (x,y,z,intensity).  Returns float32 [m,4]."""
    xyzi = np.ascontiguousarray(xyzi, dtype=np.float32)
    lin = block_linear(block_of(xyzi[:, :3], origin))
    keep = lin >= 0
    xyzi = xyzi[keep]
    lin = lin[keep]
    inv = np.float32(1.0) / np.float32(leaf)
    ijk = np.floor(xyzi[:, :3] * inv).astype(np.int64)
    # sort key: block, k, j, i  (stable -> in-voxel order = input order)
    order = np.lexsort((ijk[:, 0], ijk[:, 1], ijk[:, 2], lin))
    xyzi = xyzi[order]
    key = np.stack([lin[order], ijk[order, 2], ijk[order, 1], ijk[order, 0]], 1)
    new = np.ones(len(key), dtype=bool)
    new[1:] = (key[1:] != key[:-1]).any(1)
    seg = np.cumsum(new) - 1
    nseg = int(seg[-1]) + 1 if len(seg) else 0
    start = np.flatnonzero(new)
    rank = np.arange(len(key)) - start[seg]
    acc = np.zeros((nseg, 4), dtype=np.float32)
    for r in range(int(rank.max()) + 1 if len(rank) else 0):
        m = rank == r
        acc[seg[m]] = acc[seg[m]] + xyzi[m]           # float32 sequential accumulation
    cnt = np.bincount(seg, minlength=nseg).astype(np.float32)
    return (acc / cnt[:, None]).astype(np.float32)


def make_map(half_extent: float, leaf: float, scene_seed: int = 77, map_seed: int = 1234, half_extent_y=None, center=(0.0, 0.0)):
    scene = make_scene(half_extent, seed=scene_seed, half_extent_y=half_extent_y, center=center)
    raw = sample_surfaces(scene, leaf, seed=map_seed)
    xyzi = np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1)
    return scene, voxel_filter_blocks(xyzi, leaf)


# --------------------------------------------------------------------------
# poses  (pose7 = tx,ty,tz,qx,qy,qz,qw  -- the reference's pose_parameters layout, LidarSlam.cpp:7-9)
# --------------------------------------------------------------------------
def quat_mul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by,
                     aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx,
                     aw * bw - ax * bx - ay * by - az * bz])


def quat_from_rotvec(w):
    th = float(np.linalg.norm(w))
    if th < 1e-12:
        return np.array([0.5 * w[0], 0.5 * w[1], 0.5 * w[2], 1.0])
    s = math.sin(th / 2) / th
    return np.array([w[0] * s, w[1] * s, w[2] * s, math.cos(th / 2)])


def quat_to_R(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def random_sensor_pose(scene: Scene, seed: int, max_radius: float = 20.0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    cx = 0.5 * (scene.room[0] + scene.room[1])
    cy = 0.5 * (scene.room[2] + scene.room[3])
    for _ in range(1000):
        r = rng.uniform(0.0, max_radius)
        a = rng.uniform(0, 2 * math.pi)
        p = np.array([cx + r * math.cos(a), cy + r * math.sin(a), rng.uniform(-0.6, 0.6)])
        if scene.free(p):
            break
    else:
        raise RuntimeError("no free sensor position")
    yaw = rng.uniform(-math.pi, math.pi)
    rp = rng.uniform(-0.03, 0.03, size=2)
    q = quat_mul(quat_from_rotvec(np.array([0, 0, yaw])), quat_from_rotvec(np.array([rp[0], rp[1], 0.0])))
    q /= np.linalg.norm(q)
    return np.concatenate([p, q])


def perturb_pose(pose7: np.ndarray, seed: int, dt: float = 0.10, dth_deg: float = 1.0) -> np.ndarray:
    """T_prior = T* [+] (dt, dtheta): dt ~ U(-dt,dt) m, dtheta ~ U(-dth,dth) deg per axis."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(-dt, dt, size=3)
    w = np.deg2rad(rng.uniform(-dth_deg, dth_deg, size=3))
    q = quat_mul(pose7[3:], quat_from_rotvec(w))
    q /= np.linalg.norm(q)
    return np.concatenate([pose7[:3] + d, q])


# --------------------------------------------------------------------------
# sensors + ray casting
# --------------------------------------------------------------------------
_DIRS_CACHE = {}


def sensor_dirs(sensor: str, seed: int = 0) -> np.ndarray:
    key = (sensor, seed if sensor == "mid360" else 0)
    if key not in _DIRS_CACHE:
        _DIRS_CACHE[key] = _sensor_dirs(sensor, seed)
    return _DIRS_CACHE[key]


def _sensor_dirs(sensor: str, seed: int = 0) -> np.ndarray:
    if sensor == "vlp16":
        el = np.deg2rad(np.arange(-15.0, 15.1, 2.0))
        az = np.arange(1800) * (2 * math.pi / 1800)
    elif sensor == "os1_128":
        el = np.deg2rad(np.linspace(-22.5, 22.5, 128))
        az = np.arange(1024) * (2 * math.pi / 1024)
    elif sensor == "mid360":
        rng = np.random.default_rng(seed + 555)
        n = 240000
        azr = rng.uniform(0, 2 * math.pi, n)
        elr = np.deg2rad(rng.uniform(-7.0, 52.0, n))
        return np.stack([np.cos(elr) * np.cos(azr), np.cos(elr) * np.sin(azr), np.sin(elr)], 1)
    else:
        raise ValueError(sensor)
    # azimuth-major (column firing order), rings inner
    A, E = np.meshgrid(az, el, indexing="ij")
    return np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3)


def _raycast_numpy(room, boxes, o, d):
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        lo = np.array([room[0], room[2], room[4]])
        hi = np.array([room[1], room[3], room[5]])
        t1 = (lo - o) * inv
        t2 = (hi - o) * inv
        best = np.min(np.maximum(t1, t2), axis=1)            # inside the room: exit distance
        for b in boxes:
            lo = np.array([b[0], b[2], b[4]])
            hi = np.array([b[1], b[3], b[5]])
            t1 = (lo - o) * inv
            t2 = (hi - o) * inv
            tn = np.max(np.minimum(t1, t2), axis=1)
            tf = np.min(np.maximum(t1, t2), axis=1)
            hit = (tn <= tf) & (tn > 0)
            best = np.where(hit & (tn < best), tn, best)
    return best


try:                                                          # numba (in the image) makes scan generation ~100x faster
    import numba as _nb

    @_nb.njit(parallel=True, cache=True)
    def _raycast_numba(room, boxes, o, d):
        n = d.shape[0]
        nb = boxes.shape[0]
        out = np.empty(n, np.float64)
        # box bounds relative to the ray origin
        rel = np.empty((nb, 6), np.float64)
        for b in range(nb):
            for a in range(3):
                rel[b, 2 * a] = boxes[b, 2 * a] - o[a]
                rel[b, 2 * a + 1] = boxes[b, 2 * a + 1] - o[a]
        for i in _nb.prange(n):
            inv0 = 1.0 / d[i, 0] if d[i, 0] != 0.0 else np.inf
            inv1 = 1.0 / d[i, 1] if d[i, 1] != 0.0 else np.inf
            inv2 = 1.0 / d[i, 2] if d[i, 2] != 0.0 else np.inf
            # room (we are inside): exit distance
            best = np.inf
            for a in range(3):
                da = d[i, a]
                if da != 0.0:
                    t1 = (room[2 * a] - o[a]) / da
                    t2 = (room[2 * a + 1] - o[a]) / da
                    tm = t1 if t1 > t2 else t2
                    if tm < best:
                        best = tm
            for b in range(nb):
                # slab test; a zero direction component gives +-inf (or nan when the origin lies on the slab plane,
                # which the comparisons below treat as a miss)
                t1 = rel[b, 0] * inv0
                t2 = rel[b, 1] * inv0
                tn = t1 if t1 < t2 else t2
                tf = t1 if t1 > t2 else t2
                if tn >= best:
                    continue
                t1 = rel[b, 2] * inv1
                t2 = rel[b, 3] * inv1
                lo = t1 if t1 < t2 else t2
                hi = t1 if t1 > t2 else t2
                if lo > tn:
                    tn = lo
                if hi < tf:
                    tf = hi
                if tn > tf or tn >= best:
                    continue
                t1 = rel[b, 4] * inv2
                t2 = rel[b, 5] * inv2
                lo = t1 if t1 < t2 else t2
                hi = t1 if t1 > t2 else t2
                if lo > tn:
                    tn = lo
                if hi < tf:
                    tf = hi
                if tn <= tf and tn > 0.0 and tn < best:
                    best = tn
            out[i] = best
        return out
except Exception:                                             # pragma: no cover
    _raycast_numba = None


def raycast(scene: Scene, o: np.ndarray, d: np.ndarray) -> np.ndarray:
    """Range to the first surface along each ray (origin o [3], dirs d [n,3]); inf if none."""
    o = np.ascontiguousarray(o, dtype=np.float64)
    d = np.ascontiguousarray(d, dtype=np.float64)
    if _raycast_numba is not None:
        return _raycast_numba(np.ascontiguousarray(scene.room), np.ascontiguousarray(scene.boxes), o, d)
    return _raycast_numpy(scene.room, scene.boxes, o, d)


def make_scan(scene: Scene, sensor: str, pose7: np.ndarray, seed: int,
              range_noise: float = 0.01, rmin: float = 0.2, rmax: float = 130.0) -> np.ndarray:
    """Points in the SENSOR frame, float32 [n,4] (x,y,z,intensity)."""
    rng = np.random.default_rng(seed)
    dirs = sensor_dirs(sensor, seed)
    R = quat_to_R(pose7[3:])
    rng_true = raycast(scene, pose7[:3], dirs @ R.T)
    rn = rng_true + rng.normal(0.0, range_noise, size=rng_true.shape)
    ok = np.isfinite(rn) & (rn > rmin) & (rn < rmax)
    pts = dirs[ok] * rn[ok, None]
    inten = rng.uniform(1.0, 100.0, size=(len(pts), 1))
    return np.concatenate([pts, inten], 1).astype(np.float32)


# --------------------------------------------------------------------------
# BASELINE.json configs
# --------------------------------------------------------------------------
CONFIGS = {
    # name: half_extent, leaf(planeRes), sensor, icp iters, max_surface_features (0 = uncapped)
    "cfg1": dict(half_extent=17.5, plane_res=0.2, sensor="vlp16", max_iterations=5, max_surface_features=2000),
    "cfg1_uncapped": dict(half_extent=17.5, plane_res=0.2, sensor="vlp16", max_iterations=5, max_surface_features=0),
    "cfg2": dict(half_extent=52.0, plane_res=0.2, sensor="os1_128", max_iterations=20, max_surface_features=0),
    "cfg3": dict(half_extent=36.5, plane_res=0.1, sensor="mid360", max_iterations=20, max_surface_features=0),
    "tiny": dict(half_extent=9.0, plane_res=0.2, sensor="vlp16", max_iterations=5, max_surface_features=0),
    # x-dominant single-block hall far from the world diagonal: the layout on which the reference octree's two bugs
    # (flann/octree.h:383-385, :984-1001) cannot fire, so reference k-NN == exact k-NN (tests assert this)
    "hall": dict(half_extent=23.0, half_extent_y=9.0, center=(100.0, 0.0), plane_res=0.2, sensor="vlp16",
                 max_iterations=5, max_surface_features=0),
}


def make_case(name: str, scan_index: int = 0, max_radius: float | None = None):
    """-> dict(scene, map_xyzi [M,4] f32, scan_xyzi [N,4] f32, pose_true [7], pose_prior [7], cfg)."""
    scene, map_xyzi = make_map_for(name)
    return make_case_on(scene, map_xyzi, name, scan_index, max_radius)


def make_map_for(name: str):
    cfg = CONFIGS[name]
    return make_map(cfg["half_extent"], cfg["plane_res"], half_extent_y=cfg.get("half_extent_y"), center=cfg.get("center", (0.0, 0.0)))


def make_case_on(scene, map_xyzi, name: str, scan_index: int = 0, max_radius: float | None = None):
    cfg = CONFIGS[name]
    if max_radius is None:
        max_radius = min(20.0, min(cfg["half_extent"], cfg.get("half_extent_y") or cfg["half_extent"]) * 0.6)
    pose_true = random_sensor_pose(scene, 900 + scan_index, max_radius)
    scan = make_scan(scene, cfg["sensor"], pose_true, 1000 + scan_index)
    prior = perturb_pose(pose_true, 2000 + scan_index)
    return dict(scene=scene, map_xyzi=map_xyzi, scan_xyzi=scan, pose_true=pose_true, pose_prior=prior, cfg=cfg)


# ---------------------------------------------------------------------------------------------------------------
# Raw driver clouds for the scan-preparation rows (SURVEY 8f row 2): point_os::PointcloudXYZITR records
# {x, y, z, pad, intensity, time, ring(+pad), pad} = 8 floats, time at float index 5, plus a pose-sample buffer.
# ---------------------------------------------------------------------------------------------------------------
def _quat_axis_angle(axis, ang):
    axis = np.asarray(axis, np.float64)
    axis = axis / np.linalg.norm(axis)
    return np.r_[axis * np.sin(ang / 2), np.cos(ang / 2)]


def make_raw_sweep(n: int = 50_000, seed: int = 4000, sweep_s: float = 0.1, start_time: float = 1_700_000_000.25, rate_hz: float = 200.0,
                   with_defects: bool = True):
    """-> dict(points float32 [n,8], start_time, sample_times [m], sample_poses [m,7], T_i_l [7]).
    Points: a spinning-lidar-like shell 0.5..60 m, per-point time ascending over the sweep; with_defects adds what real
    drivers deliver and the reference's predicates react to: exact repeats of the previous point, (0,0,0) returns, a few
    NaN / inf records, points inside the blind range.  Pose samples: smooth 6-DoF motion sampled at rate_hz from before the
    sweep starts to after it ends (synchronize_measurements' precondition, featureExtraction.cpp:187-214)."""
    rng = np.random.default_rng(seed)
    az = np.linspace(0, 2 * np.pi * 1.0, n, endpoint=False)
    el = np.deg2rad(rng.uniform(-22.5, 22.5, n))
    r = rng.uniform(0.5, 60.0, n)
    pts = np.zeros((n, 8), np.float32)
    pts[:, 0] = r * np.cos(el) * np.cos(az)
    pts[:, 1] = r * np.cos(el) * np.sin(az)
    pts[:, 2] = r * np.sin(el)
    pts[:, 4] = rng.uniform(0, 255, n)
    pts[:, 5] = np.linspace(0.0, sweep_s, n)
    pts[:, 6] = rng.integers(0, 128, n).astype(np.float32)           # stands in for the ring bytes: must come back untouched
    if with_defects:
        k = rng.choice(np.arange(1, n), size=n // 50, replace=False)
        pts[k, :3] = pts[k - 1, :3]                                    # exact repeats
        k = rng.choice(np.arange(1, n), size=n // 100, replace=False)
        pts[k, :3] = 0.0                                               # zero returns
        k = rng.choice(np.arange(1, n), size=n // 100, replace=False)
        pts[k, :2] = pts[k - 1, :2]                                    # same x,y as the predecessor, different z
        pts[k, 2] = pts[k - 1, 2] + 0.05
        k2 = k[: len(k) // 2]
        pts[k2, :3] *= np.float32(0.001)                               # ... half of them inside the blind range
        pts[k2 - 1, :2] = pts[k2, :2]
        k = rng.choice(np.arange(1, n), size=8, replace=False)
        pts[k[:4], 0] = np.nan
        pts[k[4:], 1] = np.inf
    t0 = start_time - 2.5 / rate_hz
    m = int(np.ceil((sweep_s + 5.0 / rate_hz) * rate_hz)) + 1
    st = t0 + np.arange(m) / rate_hz
    sp = np.zeros((m, 7))
    for i, t in enumerate(st):
        u = t - start_time
        sp[i, :3] = [1.5 * u + 0.3 * u * u, -0.4 * u, 0.1 * np.sin(3 * u)]
        q = _quat_axis_angle([0.1, -0.2, 1.0], 0.8 * u + 0.5 * u * u)
        q2 = _quat_axis_angle([1.0, 0.3, 0.0], 0.2 * np.sin(5 * u))
        # Hamilton product q * q2 (xyzw)
        x1, y1, z1, w1 = q
        x2, y2, z2, w2 = q2
        sp[i, 3:] = [w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 + y1 * w2 + z1 * x2 - x1 * z2, w1 * z2 + z1 * w2 + x1 * y2 - y1 * x2,
                     w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2]
    T_i_l = np.r_[0.05, -0.02, 0.11, _quat_axis_angle([0.2, 1.0, -0.1], 0.35)]
    return dict(points=pts, start_time=start_time, sample_times=st, sample_poses=sp, T_i_l=T_i_l)


# ---------------------------------------------------------------------------------------------------------------
# Motion-distorted scans (within-scan motion compensation, so_register_undistort)
# ---------------------------------------------------------------------------------------------------------------
def make_moving_scan(scene: Scene, sensor: str, pose_start: np.ndarray, speed: float, yaw_rate: float, seed: int,
                     sweep_s: float = 0.1, dt: float = 0.1, imu_deskewed: bool = False, range_noise: float = 0.01,
                     rmin: float = 0.2, rmax: float = 130.0):
    """A spinning-lidar sweep taken while the sensor moves: constant forward body velocity `speed` (m/s, along the start pose's
    x axis) and yaw rate `yaw_rate` (rad/s).  Column c fires at t = c / n_cols * sweep_s and is ray-cast from the pose at t; its
    points are expressed in the sensor frame at t, with t stored in intensity.  imu_deskewed rotates every point into the start
    orientation (what so_scan_deskew with imu_only leaves: rotation removed, translation kept).
    -> dict(scan_xyzi float32 [n,4], pose_true (the pose at the sweep start), pose_prev / pose_next (the same motion at -dt / +dt),
    prior)."""
    vlp = sensor == "vlp16"
    n_cols, n_rings = (1800, 16) if vlp else (1024, 128)
    if sensor not in ("vlp16", "os1_128"):
        raise ValueError(sensor)
    rng = np.random.default_rng(seed)
    dirs = sensor_dirs(sensor).reshape(n_cols, n_rings, 3)
    q0 = np.asarray(pose_start[3:], np.float64)
    R0 = quat_to_R(q0)
    v_w = R0 @ np.array([speed, 0.0, 0.0])

    def pose_at(t):
        q = quat_mul(q0, quat_from_rotvec(np.array([0.0, 0.0, yaw_rate * t])))
        return np.concatenate([pose_start[:3] + v_w * t, q / np.linalg.norm(q)])

    out = []
    for c in range(n_cols):
        t = c / n_cols * sweep_s
        P = pose_at(t)
        d = dirs[c]
        r = raycast(scene, P[:3], d @ quat_to_R(P[3:]).T) + rng.normal(0.0, range_noise, size=len(d))
        ok = np.isfinite(r) & (r > rmin) & (r < rmax)
        pts = d[ok] * r[ok, None]
        if imu_deskewed:
            pts = pts @ quat_to_R(quat_from_rotvec(np.array([0.0, 0.0, yaw_rate * t]))).T
        out.append(np.concatenate([pts, np.full((len(pts), 1), t)], 1))
    scan = np.concatenate(out).astype(np.float32)
    prior = perturb_pose(pose_start, seed + 7, dt=0.05, dth_deg=0.5)
    return dict(scan_xyzi=scan, pose_true=np.asarray(pose_start, np.float64), pose_prev=pose_at(-dt), pose_next=pose_at(dt), prior=prior)


# ---------------------------------------------------------------------------------------------------------------
# Ring-ordered raw scans (edge extraction, so_scan_extract_edges)
# ---------------------------------------------------------------------------------------------------------------
RING_STRIDE, RING_TIME_OFFSET, RING_RING_OFFSET = 32, 20, 24     # point_os::PointcloudXYZITR: time at byte 20, uint16 ring at byte 24


def make_ring_scan(scene: Scene, sensor: str, pose7: np.ndarray, seed: int, order: str = "column", sweep_s: float = 0.1,
                   range_noise: float = 0.01, rmin: float = 0.2, rmax: float = 130.0) -> np.ndarray:
    """A spinning-lidar scan as the driver delivers it: float32 [n, 8] point_os::PointcloudXYZITR records {x, y, z, pad, intensity,
    time, ring (uint16 in the low half of float 6), pad}, sensor frame, ray-cast from the static pose7.  Ring r is the r-th lowest
    beam; column c fires at t = c / n_cols * sweep_s, so (ring, time) is unique per point.  order "column" lists the points column
    by column (the firing order), "ring" ring by ring.  Returns outside (rmin, rmax) are dropped."""
    n_cols, n_rings = {"vlp16": (1800, 16), "os1_128": (1024, 128)}[sensor]
    if order not in ("column", "ring"):
        raise ValueError(order)
    rng = np.random.default_rng(seed)
    dirs = sensor_dirs(sensor)                                        # column-major, rings inner
    rr = raycast(scene, pose7[:3], dirs @ quat_to_R(pose7[3:]).T)
    rr = rr + rng.normal(0.0, range_noise, size=rr.shape)
    col = np.repeat(np.arange(n_cols), n_rings)
    ring = np.tile(np.arange(n_rings), n_cols)
    if order == "ring":
        perm = np.lexsort((col, ring))
        dirs, rr, col, ring = dirs[perm], rr[perm], col[perm], ring[perm]
    ok = np.isfinite(rr) & (rr > rmin) & (rr < rmax)
    n = int(ok.sum())
    rec = np.zeros((n, 8), np.float32)
    rec[:, :3] = dirs[ok] * rr[ok, None]
    rec[:, 4] = rng.uniform(0.0, 255.0, n)
    rec[:, 5] = (col[ok] / n_cols * sweep_s).astype(np.float32)
    rec.view(np.uint16)[:, 12] = ring[ok].astype(np.uint16)
    return rec


def make_moving_ring_scan(scene: Scene, sensor: str, pose_start: np.ndarray, speed: float, yaw_rate: float, seed: int,
                          sweep_s: float = 0.1, dt: float = 0.1, range_noise: float = 0.01, rmin: float = 0.2, rmax: float = 130.0):
    """make_moving_scan's sweep (constant forward body velocity `speed` along the start pose's x axis, yaw rate `yaw_rate`; column c
    fires at t = c / n_cols * sweep_s from the pose at t, its points in the sensor frame at t) delivered as make_ring_scan's
    point_os::PointcloudXYZITR records {x, y, z, pad, intensity, time, ring, pad}, in firing order.
    -> dict(points float32 [n, 8], pose_true (the pose at the sweep start), pose_prev / pose_next (the same motion at -dt / +dt), prior)."""
    n_cols, n_rings = {"vlp16": (1800, 16), "os1_128": (1024, 128)}[sensor]
    rng = np.random.default_rng(seed)
    dirs = sensor_dirs(sensor).reshape(n_cols, n_rings, 3)
    q0 = np.asarray(pose_start[3:], np.float64)
    v_w = quat_to_R(q0) @ np.array([speed, 0.0, 0.0])

    def pose_at(t):
        q = quat_mul(q0, quat_from_rotvec(np.array([0.0, 0.0, yaw_rate * t])))
        return np.concatenate([pose_start[:3] + v_w * t, q / np.linalg.norm(q)])

    out = []
    for c in range(n_cols):
        t = c / n_cols * sweep_s
        P = pose_at(t)
        d = dirs[c]
        r = raycast(scene, P[:3], d @ quat_to_R(P[3:]).T) + rng.normal(0.0, range_noise, size=len(d))
        ok = np.isfinite(r) & (r > rmin) & (r < rmax)
        rec = np.zeros((int(ok.sum()), 8), np.float32)
        rec[:, :3] = d[ok] * r[ok, None]
        rec[:, 5] = np.float32(t)
        rec.view(np.uint16)[:, 12] = np.arange(n_rings)[ok].astype(np.uint16)
        out.append(rec)
    rec = np.concatenate(out)
    rec[:, 4] = rng.uniform(0.0, 255.0, len(rec))
    prior = perturb_pose(pose_start, seed + 7, dt=0.05, dth_deg=0.5)
    return dict(points=rec, pose_true=np.asarray(pose_start, np.float64), pose_prev=pose_at(-dt), pose_next=pose_at(dt), prior=prior)


def make_corridor_scene(poles: bool = True) -> Scene:
    """A 400 m x 6 m corridor (x along it, walls at y = +-3, floor -1.8, ceiling 3.2; the end walls at x = +-200 lie beyond the
    130 m range) with free-standing 0.1 m square floor-to-ceiling poles every 4 m, 1 m off each wall.  Pole centres sit at
    x = 2 + 4i, so no face plane comes within 1 m of the origin.  poles=False: the bare corridor, which constrains nothing along x."""
    room = np.array([-200.0, 200.0, -3.0, 3.0, -1.8, 3.2])
    boxes = []
    for cx in np.arange(-198.0, 199.0, 4.0) if poles else ():
        for cy in (-2.0, 2.0):
            boxes.append([cx - 0.05, cx + 0.05, cy - 0.05, cy + 0.05, -1.8, 3.2])
    return Scene(room=room, boxes=np.array(boxes, np.float64).reshape(-1, 6))

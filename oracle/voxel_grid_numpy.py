"""Restatement of pcl::VoxelGrid<PointXYZI>::applyFilter (PCL 1.12, filters/impl/voxel_grid.hpp), written from PCL's published
source and apart from the device code:

    getMinMax3D(cloud, min_p, max_p)                              finite points only (is_dense = false)
    dx = int64((max_p.x - min_p.x) * inv.x) + 1, dy, dz           float subtract, float multiply, truncate
    dx * dy * dz > INT32_MAX  ->  output = input, verbatim        ("Integer indices would overflow"), non-finite rows included
    min_b = floor(min_p * inv), max_b = floor(max_p * inv)        float multiply, floor, int
    div_b = max_b - min_b + 1, divb_mul = (1, div_b.x, div_b.x * div_b.y)
    ijk = int(floor(p * inv) - float(min_b))                      float subtraction
    idx = unsigned(ijk.x * divb_mul.x + ijk.y * divb_mul.y + ijk.z * divb_mul.z)      int arithmetic: the exact value mod 2^32
    sort by idx; one pcl::CentroidPoint per run: float sums, divided by float(n)

Choices where PCL leaves the result open:
  - the clouds are not dense (PCLPointCloud::is_dense = false, what every cloud of a sensor driver declares): points with a
    non-finite x, y or z are skipped by the bounds and by the filter, and kept only by the verbatim fall-back;
  - PCL sorts with std::sort (not stable), so the order of the points inside one voxel is unspecified; here it is cloud order;
  - a cloud without a finite point (the empty cloud included) has min_p = FLT_MAX and max_p = -FLT_MAX, so the bounds
    arithmetic is undefined; its output here is the empty cloud, which is also what the x86 conversions give;
  - the contract covers |x * (1/leaf)| < 2^20 - 1 on every axis (about 210 km at leaf 0.2); beyond it PCL's float -> int
    conversions are undefined and no output is pinned.

Also here: the per-block form of LocalMap::addSurfPointCloud / addEdgePointCloud (LocalMap.h:529-645: every touched 50 m block's
cloud is filtered on its own) and the statistic of laserMapping::adjustVoxelSize (laserMapping.cpp:600-651)."""
import numpy as np

INT32_MAX = 2 ** 31 - 1
ORIGIN0 = (10, 10, 5)


def inverse_leaf(leaf):
    """Eigen::Array4f::Ones() / leaf_size_: a float division"""
    return np.float32(1.0) / np.float32(leaf)


def bounds(xyzi):
    """getMinMax3D over the finite points: (min_p, max_p) as float32 [3], or None when there is no finite point."""
    xyz = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)[:, :3]
    fin = np.isfinite(xyz).all(1)
    if not fin.any():
        return None
    return xyz[fin].min(0), xyz[fin].max(0)


def extent(xyzi, leaf):
    """(dx, dy, dz) of the overflow test as Python ints, or None when there is no finite point."""
    b = bounds(xyzi)
    if b is None:
        return None
    lo, hi = b
    with np.errstate(over="ignore"):
        d = (hi - lo) * inverse_leaf(leaf)               # float32 subtraction and product
    return tuple(int(np.trunc(min(np.float64(v), 2.0 ** 62))) + 1 for v in d)      # (capped where a float overflows)


def falls_back(xyzi, leaf):
    """True when PCL returns the input verbatim: dx * dy * dz > INT32_MAX (exact integer product)."""
    d = extent(xyzi, leaf)
    return d is not None and d[0] * d[1] * d[2] > INT32_MAX


def voxel_index(xyzi, leaf):
    """(idx uint32 [m], rows int64 [m]): PCL's voxel index of every finite point and the row it came from, in cloud order.
    Assumes the cloud is not a fall-back case and has a finite point."""
    s = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    inv = inverse_leaf(leaf)
    lo, hi = bounds(s)
    min_b = np.floor(lo * inv).astype(np.int64)
    max_b = np.floor(hi * inv).astype(np.int64)
    div = max_b - min_b + 1
    mask = np.uint64(0xFFFFFFFF)
    mul = [np.uint64(1), np.uint64(div[0]) & mask, np.uint64(div[0] * div[1]) & mask]      # int32 products, mod 2^32
    rows = np.flatnonzero(np.isfinite(s[:, :3]).all(1))
    f = np.floor(s[rows, :3] * inv)                                                         # float32
    ijk = (f - min_b.astype(np.float32)).astype(np.int64)                                   # float subtraction, then int
    u = ijk.astype(np.uint64) & mask                                                        # two's complement bits, mod 2^32
    idx = (u[:, 0] * mul[0] + u[:, 1] * mul[1] + u[:, 2] * mul[2]) & mask
    return idx.astype(np.uint32), rows


def centroids(pts, keys):
    """One pcl::CentroidPoint per run of equal keys (keys sorted, stable): float32 sums in the given order, / float32(n)."""
    pts = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 4)
    if len(pts) == 0:
        return np.zeros((0, 4), np.float32)
    new = np.ones(len(keys), dtype=bool)
    new[1:] = keys[1:] != keys[:-1]
    seg = np.cumsum(new) - 1
    nseg = int(seg[-1]) + 1
    rank = np.arange(len(keys)) - np.flatnonzero(new)[seg]
    acc = np.zeros((nseg, 4), np.float32)
    for r in range(int(rank.max()) + 1):
        m = rank == r
        acc[seg[m]] = acc[seg[m]] + pts[m]              # float32, one point at a time per voxel, cloud order
    cnt = np.bincount(seg, minlength=nseg).astype(np.float32)
    return (acc / cnt[:, None]).astype(np.float32)


def voxel_grid(xyzi, leaf):
    """pcl::VoxelGrid<PointXYZI>(leaf) of a float32 [n, 4] {x, y, z, intensity} cloud -> float32 [m, 4]."""
    s = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    if bounds(s) is None:
        return np.zeros((0, 4), np.float32)
    if falls_back(s, leaf):
        return s.copy()
    idx, rows = voxel_index(s, leaf)
    order = np.argsort(idx, kind="stable")
    return centroids(s[rows[order]], idx[order])


def absolute_voxel_grid(xyzi, leaf):
    """The absolute-index formula: voxel floor(x * inv) per axis, output ordered by (k, j, i), no overflow test.  Equal to
    voxel_grid wherever PCL does not fall back and its index does not wrap."""
    s = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    s = s[np.isfinite(s[:, :3]).all(1)]
    ijk = np.floor(s[:, :3] * inverse_leaf(leaf)).astype(np.int64)
    order = np.lexsort((ijk[:, 0], ijk[:, 1], ijk[:, 2]))
    k = ijk[order]
    key = (k[:, 2] << 42) + (k[:, 1] << 21) + k[:, 0]
    return centroids(s[order], key)


def block_of(xyz, origin=ORIGIN0):
    """LocalMap's block of a point: int((x + 25) / 50) + origin, minus one when x + 25 < 0 (double arithmetic on floats)."""
    v = np.asarray(xyz, dtype=np.float32).astype(np.float64) + 25.0
    c = np.trunc(v / 50.0).astype(np.int64) + np.asarray(origin, dtype=np.int64)
    return c - (v < 0).astype(np.int64)


def block_linear(c):
    """cubeInd = i + 21 j + 441 k, -1 off the 21 x 21 x 11 grid"""
    ok = (c[:, 0] >= 0) & (c[:, 0] < 21) & (c[:, 1] >= 0) & (c[:, 1] < 21) & (c[:, 2] >= 0) & (c[:, 2] < 11)
    return np.where(ok, c[:, 0] + 21 * c[:, 1] + 441 * c[:, 2], -1)


def block_voxel_grid(xyzi, leaf, origin=ORIGIN0):
    """LocalMap::addSurfPointCloud / addEdgePointCloud for the touched blocks: the cloud's finite on-grid points binned to their
    blocks (cloud order inside a block), each block's cloud through voxel_grid on its own, concatenated in block order."""
    s = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    s = s[np.isfinite(s[:, :3]).all(1)]
    lin = block_linear(block_of(s[:, :3], origin))
    s, lin = s[lin >= 0], lin[lin >= 0]
    order = np.argsort(lin, kind="stable")
    s, lin = s[order], lin[order]
    cut = np.flatnonzero(np.diff(lin)) + 1
    parts = [voxel_grid(b, leaf) for b in np.split(s, cut)] if len(s) else []
    return np.concatenate(parts, 0) if parts else np.zeros((0, 4), np.float32)


def map_insert(old_xyzi, new_xyzi, leaf, origin=ORIGIN0):
    """The store after an insert: untouched blocks' points in their old order, then every touched block (old points first, then
    the new ones in input order) filtered on its own, in block order."""
    old = np.ascontiguousarray(old_xyzi, dtype=np.float32).reshape(-1, 4)
    new = np.ascontiguousarray(new_xyzi, dtype=np.float32).reshape(-1, 4)
    new = new[np.isfinite(new[:, :3]).all(1)]
    lin_old = block_linear(block_of(old[:, :3], origin))
    lin_new = block_linear(block_of(new[:, :3], origin))
    touched = np.zeros(21 * 21 * 11, dtype=bool)
    touched[lin_new[lin_new >= 0]] = True
    on = lin_old >= 0
    keep = old[on & ~touched[np.maximum(lin_old, 0)]]
    work = np.concatenate([old[on & touched[np.maximum(lin_old, 0)]], new], 0)
    return np.concatenate([keep, block_voxel_grid(work, leaf, origin)], 0)


def adjust_statistic(xyzi):
    """laserMapping::adjustVoxelSize's statistic: mean|x| * mean|y| * mean|z| with float accumulators in cloud order (every
    point, finite or not), divided by float(n), the float product widened to double."""
    s = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    a = np.zeros(3, np.float32)
    ab = np.abs(s[:, :3])
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(len(s)):
            a = a + ab[i]
        a = a / np.float32(len(s))
        return float(a[0] * a[1] * a[2])


def adjust_leaves(avg, line_res, plane_res):
    """The leaf rule: < 25 -> 0.1 / 0.2, > 65 -> 0.4 / 0.8, otherwise (NaN included) unchanged; as float32 values."""
    if avg < 25:
        line_res, plane_res = 0.1, 0.2
    elif avg > 65:
        line_res, plane_res = 0.4, 0.8
    return float(np.float32(line_res)), float(np.float32(plane_res))

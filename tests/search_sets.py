"""Seeded adversarial inputs for the neighbour searches: maps and queries where a search goes wrong if it is subtly wrong --
exact distance ties, dense clusters that overflow the search's candidate buffer, 50 m block faces, sparse maps that make the
unbounded search grow its cube, nearly empty blocks, and queries that are not finite or lie far off the grid.

Every generator returns float32 arrays; with the identity pose a scan point is exactly the float32 query it was built as."""
import numpy as np

from conftest import get_case

IDENTITY = np.array([0, 0, 0, 0, 0, 0, 1], np.float64)
KBUF_CAP = 24           # candidates the select search records before it inserts directly (so_knn.cuh kBufCap)


def cell_faces(plane_res, lo, hi):
    """float32 coordinates in [lo, hi) of the k-NN grid's cell faces (cell edge 50 / nb, nb = min(192, floor(100 / sqrt(3 planeRes)))
    cells per 50 m block, DESIGN section 2), with the float32 neighbours on either side of each."""
    nb = min(192, int(100.0 / np.sqrt(3.0 * np.float64(np.float32(plane_res)))))
    j = np.arange(int(np.floor((lo + 25.0) * nb / 50.0)), int(np.ceil((hi + 25.0) * nb / 50.0)) + 1)
    f = (-25.0 + j * (50.0 / nb)).astype(np.float32)
    f = f[(f >= lo) & (f < hi)]
    return f, np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))


def knn_case(name):
    """(map_xyzi, plane_res, queries) for test_knn_bit_exact.  lattice: voxel centres at planeRes spacing, a second lattice
    whose planes lie on the grid's cell faces (and one float32 step either side), exact distance ties everywhere; queries on lattice
    points, midpoints, faces and at random.  dense: clusters of 6-64 coincident or nearly coincident points, so that far more than
    the 24 candidates the search buffers fall inside its bound."""
    rng = np.random.default_rng(0)
    if name not in ("lattice", "dense"):
        case = get_case(name)
        base = case["map_xyzi"][::7, :3]
        q = base + rng.normal(0, 0.12, size=base.shape).astype(np.float32)
        q = np.concatenate([q, rng.uniform(-30, 30, size=(500, 3)).astype(np.float32) + q.mean(0)])     # incl. far-away queries
        return case["map_xyzi"], case["cfg"]["plane_res"], q
    pr = 0.2
    if name == "lattice":
        g = (np.arange(-30, 30) + 0.5) * pr
        a = np.stack(np.meshgrid(g, g, (np.arange(-3, 3) + 0.5) * pr, indexing="ij"), -1).reshape(-1, 3)
        fx, fxm, fxp = cell_faces(pr, 8.0, 12.0)
        fz, fzm, fzp = cell_faces(pr, -1.0, 1.0)
        xs = np.concatenate([fx, fxm[::3], fxp[1::3]])
        zs = np.concatenate([fz, fzm[::2], fzp[1::2]])
        b = np.stack(np.meshgrid(xs, np.float32(fx - 20.0), zs, indexing="ij"), -1).reshape(-1, 3)
        pts = np.concatenate([a.astype(np.float32), b.astype(np.float32)])
        q = np.concatenate([pts[rng.choice(len(pts), 3000, replace=False)],
                            (pts[rng.choice(len(a), 2000)] + np.float32(pr / 2) * rng.integers(0, 2, size=(2000, 3))).astype(np.float32),
                            np.stack([rng.choice(fx, 2000), rng.uniform(-6, 6, 2000), rng.choice(fz, 2000)], 1).astype(np.float32),
                            np.stack([rng.uniform(8, 12, 2000), rng.choice(np.float32(fx - 20.0), 2000), rng.uniform(-1, 1, 2000)], 1).astype(np.float32),
                            rng.uniform(-7, 13, size=(2000, 3)).astype(np.float32) * np.float32([1, 1, 0.2])])
    else:
        cen = rng.uniform(-5, 5, size=(600, 3)) * [1, 1, 0.3]
        pts = []
        for i, c in enumerate(cen):
            n = int(rng.integers(6, 65))
            jit = [0.0, 1e-6, 1e-4, 1e-2][i % 4]
            pts.append(c + rng.normal(0, jit, size=(n, 3)) if jit else np.repeat(c[None], n, 0))
        pts = np.concatenate(pts).astype(np.float32)
        q = np.concatenate([cen.astype(np.float32), (cen + rng.normal(0, 0.1, size=cen.shape)).astype(np.float32),
                            ((cen[:-1] + cen[1:]) / 2).astype(np.float32), rng.uniform(-6, 6, size=(2000, 3)).astype(np.float32) * np.float32([1, 1, 0.3])])
    xyzi = np.concatenate([pts, np.ones((len(pts), 1), np.float32)], 1)
    return xyzi, pr, q


def xyzi(p, intensity=1.0):
    p = np.asarray(p, np.float32).reshape(-1, 3)
    return np.concatenate([p, np.full((len(p), 1), intensity, np.float32)], 1)


# ---------------------------------------------------------------------------------------------------------------
# surf maps for the registration's search (planeRes 0.2)
# ---------------------------------------------------------------------------------------------------------------
def block_face_case(seed=4):
    """(map_xyzi, plane_res, queries): a floor and a wall straddling the 50 m block face x = 25 (relative to the grid origin), and
    queries within 1 m of it -- on the face exactly, one float32 step either side, within a few millimetres, and spread over the
    metre.  Neighbours come only from the query's own block (LocalMap.h:488-525), so a query at the face sees half a neighbourhood."""
    rng = np.random.default_rng(seed)
    n = 60000
    floor = np.stack([rng.uniform(20, 30, n), rng.uniform(-5, 5, n), rng.uniform(-1, 1, n) * 0.02 - 1.5], 1)
    m = 20000
    wall = np.stack([rng.uniform(20, 30, m), np.full(m, 4.0) + rng.uniform(-1, 1, m) * 0.02, rng.uniform(-1.5, 1.5, m)], 1)
    pts = np.concatenate([floor, wall]).astype(np.float32)
    f = np.float32(25.0)
    on = np.array([f, np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))], np.float32)
    k = 1200
    qx = np.concatenate([np.repeat(on, k // 3), rng.uniform(24.995, 25.005, k), rng.uniform(24.0, 26.0, 2 * k)]).astype(np.float32)
    nq = len(qx)
    on_wall = rng.random(nq) < 0.25
    qy = np.where(on_wall, np.float32(4.0) + rng.normal(0, 0.01, nq), rng.uniform(-4, 3.5, nq)).astype(np.float32)
    qz = np.where(on_wall, rng.uniform(-1.3, 1.3, nq), -1.5 + rng.normal(0, 0.01, nq)).astype(np.float32)
    return xyzi(pts), 0.2, np.stack([qx, qy, qz], 1).astype(np.float32)


def surf_case(name):
    """(map_xyzi, plane_res, queries) of the registration's search sets: 'lattice' and 'dense' of knn_case, 'block_face'."""
    if name == "block_face":
        return block_face_case()
    return knn_case(name)


# ---------------------------------------------------------------------------------------------------------------
# edge maps (lineRes 0.1) for the edge fit's unbounded 10-NN
# ---------------------------------------------------------------------------------------------------------------
EDGE_LINE_RES = 0.1


def edge_lattice(seed=11):
    """Lines of points on a dyadic lattice (0.125 m along x, lines 0.25 m apart in y and z): every distance is exact in float32,
    so distances tie at every rank, the 10th included.  Queries on lattice points, half-steps and at random."""
    rng = np.random.default_rng(seed)
    xs = np.arange(-40, 40) * 0.125
    ys = np.arange(-8, 8) * 0.25
    zs = np.arange(-3, 3) * 0.25
    pts = np.stack(np.meshgrid(xs, ys, zs, indexing="ij"), -1).reshape(-1, 3)
    pts = pts[rng.permutation(len(pts))]                    # ids do not follow the walk order, so the (d2, id) tie-break is exercised
    q = np.concatenate([pts[rng.choice(len(pts), 1500, replace=False)],
                        pts[rng.choice(len(pts), 1500)] + 0.0625 * rng.integers(-1, 2, size=(1500, 3)),
                        rng.uniform(-5, 5, size=(1000, 3)) * [1, 0.4, 0.15]])
    return xyzi(pts), q.astype(np.float32)


def edge_dense(seed=12):
    """Clusters of 11-64 coincident or nearly coincident points (jitter 0, 1e-6, 1e-4, 1e-2 m): with K = 10 far more than the 24
    candidates the search records fall inside its bound.  Queries at the cluster centres, near them and between them."""
    rng = np.random.default_rng(seed)
    cen = rng.uniform(-8, 8, size=(400, 3)) * [1, 1, 0.3]
    pts = []
    for i, c in enumerate(cen):
        n = int(rng.integers(11, 65))
        jit = [0.0, 1e-6, 1e-4, 1e-2][i % 4]
        pts.append(c + rng.normal(0, jit, size=(n, 3)) if jit else np.repeat(c[None], n, 0))
    pts = np.concatenate(pts)
    q = np.concatenate([cen, cen + rng.normal(0, 0.05, size=cen.shape), (cen[:-1] + cen[1:]) / 2,
                        rng.uniform(-9, 9, size=(800, 3)) * [1, 1, 0.3]])
    return xyzi(pts), q.astype(np.float32)


def edge_sparse(seed=13):
    """300 points over 40 x 40 x 10 m: the 10th neighbour lies 2-15 m away, so the unbounded search grows its cube past R = 2 and
    doubles it past R = 4.  A line of 20 points gives some queries a valid line fit."""
    rng = np.random.default_rng(seed)
    pts = np.concatenate([rng.uniform(-20, 20, size=(300, 3)) * [1, 1, 0.25],
                          np.stack([np.arange(20) * 0.09 - 0.9, np.zeros(20), np.zeros(20)], 1)])
    q = np.concatenate([rng.uniform(-22, 22, size=(1500, 3)) * [1, 1, 0.25],
                        np.stack([rng.uniform(-1, 1, 200), rng.normal(0, 0.02, 200), rng.normal(0, 0.02, 200)], 1)])
    return xyzi(pts), q.astype(np.float32)


def edge_small_blocks(seed=14):
    """Blocks holding exactly 9, 10 and 11 points (x + 1, x - 1 and y + 1 of the origin block), a few on a line, plus a populated
    origin block; queries in each."""
    rng = np.random.default_rng(seed)
    parts, qs = [], []
    for count, centre in ((9, (50.0, 0.0, 0.0)), (10, (-50.0, 0.0, 0.0)), (11, (0.0, 50.0, 0.0))):
        c = np.asarray(centre)
        line = c + np.stack([np.arange(count) * 0.08, np.zeros(count), np.zeros(count)], 1)
        line[count // 2:] += rng.normal(0, 0.5, size=(count - count // 2, 3))
        parts.append(line)
        qs.append(c + rng.normal(0, 0.3, size=(300, 3)))
        qs.append(line[:4] + 0.01)
    parts.append(rng.uniform(-10, 10, size=(2000, 3)) * [1, 1, 0.2])
    qs.append(rng.uniform(-10, 10, size=(200, 3)) * [1, 1, 0.2])
    return xyzi(np.concatenate(parts)), np.concatenate(qs).astype(np.float32)


EDGE_SETS = {"lattice": edge_lattice, "dense": edge_dense, "sparse": edge_sparse, "small_blocks": edge_small_blocks}


def edge_case(name):
    return EDGE_SETS[name]()


# ---------------------------------------------------------------------------------------------------------------
# defective queries
# ---------------------------------------------------------------------------------------------------------------
DEFECTS = np.array([np.nan, np.inf, -np.inf, 1e12, -1e12], np.float32)


def defective_points(n, seed=21):
    """n points with NaN, +-inf or +-1e12 in one, two or three coordinates (every value and coordinate count cycled), the other
    coordinates ordinary."""
    rng = np.random.default_rng(seed)
    p = rng.uniform(-5, 5, size=(n, 3)).astype(np.float32)
    for i in range(n):
        k = 1 + (i // len(DEFECTS)) % 3
        axes = rng.permutation(3)[:k]
        p[i, axes] = DEFECTS[i % len(DEFECTS)]
    return p


def mix_defective(points, frac=0.01, seed=21, min_count=30):
    """points [n, C] with defective rows inserted at random positions -> (mixed [n + m, C], boolean mask of the inserted rows)."""
    rng = np.random.default_rng(seed)
    points = np.asarray(points, np.float32)
    m = max(min_count, int(round(frac * len(points))))
    bad = np.zeros((m, points.shape[1]), np.float32)
    if points.shape[1] > 3:
        bad[:, 3:] = points[rng.integers(0, len(points), m), 3:]
    bad[:, :3] = defective_points(m, seed)
    mask = np.zeros(len(points) + m, bool)
    mask[rng.choice(len(mask), m, replace=False)] = True
    out = np.empty((len(mask), points.shape[1]), np.float32)
    out[mask] = bad
    out[~mask] = points
    return out, mask

"""Crafted neighbourhoods for the plane and line fits: inputs the synthetic scenes never produce.

plane_sets() builds a map of 5-point clusters, 2.5 m apart, so the 5-NN of a query placed near a cluster's centroid is exactly
that cluster, and returns for every cluster its class label and the float64 gate quantities of the plane fit
(LidarSlam.cpp:749-844), computed with numpy from the float32 coordinates:
  lam0        smallest eigenvalue of the scatter matrix (gate: lam0 < 1e-6 rejects)
  ratio       lam1 / lam2                               (gate: ratio < 0.1 rejects)
  dist_ratio  largest distance to the plane A n = -1 fitted by least squares, over planeRes / 2  (gate: > 1 rejects)
  gap         (lam1 - lam0) / lam2: where it is ~0 the smallest eigenvector (the PCA normal) is not defined

Classes: coincident points (5, 4 + 1, 3 + 2), exactly collinear sets (along x, y, z and a dyadic diagonal), exactly coplanar
axis-aligned sets, a dyadic square plus an apex (an exactly repeated eigenvalue), lam0 and lam1 / lam2 placed on either side of
their thresholds at relative margins of 1e-3 and 1e-7 (diagonal scatter matrices built from integer multiples of a power of
two, so the quantity is known to ~1e-12), largest plane distance on either side of planeRes / 2, planes through the world
origin (the right-hand side -1 of the fit is then nearly inconsistent), clusters near +-500 m (the edge of the block grid),
5-point subsets of a voxel-centre lattice of spacing planeRes, and generic noisy planes as a control.

edge_sets() does the same for the 10-point line fit: 10 coincident points, 10 exactly collinear points, 2 distinct points
repeated five times each."""
import numpy as np

PLANE_RES = 0.2
LINE_RES = 0.1
LAM0_MIN = 1e-6
RATIO_MIN = 0.1
MAX_DIST = float(np.float32(PLANE_RES)) / 2.0        # double(float planeRes) / 2, as the fit reads it
BAND = 1e-9                                           # sets this close (relative) to a threshold are left unclassified

_F32 = np.float32


def _slots(z_levels, x0=-21.25, n=18, step=2.5):
    """Cluster centres on a grid inside one 50 m block (multiples of 1/16, so dyadic offsets stay exact)."""
    g = x0 + step * np.arange(n)
    return [np.array([x, y, z]) for z in z_levels for y in g for x in g]


def _unit(rng):
    v = rng.normal(size=3)
    return v / np.linalg.norm(v)


def _dyadic(c, unit=1.0 / 16):
    return np.round(np.asarray(c, np.float64) / unit) * unit


def _random_frame(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q                                          # columns: in-plane u, in-plane v, normal


def _gen_planar(rng, c, ext=(0.3, 0.25), noise=0.005, frame=None):
    f = _random_frame(rng) if frame is None else frame
    uv = rng.uniform(-1, 1, size=(5, 2)) * np.asarray(ext)
    off = uv[:, :1] * f[:, 0] + uv[:, 1:] * f[:, 1] + rng.normal(0, noise, size=(5, 1)) * f[:, 2]
    return c + off


def gate_quantities(P32):
    """P32: float32 [N, 5, 3] -> dict of float64 gate quantities (module docstring), the kernel's mean and scatter order."""
    P = np.asarray(P32, np.float32).astype(np.float64)
    mean = ((((P[:, 0] + P[:, 1]) + P[:, 2]) + P[:, 3]) + P[:, 4]) / 5.0
    C = P - mean[:, None, :]
    S = np.einsum("nja,njb->nab", C, C)
    ev = np.linalg.eigvalsh(S)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = ev[:, 1] / ev[:, 2]
        gap = (ev[:, 1] - ev[:, 0]) / ev[:, 2]
    dist = np.empty(len(P))
    for i in range(len(P)):
        x = np.linalg.lstsq(P[i], -np.ones(5), rcond=None)[0]
        nn = np.sqrt(x @ x)
        dist[i] = np.abs(P[i] @ (x / nn) + 1.0 / nn).max()
    return dict(lam0=ev[:, 0], lam1=ev[:, 1], lam2=ev[:, 2], ratio=ratio, gap=gap, dist_ratio=dist / MAX_DIST)


def classify(q):
    """Expected status of each set (0 success, 3 bad PCA structure, 5 plane distance too large) and the mask of sets whose
    quantities all lie outside the BAND around their thresholds."""
    lam0, ratio, dr = q["lam0"], q["ratio"], q["dist_ratio"]
    with np.errstate(invalid="ignore"):
        bad_pca = (lam0 < LAM0_MIN) | (ratio < RATIO_MIN)             # NaN ratio (lam2 == 0) compares false, as in the reference
        status = np.where(bad_pca, 3, np.where(dr > 1.0, 5, 0))
        near = (np.abs(lam0 - LAM0_MIN) <= BAND * LAM0_MIN) | (np.abs(ratio - RATIO_MIN) <= BAND * RATIO_MIN)
        near |= ~bad_pca & (np.abs(dr - 1.0) <= BAND)
    return status, ~near


# ------------------------------------------------------------------------------------------------------------- class builders
def _coincident(rng, c, split):
    a = c + rng.uniform(-0.05, 0.05, 3)
    b = a + _unit(rng) * rng.uniform(0.05, 0.3)
    return np.array([a] * split + [b] * (5 - split))


def _collinear_axis(rng, c, axis):
    P = np.repeat(c[None], 5, 0) + rng.uniform(-0.02, 0.02, 3)
    P[:, axis] += rng.uniform(-0.3, 0.3, 5)
    return P


def _collinear_diag(rng, c):
    d = rng.integers(-2, 3, size=3)
    while not d.any():
        d = rng.integers(-2, 3, size=3)
    t = rng.permutation(np.arange(-2, 3))
    return _dyadic(c) + t[:, None] * d[None, :] / 16.0          # every coordinate a multiple of 1/16: exact in float32


def _coplanar_axis(rng, c, axis):
    P = c + rng.uniform(-0.3, 0.3, size=(5, 3))
    P[:, axis] = c[axis] + 0.01
    return P


def _square_apex(rng, c, h, t, axis, sign):
    """(+-h, 0, 0), (0, +-h, 0), (0, 0, t) around a dyadic centre: S = diag(2h^2, 2h^2, 0.8 t^2) exactly, so two eigenvalues are
    exactly equal -- the two smallest when 0.8 t^2 > 2 h^2 (the normal is then not defined)."""
    o = np.array([[h, 0, 0], [-h, 0, 0], [0, h, 0], [0, -h, 0], [0, 0, sign * t]])
    perm = [(0, 1, 2), (1, 2, 0), (2, 0, 1)][axis]
    return _dyadic(c) + o[:, perm]


def _in_window(r, rel):
    """relative distance r from a threshold is on rel's side, between rel / 2 and 3 rel / 2"""
    return (r / rel >= 0.5) & (r / rel <= 1.5)


def _lam0_margin(rng, c, rel):
    """Normal along z, c[2] in [1/4, 1/2) so z offsets are integer multiples of 2^-25 (exact): S = diag(2a^2, 2b^2, F 2^-50), with
    F = sum (k - mean k)^2 for z offsets k = (u, u, v, v, w).  Searches integers with F 2^-50 = 1e-6 (1 + rel (1 +- 1/2))."""
    assert 0.25 <= c[2] < 0.5
    unit = 2.0 ** -25
    target = LAM0_MIN * (1 + rel) / unit ** 2
    for _ in range(100):
        u = rng.integers(2000, 14000, size=100000)
        v = rng.integers(-14000, -2000, size=100000)
        # F(w) = 2u^2 + 2v^2 + w^2 - (2u + 2v + w)^2 / 5 = (4/5) w^2 - (4/5)(u + v) w + 2u^2 + 2v^2 - 4(u + v)^2 / 5
        A, B, C0 = 0.8, -0.8 * (u + v), 2.0 * u * u + 2.0 * v * v - 0.8 * (u + v) ** 2 - target
        disc = B * B - 4 * A * C0
        ok = disc >= 0
        w = np.round((-B + np.sqrt(np.where(ok, disc, 0))) / (2 * A)).astype(np.int64)
        ks = np.stack([u, u, v, v, w], 1)
        F = ((ks - ks.mean(1, keepdims=True)) ** 2).sum(1)
        hit = ok & _in_window(F * unit ** 2 / LAM0_MIN - 1, rel) & (np.abs(w) < 80000)
        if hit.any():
            k = ks[np.flatnonzero(hit)[0]]
            break
    else:
        raise RuntimeError("no lam0 set found")
    a, b = 0.25, 0.1875
    o = np.array([[a, 0, 0], [-a, 0, 0], [0, b, 0], [0, -b, 0], [0, 0, 0]], np.float64)
    o[:, 2] = k * unit
    return _dyadic(c) + o


def _ratio_margin(rng, c, rel):
    """x offsets (a, -a, 0, 0, 0), y offsets (0, 0, q2, q3, q4) 2^-18 with q2 + q3 + q4 = 0, z offsets (u, u, 0, 0, 0) 2^-18:
    S = diag(2a^2, Q 2^-36, 1.2 u^2 2^-36) up to an S_yz of rounding size.  Searches Q = q2^2 + q3^2 + q4^2 with
    lam1 / lam2 = Q 2^-36 / 2a^2 = 0.1 (1 + rel (1 +- 1/2))."""
    unit = 2.0 ** -18
    a = 0.25
    target = RATIO_MIN * (1 + rel) * 2 * a * a / unit ** 2
    for _ in range(100):
        q2 = rng.integers(-40000, 40000, size=100000)
        # Q(q3) = 2 q3^2 + 2 q2 q3 + 2 q2^2
        disc = 4.0 * q2 * q2 - 8.0 * (2.0 * q2 * q2 - target)
        ok = disc >= 0
        q3 = np.round((-2.0 * q2 + np.sqrt(np.where(ok, disc, 0))) / 4.0).astype(np.int64)
        Q = q2 * q2 + q3 * q3 + (q2 + q3) ** 2
        hit = ok & _in_window(Q * unit ** 2 / (2 * a * a) / RATIO_MIN - 1, rel) & (np.abs(q3) < 60000) & (np.abs(q2 + q3) < 60000)
        if hit.any():
            i = np.flatnonzero(hit)[0]
            qq = np.array([q2[i], q3[i], -(q2[i] + q3[i])])
            break
    else:
        raise RuntimeError("no ratio set found")
    u = int(rng.integers(2000, 3000))                              # lam0 = 1.2 u^2 2^-36 ~ 1e-4: far from both gates
    o = np.zeros((5, 3))
    o[0, 0], o[1, 0] = a, -a
    o[2:, 1] = qq * unit
    o[0, 2] = o[1, 2] = u * unit
    return _dyadic(c) + o


def _plane_dist_margin(rng, c, rel):
    """Four points on a noisy plane and a fifth lifted off it by t; t bisected (in float32) until the largest fitted-plane
    distance is planeRes / 2 * (1 + rel) to within the float32 granularity."""
    f = _random_frame(rng)
    base = _gen_planar(rng, c, ext=(0.3, 0.3), noise=0.002, frame=f)

    def make(t):
        P = base.copy()
        P[4] = c + 0.1 * f[:, 0] + t * f[:, 2]
        return P.astype(_F32)

    def dr(t):
        return gate_quantities(make(t)[None])["dist_ratio"][0]
    lo, hi = 0.0, 0.5
    if not (dr(lo) < 1 + rel < dr(hi)):
        return None
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        if dr(mid) < 1 + rel:
            lo = mid
        else:
            hi = mid
    for t in (lo, hi):
        e = dr(t) - 1
        if np.sign(e) == np.sign(rel) and abs(e) <= 10 * abs(rel):
            return make(t).astype(np.float64)
    return None


def _through_origin(rng, c):
    n = np.cross(c, rng.normal(size=3))
    n /= np.linalg.norm(n)
    u = np.cross(n, c)
    u /= np.linalg.norm(u)
    v = np.cross(n, u)
    uv = rng.uniform(-0.3, 0.3, size=(5, 2))
    return c + uv[:, :1] * u + uv[:, 1:] * v + rng.normal(0, rng.choice([0.002, 0.01, 0.03]), size=(5, 1)) * n


def _lattice(rng, c):
    """5 distinct voxel centres (i + 1/2) planeRes of a 3x3x3 neighbourhood."""
    ijk0 = np.floor(c / PLANE_RES).astype(np.int64)
    cells = np.array([(i, j, k) for i in range(3) for j in range(3) for k in range(3)])
    pick = cells[rng.choice(27, size=5, replace=False)]
    return ((ijk0 + pick).astype(np.float64) + 0.5) * np.float64(_F32(PLANE_RES))


def plane_sets(seed=0):
    """-> dict(map_xyzi float32 [5N, 4], scan_xyzi float32 [N, 4], sets float32 [N, 5, 3], label [N] str, + gate_quantities)
    Set i is map points 5i .. 5i+4; query i is scan point i."""
    rng = np.random.default_rng(seed)
    near_one = _slots([0.375])                     # z in [1/4, 1/2): the lam0-margin sets need 2^-25 steps in z
    others = _slots([-18.5, -8.5, 11.5, 21.5])
    far = [np.array([x, y, 1.5]) for x in (-520.0, -510.0, -500.0, -490.0, -480.0, 480.0, 490.0, 500.0, 510.0, 520.0)
           for y in (-20.0, -15.0, -10.0, -5.0, 0.0, 5.0, 10.0, 15.0, 20.0)]
    rng.shuffle(others)
    sets, labels = [], []

    def add(P, label):
        if P is not None:
            sets.append(np.asarray(P, np.float64).astype(_F32))
            labels.append(label)
    for c in near_one[:30 * 4]:
        i = len([lab for lab in labels if lab.startswith("lam0")])
        rel = [1e-3, -1e-3, 1e-7, -1e-7][i % 4]
        add(_lam0_margin(rng, c, rel), f"lam0_{rel:+.0e}")
    it = iter(others + near_one[30 * 4:])
    for split, name in ((5, "coincident_5"), (4, "coincident_4+1"), (3, "coincident_3+2")):
        for _ in range(60):
            add(_coincident(rng, next(it), split), name)
    for axis in range(3):
        for _ in range(40):
            add(_collinear_axis(rng, next(it), axis), "collinear_" + "xyz"[axis])
    for _ in range(60):
        add(_collinear_diag(rng, next(it)), "collinear_diag")
    for i in range(90):
        add(_coplanar_axis(rng, next(it), i % 3), "coplanar_axis")
    for i in range(108):
        h = [2.0 ** -3, 2.0 ** -4, 2.0 ** -5][i % 3]
        t = [2 * h, 3 * h, h][(i // 3) % 3]          # t = h: the repeated eigenvalue is the largest one (normal defined)
        add(_square_apex(rng, next(it), h, t, (i // 9) % 3, 1 if i % 2 else -1), "square_apex")
    for i in range(120):
        add(_ratio_margin(rng, next(it), [1e-3, -1e-3, 1e-7, -1e-7][i % 4]), f"ratio_{[1e-3, -1e-3, 1e-7, -1e-7][i % 4]:+.0e}")
    n_pd = 0
    while n_pd < 100:
        rel = [1e-3, -1e-3, 1e-5, -1e-5][n_pd % 4]
        P = _plane_dist_margin(rng, next(it), rel)
        if P is not None:
            add(P, f"plane_dist_{rel:+.0e}")
            n_pd += 1
    for _ in range(100):
        add(_through_origin(rng, next(it)), "through_origin")
    for _ in range(150):
        add(_lattice(rng, next(it)), "voxel_lattice")
    for _ in range(100):
        add(_gen_planar(rng, next(it)), "generic")
    for i, c in enumerate(far):
        kind = i % 3
        add(_gen_planar(rng, c) if kind == 0 else _coincident(rng, c, 5) if kind == 1 else _collinear_axis(rng, c, i % 2), "far_" + ["planar", "coincident", "collinear"][kind])
    P = np.stack(sets)
    q = gate_quantities(P)
    cen = P.astype(np.float64).mean(1)
    query = (cen + rng.uniform(-0.01, 0.01, size=cen.shape)).astype(_F32)
    ones = np.ones((len(P) * 5, 1), _F32)
    return dict(map_xyzi=np.concatenate([P.reshape(-1, 3), ones], 1), scan_xyzi=np.concatenate([query, ones[: len(P)]], 1), sets=P,
                label=np.array(labels), **q)


def edge_sets(seed=1, per_class=60):
    """10-point clusters for the line fit -> dict(map_xyzi [10N, 4], scan_xyzi [N, 4], label [N]); cluster i is map points 10i.."""
    rng = np.random.default_rng(seed)
    it = iter(_slots([-13.5, 6.5]))
    sets, labels = [], []
    for _ in range(per_class):
        c = next(it) + rng.uniform(-0.05, 0.05, 3)
        sets.append(np.repeat(c[None], 10, 0))
        labels.append("coincident_10")
    for i in range(per_class):
        c = next(it) + rng.uniform(-0.02, 0.02, 3)
        P = np.repeat(c[None], 10, 0)
        if i % 2:
            P[:, i % 3] += rng.uniform(-0.2, 0.2, 10)
        else:
            d = np.array([1.0, rng.integers(-1, 2), rng.integers(-1, 2)])[rng.permutation(3)]
            P = _dyadic(c) + rng.choice(np.arange(-3, 4), size=10)[:, None] * d[None, :] / 16.0
        sets.append(P)
        labels.append("collinear_10")
    for _ in range(per_class):
        a = next(it) + rng.uniform(-0.05, 0.05, 3)
        b = a + _unit(rng) * rng.uniform(0.05, 0.25)
        sets.append(np.array([a, b] * 5))
        labels.append("two_points_x5")
    P = np.stack(sets).astype(_F32)
    query = (P.astype(np.float64).mean(1) + rng.uniform(-0.01, 0.01, size=(len(P), 3))).astype(_F32)
    ones = np.ones((len(P) * 10, 1), _F32)
    return dict(map_xyzi=np.concatenate([P.reshape(-1, 3), ones], 1), scan_xyzi=np.concatenate([query, ones[: len(P)]], 1), sets=P,
                label=np.array(labels))

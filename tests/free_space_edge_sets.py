"""Hand-built free-space clearing cases whose answer is decided exactly: every scan return and map point sits at a pixel centre (or
on an axis, where atan2 is exact), the pose is the identity unless stated, and the ranges sit either far from the removal threshold
or exactly on it.  Shared by the restatement's own checks (test_free_space_edges_cpu.py) and the device's (test_free_space_edges.py).

Each case is a dict: name, opts (free_space_numpy.Opts), scan [n, 4] float32 (sensor frame), map [m, 4] float32, pose [7], want (the
counters the rule gives by hand) and on_edge: a point lies exactly on a threshold, a range gate, the azimuth seam or el_min.  The rule
decides such a case exactly here (the identity pose rotates without rounding, atan2 of +-0 is exact), but `bounds` leaves it open by
design: its slack is for rounding these cases do not have.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

import free_space_numpy as F

IDENTITY = np.array([0.0, 0, 0, 0, 0, 0, 1])
# W = 9 columns of 40 deg, H = 5 rows of 8 deg: az = 0 and el = 0 lie at the centre of pixel (2, 4), both exact in float
GRID_A = dict(az_res_deg=40.0, el_res_deg=8.0, el_min_deg=-20.0, el_max_deg=20.0)
# the same columns, H = 10 rows of 4 deg, so that a dilate 4 neighbourhood fits around rows 4 and 5
GRID_TALL = dict(az_res_deg=40.0, el_res_deg=4.0, el_min_deg=-20.0, el_max_deg=20.0)
BASE = dict(dilate=1, margin=0.25, margin_rel=0.0, min_range=0.5, max_range=100.0)
FAR, NEAR = 10.0, 3.0                   # a return past a map point at 5 m (threshold 5.25), and one in front of it


def opts(grid=GRID_A, **kw) -> F.Opts:
    d = dict(BASE)
    d.update(grid)
    d.update(kw)
    return F.Opts(**d)


def f32(v, toward=None):
    """float32(v), or the next float32 after it toward `toward`."""
    v = np.float32(v)
    return float(v if toward is None else np.nextafter(v, np.float32(toward)))


def _span(o, row, col):
    """(az, el) in degrees of the centre of pixel (row, col), the narrow last column and a partial top row included."""
    a0 = -180.0 + col * o.az_res_deg
    e0 = o.el_min_deg + row * o.el_res_deg
    return 0.5 * (a0 + min(a0 + o.az_res_deg, 180.0)), 0.5 * (e0 + min(e0 + o.el_res_deg, o.el_max_deg))


def direction(az_deg, el_deg, r):
    a, e = math.radians(az_deg), math.radians(el_deg)
    return [r * math.cos(e) * math.cos(a), r * math.cos(e) * math.sin(a), r * math.sin(e)]


def at(o, row, col, r):
    """The point at range r in the direction of the centre of pixel (row, col)."""
    return direction(*_span(o, row, col), r)


def cloud(pts) -> np.ndarray:
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    return np.c_[p, np.ones(len(p))].astype(np.float32)


def fill(o, r=FAR, skip=()):
    """One return at range r at the centre of every pixel, except the pixels in `skip`."""
    W, H = F.dims(o)
    return [at(o, i, j, r) for i in range(H) for j in range(W) if (i, j) not in set(skip)]


def case(name, o, scan, mp, want, pose=IDENTITY, on_edge=False):
    return dict(name=name, opts=o, scan=cloud(scan) if not isinstance(scan, np.ndarray) else scan, map=cloud(mp),
                pose=np.asarray(pose, np.float64), want=dict(zip(("n_image_points", "n_pixels_hit", "n_candidates", "n_removed"), want)),
                on_edge=on_edge)


# ---------------------------------------------------------------------------------------------------------------- A: decision ties
def cases_a():
    out = []
    o = opts()
    full = fill(o)                                                         # 45 returns at 10 m, one per pixel
    # margin 0.25: the threshold of the map point (4, 0, 0) is 4.25 exactly; a return at 4.25 keeps it, the next float removes it
    out.append(case("A tie margin kept", o, full + [[4.25, 0, 0]], [[4, 0, 0]], (46, 45, 1, 0), on_edge=True))
    out.append(case("A tie margin removed", o, full + [[f32(4.25, 9), 0, 0]], [[4, 0, 0]], (46, 45, 1, 1)))
    # margin_rel 0.125 * 4 = 0.5 beats margin 0.25: the tie moves to 4.5
    orel = opts(margin_rel=0.125)
    out.append(case("A tie margin_rel kept", orel, full + [[4.5, 0, 0]], [[4, 0, 0]], (46, 45, 1, 0), on_edge=True))
    out.append(case("A tie margin_rel removed", orel, full + [[f32(4.5, 9), 0, 0]], [[4, 0, 0]], (46, 45, 1, 1)))
    out.append(case("A margin beats margin_rel", orel, full + [[4.4, 0, 0]], [[4, 0, 0]], (46, 45, 1, 0)))
    # the range gate is inclusive at both ends
    out.append(case("A min_range inclusive", opts(min_range=4.0), full, [[4, 0, 0]], (45, 45, 1, 1), on_edge=True))
    out.append(case("A min_range next float", opts(min_range=f32(4.0, 9)), full, [[4, 0, 0]], (45, 45, 0, 0)))
    out.append(case("A max_range inclusive", opts(max_range=4.0), full, [[4, 0, 0]], (45, 45, 1, 1), on_edge=True))
    out.append(case("A max_range next float", opts(max_range=f32(4.0, 0)), full, [[4, 0, 0]], (45, 45, 0, 0)))
    # the neighbourhood's extent: a near return in its far corner keeps the point, one a column beyond does not; an unknown pixel in
    # the corner makes it no candidate, one beyond does not; dilate 2 reaches rows 0 and H - 1 exactly, dilate 3 leaves the image
    for d in (0, 1, 2):
        od = opts(dilate=d)
        out.append(case(f"A dilate {d} near in corner", od, full + [at(od, 2 + d, 4 + d, NEAR)], [at(od, 2, 4, 5)], (46, 45, 1, 0)))
        out.append(case(f"A dilate {d} near beyond", od, full + [at(od, 2, 5 + d, NEAR)], [at(od, 2, 4, 5)], (46, 45, 1, 1)))
        out.append(case(f"A dilate {d} unknown corner", od, fill(od, skip=[(2 - d, 4 - d)]), [at(od, 2, 4, 5)], (44, 44, 0, 0)))
        out.append(case(f"A dilate {d} unknown beyond", od, fill(od, skip=[(2, 3 - d)]), [at(od, 2, 4, 5)], (44, 44, 1, 1)))
    out.append(case("A dilate 3 leaves the image", opts(dilate=3), full, [at(o, 2, 4, 5)], (45, 45, 0, 0)))
    # row - d >= 0 and row + d < H decide at the bottom and the top of the image
    for row in (1, 3):
        out.append(case(f"A row {row} dilate 1 fits", opts(dilate=1), full, [at(o, row, 4, 5)], (45, 45, 1, 1)))
        out.append(case(f"A row {row} dilate 2 does not", opts(dilate=2), full, [at(o, row, 4, 5)], (45, 45, 0, 0)))
    return out


# ---------------------------------------------------------------------------------------------------------- B: degenerate returns
OVERFLOW = [3e38, 3e38, 0.0]            # finite, but its range 4.2e38 rounds to +inf in float
SUBNORMAL = float(np.float32(1e-40))


def degenerate_points():
    """Points that never reach the image: non-finite coordinates, the origin and its negative zeros."""
    pts = []
    for k in range(3):
        for v in (math.nan, math.inf, -math.inf):
            p = [1.0, 0.5, 0.25]
            p[k] = v
            pts.append(p)
    return pts + [[0.0, 0.0, 0.0], [-0.0, -0.0, -0.0]]


def case_b():
    """The overflowing return alone in pixel (2, 5) with known neighbours: the map point there is removed (the neighbourhood minimum
    is 10 m).  Subnormal returns alone in pixel (2, 3) make it known, with a minimum below any threshold: the map point there is a
    candidate and kept.  A subnormal point straight up lies outside the span."""
    o = opts()
    scan = fill(o, skip=[(2, 5), (2, 3)]) + degenerate_points() + [OVERFLOW]
    scan += [[SUBNORMAL, -SUBNORMAL, 0.0], [1.401298464324817e-45, -1.401298464324817e-45, 0.0], [0.0, 0.0, SUBNORMAL]]
    mp = [at(o, 2, 5, 5), at(o, 2, 3, 5)]
    return case("B degenerate returns", o, scan, mp, (46, 45, 2, 1))


def overflow_hand_example():
    """The 4 x 3 image (90 deg columns, 30 deg rows) with three ordinary returns and the overflowing one in pixel (1, 2): that pixel
    is known, so the map point in it is a candidate, and its minimum +inf exceeds any threshold."""
    o = F.Opts(az_res_deg=90.0, el_res_deg=30.0, el_min_deg=-45.0, el_max_deg=45.0, dilate=0, margin=0.1, margin_rel=0.0,
               min_range=0.0, max_range=100.0)
    scan = [direction(az, 0.0, 10.0) for az in (-135.0, -45.0, 135.0)] + [OVERFLOW]
    return case("B overflow 4x3", o, scan, [[5, 5, 0]], (4, 4, 1, 1))


# ------------------------------------------------------------------------------------------------- C: the seam and the span edges
def cases_c():
    out = []
    o = opts(dilate=0)
    # atan2(+-0, x < 0) = +-pi: +pi wraps to -pi, both are column 0; map points on the axis and at column 0's centre read it, column
    # W - 1's centre does not
    out.append(case("C seam +-0", o, [[-10, 0.0, 0], [-12, -0.0, 0]], [[-5, 0.0, 0], [-5, -0.0, 0], at(o, 2, 0, 5), at(o, 2, 8, 5)],
                    (2, 1, 3, 3), on_edge=True))
    # neighbourhoods across the seam: columns 0, 1, W - 2 and W - 1, dilate 0..4 (at dilate 4 the 9 columns are the whole row)
    ot = opts(GRID_TALL)
    W = F.dims(ot)[0]
    for c in (0, 1, W - 2, W - 1):
        for d in range(5):
            od = dataclasses.replace(ot, dilate=d)
            side = -1 if c < W / 2 else 1
            far, beyond = (c + side * d) % W, (c + side * (d + 1)) % W
            m = [at(od, 4, c, 5)]
            full = fill(od)
            out.append(case(f"C col {c} dilate {d} near across", od, full + [at(od, 4 + d, far, NEAR)], m, (91, 90, 1, 0)))
            if 2 * d + 1 < W:
                out.append(case(f"C col {c} dilate {d} near beyond", od, full + [at(od, 4, beyond, NEAR)], m, (91, 90, 1, 1)))
            out.append(case(f"C col {c} dilate {d} unknown across", od, fill(od, skip=[(4 - d, far)]), m, (89, 89, 0, 0)))
    # W = 1: every azimuth is column 0 (az_res 360 and 400)
    for az_res in (360.0, 400.0):
        o1 = opts(dict(GRID_TALL, az_res_deg=az_res), dilate=4)
        rows = [direction(37.0 * i - 150.0, _span(o1, i, 0)[1], FAR) for i in range(10)]
        m = [direction(123.0, _span(o1, 4, 0)[1], 5)]
        out.append(case(f"C W=1 az_res {az_res:g}", o1, rows, m, (10, 10, 1, 1)))
        out.append(case(f"C W=1 az_res {az_res:g} near", o1, rows + [direction(-90.0, _span(o1, 0, 0)[1], NEAR)], m, (11, 10, 1, 0)))
        out.append(case(f"C W=1 az_res {az_res:g} row 8 unknown", o1, rows[:8] + rows[9:], m, (9, 9, 0, 0)))
    # dilate 4 on W = 4: the neighbourhood covers every column, some twice
    o4 = opts(dict(GRID_TALL, az_res_deg=90.0), dilate=4)
    out.append(case("C W=4 dilate 4", o4, fill(o4), [at(o4, 4, 1, 5)], (40, 40, 1, 1)))
    out.append(case("C W=4 dilate 4 near", o4, fill(o4) + [at(o4, 8, 3, NEAR)], [at(o4, 4, 1, 5)], (41, 40, 1, 0)))
    out.append(case("C W=4 dilate 4 unknown", o4, fill(o4, skip=[(0, 2)]), [at(o4, 4, 1, 5)], (39, 39, 0, 0)))
    # el_min = 0: z = +0 and z = -0 are row 0; el_max = 0 leaves them out
    z_pm = [[10, 0, 0.0], [12, 0, -0.0]]
    m_pm = [[5, 0, 0.0], [5, 0, -0.0]]
    out.append(case("C el_min 0", opts(dict(GRID_A, el_min_deg=0.0, el_max_deg=20.0), dilate=0), z_pm, m_pm, (2, 1, 2, 2), on_edge=True))
    olo = opts(dict(GRID_A, el_min_deg=-20.0, el_max_deg=0.0), dilate=0)
    out.append(case("C el_max 0", olo, z_pm + [at(olo, 2, 4, FAR)], m_pm, (1, 1, 0, 0), on_edge=True))
    # a partial top row: [-20, 21] in 4 deg rows is 11 rows, the top one [20, 21); returns at 20.5 deg are in it, at 22 deg are not
    op = opts(dict(GRID_TALL, el_max_deg=21.0), dilate=1)
    assert F.dims(op) == (9, 11)
    low = [at(op, i, j, FAR) for i in (8, 9) for j in (3, 4, 5)]
    m = [at(op, 9, 4, 5)]
    out.append(case("C partial top row", op, low + [direction(_span(op, 10, j)[0], 20.5, FAR) for j in (3, 4, 5)], m, (9, 9, 1, 1)))
    out.append(case("C above el_max", op, low + [direction(_span(op, 10, j)[0], 22.0, FAR) for j in (3, 4, 5)], m, (6, 6, 0, 0)))
    # az_res 0.7: W = 515, the last column [179.8, 180) is narrow; its neighbourhood wraps to column 0
    on = opts(dict(GRID_TALL, az_res_deg=0.7), dilate=1)
    assert F.dims(on) == (515, 10)
    ring = [at(on, i, j, FAR) for i in (3, 4, 5) for j in (513, 514, 0)]
    m = [at(on, 4, 514, 5)]
    out.append(case("C narrow last column", on, ring, m, (9, 9, 1, 1)))
    out.append(case("C narrow last column near", on, ring + [at(on, 5, 0, NEAR)], m, (10, 9, 1, 0)))
    out.append(case("C narrow last column unknown", on, ring[:-1], m, (8, 8, 0, 0)))
    return out


# ---------------------------------------------------------------------------------------------------------------- D: column clamp
CLAMP_POINT = [-1.0, 4.5e-16, 0.0]        # atan2 = pi - 4.5e-16: the double just below pi, or pi itself


def case_d():
    """az_res 0.5 deg (W = 720): the clamp return lands in column W - 1 (the clamp) or 0 (az read as pi, wrapped) of row 2, never
    in row 3.  Map points at 0.6 m read pixels (2, 719), (2, 0) and (3, 0) alone (dilate 0); a known pixel with the 1 m return
    removes them.  Not exact: which of the first two is removed is atan2's last bit."""
    o = opts(dict(GRID_A, az_res_deg=0.5), dilate=0, min_range=0.1)
    return case("D column clamp", o, [CLAMP_POINT], [at(o, 2, 719, 0.6), at(o, 2, 0, 0.6), at(o, 3, 0, 0.6)], (1, 1, 1, 1))


def exact_cases():
    """Every hand-built case whose removal set the restatement decides exactly."""
    return cases_a() + [case_b(), overflow_hand_example()] + cases_c()

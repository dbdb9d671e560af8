"""Free-space clearing's edges in the numpy restatement (tests/free_space_numpy.py), without a GPU: the hand-built cases of
tests/free_space_edge_sets.py give the counters worked out by hand, and `bounds` decides each of them exactly, which is what lets the
device tests (test_free_space_edges.py) ask for equality.  Also the rule for a return whose float range overflows, and the bounds'
readings at the azimuth seam and at el_max."""
import math

import numpy as np
import pytest

import free_space_edge_sets as S
import free_space_numpy as F

_EXACT = S.exact_cases()


def test_overflowing_return_makes_its_pixel_known():
    """(3e38, 3e38, 0) is finite with r > 0, so it goes to its pixel; its float range is +inf.  The pixel is known, and the map point
    in it is a candidate whose neighbourhood minimum +inf exceeds the threshold."""
    c = S.overflow_hand_example()
    img, hit, n, n_hit = F.range_image(c["scan"], c["opts"])
    assert img.shape == (3, 4) and n == 4 and n_hit == 4
    assert hit[1].all() and img[1, 2] == np.float32(np.inf) and not hit[[0, 2]].any()
    rem, st = F.clear(c["map"], c["scan"], c["pose"], c["opts"])
    assert st == c["want"] and rem.tolist() == [True]
    lo, hi = F.bounds(c["map"], c["scan"], c["pose"], c["opts"])
    assert lo.tolist() == hi.tolist() == [True]


@pytest.mark.parametrize("k", range(len(_EXACT)), ids=[c["name"] for c in _EXACT])
def test_hand_case_is_decided_exactly(k):
    c = _EXACT[k]
    rem, st = F.clear(c["map"], c["scan"], c["pose"], c["opts"])
    assert st == c["want"]
    lo, hi = F.bounds(c["map"], c["scan"], c["pose"], c["opts"])
    assert not (lo & ~rem).any() and not (rem & ~hi).any()
    if not c["on_edge"]:
        assert np.array_equal(lo, hi)


def test_on_edge_cases_are_exact_by_construction():
    """The on-edge cases need no slack: the identity pose takes every map point to itself bit for bit, and the ranges on the
    threshold or the gate are exact in float."""
    for c in _EXACT:
        if c["on_edge"]:
            q = F.to_sensor(c["map"], c["pose"])
            assert np.array_equal(q, c["map"][:, :3].astype(np.float64)), c["name"]
    assert np.float32(4.25) == 4.25 and np.float32(4.0) + np.float32(0.125) * np.float32(4.0) == 4.5


def test_column_clamp_reads_column_w_minus_1_or_0():
    """(-1, 4.5e-16, 0) at az_res 0.5: (az + pi) / az_res rounds onto W = 720, clamped to column 719; were atan2 to return pi, the
    point would wrap to column 0.  The bounds read both and never row 3."""
    c = S.case_d()
    o = c["opts"]
    g = F._geom(o)
    p = c["scan"][:, :3].astype(np.float64)
    az = math.atan2(p[0, 1], p[0, 0])
    assert az < math.pi and (az + math.pi) / g["az_res"] == 720.0
    rem, st = F.clear(c["map"], c["scan"], c["pose"], o)
    assert rem.tolist() == [True, False, False] and st == c["want"]
    lo, hi = F.bounds(c["map"], c["scan"], c["pose"], o)
    assert lo.tolist() == [False, False, False] and hi.tolist() == [True, True, False]
    img, hit, _, _ = F.range_image(c["scan"], o, 1e-9, "both")
    assert np.argwhere(hit).tolist() == [[2, 0], [2, 719]]
    assert not F.range_image(c["scan"], o, 1e-9, "neither")[1].any()


def test_bounds_read_both_sides_of_a_seam_that_is_no_column_edge():
    """az_res 0.7: 360 / az_res is no integer, so az just below pi sits inside the narrow column 514, not at a column edge; the device
    may still read it as -pi, column 0."""
    o = S.opts(dict(S.GRID_TALL, az_res_deg=0.7), dilate=0)
    p = S.cloud([[-10.0, 1e-14, -0.35]])
    assert F.range_image(p, o)[1][:, 514].any()
    img, hit, _, _ = F.range_image(p, o, 1e-9, "both")
    assert sorted(np.argwhere(hit)[:, 1].tolist()) == [0, 514]


def test_bounds_at_el_max_inside_a_partial_top_row():
    """[-20, 21] in 4 deg rows: el_max = 21 deg lies inside row 10.  A return a hair below el_max may read as outside the span, one a
    hair above as inside it: "both" puts each into row 10, "neither" leaves each out, and a map point there is decided by neither."""
    o = S.opts(dict(S.GRID_TALL, el_max_deg=21.0), dilate=0)
    g = F._geom(o)
    for de in (-1e-14, 1e-14):
        el = g["el_max"] + de
        p = np.array([[10 * math.cos(el), 0.0, 10 * math.sin(el), 1.0]])
        hit_exact = F.range_image(p, o)[1]
        assert hit_exact.any() == (de < 0)
        assert F.range_image(p, o, 1e-9, "both")[1][10].any()
        assert not F.range_image(p, o, 1e-9, "neither")[1].any()
        lo, hi = F.bounds(0.5 * p, 2 * p, S.IDENTITY, o)        # FP64 clouds: float32 would move them 1e-7 pixel off the edge
        assert lo.tolist() == [False] and hi.tolist() == [True]

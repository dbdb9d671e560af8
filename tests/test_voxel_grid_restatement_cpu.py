"""The pcl::VoxelGrid restatement (oracle/voxel_grid_numpy.py) against the absolute-index formulas the map and the older tests
use, and on small clouds checked by hand: the bounding-box index, the verbatim fall-back and its threshold.  No GPU."""
import numpy as np
import pytest

from oracle import voxel_grid_numpy as vg
from conftest import get_case

LEAVES = (0.1, 0.2, 0.25, 0.3, 0.8)


def _cloud(rows):
    a = np.asarray(rows, dtype=np.float32).reshape(-1, 4)
    return a


@pytest.mark.parametrize("name", ["cfg1", "cfg2"])
@pytest.mark.parametrize("leaf", LEAVES)
def test_scan_equals_absolute_index(name, leaf):
    """Where PCL does not fall back, the bounding-box index orders voxels as (k, j, i) does: same bits as the absolute formula."""
    s = get_case(name)["scan_xyzi"].copy()
    s[::997, 1] = np.nan                              # non-finite rows are skipped by both
    assert not vg.falls_back(s, leaf)
    got = vg.voxel_grid(s, leaf)
    ref = vg.absolute_voxel_grid(s, leaf)
    assert got.dtype == np.float32 and got.shape == ref.shape and np.array_equal(got, ref)
    assert len(got) < np.isfinite(s[:, :3]).all(1).sum()


@pytest.mark.parametrize("name", ["cfg1", "cfg2"])
@pytest.mark.parametrize("leaf", LEAVES)
def test_map_blocks_equal_synth(name, leaf):
    """The per-block form (every 50 m block filtered on its own) against synth.voxel_filter_blocks, which the maps are made with."""
    from superodom_b200 import synth
    m = get_case(name)["map_xyzi"]
    if name == "cfg2":
        m = m[::4]
    got = vg.block_voxel_grid(m, leaf)
    ref = synth.voxel_filter_blocks(m, leaf)
    assert got.shape == ref.shape and np.array_equal(got, ref)


def test_map_insert_equals_oracle():
    """map_insert (old block clouds first, then the new points) against oracle.map_insert_numpy on a cfg1 scan put into its map."""
    from oracle import oracle as O
    case = get_case("cfg1")
    new = O.transform_scan_numpy(case["scan_xyzi"], case["pose_true"])
    for leaf in (0.2, 0.4):
        got = vg.map_insert(case["map_xyzi"], new, leaf)
        ref = O.map_insert_numpy(case["map_xyzi"], new, leaf)
        assert np.array_equal(got, ref), leaf


def test_far_pair_stays_two_points():
    """(0.1, 0.1, 0.1) and (26 214.5, 0.1, 0.1) at leaf 0.2: 131 073 voxels along x, no fall-back, two voxels."""
    c = _cloud([[0.1, 0.1, 0.1, 1.0], [26214.5, 0.1, 0.1, 2.0]])
    assert vg.extent(c, 0.2) == (131073, 1, 1) and not vg.falls_back(c, 0.2)
    idx, rows = vg.voxel_index(c, 0.2)
    assert list(rows) == [0, 1] and list(idx) == [0, 131072]
    assert np.array_equal(vg.voxel_grid(c, 0.2), c)


def test_overflow_threshold():
    """At leaf 0.25 every product below is exact.  dx dy dz = 1024 * 1024 * 2048 = 2^31 falls back (the input, NaN rows and order
    kept); 1024 * 1024 * 2047 is filtered."""
    nan = np.nan
    over = _cloud([[0, 0, 0, 1], [nan, 1, 1, 5], [255.75, 255.75, 511.75, 3], [0.1, 0.1, 0.1, 7]])
    assert vg.extent(over, 0.25) == (1024, 1024, 2048) and vg.falls_back(over, 0.25)
    out = vg.voxel_grid(over, 0.25)
    assert out.shape == over.shape and np.array_equal(out, over, equal_nan=True)
    under = over.copy()
    under[2, 2] = 511.5
    assert vg.extent(under, 0.25) == (1024, 1024, 2047) and not vg.falls_back(under, 0.25)
    out = vg.voxel_grid(under, 0.25)
    assert np.array_equal(out, _cloud([[0.05, 0.05, 0.05, 4], [255.75, 255.75, 511.5, 3]]))


def test_scaled_scan_falls_back():
    """A cfg1 scan with every 997th point scaled by 400 spans about 7e13 voxels at leaf 0.2: PCL returns it unchanged."""
    s = get_case("cfg1")["scan_xyzi"].copy()
    s[::1000, 0] = np.nan
    s[5::997, :3] *= np.float32(400.0)
    dx, dy, dz = vg.extent(s, 0.2)
    assert dx * dy * dz > 10 ** 13
    out = vg.voxel_grid(s, 0.2)
    assert np.array_equal(out, s, equal_nan=True)


def test_index_relative_to_bounds():
    """idx = i + j div_x + k div_x div_y from the cloud's minimum voxel, and the float subtraction it is taken with."""
    c = _cloud([[-0.3, 0.0, -0.0, 1], [0.25, 0.45, 0.25, 2], [-0.05, -0.0, 0.0, 3], [0.0, 0.2, 0.19999999, 4]])
    inv = vg.inverse_leaf(0.2)
    assert inv == np.float32(5.0)
    # floor(v * 5): x -2, 1, -1, 0; y 0, 2, -0, 1 (0.2f * 5 rounds to 1); z -0, 1, 0, 0 (0.19999999f * 5 < 1)
    idx, rows = vg.voxel_index(c, 0.2)
    # min_b = (-2, 0, 0), max_b = (1, 2, 1), div = (4, 3, 2): idx = i + 4 j + 12 k
    assert list(rows) == [0, 1, 2, 3] and list(idx) == [0, 3 + 4 * 2 + 12, 1, 2 + 4]
    out = vg.voxel_grid(c, 0.2)
    assert np.array_equal(out, c[np.argsort(idx, kind="stable")])


def test_no_finite_point():
    """The empty cloud and a cloud without a finite point give the empty cloud."""
    assert vg.voxel_grid(np.zeros((0, 4), np.float32), 0.2).shape == (0, 4)
    c = _cloud([[np.nan, 0, 0, 1], [0, np.inf, 0, 1], [0, 0, -np.inf, 1]])
    assert vg.voxel_grid(c, 0.2).shape == (0, 4) and not vg.falls_back(c, 0.2)


def test_adjust_statistic_and_leaves():
    """mean|x| mean|y| mean|z| in float, the < 25 / > 65 rule; NaN leaves the leaves as they were."""
    c = _cloud([[3, 3, 3, 0], [-3, 3, -3, 0]])
    assert vg.adjust_statistic(c) == 27.0
    assert vg.adjust_leaves(27.0, 0.2, 0.4) == (float(np.float32(0.2)), float(np.float32(0.4)))
    assert vg.adjust_leaves(25.0, 0.2, 0.4) == vg.adjust_leaves(65.0, 0.2, 0.4) == (float(np.float32(0.2)), float(np.float32(0.4)))
    assert vg.adjust_leaves(float(np.nextafter(np.float32(25), np.float32(0))), 0.2, 0.4)[1] == float(np.float32(0.2))
    assert vg.adjust_leaves(float(np.nextafter(np.float32(65), np.float32(100))), 0.2, 0.4)[1] == float(np.float32(0.8))
    c[1, 0] = np.nan
    avg = vg.adjust_statistic(c)
    assert np.isnan(avg) and vg.adjust_leaves(avg, 0.2, 0.4) == (float(np.float32(0.2)), float(np.float32(0.4)))

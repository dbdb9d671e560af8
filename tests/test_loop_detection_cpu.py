"""Properties of the loop-detection restatement (loop_detection_numpy.py), which the GPU tests compare the device against: a cloud
turned by whole sectors is found at that shift with distance 0, the distance is symmetric under swapping query and candidate with the
opposite shift, roll and pitch carried by the pose are levelled out, and an empty descriptor carries no evidence."""
import math

import numpy as np
import pytest

import loop_detection_numpy as LD

IDENT = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])


def _polar_cloud(o, seed, shift=0):
    """Points at cell centres (several per cell, random heights) of a random half of the cells; shift turns the cloud by whole
    sectors (sector j -> j + shift)."""
    rng = np.random.default_rng(seed)
    w = 2 * math.pi / o.sectors
    pts = []
    for r in range(o.rings):
        for j in range(o.sectors):
            if rng.random() < 0.5:
                continue
            rho = (r + 0.5) * o.max_range / o.rings
            az = -math.pi + ((j + shift) % o.sectors + 0.5) * w
            for z in rng.uniform(-1.5, 4.0, 3):
                pts.append([rho * math.cos(az), rho * math.sin(az), z, 1.0])
    return np.array(pts, np.float32)


def _quat(roll, pitch, yaw):
    from scipy.spatial.transform import Rotation
    return Rotation.from_euler("ZYX", [yaw, pitch, roll]).as_quat()


@pytest.mark.parametrize("k", [0, 1, 7, 30, 59])
def test_whole_sector_turn_gives_its_shift(k):
    o = LD.Opts()
    a = LD.describe(_polar_cloud(o, 3), IDENT, o)
    b = LD.describe(_polar_cloud(o, 3, shift=k), IDENT, o)
    lo, hi = LD.describe_bounds(_polar_cloud(o, 3, shift=k), IDENT, o)
    assert np.array_equal(lo, hi) and np.array_equal(lo, b)         # no point near an edge
    assert np.array_equal(np.roll(a, k, axis=1), b)
    d, s, n = LD.pair(a, b)
    assert s == k and abs(d) < 1e-12 and n == int((LD.norms(a) > 0).sum())
    assert LD.yaw_of(s, o.sectors) == pytest.approx(math.remainder(k * 2 * math.pi / o.sectors, 2 * math.pi))
    y = LD.yaw_of(s, o.sectors)
    assert -math.pi < y <= math.pi


def test_yaw_sign_follows_the_heading():
    """The same world seen from a sensor turned by +k sectors: the query's heading minus the candidate's is +k sectors."""
    o = LD.Opts()
    k = 12
    world = _polar_cloud(o, 5)
    from scipy.spatial.transform import Rotation
    yaw = k * 2 * math.pi / o.sectors
    q_pose = np.r_[0, 0, 0, _quat(0, 0, yaw)]
    seen = Rotation.from_quat(q_pose[3:]).inv().apply(world[:, :3].astype(np.float64))    # sensor frame of the turned sensor
    q_cloud = np.c_[seen, world[:, 3]].astype(np.float32)
    # the descriptor levels the heading out, so describe the turned sensor at a pose without its heading
    a = LD.describe(q_cloud, IDENT, o)
    b = LD.describe(world, IDENT, o)
    d, s, _ = LD.pair(a, b)
    assert abs(d) < 1e-12
    assert LD.yaw_of(s, o.sectors) == pytest.approx(yaw)


def test_distance_symmetry():
    rng = np.random.default_rng(1)
    o = LD.Opts(rings=8, sectors=24)
    for _ in range(5):
        a = np.where(rng.random((8, 24)) < 0.6, rng.uniform(0, 6, (8, 24)), 0).astype(np.float32)
        b = np.where(rng.random((8, 24)) < 0.6, rng.uniform(0, 6, (8, 24)), 0).astype(np.float32)
        a[:, 3] = 0                                                 # an empty column on each side
        b[:, 10] = 0
        dab, nab = LD.distances(a, b)
        dba, nba = LD.distances(b, a)
        for s in range(o.sectors):
            assert nab[s] == nba[(-s) % o.sectors]
            assert dab[s] == pytest.approx(dba[(-s) % o.sectors], abs=1e-14)


@pytest.mark.parametrize("roll,pitch", [(0.1, 0.0), (0.0, -0.12), (0.08, 0.06)])
def test_tilt_in_the_pose_is_levelled(roll, pitch):
    """A sensor tilted by roll and pitch, with a pose carrying the tilt, describes its surroundings as a level sensor does."""
    from scipy.spatial.transform import Rotation
    o = LD.Opts()
    rng = np.random.default_rng(2)
    world = np.c_[rng.uniform(-70, 70, (20000, 2)), rng.uniform(-1.8, 5.0, 20000), np.ones(20000)].astype(np.float32)
    q = _quat(roll, pitch, 0.0)
    seen = Rotation.from_quat(q).inv().apply(world[:, :3].astype(np.float64))
    tilted = LD.describe(np.c_[seen, world[:, 3]], np.r_[0, 0, 0, q], o)
    lo, hi = LD.describe_bounds(world, IDENT, o, eps=1e-6)
    tol = 1e-5
    assert np.all(lo <= tilted + tol) and np.all(tilted <= hi + tol)
    assert np.count_nonzero(lo) > 500
    # unlevelled (identity pose), the tilted view does not describe the same
    raw = LD.describe(np.c_[seen, world[:, 3]], IDENT, o)
    assert not (np.all(lo <= raw + tol) and np.all(raw <= hi + tol))


def test_empty_descriptor_has_no_evidence():
    o = LD.Opts()
    e = np.zeros((o.rings, o.sectors), np.float32)
    a = LD.describe(_polar_cloud(o, 4), IDENT, o)
    for x, y in ((e, e), (e, a), (a, e)):
        d, s, n = LD.pair(x, y)
        assert (d, s, n) == (1.0, 0, 0)


def test_cell_rules():
    """Below -height_offset reads 0; a point at max_range is left out; the seam folds to sector 0."""
    o = LD.Opts(rings=4, sectors=8, max_range=8.0, height_offset=2.0)
    pts = np.array([[1.0, 0.1, -3.0, 0], [8.0, 0.0, 1.0, 0], [-3.0, 0.0, 1.0, 0], [-3.0, -1e-300, 0.5, 0]], np.float32)
    img = LD.describe(pts, IDENT, o)
    assert img[0, 4] == 0.0 and np.count_nonzero(img) == 1
    assert img[1, 0] == np.float32(3.0)                              # (-3, 0): atan2 = pi folds to -pi, sector 0
    lo, hi = LD.describe_bounds(pts, IDENT, o)
    assert lo[1, 0] == 0 and hi[1, 0] == np.float32(3.0) and hi[1, 7] == np.float32(3.0)


def test_search_order_and_padding():
    rng = np.random.default_rng(9)
    descs = np.where(rng.random((6, 5, 12)) < 0.5, rng.uniform(0, 3, (6, 5, 12)), 0).astype(np.float32)
    descs[2] = descs[0]                                              # duplicates: equal distances, id order
    out = LD.search(descs, [5, 3, 1], 4, 1)
    keys = [(t[1], t[0]) for t in out[0]]
    assert len(keys) == 4 and keys == sorted(keys)
    full = LD.search(descs, [5], 4, 0)[0]
    assert [t[0] for t in full].index(0) + 1 == [t[0] for t in full].index(2)    # the duplicate follows its twin
    assert [t[0] for t in out[1]][2:] == [-1, -1]                    # query 3, exclude 1: ids 0, 1 eligible
    assert [t[0] for t in out[2]] == [-1] * 4                        # query 1: none


def _bits(rows):
    return [[(i, np.float64(d).tobytes(), s, n, np.float64(y).tobytes()) for i, d, s, n, y in row] for row in rows]


@pytest.mark.parametrize("rings,sectors", [(1, 2), (1, 31), (3, 32), (2, 33), (1, 65), (64, 2), (64, 33), (5, 65)])
def test_search_many_equals_search(rings, sectors):
    """search_many == search bit for bit (distances and yaws compared as bytes) on random images with crafted members: duplicates,
    images periodic in the sectors (tied shifts), an all-zero image, a single-column image, and every exclude / k edge."""
    rng = np.random.default_rng([rings, sectors])
    n = 13
    descs = np.where(rng.random((n, rings, sectors)) < 0.6, rng.uniform(0, 6, (n, rings, sectors)), 0).astype(np.float32)
    descs[4] = descs[1]                                              # duplicates
    descs[9] = descs[1]
    tile = rng.uniform(0, 3, (rings, 2 if sectors % 2 == 0 else 1)).astype(np.float32)
    descs[6] = np.tile(tile, (1, sectors // tile.shape[1]))          # periodic: the shifts of each period tie
    descs[7] = 0                                                    # empty: distance 1.0, n_pairs 0 against everything
    descs[11] = 0
    descs[11][:, sectors // 2] = 2.5                                 # one occupied column
    descs[12] = np.roll(descs[3], sectors - 1, axis=1)               # a turned copy: the shift wraps
    queries = [12, 0, 7, 9, 12, 4, 11, 6, 1]
    for k, exclude in ((1, 0), (3, 2), (5, 0), (13, 0), (16, 4), (2, 12), (4, 13)):
        want = LD.search(descs, queries, k, exclude)
        got = LD.search_many(descs, queries, k, exclude)
        assert _bits(got) == _bits(want), (k, exclude)
    # a tiny chunk size: the candidates split over several vectorised chunks give the same row
    A = descs.astype(np.float64)
    nrm = LD._norms_all(A)
    assert _bits([LD._row(A, nrm, 12, 12, 13, sectors, chunk_elems=1)]) == _bits(LD.search(descs, [12], 13, 0))

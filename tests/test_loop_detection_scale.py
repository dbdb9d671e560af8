"""Loop detection (so_loop_candidates, so_keyframe_descriptors) at the sizes it is built for and at its edges, against search_many and
describe / describe_bounds of loop_detection_numpy.py, every candidate field bit for bit.

Code paths reached (kLoopTile = 32 candidates per search CTA, k_loop_topk = 256 threads in 8 warps, kLoopPairCap = 2^20 pair entries):
  - 1 100 keyframes: up to 35 tiles per query, the last one partial; copies of one cloud at ids 5, 37, 300, 1 050 and 1 099 lie in
    tiles 0, 1, 9 and 32 and in top-k threads 5, 37, 44 and 26 (warps 0, 1, 1, 0), so their ties cross tiles and warps; top-k
    threads hold up to 5 candidates each; k = 64;
  - pair-table chunks: 1 000 repeats of query 1 099 make 2 chunks (954 + 46 rows of stride 1 099); ascending, descending and shuffled
    orders of ids 0 .. 1 099 grow the stride inside a chunk; 70 000 queries of ids 0 .. 16 make 2 chunks at the 65 535-query limit
    (65 535 x 16 <= 2^20);
  - eligible counts 0, 1, 31, 32, 33, 63, 64, 65, 256, 257 with k at, below and above each: empty, single, partial and full tiles,
    one and two candidates per top-k thread, and the padding slots;
  - shapes: rings 1 and 64 by sectors 2, 31, 32, 33, 64, 65 and 360 (lanes with 0 .. 12 shifts each), 64 x 360 on 40 keyframes;
  - descriptors of 200 000 points in one cell, of keyframes with no finite point inside max_range, of poses pitched +-90 deg (h = 0
    in the levelling) and of a non-normalised quaternion; the descriptor table copied by so_keyframe_reserve.
Not reached: one query with more than 2^20 eligible keyframes, where the pair table grows past kLoopPairCap (its descriptor table
alone would take about 5 GB)."""
import math

import numpy as np
import pytest

import loop_detection_numpy as LD
from test_keyframes import _ctx
from test_loop_detection import _add, _polar, _quat

IDENT = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
N_BIG = 1100
COPIES = (5, 37, 300, 1050, 1099)
SMALL = LD.Opts(rings=4, sectors=8)
DEFAULT = LD.Opts()


def _cloud(seed, n=300, max_range=80.0):
    rng = np.random.default_rng(seed)
    rho = rng.uniform(1.0, max_range - 1.0, n)
    az = rng.uniform(-math.pi, math.pi, n)
    return np.c_[rho * np.cos(az), rho * np.sin(az), rng.uniform(-1.5, 4.0, n), np.ones(n)].astype(np.float32)


def _four_fold(seed, n=100):
    """A cloud that maps onto itself under a quarter turn ((x, y) -> (-y, x) is exact in float): periodic images at sectors % 4 == 0."""
    c = _cloud(seed, n)
    turns = [c]
    for _ in range(3):
        t = turns[-1].copy()
        t[:, 0], t[:, 1] = -turns[-1][:, 1], turns[-1][:, 0]
        turns.append(t)
    return np.concatenate(turns, 0)


def _pose(rng):
    return np.r_[rng.uniform(-50, 50, 2), rng.uniform(-1, 1), _quat(*rng.normal(0, [0.03, 0.03, 2.0]))]


def _store(api, clouds, poses, cap_points=None, cap_frames=None):
    ctx = _ctx(api)
    ctx.keyframe_reserve(cap_points or max(sum(len(c) for c in clouds), 1), cap_frames or len(clouds))
    for c, p in zip(clouds, poses):
        _add(ctx, c, p)
    return ctx


@pytest.fixture(scope="module")
def big(gpu_api):
    rng = np.random.default_rng(11)
    clouds, poses = [], []
    for i in range(N_BIG):
        if i in COPIES[1:]:
            c, p = clouds[COPIES[0]], poses[COPIES[0]]
        elif i == 200:
            c, p = _four_fold(200), IDENT
        elif i == 400:
            c, p = np.array([[500.0, 0.0, 1.0, 1.0]], np.float32), IDENT      # nothing inside max_range: an all-zero image
        else:
            c, p = _cloud(i), _pose(rng)
        clouds.append(c)
        poses.append(p)
    ctx = _store(gpu_api, clouds, poses)
    ids = np.arange(N_BIG)
    d = {o.sectors: ctx.keyframe_descriptors(ids, **o.kw()) for o in (SMALL, DEFAULT)}
    yield ctx, d
    ctx.close()


def _want(descs, queries, k, exclude):
    """search_many's rows as the device's structured array [len(queries), k]."""
    from superodom_b200.api import LOOP_CANDIDATE_DTYPE
    queries = np.asarray(queries, np.int64)
    uq, inv = np.unique(queries, return_inverse=True)
    rows = LD.search_many(descs, uq, k, exclude)
    a = np.zeros((len(uq), k), LOOP_CANDIDATE_DTYPE)
    for i, (q, row) in enumerate(zip(uq, rows)):
        a[i]["query"] = q
        a[i]["id"], a[i]["distance"], a[i]["shift"], a[i]["n_pairs"], a[i]["yaw"] = map(np.array, zip(*row))
    return a[inv]


def _same(got, want, what):
    if got.tobytes() != want.tobytes():
        bad = np.flatnonzero([g.tobytes() != w.tobytes() for g, w in zip(got, want)])
        i = int(bad[0])
        raise AssertionError(f"{what}: {len(bad)} rows differ; first: row {i}\n got  {got[i]}\n want {want[i]}")


def _opts(o, exclude):
    return dict(o.kw(), exclude_recent=exclude)


# ------------------------------------------------------------------------------------------------------------- 1. tiles, top-k
@pytest.mark.gpu
@pytest.mark.parametrize("exclude", [0, 30])
def test_tiles_and_topk_at_scale(big, exclude):
    ctx, d = big
    every = np.arange(N_BIG)
    got = ctx.loop_candidates(every, 64, **_opts(SMALL, exclude))
    _same(got, _want(d[8], every, 64, exclude), f"4 x 8, exclude {exclude}")
    some = np.r_[1099, 1050, 1049, 1000, 777, 400, 300, 256, 200, 100, 64, 37, 31][::1 if exclude else -1]
    got = ctx.loop_candidates(some, 64, **_opts(DEFAULT, exclude))
    _same(got, _want(d[60], some, 64, exclude), f"20 x 60, exclude {exclude}")
    if exclude == 0:                                                   # the copies of 1 099: tied, in id order, ahead of all else
        for o in (SMALL, DEFAULT):
            row = ctx.loop_candidates([1099], 64, **_opts(o, 0))[0]
            assert list(row["id"][:4]) == list(COPIES[:4]) and len(set(row["distance"][:4])) == 1
            assert row["distance"][3] < row["distance"][4]
        # the empty image: distance 1.0 with no pairs against everything
        row = ctx.loop_candidates([400], 64, **_opts(DEFAULT, 0))[0]
        assert np.all(row["distance"] == 1.0) and np.all(row["n_pairs"] == 0) and np.all(row["shift"] == 0)
        assert list(row["id"]) == list(range(64))


# ------------------------------------------------------------------------------------------------------------- 2. pair-table chunks
@pytest.mark.gpu
def test_chunks_equal_single_queries(big):
    ctx, d = big
    o = _opts(SMALL, 0)
    one = ctx.loop_candidates([1099], 64, **o)[0]
    want = _want(d[8], [1099], 64, 0)[0]
    assert one.tobytes() == want.tobytes()
    rep = ctx.loop_candidates(np.full(1000, 1099), 64, **o)                 # 2 chunks: 954 + 46 rows
    assert all(r.tobytes() == one.tobytes() for r in rep)
    every = np.arange(N_BIG)
    ref = _want(d[8], every, 64, 0)
    singles = {q: ctx.loop_candidates([q], 64, **o)[0] for q in (0, 1, 500, 953, 954, 955, 1098, 1099)}
    rng = np.random.default_rng(3)
    for order in (every, every[::-1], rng.permutation(every)):
        got = ctx.loop_candidates(order, 64, **o)
        _same(got, ref[order], "ordered queries")
        for q, s in singles.items():
            assert got[int(np.flatnonzero(order == q)[0])].tobytes() == s.tobytes()


@pytest.mark.gpu
def test_more_than_65535_queries(big):
    ctx, d = big
    rng = np.random.default_rng(5)
    queries = rng.integers(0, 17, 70000)
    queries[[0, 65534, 65535, 69999]] = (16, 3, 16, 0)                      # both sides of the chunk boundary
    got = ctx.loop_candidates(queries, 17, **_opts(SMALL, 0))
    _same(got, _want(d[8], queries, 17, 0), "70 000 queries")


@pytest.mark.gpu
def test_eligible_count_boundaries(big):
    ctx, d = big
    exclude = 30
    for m in (0, 1, 31, 32, 33, 63, 64, 65, 256, 257):
        q = exclude + m
        for k in sorted({x for x in (m - 1, m, m + 1) if 1 <= x <= 64} or {1, 64}):
            got = ctx.loop_candidates([q], k, **_opts(DEFAULT, exclude))
            _same(got, _want(d[60], [q], k, exclude), f"eligible {m}, k {k}")
            pad = got[0][min(m, k):]
            assert np.all(pad["id"] == -1) and np.all(pad["distance"] == 1.0) and np.all(pad["shift"] == 0)
            assert np.all(pad["n_pairs"] == 0) and np.all(pad["yaw"] == 0.0) and np.all(pad["query"] == q)
            assert np.all(got[0][:min(m, k)]["id"] >= 0)


# ------------------------------------------------------------------------------------------------------------- 3. shapes
@pytest.fixture(scope="module")
def shapes_store(gpu_api):
    rng = np.random.default_rng(21)
    o = LD.Opts(rings=64, sectors=360)
    base = [(r, j, float(z)) for r, j, z in zip(rng.integers(0, 64, 400), rng.integers(0, 360, 400), rng.uniform(-1.5, 4.0, 400))]
    clouds = [_cloud(1000 + i, 400) for i in range(40)]
    clouds[7] = _polar(o, base)                                          # cell centres at 64 x 360
    clouds[33] = _polar(o, [(r, (j + 160) % 360, z) for r, j, z in base])   # turned by 160 sectors: found at shift 200, yaw past pi
    clouds[20] = _four_fold(20)
    poses = [_pose(rng) for _ in clouds]
    for i in (7, 33, 20):
        poses[i] = IDENT
    ctx = _store(gpu_api, clouds, poses)
    yield ctx
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rings", [1, 64])
@pytest.mark.parametrize("sectors", [2, 31, 32, 33, 64, 65, 360])
def test_shapes_equal_the_restatement(shapes_store, rings, sectors):
    ctx = shapes_store
    o = LD.Opts(rings=rings, sectors=sectors)
    n = 40
    descs = ctx.keyframe_descriptors(np.arange(n), **o.kw())
    queries = np.arange(n) if rings * sectors * sectors < 1 << 20 else np.array([39, 33, 20, 8])
    got = ctx.loop_candidates(queries, 16, **_opts(o, 0))
    _same(got, _want(descs, queries, 16, 0), f"{rings} x {sectors}")
    live = got[got["id"] >= 0]
    if rings == 1:                                                      # one ring: every cosine is 1, all shifts tie at distance 0
        assert np.all(live["shift"] == 0) and np.all(live["distance"] < 1e-12)
    elif sectors > 2:                                                   # shifts on both sides of pi, each with its yaw
        assert np.any(live["shift"] > sectors // 2) and np.any(live["yaw"] < 0)
    if (rings, sectors) == (64, 360):
        best = got[list(queries).index(33)][0]
        assert int(best["id"]) == 7 and int(best["shift"]) == 200 and best["distance"] < 1e-12
        assert float(best["yaw"]) == LD.yaw_of(200, 360) and best["yaw"] < -math.pi / 2


# ------------------------------------------------------------------------------------------------------------- 4. descriptor edges
def _edge_clouds():
    rng = np.random.default_rng(31)
    o = DEFAULT
    w = 2 * math.pi / o.sectors
    az = -math.pi + (17 + rng.uniform(0.2, 0.8, 200000)) * w            # ring 12, sector 17: well inside the cell
    rho = (12 + rng.uniform(0.2, 0.8, 200000)) * o.max_range / o.rings
    one_cell = np.c_[rho * np.cos(az), rho * np.sin(az), rng.uniform(-3.0, 6.0, 200000), np.ones(200000)].astype(np.float32)
    beyond = np.array([[500.0, 0.0, 1.0, 1.0], [0.0, -80.0, 1.0, 1.0], [-90.0, 5.0, 0.0, 1.0]], np.float32)
    bad = np.array([[np.nan, 1.0, 1.0, 1.0], [np.inf, 0.0, 0.0, 1.0], [1.0, -np.inf, 0.0, 1.0], [2.0, 3.0, np.nan, 1.0],
                    [300.0, 1.0, 1.0, 1.0]], np.float32)
    up, down = np.r_[0, 0, 0, 0.5, 0.5, -0.5, 0.5], np.r_[0, 0, 0, 0.5, -0.5, 0.5, 0.5]      # pitch -+90 deg: R00 = R10 = 0 exactly
    near = np.r_[0, 0, 0, 0.0, math.sin(math.pi / 4), 0.0, math.cos(math.pi / 4)]               # 90 deg up to rounding
    skew = np.r_[1.0, -2.0, 0.5, 0.3, -0.6, 0.9, 2.7]                                            # not normalised
    clouds = [_cloud(1), one_cell, beyond, bad, _cloud(2), _cloud(3), _cloud(4), _cloud(5), _cloud(1)]
    poses = [IDENT, IDENT, IDENT, IDENT, up, down, near, skew, skew]
    return clouds, poses


@pytest.mark.gpu
def test_descriptor_edges(gpu_api):
    clouds, poses = _edge_clouds()
    n = len(clouds)
    ctx = _store(gpu_api, clouds, poses)
    assert ctx.keyframe_info()[1] >= 200000
    for o in (DEFAULT, LD.Opts(rings=64, sectors=360)):
        dev = ctx.keyframe_descriptors(np.arange(n), **o.kw())
        for i in range(n):
            kept = ctx.keyframe_download(i, 0)
            lo, hi = LD.describe_bounds(kept, poses[i], o)
            assert np.all(lo <= dev[i]) and np.all(dev[i] <= hi), i
            sure = lo == hi
            assert sure.mean() > 0.99 and np.array_equal(dev[i][sure].view(np.uint32), lo[sure].view(np.uint32)), i
        assert not dev[2].any() and not dev[3].any()                     # no finite point inside max_range
        for i in (4, 5, 6, 7):
            assert np.count_nonzero(dev[i]) > 20
        got = ctx.loop_candidates(np.arange(n), 8, **_opts(o, 0))
        _same(got, _want(dev, np.arange(n), 8, 0), f"edges {o.rings} x {o.sectors}")
        for q in (2, 3):
            live = got[q][got[q]["id"] >= 0]
            assert np.all(live["distance"] == 1.0) and np.all(live["n_pairs"] == 0) and np.all(live["shift"] == 0)
        for q in range(4, n):
            row = {int(c["id"]): c for c in got[q]}
            assert all(row[i]["distance"] == 1.0 and row[i]["n_pairs"] == 0 for i in (2, 3) if i in row)
    # the cell's maximum of 200 000 heights (float32 of z + h, as the device rounds it)
    v = np.maximum(np.float32(0), (clouds[1][:, 2].astype(np.float64) + DEFAULT.height_offset).astype(np.float32)).max()
    dev = ctx.keyframe_descriptors([1], **DEFAULT.kw())[0]
    assert dev[12, 17] == v and np.count_nonzero(dev) == 1
    ctx.close()


@pytest.mark.gpu
def test_descriptor_table_growth(gpu_api):
    """so_keyframe_reserve copies the 64 x 360 table when it grows the frame table alone and when it grows both pools and frames."""
    clouds = [_cloud(300 + i) for i in range(24)]
    rng = np.random.default_rng(41)
    poses = [_pose(rng) for _ in clouds]
    o = _opts(LD.Opts(rings=64, sectors=360), 0)
    ids = np.arange(len(clouds))
    cap = sum(len(c) for c in clouds) + 100
    a = _store(gpu_api, clouds, poses, cap_points=cap, cap_frames=len(clouds))
    want_d = a.keyframe_descriptors(ids, **o)
    want_c = a.loop_candidates(ids[-4:], 8, **o)
    fresh = _store(gpu_api, [a.keyframe_download(i, 0) for i in ids], poses)
    for caps in ((cap, len(clouds) + 40), (2 * cap, len(clouds) + 100)):
        a.keyframe_reserve(*caps)
        got, st = a.loop_candidates(ids[-4:], 8, stats=True, **o)
        assert st["n_described"] == 0, caps                           # every descriptor came across
        assert a.keyframe_descriptors(ids, **o).tobytes() == want_d.tobytes() == fresh.keyframe_descriptors(ids, **o).tobytes()
        assert got.tobytes() == want_c.tobytes() == fresh.loop_candidates(ids[-4:], 8, **o).tobytes()
    _same(want_c, _want(want_d, ids[-4:], 8, 0), "grown table")
    a.close()
    fresh.close()

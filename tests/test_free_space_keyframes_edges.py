"""so_map_clear_free_space_keyframes at its edges on the device, every case against two references:
  R1, the definition on the device: so_map_clear_free_space of each entry's downloaded surf cloud in list order, on a second context
      with the same history: both stores (map_download order, bit for bit), k-NN on probes, 5 x 5 block counts, n_removed,
      n_image_points, n_pixels_hit and n_after;
  R2, the numpy restatement (free_space_keyframe_sets.restate): the removal set is the union of the entries' removals, n_candidates
      the size of the union of their candidate masks (each point once), n_tiles the tile plan of so_free_rule.h.  Points that
      free_space_numpy.edge_points marks as ambiguous are held between the bounds; each case prints how many it met.
Cases: keyframes spread over the window at list sizes around the cull's 32-lane warps and 128-keyframe rounds; reach at block faces;
tile seams at the largest image (4 images a tile); store states; entry lists with duplicates, empties and degenerate returns."""
import numpy as np
import pytest

import free_space_keyframe_sets as K

pytestmark = pytest.mark.gpu


def _fs(api, o):
    return api.free_space(**{n: getattr(o, n) for n, _ in api.FreeSpace._fields_})


def _ctx(api, **kw):
    """1 m cells: the spread maps fill 3 087 blocks of the dense cell table"""
    return api.Context(max_map_points=1 << 19, max_scan_points=1 << 16, plane_res=1.0, line_res=1.0, **kw)


def _src(api, keyframes):
    """A context holding keyframes [(sensor-frame cloud, pose)], imported in order (ids 0, 1, ...)"""
    s = _ctx(api)
    s.keyframe_reserve(sum(len(c) for c, _ in keyframes) + 1024, len(keyframes))
    for i, (c, p) in enumerate(keyframes):
        assert s.keyframe_import(c, p) == i
    return s


def _load(ctx, surf, edge):
    ctx.map_set_points(surf if len(surf) else np.zeros((0, 4), np.float32))
    ctx.map_set_edge_points(edge if len(edge) else np.zeros((0, 4), np.float32))


def _stores(ctx):
    """(surf, edge): map_download (getAllLocalMap) returns both stores in one cloud; with the archive off download_all is the window"""
    return ctx.map_download_all(0), ctx.map_download_all(1)


def _sequential(ctx, src, ids, poses, o, stores):
    """R1: so_map_clear_free_space of each entry's downloaded surf cloud, in list order -> summed counters"""
    tot = dict(n_image_points=0, n_pixels_hit=0, n_removed=0, n_candidates=0, n_after=tuple(len(x) for x in _stores(ctx)))
    for i, p in zip(ids, poses):
        r = ctx.map_clear_free_space(src.keyframe_download(int(i), 0), p, o, stores=stores)
        for k in ("n_image_points", "n_pixels_hit", "n_removed", "n_candidates"):
            tot[k] += r[k]
        tot["n_after"] = r["n_after"]
    return tot


def _probe(pts, n=4096, seed=3):
    rng = np.random.default_rng(seed)
    if len(pts) == 0:
        return rng.normal(0, 30.0, (n, 3)).astype(np.float32)
    m = pts[rng.choice(len(pts), n)]
    return (m[:, :3] + rng.normal(0, 0.5, (n, 3))).astype(np.float32)


def _r1(a, b, ra, rb, probe, ijks=()):
    sa, sb = _stores(a), _stores(b)
    for x, y in zip(sa, sb):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    ka, kb = a.knn(probe, 5, 0.0), b.knn(probe, 5, 0.0)
    assert all(np.array_equal(x, y) for x, y in zip(ka, kb))
    assert [a.map_counts_5x5(ijk, True) for ijk in ijks] == [b.map_counts_5x5(ijk, True) for ijk in ijks]
    for k in ("n_removed", "n_image_points", "n_pixels_hit", "n_after"):
        assert ra[k] == rb[k], (k, ra[k], rb[k])


def _gone(before, after):
    """-> mask of the rows of `before` that are gone, checking that `after` is `before` without them, bit for bit, in order"""
    keys = {r.tobytes() for r in after}
    gone = np.array([r.tobytes() not in keys for r in before], bool)
    assert np.array_equal(before[~gone].view(np.uint32), after.view(np.uint32))
    return gone


def _r2(before, after, r, clouds, poses, o, stores, label, exact_gate=False, archived=0):
    """R2 -> the restatement.  before / after: (surf, edge) of the carved context; archived: surf points in the archive (not carved,
    not in n_after)."""
    carved = [before[k] if stores & (1 << k) else None for k in range(2)]
    rs = K.restate(carved, clouds, poses, o, exact_gate=exact_gate)
    n_gone = 0
    for k in range(2):
        if carved[k] is None:
            assert np.array_equal(before[k].view(np.uint32), after[k].view(np.uint32))
            continue
        gone = _gone(before[k], after[k])
        amb = rs["ambiguous"][k]
        assert np.array_equal(gone[~amb], rs["removed"][k][~amb]), label
        assert not (rs["lower"][k] & ~gone).any() and not (gone & ~rs["upper"][k]).any(), label
        n_gone += int(gone.sum())
    n_amb = rs["n_ambiguous_map"] + rs["n_ambiguous_scan"]
    print(f"{label}: {r}; numpy removed {rs['n_removed']} candidates {rs['n_candidates']}; edge-ambiguous map points "
          f"{rs['n_ambiguous_map']}, scan points {rs['n_ambiguous_scan']}")
    assert r["n_removed"] == n_gone
    assert r["n_after"] == (len(after[0]) - archived, len(after[1]))
    if n_amb == 0:
        assert r["n_candidates"] == rs["n_candidates"], (label, r["n_candidates"], rs["n_candidates"])
        assert r["n_removed"] == rs["n_removed"]
        assert (r["n_image_points"], r["n_pixels_hit"]) == (rs["n_image_points"], rs["n_pixels_hit"])
    n = len(clouds)
    assert r["n_keyframes"] == n and r["n_tiles"] == K.tile_plan(n, o)[1]
    return rs, n_amb


def _check(api, src, ids, poses, o, stores, history, label, exact_gate=False, ijks=(), probe_pts=None, with_before=False):
    """Contexts A (batched), B (R1) and C (the store as the call finds it), each given `history`; -> (result, restatement, n_amb)"""
    a, b, c = _ctx(api), _ctx(api), _ctx(api)
    for x in (a, b, c):
        history(x)
    before = _stores(c)
    archived = c.map_archive_info(0)[0]
    fo = _fs(api, o)
    ra = a.map_clear_free_space_keyframes(src, ids, poses, fo, stores=stores)
    rb = _sequential(b, src, ids, poses, fo, stores)
    _r1(a, b, ra, rb, _probe(before[0] if probe_pts is None else probe_pts), ijks)
    clouds = [src.keyframe_download(int(i), 0) for i in ids]
    rs, n_amb = _r2(before, _stores(a), ra, clouds, poses, o, stores, label, exact_gate, archived)
    for x in (a, b, c):
        x.close()
    return (ra, rs, n_amb, before) if with_before else (ra, rs, n_amb)


# ------------------------------------------------------------------------------------------------------- 1: spread keyframes
@pytest.fixture(scope="module")
def spread(gpu_api):
    c = K.spread_case()
    src = _src(gpu_api, list(zip(c["clouds"], c["poses"])))
    c["src"] = src
    c["order"] = np.random.default_rng(11).permutation(len(c["poses"])).astype(np.int32)
    yield c
    src.close()


IJKS = [(i, j, k) for i in (0, 3, 10, 17, 20) for j in (0, 9, 20) for k in (2, 5, 8)]


@pytest.mark.parametrize("n", K.SPREAD_SIZES)
def test_spread_keyframes_one_tile(gpu_api, spread, n):
    """n keyframes from over the 21 x 21 window and five z layers (rotated, some just outside the window, some beyond reach), in
    random order, on maps that fill every block of seven z layers in both stores"""
    o = spread["opts"]
    ids = spread["order"][:n]
    poses = spread["poses"][ids]
    surf, edge = spread["surf"], spread["edge"]
    blocks = np.unique(np.r_[K.grid_block(surf), K.grid_block(edge)])
    lists = K.cull_lists(blocks[blocks >= 0], poses, o.max_range)
    cnt = lists.sum(1)
    proper = int(((cnt > 0) & (cnt < n)).sum())
    multi_warp = int(sum(len(set(np.nonzero(l)[0] % 128 // 32)) >= 2 for l in lists))
    rounds = int(sum(len(set(np.nonzero(l)[0] // 128)) >= 2 for l in lists))
    print(f"n {n}: {len(cnt)} blocks, {int((cnt == 0).sum())} reached by no entry, {proper} proper non-empty lists (longest "
          f"{int(cnt.max())}), {multi_warp} lists over two warps of a round, {rounds} over two rounds")
    if n >= 31:
        assert proper >= 200 and (cnt == 0).sum() >= 50
    if n >= 127:
        assert multi_warp >= 200
    if n >= 257:
        assert rounds >= 500
    ra, rs, n_amb = _check(gpu_api, spread["src"], ids, poses, o, 3, lambda x: _load(x, surf, edge), f"spread n={n}", ijks=IJKS)
    assert ra["n_tiles"] == 1
    if n >= 31:
        assert ra["n_removed"] > 0 and ra["n_candidates"] > ra["n_removed"]
    assert n_amb == 0


# ------------------------------------------------------------------------------------------------------- 2: reach at block faces
@pytest.mark.parametrize("axis", [0, 1], ids=["x_faces", "y_faces"])
def test_reach_at_block_faces(gpu_api, axis):
    """Points on the faces 25 + 50 k, each at FP64 r_m = float(max_range) or one FP64 or float step either side of it from a keyframe
    straight across the face (identity or 180 deg yaw: r_m exact): those in range go, the others stay, in both stores."""
    c = K.face_case(axis)
    o = c["opts"]
    src = _src(gpu_api, list(zip(c["clouds"], c["poses"])))
    ids = np.arange(len(c["poses"]), dtype=np.int32)
    surf = c["surf"]
    edge = K.xyzi(surf[:, :3], surf[:, 3] + 10 ** 6)
    ra, rs, n_amb = _check(gpu_api, src, ids, c["poses"], o, 3, lambda x: _load(x, surf, edge), f"faces axis {axis}", exact_gate=True)
    assert n_amb == 0
    assert np.array_equal(rs["removed"][0], c["want"]) and np.array_equal(rs["removed"][1], c["want"])
    assert ra["n_removed"] == 2 * int(c["want"].sum())
    src.close()


def test_reach_a_rounding_step_beyond_the_face(gpu_api):
    """Keyframes a few FP64 steps beyond max_range from a face point, under small rotations: the rotation's rounding puts some of them
    in range (r_m <= max_range, restated operation by operation), and only the box's pad and slack keep those pairs in the cull."""
    c = K.face_near_case(np.random.default_rng(5))
    o = c["opts"]
    src = _src(gpu_api, list(zip(c["clouds"], c["poses"])))
    ids = np.arange(len(c["poses"]), dtype=np.int32)
    surf = c["surf"]
    ra, rs, n_amb = _check(gpu_api, src, ids, c["poses"], o, 1, lambda x: _load(x, surf, np.zeros((0, 4), np.float32)),
                           "a rounding step beyond the face")
    in_range = np.array([K.device_range(surf[i:i + 1], p)[0] <= float(np.float32(o.max_range)) for i, p in enumerate(c["poses"])])
    print(f"{int(in_range.sum())} of {len(in_range)} points in range after the rotation; removed {ra['n_removed']}")
    assert 0 < in_range.sum() < len(in_range) and ra["n_removed"] == in_range.sum()
    src.close()


# ------------------------------------------------------------------------------------------------------- 3: tile seams
def test_tile_seams_at_the_smallest_tile(gpu_api):
    """13 entries of 2^24-pixel images, 4 a tile: empty keyframes first, in the middle and last in a tile, a tile of empty keyframes
    only, one id on both sides of a seam under two poses, clouds with NaN, inf, r = 0 and out-of-span returns.  The map equals one
    call per tile in sequence; n_candidates is the union's (each point once), below the sum over the per-tile calls."""
    c = K.seam_case()
    o = c["opts"]
    names = sorted(c["keyframes"])
    src = _src(gpu_api, [c["keyframes"][nm] for nm in names])
    ids = np.array([names.index(nm) for nm in c["ids"]], np.int32)
    poses = c["poses"]
    per, n_tiles = K.tile_plan(len(ids), o)
    assert (per, n_tiles) == (4, 4)
    hist = lambda x: _load(x, c["surf"], c["edge"])
    ra, rs, n_amb, before = _check(gpu_api, src, ids, poses, o, 3, hist, "tile seams", with_before=True)
    assert n_amb == 0 and ra["n_tiles"] == 4
    d = _ctx(gpu_api)
    hist(d)
    per_tile = [d.map_clear_free_space_keyframes(src, ids[t:t + per], poses[t:t + per], _fs(gpu_api, o), stores=3)
                for t in range(0, len(ids), per)]
    a = _ctx(gpu_api)
    hist(a)
    a.map_clear_free_space_keyframes(src, ids, poses, _fs(gpu_api, o), stores=3)
    for x, y in zip(_stores(a), _stores(d)):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    assert [r["n_tiles"] for r in per_tile] == [1, 1, 1, 1]
    tiles_sum = sum(r["n_candidates"] for r in per_tile)
    print(f"per-tile calls: candidates {[r['n_candidates'] for r in per_tile]}, removed {[r['n_removed'] for r in per_tile]}")
    assert ra["n_candidates"] == rs["n_candidates"] < tiles_sum
    assert sum(r["n_removed"] for r in per_tile) == ra["n_removed"]
    for k in range(2):                                      # every designed kind behaves as the layout says
        kinds = c["kinds"][k][before[k][:, 3].astype(np.int64) - k * 10 ** 6]   # the intensity names the point
        for kd, name in enumerate(K.SEAM_KINDS):
            m = kinds == kd
            assert rs["cand"][k][m].all(), name
            assert rs["removed"][k][m].all() == ("removed" in name), name
    for x in (a, d, src):
        x.close()


# ------------------------------------------------------------------------------------------------------- 4, 5: store states, entries
def _near(spread, r=170.0):
    """the spread keyframes within r of the origin (xy), and the map within 250 m"""
    t = spread["poses"][:, :3]
    ids = np.nonzero((np.abs(t[:, 0]) < r) & (np.abs(t[:, 1]) < r))[0].astype(np.int32)
    sel = lambda p: p[(np.abs(p[:, 0]) < 250) & (np.abs(p[:, 1]) < 250)]
    return ids, sel(spread["surf"]), sel(spread["edge"])


STATES = ["shift", "resolution", "origin", "archive", "surf_only_edge_empty", "surf_only_edge_full", "edge_only_surf_empty",
          "edge_only_surf_full", "both_surf_empty", "from_keyframes", "reversed_with_duplicates"]


@pytest.mark.parametrize("state", STATES)
def test_store_states_and_entries(gpu_api, spread, state):
    o = spread["opts"]
    src = spread["src"]
    ids, surf, edge = _near(spread)
    empty = np.zeros((0, 4), np.float32)
    stores = 3
    if state == "shift":
        hist = lambda x: (_load(x, surf, edge), x.map_shift([400.0, -420.0, 0.0]))
    elif state == "resolution":
        hist = lambda x: (_load(x, surf, edge), x.map_set_resolution(1.5, 2.0))
    elif state == "origin":
        hist = lambda x: (x.map_set_origin([120.0, -80.0, 30.0]), _load(x, surf, edge))
    elif state == "archive":
        far = surf.copy()
        far[:, 0] += 1500.0
        hist = lambda x: (x.map_archive(2 * len(surf)), _load(x, np.vstack([surf, far]), edge))
    elif state.startswith("surf_only"):
        stores = 1
        hist = lambda x: _load(x, surf, empty if state.endswith("empty") else edge)
    elif state.startswith("edge_only"):
        stores = 2
        hist = lambda x: _load(x, empty if state.endswith("empty") else surf, edge)
    elif state == "both_surf_empty":
        hist = lambda x: _load(x, empty, edge)
    elif state == "from_keyframes":
        hist = lambda x: x.map_from_keyframes(src, ids[::2], spread["poses"][ids[::2]], stores=3)
    else:
        ids = np.r_[ids[::-1], ids[:5], ids[-3:]].astype(np.int32)
        hist = lambda x: _load(x, surf, edge)
    poses = spread["poses"][ids].copy()
    if state == "reversed_with_duplicates":                   # the duplicated ids at other poses
        poses[-8:, :2] += np.array([3.0, -2.0])
    arc = {}

    def history(x):
        hist(x)
        if state == "archive" and "before" not in arc:
            arc["before"] = (x.map_archive_info(0), x.map_download_all(0))
    ra, rs, n_amb = _check(gpu_api, src, ids, poses, o, stores, history, f"state {state}", probe_pts=surf)
    assert n_amb == 0
    assert ra["n_removed"] > 0
    if state == "archive":
        a = _ctx(gpu_api)
        history(a)
        window = {p.tobytes() for p in a.map_download()}
        a.map_clear_free_space_keyframes(src, ids, poses, _fs(gpu_api, o), stores=3)
        info0, all0 = arc["before"]
        all1 = a.map_download_all(0)
        in_arc = lambda x: x[np.array([p.tobytes() not in window for p in x], bool)]
        assert a.map_archive_info(0) == info0 and info0[0] > 0
        assert np.array_equal(in_arc(all0).view(np.uint32), in_arc(all1).view(np.uint32))
        a.close()


def test_a_second_call_after_one_that_removed(gpu_api, spread):
    """Two calls in a row (the second's entries reversed, overlapping the first's) equal the per-keyframe loop of both lists; the
    second call's restatement starts from the store the first left."""
    o = spread["opts"]
    src = spread["src"]
    ids, surf, edge = _near(spread)
    first, second = ids[: len(ids) // 2 + 3], ids[len(ids) // 2:][::-1].copy()
    a, b = _ctx(gpu_api), _ctx(gpu_api)
    for x in (a, b):
        _load(x, surf, edge)
    fo = _fs(gpu_api, o)
    r1 = a.map_clear_free_space_keyframes(src, first, spread["poses"][first], fo, stores=3)
    _sequential(b, src, first, spread["poses"][first], fo, 3)
    assert r1["n_removed"] > 0
    mid = _stores(a)
    r2 = a.map_clear_free_space_keyframes(src, second, spread["poses"][second], fo, stores=3)
    rb = _sequential(b, src, second, spread["poses"][second], fo, 3)
    _r1(a, b, r2, rb, _probe(surf), IJKS)
    clouds = [src.keyframe_download(int(i), 0) for i in second]
    _, n_amb = _r2(mid, _stores(a), r2, clouds, spread["poses"][second], o, 3, "second call")
    assert n_amb == 0
    a.close()
    b.close()

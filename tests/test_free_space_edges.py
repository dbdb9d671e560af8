"""so_map_clear_free_space* at its edges on the device, against the numpy restatement (tests/free_space_numpy.py): the hand-built cases
of tests/free_space_edge_sets.py (decision ties, degenerate returns, the azimuth seam, the span edges, the column clamp) give the
restatement's removal set and counters exactly; many returns in one pixel, awkward sizes, the argument limits and the pose forms; a
carved store against the store rebuilt from the points it kept; and a randomised sweep held between the restatement's bounds."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from superodom_b200 import synth
import free_space_edge_sets as S
import free_space_numpy as F

pytestmark = pytest.mark.gpu

_EXACT = S.exact_cases()
MAX_SCAN = 262144


def _removed(before, after):
    """-> mask of the rows of `before` that are gone, and the check that `after` is `before` without them, bit for bit, in order"""
    keys_after = {r.tobytes() for r in after}
    gone = np.array([r.tobytes() not in keys_after for r in before], bool)
    assert np.array_equal(before[~gone].view(np.uint32), after.view(np.uint32))
    return gone


def _fs(api, o):
    return api.free_space(**{n: getattr(o, n) for n, _ in api.FreeSpace._fields_})


def _counters(r):
    return {k: r[k] for k in ("n_image_points", "n_pixels_hit", "n_candidates", "n_removed")}


@pytest.fixture(scope="module")
def ctx(gpu_api):
    c = gpu_api.Context(max_map_points=1 << 20, max_scan_points=MAX_SCAN, plane_res=0.2)
    yield c
    c.close()


def _carve(api, ctx, mp, scan, pose, o):
    """Load mp, clear with scan: -> (store before, store after, result)"""
    ctx.map_set_points(mp)
    before = ctx.map_download()
    r = ctx.map_clear_free_space(scan, pose, _fs(api, o))
    return before, ctx.map_download(), r


def _assert_exact(api, ctx, mp, scan, pose, o):
    """The device's removal set, order and counters are the restatement's; -> (result, removed mask)"""
    before, after, r = _carve(api, ctx, mp, scan, pose, o)
    gone = _removed(before, after)
    rem, st = F.clear(before, scan, pose, o)
    assert _counters(r) == st, (r, st)
    assert np.array_equal(gone, rem)
    assert r["n_after"] == (len(before) - st["n_removed"], 0)
    return r, gone


# --------------------------------------------------------------------------------------------------------- A, B, C: hand-built cases
@pytest.mark.parametrize("k", range(len(_EXACT)), ids=[c["name"] for c in _EXACT])
def test_hand_case_equals_the_restatement(gpu_api, ctx, k):
    c = _EXACT[k]
    lo, hi = F.bounds(c["map"], c["scan"], c["pose"], c["opts"])
    if not c["on_edge"]:
        assert np.array_equal(lo, hi)
    r, _ = _assert_exact(gpu_api, ctx, c["map"], c["scan"], c["pose"], c["opts"])
    assert _counters(r) == c["want"]


def test_degenerate_returns_in_three_layouts(gpu_api, ctx):
    """Case B as packed float4, as xyz only (stride 12) and as a 32-byte PointXYZI-like record whose padding holds NaN: one result."""
    c = S.case_b()
    xyz = c["scan"][:, :3]
    rec = np.full((len(xyz), 8), np.nan, np.float32)
    rec[:, :4] = c["scan"]
    out = []
    for scan in (c["scan"], np.ascontiguousarray(xyz), rec):
        before, after, r = _carve(gpu_api, ctx, c["map"], scan, c["pose"], c["opts"])
        out.append((r, after))
    print("case B:", out[0][0])
    assert _counters(out[0][0]) == c["want"]
    for r, after in out[1:]:
        assert r == out[0][0] and np.array_equal(after.view(np.uint32), out[0][1].view(np.uint32))


# -------------------------------------------------------------------------------------------------------------- D: the column clamp
def test_column_clamp_stays_in_its_row(gpu_api, ctx):
    c = S.case_d()
    before, after, r = _carve(gpu_api, ctx, c["map"], c["scan"], c["pose"], c["opts"])
    gone = _removed(before, after)
    lo, hi = F.bounds(before, c["scan"], c["pose"], c["opts"])
    print(f"clamp return read in column {719 if gone[0] else 0}; {r}")
    assert lo.tolist() == [False, False, False] and hi.tolist() == [True, True, False]
    assert _counters(r) == c["want"] and gone[0] != gone[1] and not gone[2]


# ------------------------------------------------------------------------------------------------------- E: order of the atomics
def test_many_returns_in_one_pixel_keep_the_true_minimum(gpu_api, ctx):
    """200 000 returns in pixel (2, 4), shuffled, with duplicates; the smallest (20 m) once.  The map point at 20 m (threshold 20.25)
    is kept only when the image holds 20 m: every other return is at least 20.5 m.  Reversed order: the same result."""
    o = S.opts(dilate=0)
    rng = np.random.default_rng(5)
    n = 200000
    az, el = rng.uniform(-15, 15, n - 1001), rng.uniform(-3, 3, n - 1001)
    rr = rng.choice(np.round(rng.uniform(20.6, 60.0, 5000), 2), n - 1001)            # many duplicate ranges
    pts = [S.direction(a, e, r) for a, e, r in zip(az, el, rr)] + [[20.5, 0, 0]] * 1000 + [[20.0, 0, 0]]
    scan = S.cloud(pts)[rng.permutation(n)]
    mp = S.cloud([[20.0, 0, 0]])
    res = []
    for s in (scan, scan[::-1]):
        r, gone = _assert_exact(gpu_api, ctx, mp, np.ascontiguousarray(s), S.IDENTITY, o)
        res.append(r)
    print("one pixel, 200 000 returns:", res[0])
    assert res[0] == res[1]
    assert _counters(res[0]) == dict(n_image_points=n, n_pixels_hit=1, n_candidates=1, n_removed=0)


# ------------------------------------------------------------------------------------------------------------ F: sizes and counters
SIZES_OPTS = S.opts(dict(S.GRID_TALL, az_res_deg=7.0), dilate=1, margin=0.3, margin_rel=0.02, max_range=60.0)   # W = 52, narrow last column


def _centres(o, n, rng, r_lo, r_hi, pose=None):
    """n points at random pixel centres and ranges; in the world frame of `pose` when given."""
    W, H = F.dims(o)
    q = np.array([S.at(o, i, j, r) for i, j, r in zip(rng.integers(0, H, n), rng.integers(0, W, n), rng.uniform(r_lo, r_hi, n))])
    q = q.reshape(-1, 3)
    if pose is not None:
        q = q @ synth.quat_to_R(np.asarray(pose[3:]) / np.linalg.norm(pose[3:])).T + np.asarray(pose[:3])
    return S.cloud(q)


def test_sizes_and_counters(gpu_api, ctx):
    o = SIZES_OPTS
    rng = np.random.default_rng(11)
    pose = np.r_[0.7, -0.4, 0.2, synth.quat_from_rotvec([0.05, -0.03, 0.4])]
    scan_all = _centres(o, MAX_SCAN, rng, 30.0, 58.0)
    map_all = _centres(o, 65537, rng, 1.0, 40.0, pose)
    for ns in (0, 1, 255, 257, MAX_SCAN):
        for nm in (1, 31, 32, 33, 255, 256, 257, 65537):
            scan, mp = scan_all[:ns], map_all[:nm]
            lo, hi = F.bounds(mp, scan, pose, o)
            assert np.array_equal(lo, hi)
            r, _ = _assert_exact(gpu_api, ctx, mp, scan, pose, o)
            assert r["n_image_points"] == ns
        print(f"scan {ns}: map 65537 -> {r}")
    ctx.map_set_points(map_all)
    before = ctx.map_download()
    big = np.concatenate([scan_all, scan_all[:1]])
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-3\)"):
        ctx.map_clear_free_space(big, pose, _fs(gpu_api, o))
    assert np.array_equal(before.view(np.uint32), ctx.map_download().view(np.uint32))


def test_empty_scan_leaves_the_store(gpu_api, ctx):
    """n = 0 with a NULL cloud, and an empty array: nothing counted, nothing removed, the store bit for bit."""
    c = _EXACT[0]
    ctx.map_set_points(c["map"])
    before = ctx.map_download()
    pose = np.ascontiguousarray(c["pose"])
    o = _fs(gpu_api, c["opts"])
    res = gpu_api.FreeSpaceResult()
    rc = ctx.L.so_map_clear_free_space(ctx.h, 1, None, 0, 16, 12, pose.ctypes.data_as(C.c_void_p), C.byref(o), C.byref(res))
    assert rc == 0
    assert ctx._free_result(res) == dict(n_image_points=0, n_pixels_hit=0, n_candidates=0, n_removed=0, n_after=(len(before), 0))
    r = ctx.map_clear_free_space(np.zeros((0, 4), np.float32), pose, o)
    assert r == ctx._free_result(res)
    assert np.array_equal(before.view(np.uint32), ctx.map_download().view(np.uint32))


def test_image_of_2_24_pixels(gpu_api, ctx):
    """4096 x 4096 pixels, all exact in float: accepted, and exact against the restatement at the seam and the top and bottom rows;
    one row more is refused."""
    o = S.opts(dict(az_res_deg=0.087890625, el_res_deg=0.0087890625, el_min_deg=-18.0, el_max_deg=18.0), dilate=2)
    assert F.dims(o) == (4096, 4096)
    scan, mp = [], []
    for row, col in ((2, 0), (4093, 4095), (2048, 1), (2, 2047)):
        scan += [S.at(o, row + i, (col + j) % 4096, S.FAR) for i in range(-2, 3) for j in range(-2, 3)]
        mp.append(S.at(o, row, col, 5.0))
    scan.append(S.at(o, 2, 2047, S.NEAR))
    scan, mp = S.cloud(scan), S.cloud(mp)
    lo, hi = F.bounds(mp, scan, S.IDENTITY, o)
    assert np.array_equal(lo, hi)
    r, gone = _assert_exact(gpu_api, ctx, mp, scan, S.IDENTITY, o)
    assert gone.tolist() == [True, True, True, False]
    ctx.map_set_points(mp)
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
        ctx.map_clear_free_space(scan, S.IDENTITY, _fs(gpu_api, dataclasses.replace(o, el_max_deg=18.0087890625)))
    assert len(ctx.map_download()) == len(mp)


_TINY = {}


def _tiny():
    if not _TINY:
        scene, mp = synth.make_map_for("tiny")
        _TINY.update(scene=scene, map=mp, cases=[synth.make_case_on(scene, mp, "tiny", k) for k in range(3)])
    return _TINY


def test_registered_form_at_max_map_points(gpu_api):
    """The registered form needs room for the scan at the surf store's tail: n + scan == max_map_points runs, one point fewer of
    room is SO_ERR_CAPACITY with both stores untouched."""
    d = _tiny()
    c = d["cases"][0]
    mp, scan = d["map"], c["scan_xyzi"]
    o = _fs(gpu_api, F.opts_for("vlp16"))
    for room, ok in ((0, True), (-1, False)):
        ctx = gpu_api.Context(max_map_points=len(mp) + len(scan) + room, max_scan_points=MAX_SCAN, plane_res=0.2)
        ctx.map_set_points(mp)
        ctx.map_set_edge_points(mp[::5])
        surf, edge = ctx.map_download_all(0), ctx.map_download_all(1)
        pose = np.array(ctx.register(scan, c["pose_prior"], 5).pose)
        if ok:
            r = ctx.map_clear_free_space_registered(pose, o, stores=3)
            print(f"registered form at max_map_points: {r}")
            assert r["n_image_points"] > 0 and sum(r["n_after"]) == len(surf) + len(edge) - r["n_removed"]
        else:
            with pytest.raises(gpu_api.SuperOdomError, match=r"\(-3\)"):
                ctx.map_clear_free_space_registered(pose, o, stores=3)
            assert np.array_equal(surf.view(np.uint32), ctx.map_download_all(0).view(np.uint32))
            assert np.array_equal(edge.view(np.uint32), ctx.map_download_all(1).view(np.uint32))
        ctx.close()


# ------------------------------------------------------------------------------------------------------------------------ G: poses
def test_quaternion_scale_and_sign_and_bad_poses(gpu_api, ctx):
    o = SIZES_OPTS
    rng = np.random.default_rng(21)
    pose = np.r_[1.5, 2.0, -0.3, synth.quat_from_rotvec([0.3, -0.2, 2.5])]
    scan = _centres(o, 3000, rng, 2.0, 40.0)
    mp = _centres(o, 5000, rng, 1.0, 40.0, pose)
    lo, hi = F.bounds(mp, scan, pose, o)
    assert np.array_equal(lo, hi)
    r0, gone0 = _assert_exact(gpu_api, ctx, mp, scan, pose, o)
    assert r0["n_removed"] > 0
    for s in (1e-3, 1e3, -1.0):
        p = np.r_[pose[:3], s * pose[3:]]
        before, after, r = _carve(gpu_api, ctx, mp, scan, p, o)
        assert r == r0 and np.array_equal(_removed(before, after), gone0)
    ctx.map_set_points(mp)
    ctx.map_set_edge_points(mp[::3])
    surf, edge = ctx.map_download_all(0), ctx.map_download_all(1)
    bad = [np.r_[pose[:3], 0.0, 0.0, 0.0, 0.0]]
    for k in range(7):
        for v in (np.nan, np.inf):
            p = pose.copy()
            p[k] = v
            bad.append(p)
    for p in bad:
        with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
            ctx.map_clear_free_space(scan, p, _fs(gpu_api, o), stores=3)
    assert np.array_equal(surf.view(np.uint32), ctx.map_download_all(0).view(np.uint32))
    assert np.array_equal(edge.view(np.uint32), ctx.map_download_all(1).view(np.uint32))
    ctx.map_set_edge_points(np.zeros((0, 4), np.float32))


def _sensor_cloud(o, n, rng, r_lo, r_hi, el_pad=1.0):
    """n points in uniform random directions over the span (el_pad degrees beyond it) at uniform ranges"""
    az = rng.uniform(-180.0, 180.0, n)
    el = rng.uniform(o.el_min_deg - el_pad, o.el_max_deg + el_pad, n)
    r = rng.uniform(r_lo, r_hi, n)
    a, e = np.radians(az), np.radians(el)
    return np.c_[r * np.cos(e) * np.cos(a), r * np.cos(e) * np.sin(a), r * np.sin(e)]


def _to_world(q, pose):
    return q @ synth.quat_to_R(np.asarray(pose[3:]) / np.linalg.norm(pose[3:])).T + np.asarray(pose[:3])


def test_rotated_pose_10_km_out_with_the_archive(gpu_api):
    """The window sits 10 km from the origin of the world, the block archive on and holding a copy of the map 2 km further: the
    removal set lies between the bounds, and the archive is never carved."""
    o = F.Opts(az_res_deg=0.4, el_res_deg=0.4, el_min_deg=-23.0, el_max_deg=23.0, dilate=2)
    rng = np.random.default_rng(31)
    pose = np.r_[10000.3, -7000.7, 12.5, synth.quat_from_rotvec([0.05, 0.02, 1.2])]
    scan = S.cloud(_sensor_cloud(o, 200000, rng, 30.0, 50.0))
    mp = S.cloud(_to_world(_sensor_cloud(o, 30000, rng, 1.0, 50.0), pose))
    far = mp.copy()
    far[:, 0] += 2000.0
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=MAX_SCAN, plane_res=0.2)
    ctx.map_archive(len(mp) + len(far))
    ctx.map_set_origin(pose[:3])
    ctx.map_set_points(np.vstack([mp, far]))
    before = ctx.map_download()
    n_arc = ctx.map_archive_info(0)[0]
    arc0 = ctx.map_download_all(0)
    r = ctx.map_clear_free_space(scan, pose, _fs(gpu_api, o))
    gone = _removed(before, ctx.map_download())
    lo, hi = F.bounds(before, scan, pose, o)
    print(f"10 km out: {r}; numpy lower {lo.sum()} upper {hi.sum()}")
    assert len(before) + n_arc == len(mp) + len(far) and len(before) > len(mp) // 2 and ctx.map_archive_info(0)[0] == n_arc
    arc1 = ctx.map_download_all(0)
    window = {p.tobytes() for p in before}
    in_arc = lambda x: x[np.array([p.tobytes() not in window for p in x], bool)]
    assert np.array_equal(in_arc(arc0).view(np.uint32), in_arc(arc1).view(np.uint32))
    assert not (lo & ~gone).any() and not (gone & ~hi).any()
    assert r["n_removed"] == gone.sum() > 100
    ctx.close()


# ---------------------------------------------------------------------------------------- H: a carved store and the rebuilt one
def _icp_bytes(r):
    """the bytes of every field of an IcpResult but the timings"""
    b = bytes(r)
    return [b[f.offset:f.offset + f.size] for f in (getattr(type(r), n) for n, _ in type(r)._fields_ if not n.startswith("time"))]


def _try(f, *a, **kw):
    try:
        return f(*a, **kw)
    except Exception as e:                          # the same error on both sides counts as the same result
        return ("error", str(e))


def _same(a, b):
    if isinstance(a, tuple) and a and isinstance(a[0], np.ndarray):
        return all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))
    return a == b


def _carve_scan(o, r):
    """a return at range r at the centre of every pixel"""
    return S.cloud(S.fill(o, r))


CARVE_WIDE = F.Opts(az_res_deg=2.0, el_res_deg=2.0, el_min_deg=-60.0, el_max_deg=60.0, dilate=1, margin=0.3, margin_rel=0.0,
                    min_range=0.5, max_range=100.0)
CARVE_ALL = F.Opts(az_res_deg=2.0, el_res_deg=2.0, el_min_deg=-90.0, el_max_deg=90.0, dilate=0, margin=0.3, margin_rel=0.0,
                   min_range=0.1, max_range=300.0)
AT_GHOST = np.array([60.0, 0, 0, 0, 0, 0, 1])        # in block (+1, 0, 0) of the origin's, beyond the ghost copy
AT_ROOM_SIDE = np.array([20.0, 0, 0, 0, 0, 0, 1])


@pytest.mark.parametrize("carve", ["partial", "empty_block", "whole_surf", "whole_edge"])
def test_carved_store_equals_the_store_rebuilt_from_what_it_kept(gpu_api, carve):
    """The tiny room in block (0, 0, 0) plus a copy of it 40 m along x, alone in block (1, 0, 0).  Carves from 60 m along x: returns
    at 20 m take part of the copy, at 45 m all of it (its block's slot goes); from 20 m, returns at 200 m over the whole sphere take
    the whole surf store, or the whole edge store (stores=2).  The carved context and a fresh one loaded with the kept cloud then give
    the same k-NN, 5 x 5 block counts, registration, insert and registration after it, bit for bit."""
    d = _tiny()
    room = d["map"]
    ghost = room.copy()
    ghost[:, 0] += 40.0
    mp = np.vstack([room, ghost])
    edge = mp[::3]
    pose, o, r_scan, stores = {"partial": (AT_GHOST, CARVE_WIDE, 20.0, 1), "empty_block": (AT_GHOST, CARVE_WIDE, 45.0, 1),
                               "whole_surf": (AT_ROOM_SIDE, CARVE_ALL, 200.0, 1), "whole_edge": (AT_ROOM_SIDE, CARVE_ALL, 200.0, 2)}[carve]
    mk = lambda: gpu_api.Context(max_map_points=1 << 20, max_scan_points=MAX_SCAN, plane_res=0.2, line_res=0.1)
    a, b = mk(), mk()
    a.map_set_points(mp)
    a.map_set_edge_points(edge)
    r = a.map_clear_free_space(_carve_scan(o, r_scan), pose, _fs(gpu_api, o), stores=stores)
    kept_s, kept_e = a.map_download_all(0), a.map_download_all(1)
    print(f"{carve}: {r}")
    if carve == "partial":
        assert 0 < r["n_removed"] < len(ghost) and len(kept_s) == len(mp) - r["n_removed"]
    elif carve == "empty_block":
        assert r["n_removed"] == len(ghost) and np.array_equal(kept_s.view(np.uint32), room.view(np.uint32))
    elif carve == "whole_surf":
        assert r["n_after"] == (0, len(edge)) and len(kept_s) == 0
    else:
        assert r["n_after"] == (len(mp), 0) and len(kept_e) == 0
    b.map_set_points(kept_s)
    b.map_set_edge_points(kept_e)
    qrng = np.random.default_rng(41)
    queries = np.vstack([room[qrng.integers(0, len(room), 2000), :3] + qrng.normal(0, 0.3, (2000, 3)),
                         ghost[qrng.integers(0, len(ghost), 1000), :3] + qrng.normal(0, 0.3, (1000, 3))]).astype(np.float32)
    assert _same(_try(a.knn, queries, 5, 0.0), _try(b.knn, queries, 5, 0.0))
    blocks = [(i, j, k) for i in range(9, 13) for j in range(9, 12) for k in range(4, 7)]
    assert [_try(a.map_counts_5x5, ijk, True) for ijk in blocks] == [_try(b.map_counts_5x5, ijk, True) for ijk in blocks]
    c1, c2 = d["cases"][1], d["cases"][2]
    e1 = c1["scan_xyzi"][::7] if carve == "whole_edge" else None
    reg = lambda x, c, e: _try(lambda: _icp_bytes(x.register(c["scan_xyzi"], c["pose_prior"], 5, edge_xyzi=e)))
    ra, rb = reg(a, c1, e1), reg(b, c1, e1)
    assert ra == rb
    for x in (a, b):
        x.map_add_scan(c1["scan_xyzi"], c1["pose_true"])
    for k in (0, 1):
        assert np.array_equal(a.map_download_all(k).view(np.uint32), b.map_download_all(k).view(np.uint32))
    assert reg(a, c2, e1) == reg(b, c2, e1)
    a.close()
    b.close()


# -------------------------------------------------------------------------------------------------------- I: randomised sweep
AZ_RES = [0.1, 0.35, 0.4, 0.7, 1.3, 7.0, 90.0, 400.0]


def _sweep_set(seed):
    rng = np.random.default_rng(1000 + seed)
    az_res = AZ_RES[seed % len(AZ_RES)]
    el_res = float(rng.choice([0.2, 0.4, 1.0, 2.0, 4.3]))
    W = int(np.ceil(360.0 / float(np.float32(az_res))))
    h = int(rng.integers(1, max(2, min(60, 60000 // W))))
    span = el_res * (h + rng.uniform(0.05, 0.95))                         # a partial top row
    el_min = float(rng.uniform(-30.0, 0.0))
    o = F.Opts(az_res_deg=az_res, el_res_deg=el_res, el_min_deg=el_min, el_max_deg=el_min + span, dilate=int(rng.integers(0, 5)),
               margin=float(rng.uniform(0.0, 1.0)), margin_rel=float(rng.uniform(0.0, 0.05)), min_range=float(rng.uniform(0.0, 3.0)),
               max_range=float(rng.uniform(20.0, 60.0)))
    g = F._geom(o)
    Wd, Hd = F.dims(o)
    n_scan = min(150000, 6 * Wd * Hd + 1000)
    q_scan = _sensor_cloud(o, n_scan, rng, 3.0, 50.0, el_pad=0.2 * span)
    q_map = _sensor_cloud(o, 10000, rng, 0.5, 55.0, el_pad=0.2 * span)

    def edges(n, r_lo, r_hi):
        """n points within 1e-6 pixel of the seam, el_min or el_max"""
        u = rng.uniform(-1e-6, 1e-6, n)
        az = np.where(rng.random(n) < 0.5, rng.uniform(-np.pi, np.pi, n), np.pi + u * g["az_res"])
        el = np.select([rng.random(n) < 0.33, rng.random(n) < 0.5], [g["el_min"] + u * g["el_res"], g["el_max"] + u * g["el_res"]],
                       rng.uniform(g["el_min"], g["el_max"], n))
        r = rng.uniform(r_lo, r_hi, n)
        return np.c_[r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)]

    pose = np.r_[rng.normal(0, 2.0, 3), synth.quat_from_rotvec(rng.normal(0, 0.3, 3))]
    scan = S.cloud(np.vstack([q_scan, edges(2000, 3.0, 50.0)]))
    mp = S.cloud(_to_world(np.vstack([q_map, edges(1000, 0.5, 55.0)]), pose))
    return o, scan, mp, pose


def test_randomised_sweep_lies_between_the_bounds(gpu_api, ctx):
    exact_sets = 0
    for seed in range(40):
        o, scan, mp, pose = _sweep_set(seed)
        before, after, r = _carve(gpu_api, ctx, mp, scan, pose, o)
        gone = _removed(before, after)
        lo, hi = F.bounds(before, scan, pose, o)
        _, st = F.clear(before, scan, pose, o)
        n_amb_scan = int(F.edge_points(scan, o).sum())
        n_amb_map = int((F.edge_points(before, o, pose) | (hi & ~lo)).sum())
        W, H = F.dims(o)
        print(f"set {seed:2d}: {W} x {H}, dilate {o.dilate}, {len(scan)} returns, {len(before)} map points; ambiguous scan points "
              f"{n_amb_scan}, map points {n_amb_map}; removed {int(gone.sum())} (numpy {int(lo.sum())}..{int(hi.sum())})")
        assert not (lo & ~gone).any() and not (gone & ~hi).any()
        assert r["n_removed"] == gone.sum() and r["n_after"] == (len(after), 0)
        if n_amb_scan == 0 and n_amb_map == 0:
            exact_sets += 1
            assert _counters(r) == st
    print(f"{exact_sets} of 40 sets without an ambiguous point, their counters exact")

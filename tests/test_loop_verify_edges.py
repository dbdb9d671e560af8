"""Loop verification (so_loop_verify) at its edges, every score against the numpy restatement (loop_verify_numpy.py): inliers, overlap
and rmse bit for bit, the conflict counts exact or inside the restatement's pixel-edge sandwich, the submap ids and sizes exact.

  - the inlier bound: d^2 == float(inlier_dist^2) counts, the next float below does not; on the select walk, on the knn_cube path
    (inlier_dist above R * cs), past the 50 m block, and at a subnormal bound where only coincident points count;
  - the in-block rule: a candidate near a block face, its query partly off the window or across the face;
  - the fixed-order sum at grid sizes 1, 256, 257 and 2048+ and nq % 64 != 0;
  - many images: half_window 0 and 8, windows cut at id 0 and at the range's end, the query inside the range, empty submap
    keyframes first, in the middle and last, a submap of empty keyframes only, each keyframe's points in its own image, and the
    256 MiB image limit at its boundary;
  - degenerate queries: an empty query keyframe, NaN and inf points;
  - scratch independence: one mixed batch on a fresh scratch, one that verified a much larger candidate and one used for mapping;
  - an error in the middle of a batch.

Keyframes are imported (so_keyframe_import) from the cfg2 VLP-16 loop of test_loop_detection.py at their true poses."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

import loop_verify_numpy as V
from test_keyframes import _ctx, _err
from test_loop_detection import _loop_scans, _loop_truth
from test_loop_verify import VLP16, _bytes

pytestmark = pytest.mark.gpu

SO_ERR_ARG = -1
REG_FIELDS = ("pose", "pose_opt", "cov", "iter_cost", "hist_obs", "hist_reject_plane")


def _store(api, clouds, poses, cap_points=1 << 22):
    ctx = _ctx(api)
    ctx.keyframe_reserve(cap_points, len(clouds) + 4)
    for c, p in zip(clouds, poses):
        assert ctx.keyframe_import(np.asarray(c, np.float32).reshape(-1, 4), p) >= 0
    return ctx


def _cand(query, cid, yaw=0.0):
    from superodom_b200 import api
    c = np.zeros(1, api.LOOP_CANDIDATE_DTYPE)
    c[0]["query"], c[0]["id"], c[0]["yaw"] = query, cid, yaw
    return c


def _opts(api, **kw):
    image = kw.pop("image", VLP16)
    return api.loop_verify_opts(image=image, **kw)


def _reg_bytes(r):
    return tuple(bytes(getattr(r.reg, f)) for f in REG_FIELDS) + ((r.reg.status, r.reg.n_iterations),)


def _f64(x):
    return struct.pack("<d", float(x))


def _check(ctx, scratch, r, o, reach=None, tag=""):
    """r: the result of the last candidate scratch verified.  Every field against the restatement -> the restatement's scores."""
    q, cid = int(r.query), int(r.id)
    poses = ctx.keyframe_poses()
    ids = V.submap_ids(q, cid, o.half_window, o.id_begin, o.id_end, o.exclude_recent)
    surf = scratch.map_download_all(0)
    assert r.skipped == 0 and r.n_submap_keyframes == len(ids) and r.n_submap_points == len(surf), (tag, ids)
    reg_pose = np.array(r.reg.pose)
    s = V.scores(ctx.keyframe_download(q, 0, reg_pose), ctx.keyframe_download(q, 0), surf, scratch.map_origin(),
                 [ctx.keyframe_download(i, 0) for i in ids], poses[ids], reg_pose, o.inlier_dist, o.image, reach=reach)
    assert (r.n_query_points, r.n_inliers) == (s["n_query"], s["n_inliers"]), tag
    assert _f64(r.overlap) == _f64(s["overlap"]) and _f64(r.rmse) == _f64(s["rmse"]), (tag, r.rmse, s["rmse"])
    for side, dev in (("query", (r.n_cand_query, r.n_conflict_query)), ("map", (r.n_cand_map, r.n_conflict_map))):
        b = s[side]
        assert b["cand"][0] <= dev[0] <= b["cand"][1] and b["conflict"][0] <= dev[1] <= b["conflict"][1], (tag, side, dev, b)
    assert r.conflict_query == V.fraction(r.n_conflict_query, r.n_cand_query)
    assert r.conflict_map == V.fraction(r.n_conflict_map, r.n_cand_map)
    assert r.accepted == V.accept(r.reg.status, s["overlap"], r.conflict_query, r.conflict_map, o.min_overlap, o.max_conflict)
    print(f"{tag}: q {q} id {cid} submap {ids} pts {len(surf)} nq {s['n_query']} grid {s['grid']} inliers {s['n_inliers']} "
          f"rmse {s['rmse']:.6f} cand/conf q {r.n_cand_query}/{r.n_conflict_query} map {r.n_cand_map}/{r.n_conflict_map} "
          f"sandwiched points q {s['query']['open']} map {s['map']['open']}")
    return s


def _verify_one(ctx, scratch, cand, o, **kw):
    r = ctx.loop_verify(scratch, cand, o)[0]
    return r, _check(ctx, scratch, r, o, **kw)


def _scene(n=30):
    return list(_loop_scans(False)[:n]), list(_loop_truth(False)[:n])


def _near(scan, pose, n, seed, sigma=0.03):
    """n points of scan (sensor frame), repeated and jittered: a query keyframe of any size at the same place."""
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, len(scan), n)
    out = scan[idx].copy()
    out[:, :3] += rng.normal(0, sigma, (n, 3)).astype(np.float32)
    return out


# ------------------------------------------------------------------------------------------------------------- 1. the inlier bound
def _largest_at_most(t32):
    """The largest positive double x with float(x * x) <= t32."""
    lo, hi = 0, int(np.float64(np.inf).view(np.int64)) - 1
    with np.errstate(over="ignore"):
        while lo < hi:
            mid = (lo + hi + 1) // 2
            x = float(np.int64(mid).view(np.float64))
            if np.float32(x * x) <= t32:
                lo = mid
            else:
                hi = mid - 1
    return float(np.int64(lo).view(np.float64))


@pytest.fixture(scope="module")
def loop_store(gpu_api):
    scans, poses = _scene()
    ctx = _store(gpu_api, scans + [_loop_scans(False)[59]], poses + [_loop_truth(False)[59]])
    yield ctx, len(scans)
    ctx.close()


@pytest.mark.parametrize("mode,dist,lo,hi", [("select", 0.5, 0.05, 0.25), ("cube", 1.2, 0.7, 1.44), ("past_block", 60.0, 4.0, 3600.0)])
def test_inlier_bound_tie(gpu_api, loop_store, mode, dist, lo, hi):
    ctx, q = loop_store
    cand = _cand(q, 1)
    base = dict(id_begin=0, id_end=q, half_window=2)
    scratch = _ctx(gpu_api)
    r0, s0 = _verify_one(ctx, scratch, cand, _opts(gpu_api, inlier_dist=dist, **base), reach=dist, tag=f"{mode} {dist}")
    d2 = s0["d2"][s0["inlier"] & (s0["d2"] > lo) & (s0["d2"] <= hi)]
    assert len(d2), (mode, "no inlier in the band")
    t = np.float32(np.sort(d2)[len(d2) // 2] if mode != "past_block" else d2.max())
    at, below = _largest_at_most(t), _largest_at_most(np.nextafter(t, np.float32(0)))
    assert np.float32(at * at) == t and np.float32(below * below) == np.nextafter(t, np.float32(0))
    n_tie = int((s0["d2"] == t).sum())
    got = {}
    for name, x in (("at", at), ("below", below)):
        o = _opts(gpu_api, inlier_dist=x, **base)
        r, s = _verify_one(ctx, scratch, cand, o, reach=max(x, 1e-3), tag=f"{mode} {name}")
        assert _reg_bytes(r) == _reg_bytes(r0), (mode, name)                  # the alignment does not depend on inlier_dist
        got[name] = (r, s)
    assert got["at"][0].n_inliers - got["below"][0].n_inliers == n_tie >= 1, mode
    assert got["at"][1]["inlier"][s0["d2"] == t].all() and not got["below"][1]["inlier"][s0["d2"] == t].any()
    scratch.close()


def test_subnormal_bound_counts_only_coincident_points(gpu_api):
    """A sparse lattice (3 m pitch: no point has a neighbour within the plane fit's radius, so the alignment finds no correspondence
    and keeps its prior) imported as both the candidate and the query at the same pose: the query lands on the map's points, d^2 = 0
    exactly, and the smallest inlier_dist with a nonzero float square (a subnormal bound) counts exactly those."""
    g = np.arange(-12.0, 12.1, 3.0)
    lat = np.array([[x, y, z, 1.0] for x in g for y in g for z in (-1.5, 1.5)], np.float32)
    lat[:, :3] += np.float32(0.1)
    pose = np.array([2.0, -3.0, 0.5, 0.0, 0.0, 0.0, 1.0])
    ctx = _store(gpu_api, [lat, lat], [pose, pose])
    scratch = _ctx(gpu_api)
    x = _largest_at_most(np.float32(1e-44))
    assert 0 < np.float32(x * x) < np.finfo(np.float32).tiny
    o = _opts(gpu_api, inlier_dist=x, id_begin=0, id_end=1, half_window=0)
    r, s = _verify_one(ctx, scratch, _cand(1, 0), o, reach=1e-3, tag="subnormal")
    assert np.array_equal(np.array(r.reg.pose), pose), "the alignment moved: the lattice no longer lands on the map"
    assert r.n_inliers == len(lat) == int((s["d2"] == 0).sum()) and r.rmse == 0.0
    # a query half a millimetre off: no d^2 is 0, so nothing counts at the subnormal bound, everything at 1 cm
    off = lat.copy()
    off[:, 0] += np.float32(5e-4)
    ctx2 = _store(gpu_api, [lat, off], [pose, pose])
    r, s = _verify_one(ctx2, scratch, _cand(1, 0), o, reach=1e-3, tag="subnormal off")
    assert r.n_inliers == 0 and r.rmse == 0.0
    r, s = _verify_one(ctx2, scratch, _cand(1, 0), _opts(gpu_api, inlier_dist=0.01, id_begin=0, id_end=1, half_window=0),
                       tag="off 1 cm")
    assert r.n_inliers == len(lat)
    for c in (ctx, ctx2, scratch):
        c.close()


# ------------------------------------------------------------------------------------------------------------- 2. the in-block rule
def test_block_faces_and_window(gpu_api):
    """A candidate a few metres inside a block face: so_map_set_origin puts the candidate's block at the window's lower corner, so
    the query's part below it falls off the window, and query points near the faces have their true nearest neighbour across them."""
    from superodom_b200 import synth
    scans, poses = _scene(12)
    shift = np.array([-22.5 - poses[4][0], 0.0, 0.0])                  # keyframe 4 2.5 m inside the face x = -25
    moved = [np.r_[p[:3] + shift, p[3:]] for p in poses]
    ctx = _store(gpu_api, scans + [scans[4]], moved + [moved[4]])
    scratch = _ctx(gpu_api)
    n = len(scans)
    for cid in (3, 4, 5):
        for dist in (0.5, 3.0):
            o = _opts(gpu_api, id_begin=0, id_end=n, half_window=2, inlier_dist=dist)
            r, s = _verify_one(ctx, scratch, _cand(n, cid), o, reach=dist, tag=f"face cand {cid} dist {dist}")
            qw = ctx.keyframe_download(n, 0, np.array(r.reg.pose))[:, :3]
            off = synth.block_linear(synth.block_of(qw, scratch.map_origin())) < 0
            print(f"  origin {scratch.map_origin()}, query points off the window {int(off.sum())}")
            assert off.any() and not s["inlier"][off].any()
    scratch.close()
    ctx.close()


def _lattice(lo, hi, pitch, z=(-1.5, 1.5)):
    g = np.arange(lo, hi + 1e-9, pitch)
    return np.array([[x, y, zz] for x in g for y in g for zz in z], np.float64)


def test_points_on_block_faces(gpu_api):
    """Query points exactly on block faces, at a candidate whose block lies below the world origin, so that the window holds blocks
    of negative x + 25: LocalMap's truncate-then-decrement rule sends x + 25 = -50 to the block below (with the candidate), x + 25 = 0
    to the block above.  Map points on both sides of each face, nearer across it.  Sparse lattices (3 m pitch) keep the alignment at
    its prior, so every query point lands where it was placed."""
    P = np.array([-80.0, -80.0, 0.5, 0.0, 0.0, 0.0, 1.0])
    faces = np.array([[-75.0, -80.0, 0.5], [-25.0, -80.0, 0.5], [-80.0, -75.0, 0.5], [-80.0, -25.0, 0.5], [-75.0, -75.0, 0.5],
                      [-75.0, -25.0, -1.0]])
    near = np.concatenate([faces + [1.0, 0, 0], faces - [1.5, 0, 0], faces + [0, 1.0, 0], faces - [0, 1.5, 0]])
    m = np.concatenate([_lattice(-92.0, -68.0, 3.0) + [0.25, 0.25, 0.0], near])
    sensor = lambda w: np.c_[(w - P[:3]).astype(np.float32), np.ones(len(w), np.float32)]
    ctx = _store(gpu_api, [sensor(m), sensor(faces)], [P, P])
    scratch = _ctx(gpu_api)
    o = _opts(gpu_api, id_begin=0, id_end=1, half_window=0, inlier_dist=30.0)
    r, s = _verify_one(ctx, scratch, _cand(1, 0), o, reach=30.0, tag="block faces")
    assert np.array_equal(np.array(r.reg.pose), P), "the alignment moved: the face points are no longer on the faces"
    assert np.array_equal(ctx.keyframe_download(1, 0, P)[:, :3], faces.astype(np.float32))
    assert r.n_query_points == len(faces) and r.n_inliers == int(np.isfinite(s["d2"]).sum()) > 0
    print("  face d2", s["d2"])
    scratch.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------------------- 3. the sum's sizes
def test_fixed_order_sum_at_every_grid_size(gpu_api):
    scans, poses = _scene(12)
    sizes = [1, 63, 64, 65, 64 * 256, 64 * 256 + 1, 131101]
    queries = [_near(scans[5], poses[5], n, 100 + n) for n in sizes]
    ctx = _store(gpu_api, scans + queries, poses + [poses[5]] * len(sizes))
    scratch = _ctx(gpu_api)
    grids = []
    for k, n in enumerate(sizes):
        o = _opts(gpu_api, id_begin=0, id_end=len(scans), half_window=3)
        r, s = _verify_one(ctx, scratch, _cand(len(scans) + k, 5), o, tag=f"nq {n}")
        assert r.n_query_points == n and s["n_inliers"] > 0
        grids.append(s["grid"])
    assert {1, 256, 257}.issubset(grids) and max(grids) >= 2048
    scratch.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------------------- 4. many images
def test_windows_and_empty_keyframes(gpu_api):
    scans, poses = _scene(20)
    empty = np.zeros((0, 4), np.float32)
    holes = [s if i not in (2, 10, 18) else empty for i, s in enumerate(scans)]
    ctx = _store(gpu_api, holes + [scans[10]], poses + [poses[10]])
    scratch = _ctx(gpu_api)
    q = len(scans)
    cases = [(10, 0, 0, q), (10, 8, 0, q), (2, 8, 0, q), (0, 8, 0, q), (18, 8, 0, q), (19, 8, 0, q), (10, 8, 4, 17)]
    for cid, w, b, e in cases:
        o = _opts(gpu_api, id_begin=b, id_end=e, half_window=w)
        _verify_one(ctx, scratch, _cand(q, cid), o, tag=f"window c {cid} w {w} [{b},{e})")
    # the query inside the range: never in its own submap
    o = _opts(gpu_api, id_begin=0, id_end=q, half_window=8)
    r, _ = _verify_one(ctx, scratch, _cand(12, 9), o, tag="query inside")
    assert r.n_submap_keyframes == 16
    ctx.close()
    # a submap of empty keyframes only
    ctx = _store(gpu_api, [empty] * 5 + [scans[3]], poses[:6])
    r, s = _verify_one(ctx, scratch, _cand(5, 2), _opts(gpu_api, id_begin=0, id_end=5, half_window=2), tag="all empty")
    assert r.n_submap_points == 0 and r.n_inliers == 0 and r.n_cand_map == 0 and r.n_cand_query == 0 and not r.accepted
    scratch.close()
    ctx.close()


def test_each_image_holds_its_own_keyframe(gpu_api):
    """Three one-point submap keyframes 20 m apart, each point the only return that makes one query point a conflict (dilate 0, the
    query point half way along the keyframe's ray): every keyframe's first point must land in its own image, or a conflict is lost.
    One-point clouds give the alignment no correspondence, so it keeps its prior and every query point lands where it was placed."""
    pos = [np.array([0.0, 20.0 * k, 0.0]) for k in range(3)]
    dirs = [np.array([math.cos(a), math.sin(a), 0.1]) for a in (0.1, 0.1 + math.pi / 2, 0.1 + math.pi)]
    ident = [0.0, 0.0, 0.0, 1.0]
    clouds = [np.array([[*(10.0 * d), 1.0]], np.float32) for d in dirs]
    query = np.array([[*(p + 5.0 * d - pos[1]), 1.0] for p, d in zip(pos, dirs)], np.float32)
    ctx = _store(gpu_api, clouds + [query], [np.r_[p, ident] for p in pos] + [np.r_[pos[1], ident]])
    scratch = _ctx(gpu_api)
    o = _opts(gpu_api, image=dict(VLP16, dilate=0), id_begin=0, id_end=3, half_window=1)
    r, s = _verify_one(ctx, scratch, _cand(3, 1), o, tag="one point per image")
    assert np.array_equal(np.array(r.reg.pose), np.r_[pos[1], ident]), "the alignment moved"
    assert (r.n_cand_query, r.n_conflict_query) == (3, 3) and s["query"]["open"] == 0
    scratch.close()
    ctx.close()


def test_image_limit_at_its_boundary(gpu_api):
    """17 images of 900 x 4386 pixels fit in 256 MiB (268 423 200 bytes), 900 x 4387 do not; the limit counts 2w + 1 images."""
    scans, poses = _scene(20)
    ctx = _store(gpu_api, scans + [scans[10]], poses + [poses[10]])
    q = len(scans)
    fit = dict(az_res_deg=0.4, el_res_deg=0.015625, el_min_deg=-34.265625, el_max_deg=34.265625, dilate=0)
    past = dict(fit, el_max_deg=34.28125)
    assert 17 * 900 * 4386 * 4 <= 256 << 20 < 17 * 900 * 4387 * 4
    scratch = _ctx(gpu_api)
    o = _opts(gpu_api, image=fit, id_begin=0, id_end=q, half_window=8)
    r, s = _verify_one(ctx, scratch, _cand(q, 10), o, tag="at the image limit")
    assert r.n_submap_keyframes == 17 and r.n_cand_query > 0 and r.n_cand_map > 0
    for c in (ctx, scratch):
        c.kernel_launches(reset=True)
    assert _err(gpu_api, lambda: ctx.loop_verify(scratch, _cand(q, 10), _opts(gpu_api, image=past, id_begin=0, id_end=q,
                                                                                    half_window=8))) == SO_ERR_ARG
    assert ctx.kernel_launches() == 0 and scratch.kernel_launches() == 0
    # 16 images (half_window 7 and 2w + 1 = 15, or 2w = 16) of the larger image fit: the smaller window is accepted
    r = ctx.loop_verify(scratch, _cand(q, 10), _opts(gpu_api, image=past, id_begin=0, id_end=q, half_window=7))[0]
    _check(ctx, scratch, r, _opts(gpu_api, image=past, id_begin=0, id_end=q, half_window=7), tag="past the limit, w 7")
    scratch.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------------------- 5. degenerate queries
def test_empty_query_equals_its_manual_alignment(gpu_api):
    scans, poses = _scene(8)
    ctx = _store(gpu_api, scans + [np.zeros((0, 4), np.float32)], poses + [poses[4]])
    q = len(scans)
    scratch = _ctx(gpu_api)
    o = _opts(gpu_api, id_begin=0, id_end=q, half_window=2)
    r, s = _verify_one(ctx, scratch, _cand(q, 4), o, tag="empty query")
    sub = _ctx(gpu_api)
    ids = [2, 3, 4, 5, 6]
    sub.map_set_origin(poses[4][:3])
    sub.map_from_keyframes(ctx, ids, ctx.keyframe_poses()[ids], 1)
    prior = ctx.loop_prior(_cand(q, 4)[0])
    reg = sub.register_keyframes(ctx, [q], [prior], 20, 0)[0]
    for f in REG_FIELDS:
        assert bytes(getattr(reg, f)) == bytes(getattr(r.reg, f)), f
    assert (reg.status, reg.n_iterations) == (r.reg.status, r.reg.n_iterations)
    assert (r.n_query_points, r.n_inliers, r.n_cand_query, r.n_conflict_query, r.n_cand_map, r.n_conflict_map) == (0,) * 6
    assert r.overlap == 0.0 and r.rmse == 0.0 and not r.accepted
    for c in (ctx, scratch, sub):
        c.close()


def test_non_finite_points_are_not_counted(gpu_api):
    scans, poses = _scene(8)
    rng = np.random.default_rng(3)
    bad = np.array([[np.nan, 1, 1, 1], [1, np.inf, 1, 1], [1, 1, -np.inf, 1], [np.nan] * 4, [np.inf, -np.inf, np.nan, 1]], np.float32)

    def spoil(s):
        idx = np.sort(rng.choice(len(s) + len(bad), len(bad), replace=False))
        out = np.insert(s, idx - np.arange(len(bad)), bad, axis=0)
        return out

    dirty = [spoil(s) if i in (3, 5) else s for i, s in enumerate(scans)]
    ctx = _store(gpu_api, dirty + [spoil(scans[4])], poses + [poses[4]])
    q = len(scans)
    scratch = _ctx(gpu_api)
    o = _opts(gpu_api, id_begin=0, id_end=q, half_window=2)
    r, s = _verify_one(ctx, scratch, _cand(q, 4), o, tag="non-finite")
    assert r.n_query_points == len(scans[4]) and r.n_inliers > 0 and r.n_cand_query > 0
    for c in (ctx, scratch):
        c.close()


# ------------------------------------------------------------------------------------------------------------- 6. scratch independence
def test_results_independent_of_the_scratch(gpu_api):
    from superodom_b200 import api
    scans, poses = _scene(24)
    big = _near(scans[6], poses[6], 120000, 9)
    ctx = _store(gpu_api, scans + [scans[5], scans[12], scans[20], big], poses + [poses[5], poses[12], poses[20], poses[6]])
    n = len(scans)
    o = _opts(gpu_api, id_begin=0, id_end=n, half_window=3)
    rows = [(n, -1), (n, 4), (n + 1, 12), (n + 1, -1), (n + 2, 19), (n, 4), (n + 2, 22), (n + 1, -1)]
    batch = np.zeros(len(rows), api.LOOP_CANDIDATE_DTYPE)
    for k, (qq, c) in enumerate(rows):
        batch[k]["query"], batch[k]["id"], batch[k]["yaw"] = qq, c, 0.01 * rows.index((qq, c))      # the repeated candidate alike
    before = (ctx.keyframe_poses().tobytes(), ctx.keyframe_info(), [ctx.keyframe_download(i, 0).tobytes() for i in range(n + 4)])
    fresh = _ctx(gpu_api)
    larger = _ctx(gpu_api)
    ctx.loop_verify(larger, _cand(n + 3, 6), _opts(gpu_api, id_begin=0, id_end=n, half_window=8))
    used = _ctx(gpu_api)
    m = scans[7].copy()
    used.map_set_points(np.c_[m[:, :3] + poses[7][:3].astype(np.float32), m[:, 3:]])
    used.map_set_edge_points(np.c_[m[::3, :3] + poses[7][:3].astype(np.float32), m[::3, 3:]])
    used.register(scans[8], poses[8], 5)
    used.map_add_registered_scan(poses[8])
    outs = [_bytes(api, ctx.loop_verify(s, batch, o)) for s in (fresh, larger, used)]
    assert outs[0] == outs[1] == outs[2]
    alone = []
    for k in range(len(batch)):
        s = _ctx(gpu_api)
        r = ctx.loop_verify(s, batch[k:k + 1], o)[0]
        if not r.skipped:
            _check(ctx, s, r, o, tag=f"alone {k}")
        alone.append(_bytes(api, [r])[0])
        s.close()
    assert outs[0] == alone
    res = ctx.loop_verify(fresh, batch, o)
    assert [r.skipped for r in res] == [int(c == -1) for _, c in rows] and _bytes(api, res[1:2]) == _bytes(api, res[5:6])
    after = (ctx.keyframe_poses().tobytes(), ctx.keyframe_info(), [ctx.keyframe_download(i, 0).tobytes() for i in range(n + 4)])
    assert before == after
    for c in (ctx, fresh, larger, used):
        c.close()


# ------------------------------------------------------------------------------------------------------------- 7. an error mid-batch
def test_error_mid_batch_keeps_the_results_before_it(gpu_api):
    from superodom_b200 import api
    scans, poses = _scene(12)
    big = _near(scans[6], poses[6], 40000, 4)
    ctx = _store(gpu_api, scans + [scans[5], big, scans[7]], poses + [poses[5], poses[6], poses[7]])
    n = len(scans)
    o = _opts(gpu_api, id_begin=0, id_end=n, half_window=2)
    batch = np.concatenate([_cand(n, 4), _cand(n + 2, 8), _cand(n + 1, 6), _cand(n + 2, 7)])
    small = dict(max_scan_points=1 << 15)
    assert max(len(scans[5]), len(scans[7])) <= 1 << 15 < len(big)
    before = (ctx.keyframe_poses().tobytes(), ctx.keyframe_info())
    scratch, alone, pair = (_ctx(gpu_api, **small) for _ in range(3))
    res = (api.LoopVerifyResult * 4)()
    rc = ctx.L.so_loop_verify(ctx.h, scratch.h, api._p(batch), 4, C.byref(o), res)
    alone_rc = _err(gpu_api, lambda: ctx.loop_verify(alone, batch[2:3], o))
    assert rc < 0 and rc == alone_rc, (rc, alone_rc)
    two = ctx.loop_verify(pair, batch[:2], o)
    assert _bytes(api, list(res)[:2]) == _bytes(api, two)
    assert (ctx.keyframe_poses().tobytes(), ctx.keyframe_info()) == before
    for c in (ctx, scratch, alone, pair):
        c.close()

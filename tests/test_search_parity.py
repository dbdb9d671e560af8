"""The registration's own neighbour searches against the exact in-block search of the oracle, on the inputs where searches go wrong
(tests/search_sets.py): the scan search of ICP iteration 0 (warp-per-query and lane-per-query kernels), the seeded search of later
iterations (so_correspond_seeded), the edge fit's unbounded 10-NN, and queries that are not finite or lie far off the grid.

Bars: neighbour ids, float d2, statuses, selection masks and histograms bit for bit; the seed is a pruning aid only, so a seeded
search is bit-equal to an unseeded one in every reported field."""
import numpy as np
import pytest

import search_sets as S
from conftest import get_case, quat_angle

pytestmark = pytest.mark.gpu

NONE = 0xFFFFFFFF
POSE_TOL_M = 1e-4
POSE_TOL_RAD = 1e-4
COOP_MAX_QUERIES = 32 * 256            # so_icp.cuh kCoopMaxGrid x kThreads: larger scans take the lane-per-query search


def _ctx(api, map_xyzi, plane_res, lane=False, monkeypatch=None, **kw):
    """A context on map_xyzi; lane: SO_NO_COOP_KNN, one query per thread whatever the scan size (read when the context is made)."""
    if lane:
        monkeypatch.setenv("SO_NO_COOP_KNN", "1")
    try:
        ctx = api.Context(max_map_points=max(1 << 20, len(map_xyzi) + 1024), max_scan_points=262144, plane_res=plane_res, **kw)
    finally:
        if lane:
            monkeypatch.delenv("SO_NO_COOP_KNN")
    ctx.map_set_points(map_xyzi)
    return ctx


def _translation(t):
    return np.array([t[0], t[1], t[2], 0, 0, 0, 1], np.float64)


def _moved(pose, dt, drot, axis=(0.3, -0.5, 0.8)):
    """pose with its translation moved by dt and its rotation by drot radians about `axis` (right-multiplied)."""
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    dq = np.concatenate([a * np.sin(drot / 2), [np.cos(drot / 2)]])
    x1, y1, z1, w1 = pose[3:]
    x2, y2, z2, w2 = dq
    q = np.array([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                  w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2])
    return np.concatenate([np.asarray(pose[:3], np.float64) + np.asarray(dt, np.float64), q / np.linalg.norm(q)])


def _ostatus(oc):
    st = oc["status"].astype(np.int64)
    st[st < 0] = 255
    return st


def _assert_matches_oracle(got, want, plane_res, what):
    """so_correspond output against the oracle's exact correspondences: statuses and histograms; neighbour ids and d2 bit for bit
    wherever five neighbours were found; a point with fewer than five inside the 3 planeRes gate reports exactly the oracle's
    neighbours inside the gate; the plane fit of accepted points."""
    gc, gho, ghr = got
    oc, oho, ohr = want
    ost = _ostatus(oc)
    assert np.array_equal(gc["status"].astype(np.int64), ost), (what, np.flatnonzero(gc["status"].astype(np.int64) != ost)[:10])
    assert np.array_equal(gho, oho) and np.array_equal(ghr, ohr), (what, gho, oho, ghr, ohr)
    found5 = ~np.isin(ost, (1, 2, 255))
    assert np.array_equal(gc["nn"][found5].astype(np.int64), oc["nn"][found5]), what
    assert np.array_equal(gc["nn_d2"][found5], oc["nn_d2"][found5]), what
    bound = np.float32(3 * np.float32(plane_res))
    far = ost == 2
    want_far = np.where(oc["nn_d2"][far] <= bound, oc["nn"][far], NONE)
    assert np.array_equal(gc["nn"][far].astype(np.int64), want_far), what
    assert (gc["nn"][ost == 1] == NONE).all(), what
    ok = ost == 0
    assert np.array_equal(gc["obs"][ok], oc["obs"][ok].astype(np.uint8)), what
    assert np.allclose(gc["n"][ok], oc["n"][ok], rtol=0, atol=1e-8) and np.allclose(gc["w"][ok], oc["w"][ok], rtol=1e-10, atol=0), what


def _same_bits(a, b):
    """two so_correspond outputs (corr, hist_obs, hist_rej) are identical in every byte"""
    return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------------------
# B. ICP iteration 0: both search kernels on lattice ties, dense clusters and 50 m block faces
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lattice", "dense", "block_face"])
def test_iteration0_search_on_adversarial_sets(gpu_api, oracle_mod, monkeypatch, name):
    mp, pr, q = S.surf_case(name)
    rng = np.random.default_rng(1)
    scan = S.xyzi(q)
    small = scan[rng.permutation(len(scan))[:COOP_MAX_QUERIES]]           # the warp search serves scans up to 8 192 points
    reps = COOP_MAX_QUERIES // len(scan) + 1
    big = np.concatenate([scan] * reps)                                   # > 8 192 points: the lane search
    assert len(small) <= COOP_MAX_QUERIES < len(big)
    om = oracle_mod.OracleMap(mp)
    warp = _ctx(gpu_api, mp, pr)
    lane = _ctx(gpu_api, mp, pr, lane=True, monkeypatch=monkeypatch)
    # identity, then a translation by dyadic amounts: the transformed queries stay the float32 points the set was built with
    for pose in (S.IDENTITY, _translation([0.25, -0.5, 0.125])):
        want_small = om.correspond(small, pose, pr, 0, 0, n_threads=8)
        got_warp = warp.correspond(small, pose)
        _assert_matches_oracle(got_warp, want_small, pr, (name, "warp"))
        got_lane = lane.correspond(small, pose)
        _assert_matches_oracle(got_lane, want_small, pr, (name, "lane"))
        assert _same_bits(got_warp, got_lane), name
        oc, oho, ohr = om.correspond(scan, pose, pr, 0, 0, n_threads=8)
        want_big = (np.concatenate([oc] * reps), oho * reps, ohr * reps)
        _assert_matches_oracle(warp.correspond(big, pose), want_big, pr, (name, "lane, large scan"))
        assert (_ostatus(oc) == 0).sum() > 100 or name == "dense"
    warp.close()
    lane.close()


# ---------------------------------------------------------------------------------------------------------------
# C. Later ICP iterations: the search seeded with the previous iteration's neighbours
# ---------------------------------------------------------------------------------------------------------------
def _seed_branches(map_xyz, scan, pose, first, second_status):
    """seed_bound (so_icp.cu) restated: for every point whose first search found five neighbours and whose second search runs in a
    block of >= 5 points, is the seed taken (all five old neighbours in the query's new block and u <= 1.3 d5), rejected by the 1.3
    rule, or void because the old neighbours lie in another block?  u = the largest of the old neighbours' distances to the moved
    query with the reference's rounding (float differences, double sum, float result).  -> dict of boolean masks."""
    from oracle.oracle import transform_scan_numpy
    from superodom_b200 import synth
    st0 = first["status"].astype(np.int64)
    eligible = ~np.isin(st0, (1, 2, 255)) & ~np.isin(second_status.astype(np.int64), (1, 255))
    qf = transform_scan_numpy(scan, pose)[:, :3]
    qb = synth.block_linear(synth.block_of(qf))
    nn = np.where(eligible[:, None], first["nn"].astype(np.int64), 0)
    c = map_xyz[nn]                                                       # float32 [n, 5, 3]
    nb_block = synth.block_linear(synth.block_of(c.reshape(-1, 3))).reshape(-1, 5)
    same = (nb_block == qb[:, None]).all(1)
    d = (qf[:, None, :] - c).astype(np.float64)                           # float32 differences, widened
    u = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]).astype(np.float32).max(1)
    rule = u <= np.float32(1.3) * first["nn_d2"][:, 4]
    return {"take": eligible & same & rule, "reject": eligible & same & ~rule, "crossed": eligible & ~same}


# (set, move name, pose_prev, pose, branch that must run, its minimum count)
def _seed_moves():
    cfg1 = get_case("cfg1")["pose_prior"]
    return [
        ("cfg1", "none", cfg1, cfg1, "take", 20000),
        ("cfg1", "small", cfg1, _moved(cfg1, [0.003, -0.002, 0.001], 1e-4), "take", 10000),
        ("cfg1", "small_5mm", cfg1, _moved(cfg1, [-0.004, 0.003, 0.0], -1e-4, axis=(0, 0, 1)), "take", 10000),
        ("cfg1", "large", cfg1, _moved(cfg1, [0.15, -0.1, 0.05], 0.02), "reject", 2000),
        ("block_face", "cross", _translation([-0.004, 0.0, 0.0]), S.IDENTITY, "crossed", 300),
        ("block_face", "small", _translation([0.0, 0.001, -0.002]), S.IDENTITY, "take", 3000),
        ("lattice", "faces", _translation([2.0 ** -9, -2.0 ** -10, 2.0 ** -11]), S.IDENTITY, "take", 3000),
        ("dense", "small", _translation([0.0, 2.0 ** -9, 0.0]), S.IDENTITY, "take", 300),
    ]


def _seed_case(name):
    if name == "cfg1":
        case = get_case("cfg1")
        return case["map_xyzi"], case["cfg"]["plane_res"], case["scan_xyzi"]
    mp, pr, q = S.surf_case(name)
    return mp, pr, S.xyzi(q)


@pytest.mark.parametrize("name,move", [(m[0], m[1]) for m in [("cfg1", "none"), ("cfg1", "small"), ("cfg1", "small_5mm"), ("cfg1", "large"),
                                                                ("block_face", "cross"), ("block_face", "small"), ("lattice", "faces"),
                                                                ("dense", "small")]])
def test_seeded_search_equals_unseeded_and_oracle(gpu_api, oracle_mod, monkeypatch, name, move):
    spec = [m for m in _seed_moves() if m[:2] == (name, move)][0]
    _, _, prev, pose, branch, minimum = spec
    mp, pr, scan = _seed_case(name)
    om = oracle_mod.OracleMap(mp)
    ctx = _ctx(gpu_api, mp, pr, lane=True, monkeypatch=monkeypatch)      # the warp search ignores seeds
    first = ctx.correspond(scan, prev)                                    # what iteration 0 at pose_prev leaves for the seed
    _assert_matches_oracle(first, om.correspond(scan, prev, pr, 0, 0, n_threads=8), pr, (name, move, "iteration 0"))
    plain = ctx.correspond(scan, pose)
    seeded = ctx.correspond(scan, pose, seed_pose=prev)
    assert _same_bits(seeded, plain), (name, move)
    want = om.correspond(scan, pose, pr, 0, 0, n_threads=8)
    _assert_matches_oracle(seeded, want, pr, (name, move, "seeded"))
    # so_evaluate sees the seeded search's correspondences
    H, g, cost = ctx.evaluate(pose)
    oH, og, ocost, _ = oracle_mod.evaluate(want[0], pose, pr)
    assert np.abs(H - oH).max() <= 1e-10 * np.abs(oH).max() and abs(cost - ocost) <= 1e-10 * ocost
    br = _seed_branches(mp[:, :3], scan, pose, first[0], seeded[0]["status"])
    counts = {k: int(v.sum()) for k, v in br.items()}
    counts["crossed_found5"] = int((br["crossed"] & ~np.isin(seeded[0]["status"], (1, 2, 255))).sum())
    print(f"seed branches {name}/{move}: {counts}")
    key = "crossed_found5" if branch == "crossed" else branch
    assert counts[key] >= minimum, counts
    # a large scan takes the lane search without the switch, and so does the seeded search on it
    if len(scan) > COOP_MAX_QUERIES:
        warp = _ctx(gpu_api, mp, pr)
        assert _same_bits(warp.correspond(scan, pose, seed_pose=prev), plain), (name, move)
        warp.close()
    ctx.close()


def test_seeded_hook_arguments_and_side_effects(gpu_api, monkeypatch):
    import ctypes as C
    case = get_case("tiny")
    ctx = _ctx(gpu_api, case["map_xyzi"], 0.2)
    s = np.ascontiguousarray(case["scan_xyzi"])
    pose = np.ascontiguousarray(case["pose_prior"])
    corr = np.zeros(len(s), gpu_api.CORR_DTYPE)
    p = lambda a: a.ctypes.data_as(C.c_void_p)                           # noqa: E731
    assert ctx.L.so_correspond_seeded(ctx.h, p(s), len(s), 16, 12, p(pose), 0, p(corr), None, None, None) < 0
    assert b"bad args" in ctx.L.so_last_error()
    assert ctx.L.so_correspond_seeded(ctx.h, p(s), 0, 16, 12, p(pose), 0, p(corr), None, None, p(pose)) < 0
    assert b"bad args" in ctx.L.so_last_error()
    big = np.zeros((300000, 4), np.float32)
    with pytest.raises(gpu_api.SuperOdomError):
        ctx.correspond(big, pose, seed_pose=pose)
    # the registered-scan record is invalidated, as by so_correspond
    r = ctx.register(s, pose, 5)
    assert r.status == 0
    ctx.correspond(s, pose, seed_pose=pose)
    with pytest.raises(gpu_api.SuperOdomError):
        ctx.map_add_registered_scan(np.array(r.pose))
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# D. The edge fit's unbounded 10-NN on ties, dense clusters, sparse maps and nearly empty blocks
# ---------------------------------------------------------------------------------------------------------------
def _edge_ctx(api, em):
    mp, _, _ = S.block_face_case()
    ctx = api.Context(max_map_points=1 << 20, max_scan_points=262144, plane_res=0.2)
    ctx.map_set_points(mp)
    ctx.map_set_resolution(S.EDGE_LINE_RES, 0.2)
    ctx.map_set_edge_points(em)
    return ctx


def _brute_d2(map_xyz, q, k):
    """the k smallest distances of every query to the map points of its own block, with the reference's rounding, ascending
    (inf where the block has fewer)"""
    from superodom_b200 import synth
    mb = synth.block_linear(synth.block_of(map_xyz))
    qb = synth.block_linear(synth.block_of(q))
    out = np.full((len(q), k), np.inf, np.float32)
    for i0 in range(0, len(q), 256):
        d = (q[i0:i0 + 256, None, :] - map_xyz[None, :, :]).astype(np.float64)
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]).astype(np.float32)
        d2[mb[None, :] != qb[i0:i0 + 256, None]] = np.inf
        out[i0:i0 + 256] = np.sort(d2, 1)[:, :k] if d2.shape[1] >= k else np.pad(np.sort(d2, 1), ((0, 0), (0, k - d2.shape[1])), constant_values=np.inf)
    return out


@pytest.mark.parametrize("name", list(S.EDGE_SETS))
def test_edge_10nn_on_adversarial_sets(gpu_api, oracle_mod, name):
    from superodom_b200 import synth
    em, q = S.edge_case(name)
    ctx = _edge_ctx(gpu_api, em)
    om = oracle_mod.OracleMap(S.block_face_case()[0])
    om.set_edge_points(em)
    scan = S.xyzi(q)
    for pose in (S.IDENTITY, _translation([0.0625, 0.0, -0.125])):
        gc, ghr = ctx.correspond_edge(scan, pose)
        oc, ohr = om.correspond_edge(scan, pose, S.EDGE_LINE_RES)
        assert np.array_equal(ghr, ohr), (name, ghr, ohr)
        assert np.array_equal(gc["status"].astype(np.int32), oc["status"]), name
        searched = oc["nn"][:, 0] >= 0
        assert np.array_equal(gc["nn"][searched].astype(np.int64), oc["nn"][searched]), name       # all ten, in order
        assert (gc["nn"][~searched] == NONE).all() and (gc["selected_mask"][~searched] == 0).all(), name
        omask = np.zeros(len(oc), np.uint32)
        for j in range(10):
            omask |= np.where(np.arange(10)[None, :] < oc["n_sel"][:, None], (oc["sel"] == j), False).any(1).astype(np.uint32) << np.uint32(j)
        assert np.array_equal(gc["selected_mask"][searched], omask[searched]), name
        ok = oc["status"] == 0
        same = np.abs(gc["a"][ok] - oc["a"][ok]).max(1, initial=0) + np.abs(gc["b"][ok] - oc["b"][ok]).max(1, initial=0)
        swap = np.abs(gc["a"][ok] - oc["b"][ok]).max(1, initial=0) + np.abs(gc["b"][ok] - oc["a"][ok]).max(1, initial=0)
        assert (np.minimum(same, swap) < 1e-7).all() and np.allclose(gc["w"][ok], oc["w"][ok], rtol=1e-9), name
    # coverage, from the exact distances (identity pose: the queries are the set's float32 points)
    d = _brute_d2(em[:, :3], q, 11)
    nb = min(192, int(100.0 / np.sqrt(3.0 * np.float64(np.float32(S.EDGE_LINE_RES)))))
    cs = np.float32(50.0 / nb)
    ring = np.float32(2 * cs) ** 2                                       # R = 2 at lineRes 0.1: the select search's complete radius
    qb = synth.block_linear(synth.block_of(q))
    mb = synth.block_linear(synth.block_of(em[:, :3]))
    cover = {
        "tie_at_10": int(((d[:, 9] == d[:, 10]) | (d[:, 8] == d[:, 9]))[np.isfinite(d[:, 9])].sum()),
        "over_buffer": 0,
        "grown": int((d[:, 9] > ring)[np.isfinite(d[:, 9])].sum()),
        "doubled": int((d[:, 9] > np.float32(4 * cs) ** 2)[np.isfinite(d[:, 9])].sum()),
    }
    fin = np.isfinite(d[:, 9])
    for i0 in range(0, len(q), 256):
        dd = (q[i0:i0 + 256, None, :] - em[None, :, :3]).astype(np.float64)
        dd = (dd ** 2).sum(-1)
        inside = (dd <= d[i0:i0 + 256, 9:10].astype(np.float64) * 1.00001) & (mb[None, :] == qb[i0:i0 + 256, None])
        cover["over_buffer"] += int(((inside.sum(1) > S.KBUF_CAP) & fin[i0:i0 + 256]).sum())
    for count in (9, 10, 11):
        blocks = [b for b in np.unique(mb) if (mb == b).sum() == count]
        cover[f"block_{count}"] = int(np.isin(qb, blocks).sum())
    print(f"edge coverage {name}: {cover}")
    need = {"lattice": ["tie_at_10"], "dense": ["over_buffer"], "sparse": ["grown", "doubled"],
            "small_blocks": ["block_9", "block_10", "block_11"]}[name]
    for k in need:
        assert cover[k] >= 50, (k, cover)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# E. Queries that are not finite or lie far off the grid have no block
# ---------------------------------------------------------------------------------------------------------------
def _check_defective_corr(mixed, clean, bad, what):
    """so_correspond output of a scan with defective rows against the same call without them: the defective rows are
    NOT_ENOUGH_NEIGHBORS with no neighbours, every other row is bit-equal, the histograms differ by the defective count only"""
    mc, mho, mhr = mixed
    cc, cho, chr_ = clean
    assert (mc["status"][bad] == 1).all(), (what, np.unique(mc["status"][bad], return_counts=True))
    assert (mc["nn"][bad] == NONE).all() and (mc["w"][bad] == 0).all(), what
    assert mc[~bad].tobytes() == cc.tobytes(), what
    assert np.array_equal(mho, cho), what
    want = chr_.copy()
    want[1] += int(bad.sum())
    assert np.array_equal(mhr, want), what


@pytest.mark.parametrize("lane", [False, True])
def test_defective_queries_in_the_scan_search(gpu_api, oracle_mod, monkeypatch, lane):
    mp, pr, q = S.block_face_case()
    clean = S.xyzi(q)
    mixed, bad = S.mix_defective(clean, frac=0.02)
    om = oracle_mod.OracleMap(mp)
    ctx = _ctx(gpu_api, mp, pr, lane=lane, monkeypatch=monkeypatch)
    for pose in (S.IDENTITY, _moved(S.IDENTITY, [0.01, 0.0, 0.0], 0.001)):
        got = ctx.correspond(mixed, pose)
        _check_defective_corr(got, ctx.correspond(clean, pose), bad, ("so_correspond", lane))
        _assert_matches_oracle(got, om.correspond(mixed, pose, pr, 0, 0, n_threads=8), pr, ("so_correspond", lane))
        prev = _moved(pose, [0.002, -0.001, 0.0], 1e-4)
        got = ctx.correspond(mixed, pose, seed_pose=prev)
        _check_defective_corr(got, ctx.correspond(clean, pose, seed_pose=prev), bad, ("so_correspond_seeded", lane))
        _assert_matches_oracle(got, om.correspond(mixed, pose, pr, 0, 0, n_threads=8), pr, ("so_correspond_seeded", lane))
    ctx.close()


def test_defective_queries_in_the_edge_search(gpu_api, oracle_mod):
    em, q = S.edge_case("dense")
    clean = S.xyzi(q)
    mixed, bad = S.mix_defective(clean, frac=0.05)
    ctx = _edge_ctx(gpu_api, em)
    om = oracle_mod.OracleMap(S.block_face_case()[0])
    om.set_edge_points(em)
    gc, ghr = ctx.correspond_edge(mixed, S.IDENTITY)
    cc, chr_ = ctx.correspond_edge(clean, S.IDENTITY)
    oc, ohr = om.correspond_edge(mixed, S.IDENTITY, S.EDGE_LINE_RES)
    assert np.array_equal(gc["status"].astype(np.int32), oc["status"]) and np.array_equal(ghr, ohr), (ghr, ohr)
    assert (gc["status"][bad] == 1).all() and (gc["nn"][bad] == NONE).all() and (gc["selected_mask"][bad] == 0).all()
    assert gc[~bad].tobytes() == cc.tobytes()
    want = chr_.copy()
    want[1] += int(bad.sum())
    assert np.array_equal(ghr, want)
    ctx.close()


def test_defective_queries_in_the_knn(gpu_api, oracle_mod):
    import torch
    mp, pr, q = S.block_face_case()
    qs = np.concatenate([q] * 8)                                          # >= 32 768 queries: so_knn orders them by cell first
    for clean in (q, qs):
        mixed, bad = S.mix_defective(clean, frac=0.01)
        om = oracle_mod.OracleMap(mp)
        ctx = _ctx(gpu_api, mp, pr)
        _, _, of = om.knn(mixed, 5, 0)
        assert not of[bad].any()
        for k in (1, 5, 8):
            for b in (0.0, float(np.float32(3 * np.float32(pr)))):
                gi, gd = ctx.knn(mixed, k, b)
                ci, cd = ctx.knn(clean, k, b)
                assert (gi[bad] == NONE).all() and (gd[bad] == 0).all(), (k, b)
                assert np.array_equal(gi[~bad], ci) and np.array_equal(gd[~bad], cd), (k, b)
                dq = torch.from_numpy(np.concatenate([mixed, np.ones((len(mixed), 1), np.float32)], 1)).cuda()
                di = torch.empty((len(mixed), k), dtype=torch.int32, device="cuda")
                dd = torch.empty((len(mixed), k), dtype=torch.float32, device="cuda")
                ctx.knn_device(dq.data_ptr(), len(mixed), k, b, di.data_ptr(), dd.data_ptr())
                torch.cuda.synchronize()
                assert np.array_equal(di.cpu().numpy().view(np.uint32), gi) and np.array_equal(dd.cpu().numpy(), gd), (k, b)
        ctx.close()


@pytest.mark.parametrize("cap", [0, 2000])
def test_defective_points_in_a_registration(gpu_api, oracle_mod, cap):
    case = get_case("cfg1")
    cfg = case["cfg"]
    mixed, bad = S.mix_defective(case["scan_xyzi"], frac=0.01)
    ctx = _ctx(gpu_api, case["map_xyzi"], cfg["plane_res"], max_batch=2)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    ro = om.register(mixed, case["pose_prior"], cfg["plane_res"], cfg["max_iterations"], cap, knn_mode=0, n_threads=8)
    single = ctx.register(mixed, case["pose_prior"], cfg["max_iterations"], cap)
    batch = ctx.register_batch(np.concatenate([mixed, mixed]), [len(mixed)] * 2, np.stack([case["pose_prior"]] * 2), cfg["max_iterations"], cap)
    for r in [single] + list(batch):
        assert r.status == 0 and ro.status == 0
        n = ro.n_iterations
        assert r.n_iterations == n
        assert list(r.iter_n_surf[:n]) == list(ro.iter_n_surf[:n])
        assert list(r.hist_obs) == list(ro.hist_obs) and list(r.hist_reject_plane) == list(ro.hist_reject_plane), \
            (list(r.hist_reject_plane), list(ro.hist_reject_plane))
        pg, po = np.array(r.pose), np.array(ro.pose)
        assert np.abs(pg[:3] - po[:3]).max() <= POSE_TOL_M and quat_angle(pg[3:], po[3:]) <= POSE_TOL_RAD, (pg, po)
    if cap == 0:
        assert ro.hist_reject_plane[1] >= bad.sum()                   # every defective point is NOT_ENOUGH_NEIGHBORS
    ctx.close()

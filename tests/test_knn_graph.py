"""The neighbour graph of the surf store (so_knn.cuh: knn_graph_rank; so_map.cu: k_knn_graph): its rows and radii against an exact
in-block K-NN in numpy, registrations and correspondences bit-equal with the graph forced on and forced off, no stale graph after
the map changes, and the graph actually answering queries.  The certificate and the build rule are tested on the CPU
(tests/cpp/graph_rule_test.cpp)."""
import os
import subprocess

import numpy as np
import pytest

import search_sets as S
from conftest import get_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 0xFFFFFFFF


def test_certificate_and_build_rule_cpu(tmp_path):
    exe = tmp_path / "graph_rule_test"
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cpp", "graph_rule_test.cpp"), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout


def _ctx(api, map_xyzi, plane_res, graph, monkeypatch, **kw):
    """graph: 'on' (built for every search call), 'off' (never used) or None (the build rule); read when the context is made"""
    if graph:
        monkeypatch.setenv("SO_KNN_GRAPH", graph)
    try:
        ctx = api.Context(max_map_points=max(1 << 20, len(map_xyzi) + 1024), max_scan_points=262144, plane_res=plane_res, **kw)
    finally:
        if graph:
            monkeypatch.delenv("SO_KNN_GRAPH")
    ctx.map_set_points(map_xyzi)
    return ctx


def _exact_d2(a, b):
    d = (a[:, None, :] - b[None, :, :]).astype(np.float32).astype(np.float64)       # float32 differences, double squares
    return (d * d).sum(-1).astype(np.float32)


def _block(p):
    return np.floor((p.astype(np.float64) + 25.0) / 50.0).astype(np.int64)


def _check_graph(ctx, map_xyzi, rng, n_check=1500):
    ids, nbr, rad = ctx.knn_graph()
    k = nbr.shape[1]
    assert len(ids) > 0 and k % 4 == 0
    pts = map_xyzi[:, :3].astype(np.float32)
    blk = _block(pts)
    rows = rng.choice(len(ids), min(n_check, len(ids)), replace=False)
    for t in rows:
        a = int(ids[t])
        same = np.flatnonzero((blk == blk[a]).all(1))
        others = same[same != a]
        d2 = _exact_d2(pts[a:a + 1], pts[others])[0]
        order = np.lexsort((others, d2))                                              # (d2, id)
        want = others[order[:k]]
        # the row's own search ranks a first among its coincident duplicates only when its id is the smallest of them
        dup_before = np.count_nonzero((d2 == 0) & (others < a))
        if len(others) <= k:
            assert rad[t] == np.inf and sorted(nbr[t][nbr[t] != NONE].tolist()) == sorted(want.tolist()), t
        elif dup_before + 1 > k:
            assert rad[t] == 0, t
        else:
            assert np.array_equal(nbr[t].astype(np.int64), want), (t, nbr[t], want)
            assert rad[t] == np.float32(np.float32(0.99999) * np.sqrt(d2[order[k - 1]])), (t, rad[t])
    return ids, nbr, rad


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lattice", "dense", "block_face", "sparse", "small_blocks"])
def test_graph_rows_and_radii_against_numpy(gpu_api, monkeypatch, name):
    if name in ("sparse", "small_blocks"):
        e = S.edge_sparse() if name == "sparse" else S.edge_small_blocks()
        mp, pr = (e[0] if isinstance(e, tuple) else e), 0.2
    else:
        mp, pr, _ = S.surf_case(name)
    mp = np.asarray(mp, np.float32)
    if mp.shape[1] == 3:
        mp = S.xyzi(mp)
    ctx = _ctx(gpu_api, mp, pr, "on", monkeypatch)
    _check_graph(ctx, mp, np.random.default_rng(3))
    ctx.close()


def _fields(results):
    """every result field except the wall-clock times"""
    out = []
    for r in results:
        out.append((bytes(memoryview(r.pose_opt).cast("B")), r.status, r.n_iterations, list(r.iter_n_surf), list(r.iter_cost), list(r.cov),
                    list(r.iter_dtrans), list(r.iter_drot), list(r.hist_obs), list(r.hist_reject_plane)))
    return out


def _batch(case_names, n_each):
    scans, poses = [], []
    for name in case_names:
        for i in range(n_each):
            c = get_case(name, i)
            scans.append(c["scan_xyzi"])
            poses.append(c["pose_prior"])
    return scans, np.array(poses)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny", "cfg1", "cfg2"])
def test_registration_same_bits_with_graph_on_and_off(gpu_api, monkeypatch, name):
    scans, poses = _batch([name], 3)
    cfg = get_case(name)["cfg"]
    mp = get_case(name)["map_xyzi"]
    # non-finite and far-off points in the first scan
    bad = S.defective_points(64)
    scans[0] = np.concatenate([scans[0], S.xyzi(bad) if bad.shape[1] == 3 else bad]).astype(np.float32)
    flat = np.ascontiguousarray(np.concatenate(scans), np.float32)
    n_points = np.array([len(s) for s in scans], np.uint32)
    res = {}
    for mode in ("on", "off"):
        ctx = _ctx(gpu_api, mp, cfg["plane_res"], mode, monkeypatch, max_batch=8)
        ctx.knn_graph_stats(True)
        batch = ctx.register_batch(flat, n_points, poses, cfg["max_iterations"], cfg["max_surface_features"])
        single = ctx.register(scans[1], poses[1], cfg["max_iterations"], cfg["max_surface_features"])
        st = ctx.knn_graph_stats(False)
        res[mode] = (_fields(batch), _fields([single]), st)
        ctx.close()
    assert res["on"][0] == res["off"][0] and res["on"][1] == res["off"][1]
    assert res["off"][2][:, 1].sum() == 0
    assert res["on"][2][:, 1].sum() > 0, res["on"][2][:4]                             # the graph answered queries


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lattice", "dense", "block_face"])
def test_correspond_same_bits_with_graph_on_and_off(gpu_api, monkeypatch, name):
    mp, pr, q = S.surf_case(name)
    scan, _ = S.mix_defective(S.xyzi(q))
    scan = np.concatenate([scan] * (8192 // len(scan) + 1))                           # > 8 192 points: the lane-per-query search
    got = {}
    for mode in ("on", "off"):
        ctx = _ctx(gpu_api, mp, pr, mode, monkeypatch)
        ctx.knn_graph_stats(True)
        a = ctx.correspond(scan, S.IDENTITY)
        b = ctx.correspond(scan, np.array([0.03, -0.02, 0.01, 0, 0, 0, 1.0]), seed_pose=S.IDENTITY)
        got[mode] = (a, b, ctx.knn_graph_stats(False))
        ctx.close()
    for x, y in zip(got["on"][:2], got["off"][:2]):
        assert all(u.tobytes() == v.tobytes() for u, v in zip(x, y)), name
    assert got["on"][2][:, 1].sum() > 0


@pytest.mark.gpu
def test_no_stale_graph_after_the_map_changes(gpu_api, monkeypatch):
    c0, c1 = get_case("tiny", 0), get_case("tiny", 1)
    cfg = c0["cfg"]
    out = {}
    for mode in ("on", "off"):
        ctx = _ctx(gpu_api, c0["map_xyzi"], cfg["plane_res"], mode, monkeypatch)
        r0 = ctx.register(c0["scan_xyzi"], c0["pose_prior"], cfg["max_iterations"])
        g0 = ctx.knn_graph()[2].copy() if mode == "on" else None
        ctx.map_add_scan(c0["scan_xyzi"], np.array(r0.pose_opt))                    # insert: the index and the sorted order change
        r1 = ctx.register(c1["scan_xyzi"], c1["pose_prior"], cfg["max_iterations"])
        if mode == "on":
            ids, nbr, rad = ctx.knn_graph()
            assert len(rad) != len(g0) or not np.array_equal(rad, g0)
        ctx.map_set_points(c0["map_xyzi"][::2])                                       # replace the map
        r2 = ctx.register(c1["scan_xyzi"], c1["pose_prior"], cfg["max_iterations"])
        out[mode] = _fields([r0, r1, r2])
        ctx.close()
    assert out["on"] == out["off"]


@pytest.mark.gpu
def test_build_rule_builds_for_large_calls_only(gpu_api, monkeypatch):
    """Without the switch: a call of fewer queries than 8 x the map's points searches without the graph, a larger one builds it."""
    c = get_case("tiny")
    cfg = c["cfg"]
    mp = c["map_xyzi"]
    scan = c["scan_xyzi"]
    ctx = _ctx(gpu_api, mp, cfg["plane_res"], None, monkeypatch, max_batch=64)
    ctx.knn_graph_stats(True)
    ctx.register(scan, c["pose_prior"], cfg["max_iterations"])
    assert ctx.knn_graph_stats(True)[:, 1].sum() == 0
    reps = int(np.ceil(8 * len(mp) / len(scan))) + 1
    assert reps <= 64
    flat = np.ascontiguousarray(np.concatenate([scan] * reps), np.float32)
    ctx.register_batch(flat, np.full(reps, len(scan), np.uint32), np.tile(c["pose_prior"], (reps, 1)), cfg["max_iterations"])
    assert ctx.knn_graph_stats(False)[:, 1].sum() > 0
    ctx.close()

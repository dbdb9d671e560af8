"""Loop verification on the device (so_loop_verify): equal to the manual sequence it replaces and to the existing calls that define its
scores, deterministic, per candidate, and leaving the keyframe context alone; its decisions on the loop scenarios of
test_loop_detection.py (true revisits accepted, look-alike places rejected); its argument errors; and the shim's loop closure."""
import functools
import math
import subprocess

import numpy as np
import pytest

from conftest import get_case
from test_keyframes import _compose, _ctx, _err, _inverse
from test_loop_detection import LOOP_OPTS, _closure, _drive, _heading, _loop_scans, _loop_truth, _scans, _wrap

SO_ERR_ARG = -1
VLP16 = dict(el_res_deg=2.0, el_min_deg=-16.0, el_max_deg=16.0)


def _opts(api, **kw):
    return api.loop_verify_opts(image=VLP16, **kw)


def _bytes(api, res):
    """A result's bytes with its timings zeroed (everything else must repeat bit for bit)."""
    out = []
    for r in res:
        c = api.LoopVerifyResult.from_buffer_copy(r)
        c.time_ms = 0.0
        c.reg.time_ms = 0.0
        c.reg.time_total_ms = 0.0
        out.append(bytes(c))
    return out


def _true_rel_err(rel7, truth, c, q):
    e = _compose(_inverse(_compose(_inverse(truth[c]), truth[q])), np.asarray(rel7))
    return float(np.linalg.norm(e[:3])), abs(_wrap(_heading(e)))


@functools.lru_cache(maxsize=None)
def _aisle_truth():
    """A straight path along the aisle between two shelving rows (rows every 5 m at y = 3 and 8): the look-alike case of DESIGN.md,
    "Loop detection", where false matches reach distance 0.17."""
    from superodom_b200 import synth
    scene = get_case("cfg2", 0)["scene"]
    out = []
    for i in range(45):
        p = np.array([-20.0 + 0.9 * i, 5.5, 0.0])
        for dy in (0.0, 0.5, -0.5, 1.0, -1.0):
            if scene.free(p + [0.0, dy, 0.0]):
                p = p + [0.0, dy, 0.0]
                break
        out.append(np.r_[p, synth.quat_from_rotvec(np.zeros(3))])
    return np.array(out)


def _report(tag, truth, res):
    for r in res:
        if r.skipped:
            continue
        d = float(np.linalg.norm(truth[r.id, :3] - truth[r.query, :3]))
        print(f"{tag}: q {r.query} id {r.id} true dist {d:.2f} m status {r.reg.status} overlap {r.overlap:.3f} rmse {r.rmse:.3f} "
              f"conflict q {r.conflict_query:.4f} ({r.n_conflict_query}/{r.n_cand_query}) map {r.conflict_map:.4f} "
              f"({r.n_conflict_map}/{r.n_cand_map}) accepted {r.accepted} {r.time_ms:.2f} ms")


# ------------------------------------------------------------------------------------------------------------- 1. equalities
@pytest.mark.gpu
def test_equals_the_calls_that_define_it(gpu_api):
    api = gpu_api
    scene, truth, est, q, off, ctx, true_near = _closure(api, False)
    cands = ctx.loop_candidates([q], 5, **LOOP_OPTS)[0]
    o = _opts(api)
    scratch = _ctx(api)
    res = ctx.loop_verify(scratch, cands, o)
    poses = ctx.keyframe_poses()
    bound = np.float32(np.float64(o.inlier_dist) ** 2)
    for cand, r in zip(cands, res):
        c = int(cand["id"])
        assert (r.query, r.id, r.skipped) == (q, c, 0)
        ids = [i for i in range(c - 2, c + 3) if 0 <= i < q - 30]
        sub = _ctx(api)
        sub.map_set_origin(poses[c][:3])
        sub.map_from_keyframes(ctx, ids, poses[ids], 1)
        prior = api.loop_prior(poses[c], poses[q], float(cand["yaw"]))
        assert np.array_equal(prior, ctx.loop_prior(cand))
        reg = sub.register_keyframes(ctx, [q], [prior], 20, 0)[0]
        for f in ("pose", "pose_opt", "cov", "iter_cost", "hist_obs", "hist_reject_plane"):
            assert bytes(getattr(reg, f)) == bytes(getattr(r.reg, f)), f
        assert (reg.status, reg.n_iterations, reg.pos_inv_cond) == (r.reg.status, r.reg.n_iterations, r.reg.pos_inv_cond)
        assert r.n_submap_keyframes == len(ids) and r.n_submap_points == sub.map_size()
        assert np.allclose(r.rel7, _compose(_inverse(poses[c]), np.array(reg.pose)), atol=1e-12)
        # overlap: so_knn(k = 1, max_d2 = inlier_dist^2) of the query at reg.pose
        pts = ctx.keyframe_download(q, 0, np.array(reg.pose))
        pts = pts[np.isfinite(pts[:, :3]).all(axis=1)]
        idx, d2 = sub.knn(pts[:, :3], 1, float(bound))
        hit = idx[:, 0] != 0xFFFFFFFF
        assert r.n_query_points == len(pts) and r.n_inliers == int(hit.sum())
        assert r.overlap == r.n_inliers / r.n_query_points
        assert math.isclose(r.rmse, math.sqrt(d2[hit, 0].astype(np.float64).sum() / hit.sum()), rel_tol=1e-12)
        # the map conflict: so_map_clear_free_space of the query at reg.pose on this copy of the submap
        fs = sub.map_clear_free_space(ctx.keyframe_download(q, 0), np.array(reg.pose), api.free_space(**VLP16), stores=1)
        assert (r.n_conflict_map, r.n_cand_map) == (fs["n_removed"], fs["n_candidates"])
        # the query conflict: so_map_clear_free_space_keyframes over the submap ids, on a map of the aligned query points
        t = _ctx(api)                                                  # the default window, centred on the world origin, holds them all
        t.map_set_points(pts)
        assert t.map_size() == len(pts)
        fk = t.map_clear_free_space_keyframes(ctx, ids, poses[ids], api.free_space(**VLP16), stores=1)
        assert (r.n_conflict_query, r.n_cand_query) == (fk["n_removed"], fk["n_candidates"])
        assert r.conflict_query == (r.n_conflict_query / r.n_cand_query if r.n_cand_query else 0.0)
        assert r.conflict_map == (r.n_conflict_map / r.n_cand_map if r.n_cand_map else 0.0)
        assert r.time_ms > 0
        sub.close()
        t.close()
    _report("drift", truth, res)
    # two calls give the same bytes; k candidates in one call equal k calls of one
    again = ctx.loop_verify(scratch, cands, o)
    assert _bytes(api, res) == _bytes(api, again)
    one = [ctx.loop_verify(scratch, cands[i:i + 1], o)[0] for i in range(len(cands))]
    assert _bytes(api, res) == _bytes(api, one)
    scratch.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------------------- 2. decisions
@pytest.mark.gpu
@pytest.mark.parametrize("reverse", [False, True])
def test_true_revisits_accepted(gpu_api, reverse):
    scene, truth, est, q, off, ctx, true_near = _closure(gpu_api, reverse)
    cands = ctx.loop_candidates([q], 5, **LOOP_OPTS)[0]
    scratch = _ctx(gpu_api)
    res = ctx.loop_verify(scratch, cands, _opts(gpu_api))
    _report("reverse" if reverse else "forward", truth, res)
    best = res[0]
    assert abs(best.id - true_near) <= 1 and best.accepted
    for r in res:
        if r.accepted:
            t_err, y_err = _true_rel_err(r.rel7, truth, r.id, q)
            print(f"  accepted {r.id}: {t_err:.3f} m, {math.degrees(y_err):.3f} deg from the true relative pose")
            assert t_err < 0.3 and y_err < math.radians(1.0)
    scratch.close()
    ctx.close()


def _no_false_loop(api, tag, truth, scans):
    ctx = _drive(api, get_case("cfg2", 0)["scene"], truth, truth, 7000, scans)
    scratch = _ctx(api)
    qs = np.arange(31, len(truth))
    cands = ctx.loop_candidates(qs, 5, **LOOP_OPTS)
    res = ctx.loop_verify(scratch, cands, _opts(api))
    _report(tag, truth, res)
    checked = 0
    for r in res:
        if r.skipped:
            continue
        checked += 1
        if np.linalg.norm(truth[r.id, :3] - truth[r.query, :3]) > 3.0:
            assert not r.accepted, (tag, r.query, r.id)
        elif r.accepted:
            t_err, y_err = _true_rel_err(r.rel7, truth, r.id, r.query)
            assert t_err < 0.3 and y_err < math.radians(1.0)
    assert checked == sum(int(c["id"]) >= 0 for c in cands.reshape(-1))
    print(f"{tag}: {checked} candidates checked, min distance {cands['distance'][cands['id'] >= 0].min():.3f}")
    scratch.close()
    ctx.close()


@pytest.mark.gpu
def test_no_loop_path_rejected(gpu_api):
    """The first 45 keyframes of the loop (half way round, never revisiting): every candidate is a false loop."""
    _no_false_loop(gpu_api, "no loop", _loop_truth(False)[:45], _loop_scans(False)[:45])


@pytest.mark.gpu
def test_aisle_path_rejected(gpu_api):
    """A straight aisle between look-alike shelving rows, where Scan Context distances of false matches are smallest."""
    truth = _aisle_truth()
    _no_false_loop(gpu_api, "aisle", truth, _scans(get_case("cfg2", 0)["scene"], truth, 9100))


# ------------------------------------------------------------------------------------------------------------- 3. nothing else changes
@pytest.mark.gpu
def test_keyframe_context_unchanged(gpu_api):
    truth = _loop_truth(False)
    outs = []
    for verify in (False, True):
        ctx = _drive(gpu_api, get_case("cfg2", 0)["scene"], truth, truth, 7000, _loop_scans(False))
        q = len(truth) - 1
        cands = ctx.loop_candidates([q], 3, **LOOP_OPTS)[0]
        if verify:
            scratch = _ctx(gpu_api)
            ctx.loop_verify(scratch, cands, _opts(gpu_api))
            scratch.close()
        desc = ctx.keyframe_descriptors(np.arange(q + 1), **LOOP_OPTS)
        again = ctx.loop_candidates([q], 3, stats=True, **LOOP_OPTS)
        ctx.map_add_registered_scan(ctx.keyframe_poses()[q])
        outs.append((ctx.map_download(0).tobytes(), ctx.keyframe_poses().tobytes(), desc.tobytes(), again[0].tobytes(),
                     again[1]["n_described"], ctx.keyframe_info(), [ctx.keyframe_download(i, 0).tobytes() for i in (0, q)]))
        ctx.close()
    assert outs[0] == outs[1]


# ------------------------------------------------------------------------------------------------------------- 4. errors
@pytest.mark.gpu
def test_argument_errors_before_device_work(gpu_api):
    api = gpu_api
    from test_loop_detection import _random_polar, _store, IDENT
    import loop_detection_numpy as LD
    o = LD.Opts(rings=4, sectors=8, max_range=8.0)
    ctx = _store(api, [_random_polar(o, k) for k in range(6)], [IDENT] * 6)
    scratch = _ctx(api)
    bare = _ctx(api)
    cand = np.zeros(1, api.LOOP_CANDIDATE_DTYPE)
    cand[0]["query"], cand[0]["id"] = 5, 0
    good = dict(exclude_recent=2)
    for c in (ctx, scratch, bare):
        c.kernel_launches(reset=True)
    assert _err(api, lambda: ctx.loop_verify(ctx, cand, **good)) == SO_ERR_ARG                 # scratch == ctx
    assert _err(api, lambda: bare.loop_verify(scratch, cand, **good)) == SO_ERR_ARG            # no keyframe store
    for q, i in ((6, 0), (-1, 0), (5, 6), (5, -2), (5, 5), (5, 3), (2, 0)):                   # ids: held, -1 only, distinct, eligible
        bad = cand.copy()
        bad[0]["query"], bad[0]["id"] = q, i
        assert _err(api, lambda: ctx.loop_verify(scratch, bad, **good)) == SO_ERR_ARG, (q, i)
    bad_opts = [dict(half_window=-1), dict(half_window=9), dict(exclude_recent=-1), dict(id_begin=-1, id_end=3), dict(id_begin=3, id_end=2),
                dict(id_begin=0, id_end=7), dict(icp=dict(max_icp_iters=0)), dict(icp=dict(max_icp_iters=33)), dict(inlier_dist=0.0),
                dict(inlier_dist=float("nan")), dict(inlier_dist=float("inf")), dict(inlier_dist=1e30), dict(min_overlap=-0.1),
                dict(min_overlap=1.5), dict(max_conflict=float("nan")), dict(image=dict(dilate=5)), dict(image=dict(az_res_deg=0.0)),
                dict(image=dict(az_res_deg=0.01, el_res_deg=0.05, el_min_deg=-40.0, el_max_deg=40.0))]
    for kw in bad_opts:
        assert _err(api, lambda: ctx.loop_verify(scratch, cand, **dict(good, **kw))) == SO_ERR_ARG, kw
    for c in (ctx, scratch, bare):
        assert c.kernel_launches() == 0
    # an unused slot: skipped, nothing launched; the range form accepts what the default form refuses
    skip = cand.copy()
    skip[0]["id"] = -1
    r = ctx.loop_verify(scratch, skip, **good)[0]
    assert r.skipped == 1 and r.query == 5 and r.id == -1 and r.accepted == 0 and r.n_query_points == 0
    assert scratch.kernel_launches() == 0 and ctx.kernel_launches() == 0
    assert ctx.loop_verify(scratch, cand[:0], **good) == []
    r = ctx.loop_verify(scratch, cand, **good)[0]
    assert r.skipped == 0 and r.n_submap_keyframes == 3 and scratch.kernel_launches() > 0
    wide = cand.copy()
    wide[0]["id"] = 4
    r = ctx.loop_verify(scratch, wide, id_begin=2, id_end=6, half_window=1)[0]
    assert r.n_submap_keyframes == 2                                   # ids 3 and 4: the query 5 is never in its submap
    for c in (ctx, scratch, bare):
        c.close()


# ------------------------------------------------------------------------------------------------------------- 5. shim
@pytest.mark.gpu
def test_loop_verify_shim_closes_the_loop(gpu_api, tmp_path):
    """tests/cpp/loop_verify_test.cpp on the drifted loop: loopCandidates -> verifyLoop -> optimizeKeyframes -> rebuildFromKeyframes."""
    from test_cpp_shim import _build
    from test_sessions_cpu import _file
    scene, truth, est, q, off, ctx, true_near = _closure(gpu_api, False)
    frames = [(est[i], ctx.keyframe_download(i, 0), np.zeros((0, 4), np.float32)) for i in range(q + 1)]
    ctx.close()
    path = tmp_path / "session.bin"
    path.write_bytes(_file(frames))
    exe = _build(tmp_path, "loop_verify_test")
    out = subprocess.run([exe, str(path), str(q)], capture_output=True, text=True)
    print(out.stdout[:3000])
    assert out.returncode == 0, out.stderr
    lines = [ln.split() for ln in out.stdout.strip().splitlines()]
    loop = [int(ln[1]) for ln in lines if ln[0] == "loop"][0]
    assert abs(loop - true_near) <= 1
    v = [ln for ln in lines if ln[0] == "verify" and int(ln[1]) == loop][0]
    rel = np.array([float(x) for x in v[8:15]])
    t_err, y_err = _true_rel_err(rel, truth, loop, q)
    assert t_err < 0.3 and y_err < math.radians(1.0)
    opt = np.array([[float(x) for x in ln[2:]] for ln in lines if ln[0] == "pose"])
    before = np.linalg.norm(est[:, :3] - truth[:, :3], axis=1)
    after = np.linalg.norm(opt[:, :3] - truth[:, :3], axis=1)
    print(f"shim: keyframe error mean {before.mean():.3f} -> {after.mean():.3f} m, max {before.max():.3f} -> {after.max():.3f} m")
    assert after.mean() < 0.6 * before.mean() and after.max() < 0.7 * before.max()
    assert int([ln for ln in lines if ln[0] == "map"][0][1]) > 1000

"""so_pose_graph_solve on the device against the restatements in pose_graph_numpy.py (the dense solve_full and the exact sparse step),
the preconditioner's exactness on chain graphs, a graph with a direction no edge observes, the Cauchy loss against a false loop
closure, run-to-run determinism, and the drifted loop of tests/test_keyframes.py closed with the device solve."""
import numpy as np
import pytest

import pose_graph_numpy as PG
import test_ceres_restatement as CR
import trust_region_sets as TRS


def _ctx(api):
    return api.Context(max_map_points=1 << 20, max_scan_points=1 << 16)


def _family(rng, name, n):
    if name == "chain":
        return PG.drifted(rng, n, loops=0, drift=(0.05, 0.01))
    if name == "loop":
        return PG.drifted(rng, n, loops=1, drift=(0.05, 0.01))
    if name == "loops":
        return PG.drifted(rng, n, loops=max(2, n // 3), drift=(0.1, 0.03))
    if name == "dup":
        return PG.drifted(rng, n, loops=1, dup=True, drift=(0.05, 0.01))
    if name == "full":
        return PG.drifted(rng, n, loops=2, full_info=True, drift=(0.05, 0.01))
    if name == "rankdef":
        return PG.drifted(rng, n, loops=2, full_info=True, rank_def=True, drift=(0.05, 0.01))
    if name == "cauchy":
        return PG.drifted(rng, n, loops=2, false_loops=1, cauchy=1.0, drift=(0.1, 0.03))
    if name == "far":                                                   # large drift: the model over-predicts, steps are rejected
        return PG.drifted(rng, n, loops=2, drift=(0.4, 0.25))
    if name == "exact":                                                 # start at the truth of exact measurements: g = 0
        init, edges, truth = PG.drifted(rng, n, loops=1, noise=(0.0, 0.0), drift=(0.0, 0.0), sqrt_info=np.r_[50, 50, 50, 200, 200, 200.0])
        return truth, edges, truth
    raise ValueError(name)


FAMILIES = ("chain", "loop", "loops", "dup", "full", "rankdef", "cauchy", "far", "exact")


def _compare(api, ctx, init, edges, fixed, iters, sparse, stats):
    E = PG.to_array(edges)
    prob = PG.PoseGraph(init, E, fixed)
    ref = (PG.solve_sparse if sparse else CR.solve_full)(prob, prob.x0(), iters)
    if not TRS.fair(ref, max_radius_error=1e-10 if not sparse else np.inf):
        stats["unfair"] += 1
        return None
    X, r = ctx.pose_graph_solve(init, E, fixed=fixed, max_iterations=iters)
    Xr = prob.nodes(ref["x"])
    assert (r["iterations"], r["successful"], r["unsuccessful"], r["termination"]) == \
        (ref["iterations"], ref["successful"], ref["unsuccessful"], ref["termination"]), (r, ref["steps"])
    # relative to the value, with floors for the "exact" family, whose cost and gmax are rounding of zero (a 1e-20 floor on the cost
    # measured 3.2e-5 there)
    rel = lambda a, b, floor: abs(a - b) / max(abs(b), floor)
    stats["cost"] = max(stats["cost"], rel(r["final_cost"], ref["final_cost"], 1e-12), rel(r["initial_cost"], ref["initial_cost"], 1e-12))
    stats["gmax"] = max(stats["gmax"], rel(r["gmax"], ref["gmax"], 1e-9))
    stats["pose"] = max(stats["pose"], np.abs(X - Xr).max())
    stats["terms"].add(r["termination"])
    stats["rejected"] += "r" in ref["steps"]
    stats["n"] += 1
    return r


def _check(stats, what, cost_tol, pose_tol, gmax_tol):
    print(f"{what}: {stats['n']} solves compared ({stats['unfair']} near a threshold skipped), exits {sorted(stats['terms'])}, "
          f"solves with a rejected step {stats['rejected']}; max relative cost {stats['cost']:.2e}, gmax {stats['gmax']:.2e}, "
          f"max pose difference {stats['pose']:.2e}")
    assert stats["cost"] <= cost_tol and stats["pose"] <= pose_tol
    # gmax is the gradient at the final iterate: near a minimum it is a small difference of large terms, so its relative error is the
    # pose error times the largest information over gmax, not rounding of gmax itself (measured 4.2e-3 dense, 2.25e-3 sparse)
    assert stats["gmax"] <= gmax_tol


def _stats():
    return dict(n=0, unfair=0, cost=0.0, gmax=0.0, pose=0.0, terms=set(), rejected=0)


@pytest.mark.gpu
def test_against_the_dense_restatement(gpu_api):
    ctx = _ctx(gpu_api)
    st = _stats()
    rng = np.random.default_rng(1)
    for fam in FAMILIES:
        for n in (2, 3, 4, 5, 7, 8, 9):
            for iters in (50, 3):
                init, edges, _ = _family(rng, fam, n)
                fixed = int(rng.integers(0, n)) if n > 3 and rng.integers(0, 2) else 0
                _compare(gpu_api, ctx, init, edges, fixed, iters, False, st)
    # bounds: three times the measured values (cost 1.06e-9: PCG's step against the dense QR's last bits; poses 1.3e-10)
    _check(st, "dense", cost_tol=3e-9, pose_tol=1e-8, gmax_tol=1.3e-2)
    # every exit these families reach: 0 (iteration limit), 1 (gradient), 2 (parameter), 3 (function); 4 and 5 need a radius of 1e-32
    # or five invalid steps in a row, which no family here produces
    assert {0, 1, 2, 3} <= st["terms"] and st["rejected"] > 0
    ctx.close()


@pytest.mark.gpu
def test_against_the_sparse_restatement(gpu_api):
    ctx = _ctx(gpu_api)
    st = _stats()
    rng = np.random.default_rng(2)
    for n, loops, fam in ((1023, 20, "loops"), (1024, 0, "chain"), (1025, 50, "cauchy"), (1000, 100, "loops"), (10000, 100, "loops")):
        init, edges, _ = PG.drifted(rng, n, loops=loops, false_loops=5 if fam == "cauchy" else 0, cauchy=1.0 if fam == "cauchy" else 0.0,
                                    drift=(0.05, 0.01))
        _compare(gpu_api, ctx, init, edges, int(rng.integers(0, n)), 50, True, st)
    # identical decisions, but not the 1e-9 / 1e-8 of the small graphs: PCG's step differs from the exact one by up to kPcgTol
    # (1e-10) relative in the preconditioner's norm, and on the 10 000-node chain 50 iterations that end at the iteration limit carry
    # that difference along the trajectory.  Bounds: three times the measured cost 7.3e-5 relative, poses 1.1e-4, gmax 2.25e-3
    _check(st, "sparse", cost_tol=2.2e-4, pose_tol=3.3e-4, gmax_tol=6.8e-3)
    ctx.close()


@pytest.mark.gpu
def test_chain_graphs_take_one_pcg_iteration_per_trial(gpu_api):
    """The preconditioner is the whole system of a graph of consecutive edges (duplicates included): PCG ends after one iteration on
    short chains.  On chains of 1 000 nodes and more the damped system's condition number times machine epsilon exceeds the stopping
    tolerance (1e-10) late in the solve, when the radius is large, so a trial can take a second iteration that only removes rounding
    (measured at n = 1024: 42 PCG iterations over 31 trials); there the bound is two per trial."""
    ctx = _ctx(gpu_api)
    rng = np.random.default_rng(4)
    for n in (2, 3, 17, 1024, 1025, 5000):
        init, edges, _ = PG.drifted(rng, n, loops=0, dup=n % 2 == 1, drift=(0.05, 0.01))
        _, r = ctx.pose_graph_solve(init, edges, fixed=int(rng.integers(0, n)))
        print(f"chain n={n}: {r['iterations']} trust-region iterations, {r['pcg_iterations']} PCG iterations")
        assert r["iterations"] > 0
        if n <= 17:
            assert r["pcg_iterations"] == r["iterations"], (n, r)
        else:
            assert r["iterations"] <= r["pcg_iterations"] <= 2 * r["iterations"], (n, r)
    ctx.close()


@pytest.mark.gpu
def test_results_are_bit_identical_run_to_run(gpu_api):
    ctx = _ctx(gpu_api)
    rng = np.random.default_rng(6)
    init, edges, _ = PG.drifted(rng, 3000, loops=200, false_loops=10, cauchy=1.0, drift=(0.05, 0.01))
    a = ctx.pose_graph_solve(init, edges, weights=True)
    b = ctx.pose_graph_solve(init, edges, weights=True)
    scan = np.random.default_rng(0).uniform(-20, 20, (4000, 4)).astype(np.float32)      # a registration, keyframes and a loop search
    ctx.map_set_points(scan)                                                             # in between
    ctx.keyframe_reserve(1 << 16, 8)
    for k in range(3):
        ctx.register(scan, np.r_[0.1 * k, 0, 0, 0, 0, 0, 1.0], 3, 0)
        ctx.keyframe_add_registered(np.r_[0.1 * k, 0, 0, 0, 0, 0, 1.0])
    ctx.loop_candidates([2], 1, exclude_recent=0)
    c = ctx.pose_graph_solve(init, edges, weights=True)
    for o in (b, c):
        assert a[0].tobytes() == o[0].tobytes() and a[2].tobytes() == o[2].tobytes()
        assert {k: v for k, v in a[1].items() if k != "time_ms"} == {k: v for k, v in o[1].items() if k != "time_ms"}
    ctx.close()


@pytest.mark.gpu
def test_unobserved_direction(gpu_api):
    """Edges whose S leaves a direction unobserved (zero rows: here no edge constrains yaw or z), which so_pose_graph_check accepts:
    late in a solve the damping falls to diag / 1e16 and a cyclic-reduction pivot can lose positivity to rounding in one thread's rows
    only.  The solve must end with a termination code and finite poses, and the same outputs on a second call."""
    ctx = _ctx(gpu_api)
    rng = np.random.default_rng(8)
    for n in (9, 300):
        init, edges, _ = PG.drifted(rng, n, loops=n // 5, drift=(0.05, 0.01))
        planar = [(i, j, z, S * np.r_[1, 1, 0, 1, 1, 0][:, None], c) for i, j, z, S, c in edges]
        gpu_api.pose_graph_check(n, PG.to_array(planar))
        a = ctx.pose_graph_solve(init, planar)
        b = ctx.pose_graph_solve(init, planar)
        print(f"unobserved direction, n={n}: {a[1]['iterations']} iterations, termination {a[1]['termination']}")
        assert np.isfinite(a[0]).all() and a[1]["termination"] in (0, 1, 2, 3, 4, 5)
        assert a[0].tobytes() == b[0].tobytes()
        if n < 10:                                                      # the dense restatement takes the same decisions
            prob = PG.PoseGraph(init, PG.to_array(planar))
            ref = CR.solve_full(prob, prob.x0(), 50)
            if TRS.fair(ref):
                assert (a[1]["iterations"], a[1]["termination"]) == (ref["iterations"], ref["termination"])
    ctx.close()


@pytest.mark.gpu
def test_cauchy_rejects_a_false_loop(gpu_api):
    """A 500-node drifted walk (1.42 m mean position error) with one true closure (first to last keyframe) and one false one (Z =
    identity between keyframes 23.7 m apart); loop edges sigma 0.1 m / 0.01 rad.  Measured: Cauchy c = 10 ends at 0.389 m mean error,
    the false edge's rho' 9.8e-4 and the true edge's 0.999; without a loss the false edge bends the walk to 10.8 m.  c = 5 to 20 behave
    alike (0.41 to 0.51 m); c = 40 lets the false edge pull (2.1 m)."""
    ctx = _ctx(gpu_api)
    rng = np.random.default_rng(5)
    n = 500
    init, edges, truth = PG.drifted(rng, n, loops=0, drift=(0.03, 0.004))
    si = np.r_[np.full(3, 1 / 0.1), np.full(3, 1 / 0.01)]
    true_z = PG.compose(PG.inverse(truth[0]), truth[n - 1])
    false_z = np.r_[0, 0, 0, 0, 0, 0, 1.0]
    err = lambda X: float(np.linalg.norm(X[:, :3] - truth[:, :3], axis=1).mean())
    out = {}
    for c in (10.0, 0.0):
        e = edges + [PG.edge(0, n - 1, true_z, si, c), PG.edge(100, 350, false_z, si, c)]
        X, r, w = ctx.pose_graph_solve(init, e, weights=True)
        out[c] = (err(X), w[-2], w[-1])
        print(f"cauchy {c}: mean position error {out[c][0]:.3f} m (start {err(init):.3f} m), true edge rho' {w[-2]:.3g}, "
              f"false edge rho' {w[-1]:.3g}, {r['iterations']} iterations, termination {r['termination']}")
    assert out[10.0][2] < 0.01 and out[10.0][1] > 0.9
    assert out[10.0][0] < 0.6                                           # 1.5 x the measured 0.389 m
    assert out[0.0][0] > 5.0                                            # measured 10.8 m
    ctx.close()


@pytest.mark.gpu
def test_loop_closure_end_to_end_on_the_device(gpu_api):
    """The drifted loop of tests/test_keyframes.py::test_loop_closure_end_to_end, closed with so_pose_graph_solve in place of the scipy
    helper: the same edges, the same error, map and next-registration bounds; poses against the dense restatement as in the
    comparisons above, and the largest difference from the helper's solution printed."""
    from superodom_b200 import synth
    from test_keyframes import _ctx as kf_ctx, _loop_poses, _compose, _inverse, _pose_graph, _share_far
    from conftest import get_case
    scene = get_case("cfg2", 0)["scene"]
    n_max, mf = 60, 0
    truth = _loop_poses(scene, n_max, 16.0)
    drift = np.r_[0.02, 0.01, 0.0, 0.0, 0.0, 0.0, 1.0]
    ctx = kf_ctx(gpu_api)
    ctx.map_set_origin(truth[0][:3])
    ctx.keyframe_reserve(n_max << 15, n_max)
    est = [truth[0]]
    ctx.register(synth.make_scan(scene, "vlp16", truth[0], 5000, rmax=20.0), truth[0], 10, mf)
    ctx.keyframe_add_registered(truth[0])
    ctx.map_add_registered_scan(truth[0])
    n = n_max
    for i in range(1, n_max):
        prior = _compose(est[-1], _compose(_inverse(truth[i - 1]), truth[i]))
        r = ctx.register(synth.make_scan(scene, "vlp16", truth[i], 5000 + i, rmax=20.0), prior, 10, mf)
        assert r.status == 0, (i, r.status)
        p = _compose(drift, np.array(r.pose))
        est.append(p)
        ctx.keyframe_add_registered(p)
        ctx.map_add_registered_scan(p)
        if i > n_max // 2 and np.linalg.norm(p[:3] - est[0][:3]) < 6.0:
            n = i + 1
            break
    est = np.array(est)
    truth = truth[:n]
    err_before = np.linalg.norm(est[:, :3] - truth[:, :3], axis=1)
    assert n < n_max and err_before[-1] > 0.2
    live_map = ctx.map_download(0)
    sub = kf_ctx(gpu_api)
    sub.map_set_origin(truth[0][:3])
    sub.map_from_keyframes(ctx, [0, 1, 2], est[:3], 1)
    loop = sub.register_keyframes(ctx, [n - 1], [est[n - 1]], 20, mf)[0]
    assert loop.status == 0
    t_loop = np.array(loop.pose)
    w_odo = np.r_[np.full(3, 1 / 0.02), np.full(3, 1 / np.deg2rad(0.05))]
    w_loop = np.r_[np.full(3, 1 / 0.01), np.full(3, 1 / np.deg2rad(0.05))]
    edges = [(i, i + 1, _compose(_inverse(est[i]), est[i + 1]), w_odo) for i in range(n - 1)]
    edges.append((0, n - 1, _compose(_inverse(est[0]), t_loop), w_loop))
    opt, res = ctx.pose_graph_solve(est, edges)
    E = PG.to_array([PG.edge(i, j, z, w) for i, j, z, w in edges])
    prob = PG.PoseGraph(est, E)
    ref = CR.solve_full(prob, prob.x0(), 50)
    assert (res["iterations"], res["termination"]) == (ref["iterations"], ref["termination"])
    d_ref = np.abs(opt - prob.nodes(ref["x"])).max()
    helper = _pose_graph(est, edges)
    d_helper = np.abs(opt[:, :3] - helper[:, :3]).max()
    err_after = np.linalg.norm(opt[:, :3] - truth[:, :3], axis=1)
    print(f"loop on the device: {n} keyframes, {res['iterations']} iterations ({res['pcg_iterations']} PCG), {res['time_ms']:.2f} ms; "
          f"error mean {err_before.mean():.3f} -> {err_after.mean():.3f} m, max {err_before.max():.3f} -> {err_after.max():.3f} m; "
          f"poses vs the restatement {d_ref:.2e}, largest position difference from the scipy helper {d_helper:.2e} m")
    if TRS.fair(ref):
        assert d_ref <= 1e-8
    assert err_after.mean() < 0.6 * err_before.mean() and err_after.max() < 0.7 * err_before.max()
    ids = np.arange(n, dtype=np.int32)
    ctx.map_from_keyframes(ctx, ids, opt, 1)
    gt = kf_ctx(gpu_api)
    gt.map_set_origin(truth[0][:3])
    gt.map_from_keyframes(ctx, ids, truth, 1)
    gt_map = gt.map_download(0)
    far_live, far_rebuilt = _share_far(live_map, gt_map, 0.2), _share_far(ctx.map_download(0), gt_map, 0.2)
    print(f"loop on the device: map points farther than planeRes from the ground-truth rebuild {far_live:.4f} -> {far_rebuilt:.4f}")
    assert far_rebuilt < 0.6 * far_live
    prior = _compose(opt[-1], _compose(_inverse(truth[n - 1]), truth[0]))
    r = ctx.register(synth.make_scan(scene, "vlp16", truth[0], 6000, rmax=20.0), prior, 10, mf)
    nxt_err = np.linalg.norm(np.array(r.pose)[:3] - truth[0, :3])
    print(f"loop on the device: next registration error {nxt_err:.3f} m")
    assert r.status == 0 and nxt_err < 0.1
    for x in (ctx, sub, gt):
        x.close()

"""so_kernel_launches against CUDA's own record of the kernels: torch.profiler (CUDA activities) around one call counts the kernels of
namespace so::, and that number must equal the change of Context.kernel_launches() over the call.  The calls run no cub primitive
(cub's kernels are outside so:: and are counted by fixed tallies): the stage hooks, the given-correspondence solves, and capped
registrations of one and two scans, whose ordering is the one-CTA k_prepare_small, in every mode and in the schedule's unrolled,
profiled and neighbour-graph forms.  Every registration is run once before it is recorded, so that the map index and the neighbour
graph are built outside the window.  The default form, a CUDA-graph WHILE node, is not among them: torch.profiler (torch 2.11,
CUDA 12.8, on an H100) lists the kernels of the WHILE body once, not once per pass, so it cannot count that form."""
import re

import numpy as np
import pytest

from test_undistortion import _moving_case

pytestmark = pytest.mark.gpu

ITERS, MF = 4, 2000
SO_KERNEL = re.compile(r"^(void )?so::")


def _device_kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and SO_KERNEL.match(e.name)]


def _check(ctx, fn):
    ctx.kernel_launches(reset=True)
    names = _device_kernels(fn)
    assert ctx.kernel_launches() == len(names), names
    return names


@pytest.fixture(scope="module")
def scene():
    from superodom_b200 import synth
    d = _moving_case("cfg1", 1.5, 0.3)
    d2 = _moving_case("cfg1", 1.5, 0.3, k=1)
    em = synth.make_edge_map(d["case"]["scene"], 0.1)
    return {"map": d["case"]["map_xyzi"], "edge_map": em, "scans": [d["scan_xyzi"], d2["scan_xyzi"]],
            "priors": [d["prior"], d2["prior"]], "prev": [d["pose_prev"], d2["pose_prev"]],
            "edges": [synth.make_edge_scan(em, d["pose_true"], 17), synth.make_edge_scan(em, d2["pose_true"], 18)]}


def _ctx(api, scene, monkeypatch, env=()):
    for k, v in env:
        monkeypatch.setenv(k, v)
    ctx = api.Context(max_map_points=1 << 20, max_scan_points=65536, max_batch=4, plane_res=0.2)
    for k, _ in env:
        monkeypatch.delenv(k)
    ctx.map_set_points(scene["map"])
    ctx.map_set_edge_points(scene["edge_map"])
    return ctx


def _registration(api, ctx, scene, mode, n_scans, edges):
    s, p, pp, e = scene["scans"][:n_scans], scene["priors"][:n_scans], scene["prev"][:n_scans], scene["edges"][:n_scans]
    flat, n, poses = np.concatenate(s), [len(x) for x in s], np.stack(p)
    if n_scans == 1:
        edge = e[0] if edges else None
        if mode == "none":
            return lambda: ctx.register(s[0], p[0], ITERS, MF, edge_xyzi=edge)
        if mode == "approximated":
            u = api.undistort(pp[0], 0.1)
            if edges:
                return lambda: ctx.register_undistort_edges(s[0], edge, p[0], u, ITERS, MF)
            return lambda: ctx.register_undistort(s[0], p[0], u, ITERS, MF)
        m = api.motion(0.1)
        if edges:
            return lambda: ctx.register_optimized_edges(s[0], edge, p[0], m, ITERS, MF)
        return lambda: ctx.register_optimized(s[0], p[0], m, ITERS, MF)
    if mode == "none":
        if edges:
            return lambda: ctx.register_batch_edges(flat, n, np.concatenate(e), [len(x) for x in e], poses, ITERS, MF)
        return lambda: ctx.register_batch(flat, n, poses, ITERS, MF)
    if mode == "approximated":
        return lambda: ctx.register_batch_undistort(flat, n, poses, [api.undistort(x, 0.1) for x in pp], ITERS, MF)
    return lambda: ctx.register_batch_optimized(flat, n, poses, [api.motion(0.1)] * n_scans, ITERS, MF)


FORMS = {
    "unrolled": (("SO_NO_COND_GRAPH", "1"),),
    "profiled": (),
    "graph_search": (("SO_NO_COND_GRAPH", "1"), ("SO_KNN_GRAPH", "on"), ("SO_NO_COOP_KNN", "1")),
}
CASES = [("none", 1, False), ("none", 1, True), ("approximated", 1, False), ("approximated", 1, True), ("optimized", 1, False),
         ("optimized", 1, True), ("none", 2, False), ("none", 2, True), ("approximated", 2, False), ("optimized", 2, False)]


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("mode,n_scans,edges", CASES)
def test_registration(gpu_api, scene, monkeypatch, form, mode, n_scans, edges):
    ctx = _ctx(gpu_api, scene, monkeypatch, FORMS[form])
    if form == "profiled":
        ctx.profile_enable(True)
    call = _registration(gpu_api, ctx, scene, mode, n_scans, edges)
    call()
    names = _check(ctx, call)
    assert any("k_prepare_small" in k for k in names)
    if form == "graph_search":
        assert any("k_knn_round2" in k for k in names)
    ctx.close()


def test_stage_hooks(gpu_api, scene, monkeypatch):
    ctx = _ctx(gpu_api, scene, monkeypatch)
    s, p, e = scene["scans"][0][:4000], scene["priors"][0], scene["edges"][0]
    ctx.correspond(s, p)                                               # builds the map index
    # so_correspond and so_correspond_seeded run one cub ordering each: the difference is the seeded call's second correspondence pass
    ctx.kernel_launches(reset=True)
    plain = _device_kernels(lambda: ctx.correspond(s, p))
    n_plain = ctx.kernel_launches(reset=True)
    seeded = _device_kernels(lambda: ctx.correspond(s, p, seed_pose=scene["prev"][0]))
    assert ctx.kernel_launches() - n_plain == len(seeded) - len(plain) > 0
    _check(ctx, lambda: ctx.evaluate(p))                               # plane rows
    names = _check(ctx, lambda: ctx.correspond_edge(e, p))
    assert any("k_edge_fit" in k for k in names)
    _check(ctx, lambda: ctx.evaluate(p))                               # edge rows: so_correspond_edge replaced the plane rows
    ctx.register(scene["scans"][0], p, ITERS, MF, edge_xyzi=e)
    names = _check(ctx, lambda: ctx.evaluate(p))                       # the registration's last plane and edge rows
    assert any("k_edge_evaluate" in k for k in names) and any("k_evaluate" in k for k in names)
    ctx.close()


def test_covariance_and_degeneracy(gpu_api, scene, monkeypatch):
    ctx = _ctx(gpu_api, scene, monkeypatch)
    rng = np.random.default_rng(3)
    for n in (6, 12):
        a = rng.standard_normal((n, n))
        _check(ctx, lambda: ctx.covariance(a @ a.T + n * np.eye(n)))
    a = rng.standard_normal((6, 6))
    _check(ctx, lambda: ctx.degeneracy_analysis(a @ a.T + np.eye(6), gpu_api.degeneracy(0.2, 0.1)))
    ctx.close()


def test_solves(gpu_api, scene, monkeypatch):
    import motion_solve_sets as MS
    import trust_region_sets as TS
    from test_motion_solve import _pack
    from test_trust_region import _rows
    ctx = _ctx(gpu_api, scene, monkeypatch)
    problems = TS.sample(5, 1, lms=(4,), row_counts=(4097,))
    for b in (1, 3):
        rows, pr = _rows(problems[:b])
        _check(ctx, lambda: ctx.solve(rows, pr))
        ds = [gpu_api.degeneracy(0.2, 0.1)] * b
        _check(ctx, lambda: ctx.solve(rows, pr, ds))
    mp = MS.sample(5, 1, lms=(4,), row_counts=(4097,))
    _check(ctx, lambda: ctx.solve_optimized(*_pack(mp[:2])))
    ctx.close()

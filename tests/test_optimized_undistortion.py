"""Within-scan motion estimated by the registration (so_register_optimized*, mode OPTIMIZED).

CPU: the numpy restatement's Jacobian against central differences, its two-block solve on its own terms, the ABI layout.
GPU: the stage hook against the restatement, one ICP iteration against the restatement's solve on the same correspondences, batches
against single calls, packed against strided uploads, repeatability, the map insert, the prefiltered path, argument errors, the
profile classes, and the accuracy against APPROXIMATED when the previous registration's velocity is wrong."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest

import optimized_numpy as ON
from conftest import get_case, quat_angle
from test_ceres_restatement import _plus, _rot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDENTITY = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])


def _unit(q):
    return q / np.linalg.norm(q)


def _rand_pose(rng, t=3.0, r=0.4):
    from superodom_b200 import synth
    return np.concatenate([rng.normal(0, t, 3), _unit(synth.quat_from_rotvec(rng.normal(0, r, 3)))])


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("kind", ["plain", "alpha_outside", "small_angle", "negative_w", "tiny_angle"])
def test_jacobian_matches_central_differences(kind):
    rng = np.random.default_rng(hash(kind) % 1000)
    for trial in range(6):
        T = _rand_pose(rng)
        D = _rand_pose(rng, 0.5, 0.3)
        if kind == "small_angle":
            D[3:] = _unit(np.r_[rng.normal(0, 2e-3, 3), 1.0])                # |phi| < 1e-2: the series branch
        if kind == "tiny_angle":
            D[3:] = _unit(np.r_[rng.normal(0, 1e-7, 3), 1.0])
        if kind == "negative_w":
            D[3:] = -D[3:]
        n = 40
        P = rng.uniform(-30, 30, (n, 3))
        A = rng.uniform(-0.5, 1.5, n) if kind == "alpha_outside" else rng.uniform(0, 1, n)
        N = np.stack([_unit(v) for v in rng.normal(size=(n, 3))])
        Dd = rng.normal(0, 5, n)
        J = ON.jacobian(P, A, N, T, D)
        num = np.zeros_like(J)
        for k in range(12):
            h = 1e-6
            d = np.zeros(12)
            d[k] = h
            rp = ON.residuals(P, A, N, Dd, _plus(T, d[:6]), _plus(D, d[6:]))
            rm = ON.residuals(P, A, N, Dd, _plus(T, -d[:6]), _plus(D, -d[6:]))
            num[:, k] = (rp - rm) / (2 * h)
        scale = np.abs(J).max() + 1.0
        assert np.abs(J - num).max() < 2e-6 * scale, (kind, trial, np.abs(J - num).max())


def _random_problem(rng, n, info):
    """planes seen by a moving sensor: correspondences {p, alpha, n, d, w} exact at a ground-truth (T, D)"""
    T = _rand_pose(rng, 5.0, 0.15)
    D = np.r_[rng.normal(0, 0.4, 3), _unit(np.r_[rng.normal(0, 0.03, 3), 1.0])]
    normals = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    P = rng.uniform(-20, 20, (n, 3))
    A = rng.uniform(0, 1, n)
    k = rng.integers(0, 3, n)
    N = normals[k] * rng.choice([-1.0, 1.0], n)[:, None]
    world = ON.warp_double(P, A, D) @ _rot(T[3:]).T + T[:3]
    Dd = -(N * world).sum(1) + rng.normal(0, 0.005, n)
    W = rng.uniform(0.5, 1.0, n)
    return T, D, ON.Problem(P, A, N, Dd, W, 0.6, D, info)


def test_numpy_two_block_solve_recovers_the_motion():
    rng = np.random.default_rng(3)
    for trial in range(8):
        T, D, prob = _random_problem(rng, 300, np.zeros(6))
        T0 = _plus(T, np.r_[rng.uniform(-1, 1, 3) * 0.05, rng.uniform(-1, 1, 3) * 0.01])
        Tn, Dn, it, succ, unsucc, term = ON.solve(prob, T0, IDENTITY, 12)
        assert np.abs(Tn[:3] - T[:3]).max() < 0.02 and np.abs(Dn[:3] - D[:3]).max() < 0.05, (trial, Tn - T, Dn - D)
        # a strong prior at the truth pins D there
        prob.sqrt_info = np.sqrt(len(prob.P) * np.full(6, 1e4))
        Tn, Dn, *_ = ON.solve(prob, T0, D, 12)
        assert np.abs(Dn - D).max() < 1e-3


def test_motion_struct_layout():
    from superodom_b200 import api
    assert C.sizeof(api.Motion) == 112 and api.Motion.motion_prior.offset == 8 and api.Motion.motion_info.offset == 64
    assert api.MotionResult.motion.offset == C.sizeof(api.IcpResult)
    assert C.sizeof(api.MotionResult) == C.sizeof(api.IcpResult) + 112


def test_motion_struct_layout_in_c(tmp_path):
    from superodom_b200 import api
    src = tmp_path / "l.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "superodom_b200.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu\\n", '
                   'sizeof(so_motion), offsetof(so_motion, motion_prior), offsetof(so_motion, motion_info), sizeof(so_motion_result), '
                   'offsetof(so_motion_result, motion), offsetof(so_motion_result, pose_end)); return 0;}\n')
    exe = tmp_path / "l"
    subprocess.check_call(["cc", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).decode().split()]
    assert got == [C.sizeof(api.Motion), 8, 64, C.sizeof(api.MotionResult), api.MotionResult.motion.offset, api.MotionResult.pose_end.offset]


# ------------------------------------------------------------------------------------------------------------------ GPU
def _ctx(api, case, **kw):
    ctx = api.Context(max_map_points=max(1 << 20, len(case["map_xyzi"]) * 2 + 1024), max_scan_points=262144, plane_res=case["cfg"]["plane_res"], **kw)
    ctx.map_set_points(case["map_xyzi"])
    return ctx


_moving = {}


def _moving_case(name, speed, yaw_rate, k=0):
    from superodom_b200 import synth
    key = (name, speed, yaw_rate, k)
    if key not in _moving:
        case = get_case(name)
        pose = synth.random_sensor_pose(case["scene"], 950 + k, 8.0)
        d = synth.make_moving_scan(case["scene"], case["cfg"]["sensor"], pose, speed, yaw_rate, 60 + k)
        d["case"] = case
        d["motion_true"] = ON.compose(ON.inverse(d["pose_true"]), d["pose_next"])
        _moving[key] = d
    return _moving[key]


def _res_equal(a, b):
    for f, _ in a._fields_:
        va, vb = getattr(a, f), getattr(b, f)
        if isinstance(va, C.Structure):
            _res_equal(va, vb)
            continue
        if f.startswith("time"):
            continue
        if hasattr(va, "__len__"):
            assert bytes(va) == bytes(vb), f
        else:
            assert va == vb or (isinstance(va, float) and math.isnan(va) and math.isnan(vb)), f


def _plane_rows(ctx, scan, T, D, dt, mf, a2):
    """the restatement's Problem over the correspondences at T of float(u(D)) (so_correspond on the numpy warp)"""
    u = ON.warp_points(scan, D, dt)
    corr, _, hr = ctx.correspond(np.concatenate([u, scan[:, 3:4]], 1), T, mf)
    ok = corr["w"] != 0.0
    return ON.Problem(scan[ok, :3].astype(np.float64), ON.alphas(scan[ok, 3], dt), corr["n"][ok], corr["d"][ok], corr["w"][ok], a2,
                      IDENTITY, np.zeros(6)), int(hr[0])


def _a2(case):
    a = float(np.sqrt(np.float32(3 * np.float32(case["cfg"]["plane_res"]))))
    return a * a


@pytest.mark.gpu
@pytest.mark.parametrize("mf", [0, 2000])
def test_stage_hook_matches_numpy(gpu_api, mf):
    d = _moving_case("cfg1", 5.0, 0.5)
    case = d["case"]
    ctx = _ctx(gpu_api, case)
    scan = d["scan_xyzi"]
    for D in (d["motion_true"], IDENTITY, np.r_[0.3, -0.05, 0.01, -_unit(np.r_[0.01, -0.02, 0.05, 1.0])]):
        H, g, cost = ctx.evaluate_optimized(scan, d["prior"], D, 0.1, mf)
        prob, n_ok = _plane_rows(ctx, scan, d["prior"], D, 0.1, mf, _a2(case))
        assert n_ok == len(prob.P) > 100
        Hn, gn, cn = prob.normal_equations(np.asarray(d["prior"]), np.asarray(D))
        assert np.abs(H - Hn).max() <= 1e-10 * np.abs(Hn).max()
        assert np.abs(g - gn).max() <= 1e-10 * np.abs(gn).max() + 1e-12
        assert abs(cost - cn) <= 1e-10 * abs(cn)


@pytest.mark.gpu
@pytest.mark.parametrize("name,speed,D0kind,info", [("cfg1", 5.0, "true", 0.0), ("cfg1", 1.5, "identity", 0.0), ("cfg1", 5.0, "identity", 0.01),
                                                    ("cfg2", 10.0, "identity", 0.0), ("cfg2", 0.0, "fast", 0.01)])
def test_one_iteration_matches_numpy_solve(gpu_api, name, speed, D0kind, info):
    """max_icp_iters = 1: the device's solve on its own correspondences == the restatement's solve on so_correspond's at (T0, D0)."""
    d = _moving_case(name, speed, 0.3 if speed else 0.0)
    case = d["case"]
    fast = ON.compose(ON.inverse(_moving_case(name, 5.0, 0.3)["pose_true"]), _moving_case(name, 5.0, 0.3)["pose_next"])
    D0 = {"true": d["motion_true"], "identity": IDENTITY, "fast": fast}[D0kind]
    ctx = _ctx(gpu_api, case)
    scan = d["scan_xyzi"]
    lm = 4
    r = ctx.register_optimized(scan, d["prior"], gpu_api.motion(0.1, D0, [info] * 6), 1, 0, lm_max_iterations=lm)
    prob, n_ok = _plane_rows(ctx, scan, d["prior"], D0, 0.1, 0, _a2(case))
    prob.D0 = _unit_pose(D0)
    prob.sqrt_info = np.sqrt(n_ok * np.full(6, info))
    T, D, it, succ, unsucc, term = ON.solve(prob, d["prior"], D0, lm)
    assert r.icp.iter_n_surf[0] == n_ok
    assert (r.icp.iter_lm_steps[0], r.icp.iter_lm_successful[0], r.icp.iter_lm_termination[0]) == (it, succ, term)
    assert np.abs(np.array(r.icp.pose_opt) - T).max() < 1e-8
    assert np.abs(np.array(r.motion) - D).max() < 1e-8


def _unit_pose(p):
    p = np.array(p, np.float64)
    p[3:] = _unit(p[3:])
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("mf", [2000, 0])
def test_batch_equals_single_calls_and_repeats(gpu_api, mf):
    ds = [_moving_case("cfg1", v, 0.3, k) for k, v in enumerate([0.0, 1.5, 5.0, 3.0, 5.0])]
    case = ds[0]["case"]
    ms = [gpu_api.motion(0.1, IDENTITY if k % 2 else ds[k]["motion_true"], [0.01 * k] * 6) for k in range(len(ds))]
    single = _ctx(gpu_api, case)
    ref = [single.register_optimized(d["scan_xyzi"], d["prior"], m, 5, mf, skip_map_checks=True) for d, m in zip(ds, ms)]
    again = [single.register_optimized(d["scan_xyzi"], d["prior"], m, 5, mf, skip_map_checks=True) for d, m in zip(ds, ms)]
    for a, b in zip(ref, again):
        _res_equal(a, b)
    # a strided upload (x, y, z, pad, time) gives the same bits
    d = ds[2]
    strided = np.concatenate([d["scan_xyzi"][:, :3], np.zeros((len(d["scan_xyzi"]), 1), np.float32), d["scan_xyzi"][:, 3:]], 1)
    _res_equal(single.register_optimized(strided, d["prior"], ms[2], 5, mf, time_col=4, skip_map_checks=True), ref[2])
    for mb in (2, 5):
        ctx = _ctx(gpu_api, case, max_batch=mb)
        for f in range(0, len(ds), mb):
            sub = ds[f:f + mb]
            res = ctx.register_batch_optimized(np.concatenate([x["scan_xyzi"] for x in sub]), [len(x["scan_xyzi"]) for x in sub],
                                               np.stack([x["prior"] for x in sub]), ms[f:f + mb], 5, mf, skip_map_checks=True)
            for a, b in zip(res, ref[f:f + mb]):
                _res_equal(a, b)
            sres = ctx.register_batch_optimized(np.concatenate([strided if x is d else np.concatenate([x["scan_xyzi"][:, :3], np.zeros((len(x["scan_xyzi"]), 1), np.float32), x["scan_xyzi"][:, 3:]], 1) for x in sub]),
                                                [len(x["scan_xyzi"]) for x in sub], np.stack([x["prior"] for x in sub]), ms[f:f + mb], 5, mf,
                                                time_col=4, skip_map_checks=True)
            for a, b in zip(sres, ref[f:f + mb]):
                _res_equal(a, b)


@pytest.mark.gpu
def test_result_fields(gpu_api):
    d = _moving_case("cfg1", 5.0, 0.5)
    ctx = _ctx(gpu_api, d["case"])
    r = ctx.register_optimized(d["scan_xyzi"], d["prior"], gpu_api.motion(0.1), 5, 2000)
    assert r.icp.status == 0
    T, D = np.array(r.icp.pose_opt), np.array(r.motion)
    assert np.abs(np.array(r.pose_end) - ON.compose(T, D)).max() < 1e-12
    cov = np.array(r.icp.cov).reshape(6, 6)
    assert np.allclose(cov, cov.T) and np.all(np.linalg.eigvalsh(cov) > 0) and r.icp.pos_err > 0


@pytest.mark.gpu
def test_insert_equals_insert_of_the_warped_cloud(gpu_api):
    d = _moving_case("cfg1", 5.0, 0.5)
    a, b = _ctx(gpu_api, d["case"]), _ctx(gpu_api, d["case"])
    r = a.register_optimized(d["scan_xyzi"], d["prior"], gpu_api.motion(0.1), 5, 2000)
    pose = np.array(r.icp.pose)
    a.map_add_registered_scan(pose)
    u = ON.warp_points(d["scan_xyzi"], np.array(r.motion), 0.1)
    b.map_add_scan(np.concatenate([u, d["scan_xyzi"][:, 3:]], 1), pose)
    assert np.array_equal(a.map_download(), b.map_download())
    # a plain so_register afterwards inserts its cloud as before
    a.register(d["scan_xyzi"], d["prior"], 5, 2000)
    b.register(d["scan_xyzi"], d["prior"], 5, 2000)
    a.map_add_registered_scan(pose)
    b.map_add_scan(d["scan_xyzi"], pose)
    assert np.array_equal(a.map_download(), b.map_download())


@pytest.mark.gpu
def test_prefiltered_equals_host_path(gpu_api):
    d = _moving_case("cfg2", 1.5, 0.3)
    case = d["case"]
    m = gpu_api.motion(0.1)
    a, b = _ctx(gpu_api, case), _ctx(gpu_api, case)
    filt, _, _, _ = a.scan_prefilter(d["scan_xyzi"], 0.2, case["cfg"]["plane_res"], auto_voxel_size=False)
    ra = a.register_prefiltered_optimized(d["prior"], m, 10)
    rb = b.register_optimized(filt, d["prior"], m, 10)
    _res_equal(ra, rb)
    a.map_add_registered_scan(np.array(ra.icp.pose))
    b.map_add_registered_scan(np.array(rb.icp.pose))
    assert np.array_equal(a.map_download(), b.map_download())


@pytest.mark.gpu
def test_argument_errors_before_device_work(gpu_api):
    d = _moving_case("cfg1", 1.5, 0.3)
    ctx = _ctx(gpu_api, d["case"])
    ctx.kernel_launches(reset=True)
    nan = float("nan")
    bad = [gpu_api.motion(0.0), gpu_api.motion(-0.1), gpu_api.motion(nan), gpu_api.motion(float("inf")),
           gpu_api.motion(0.1, np.r_[IDENTITY[:6], nan]), gpu_api.motion(0.1, np.zeros(7)), gpu_api.motion(0.1, info=[0, 0, -1, 0, 0, 0]),
           gpu_api.motion(0.1, info=[0, 0, 0, nan, 0, 0]), gpu_api.motion(0.1, info=[0, 0, 0, 0, float("inf"), 0])]
    scan = d["scan_xyzi"]
    for m in bad:
        for call in (lambda: ctx.register_optimized(scan, d["prior"], m, 5, 2000),
                     lambda: ctx.register_batch_optimized(scan, [len(scan)], d["prior"][None], [m], 5, 2000),
                     lambda: ctx.register_prefiltered_optimized(d["prior"], m, 5)):
            with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
                call()
    good = gpu_api.motion(0.1)
    for call in (lambda: ctx.register_optimized(scan, d["prior"], good, 5, 2000, pose_prior=(1.0, (0.0, 0.0, 0.0))),
                 lambda: ctx.register_optimized(scan, d["prior"], good, 0, 2000),
                 lambda: ctx.register_prefiltered_optimized(d["prior"], good, 5),
                 lambda: ctx.evaluate_optimized(scan, d["prior"], np.zeros(7), 0.1),
                 lambda: ctx.evaluate_optimized(scan, d["prior"], IDENTITY, 0.0),
                 lambda: ctx.register_undistort(scan, d["prior"], gpu_api.undistort(d["pose_prev"], 0.1, mode=2), 5, 2000)):
        with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
            call()
    with pytest.raises(gpu_api.SuperOdomError, match="so_register_optimized"):
        ctx.register_undistort(scan, d["prior"], gpu_api.undistort(d["pose_prev"], 0.1, mode=2), 5, 2000)
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-3\)"):
        ctx.register_optimized(np.zeros((262145, 4), np.float32), d["prior"], good, 5, 2000)
    assert ctx.kernel_launches() == 0


@pytest.mark.gpu
def test_profile_classes_7_and_8(gpu_api):
    d = _moving_case("cfg1", 1.5, 0.3)
    ctx = _ctx(gpu_api, d["case"])
    ctx.profile_enable(True)
    r = ctx.register_optimized(d["scan_xyzi"], d["prior"], gpu_api.motion(0.1), 5, 2000)
    ms7, n7 = ctx.profile_get(7)
    ms8, n8 = ctx.profile_get(8)
    assert n7 == r.icp.n_iterations and ms7 > 0.0
    assert n8 == sum(1 + r.icp.iter_lm_steps[i] for i in range(r.icp.n_iterations)) and ms8 > 0.0
    ctx.profile_enable(False)
    ref = _ctx(gpu_api, d["case"]).register_optimized(d["scan_xyzi"], d["prior"], gpu_api.motion(0.1), 5, 2000)
    assert np.array_equal(np.array(r.icp.pose_opt), np.array(ref.icp.pose_opt))


# ------------------------------------------------------------------------------------------------------------------ accuracy
def _err(pose, truth):
    return float(np.linalg.norm(np.asarray(pose[:3]) - truth[:3])), quat_angle(_unit(np.asarray(pose[3:])), truth[3:])


def _accuracy_row(api, name, scenario, speed, mf, it, info):
    """(scenario, speed) -> pose errors of so_register, APPROXIMATED and OPTIMIZED against the sweep-start truth, and OPTIMIZED's
    motion error.  The previous registration APPROXIMATED takes its velocity from, and OPTIMIZED's D0:
      constant  -- the scan's own motion (pose_prev, the true D)
      start     -- at rest before the sweep (pose_prev = pose_true, D0 = identity), the sweep at `speed`
      brake     -- 5 m/s before (pose_prev 0.5 m behind, D0 the 5 m/s motion), the sweep at rest
      still     -- at rest throughout"""
    sweep_speed = 0.0 if scenario in ("brake", "still") else speed
    yaw = 0.3 if sweep_speed else 0.0
    d = _moving_case(name, sweep_speed, yaw)
    truth = d["pose_true"]
    if scenario == "constant":
        prev, D0 = d["pose_prev"], d["motion_true"]
    elif scenario == "brake":
        fast = _moving_case(name, 5.0, 0.0)
        D0 = ON.compose(ON.inverse(fast["pose_true"]), fast["pose_next"])
        prev = ON.compose(truth, ON.inverse(D0))
    else:
        prev, D0 = truth, IDENTITY
    ctx = _ctx(api, d["case"])
    rn = ctx.register(d["scan_xyzi"], d["prior"], it, mf)
    ra = ctx.register_undistort(d["scan_xyzi"], d["prior"], api.undistort(prev, 0.1), it, mf)
    ro = ctx.register_optimized(d["scan_xyzi"], d["prior"], api.motion(0.1, D0, [info] * 6), it, mf)
    Dt = d["motion_true"]
    return dict(name=name, scenario=scenario, speed=speed, info=info, none=_err(rn.pose, truth), approx=_err(ra.pose, truth),
                opt=_err(ro.icp.pose, truth), motion=_err(np.array(ro.motion), Dt))


ACCURACY = [("cfg1", 2000, 5), ("cfg2", 0, 20)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,mf,it", ACCURACY)
def test_optimized_beats_approximated_when_the_velocity_changes(gpu_api, name, mf, it):
    rows = []
    for scenario, speeds in (("constant", (5.0,)), ("start", (1.5, 5.0, 10.0)), ("brake", (5.0,)), ("still", (0.0,))):
        for v in speeds:
            rows.append(_accuracy_row(gpu_api, name, scenario, v, mf, it, 0.0))
    out = os.environ.get("SO_ACCURACY_OUT")
    if out:
        with open(out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
    # measured (DESIGN.md §4, motion_info 0): OPTIMIZED 0.013-0.031 m in every scenario; APPROXIMATED 0.003-0.008 m with the right
    # velocity, 0.06 / 0.17-0.18 / 0.33-0.35 m starting at 1.5 / 5 / 10 m/s and 0.17 m braking from 5 m/s
    for r in rows:
        eo, ea = r["opt"][0], r["approx"][0]
        assert eo < 0.05 and r["opt"][1] < 0.005, r
        if r["scenario"] in ("constant", "still"):
            assert eo < 0.04, r                                   # measured 0.013-0.031 m on these scans
        if r["scenario"] == "brake" or (r["scenario"] == "start" and r["speed"] >= 5.0):
            assert eo < 0.3 * ea, r
        elif r["scenario"] == "start":
            assert eo < ea, r


# ------------------------------------------------------------------------------------------------------------------ whole ICP loop
def _numpy_register(ctx, scan, T0, D0, dt, info, iters, mf, a2, lm=4):
    """so_register_optimized's ICP loop restated: every iteration re-corresponds at T on float(u(D)) (so_correspond on the numpy
    warp), solves over two blocks, and stops after a solve with one successful step or on the last iteration.  -> (T, D, per-iteration
    (n_ok, lm steps, successful, termination, hist_obs, hist_reject_plane), H of the last solve with the prior rows)"""
    T, D = np.array(T0, float), _unit_pose(D0)
    its = []
    for k in range(iters):
        u = ON.warp_points(scan, D, dt)
        corr, ho, hr = ctx.correspond(np.concatenate([u, scan[:, 3:4]], 1), T, mf)
        ok = corr["w"] != 0.0
        prob = ON.Problem(scan[ok, :3].astype(np.float64), ON.alphas(scan[ok, 3], dt), corr["n"][ok], corr["d"][ok], corr["w"][ok], a2,
                          _unit_pose(D0), np.full(6, info))
        prob.sqrt_info = np.sqrt(int(hr[0]) * np.full(6, info))
        T, D, it, succ, unsucc, term = ON.solve(prob, T, D, lm)
        its.append((int(hr[0]), it, succ, term, list(ho), list(hr)))
        if succ == 1:
            break
    _, _, J = prob.linearise(T, D)
    return T, D, its, J.T @ J


def _cov_T(H):
    """T's 6x6 block of ceres::Covariance (DENSE_SVD): the pseudo-inverse dropping directions with s_i / s_max < sqrt(1e-14)"""
    w, V = np.linalg.eigh(H)
    keep = np.sqrt(np.clip(w, 0, None) / w.max()) >= 1e-7
    return ((V[:, keep] / w[keep]) @ V[:, keep].T)[:6, :6]


@pytest.mark.gpu
@pytest.mark.parametrize("name,scenario,mf,info", [("cfg1", "start", 2000, 0.0), ("cfg1", "brake", 2000, 0.01), ("cfg1", "constant", 0, 0.01),
                                                   ("cfg2", "start", 4000, 0.01)])
def test_icp_loop_matches_numpy(gpu_api, name, scenario, mf, info):
    """The whole registration (re-warp at the updated D every iteration, the break rule, the per-iteration statistics and histograms,
    the covariance of T) against the numpy ICP loop on the device's own search and fit."""
    case = get_case(name)
    sweep = 0.0 if scenario == "brake" else 5.0
    d = _moving_case(name, sweep, 0.3 if sweep else 0.0)
    fast = _moving_case(name, 5.0, 0.0)
    D0 = {"start": IDENTITY, "brake": ON.compose(ON.inverse(fast["pose_true"]), fast["pose_next"]), "constant": d["motion_true"]}[scenario]
    it = 5 if name == "cfg1" else 10
    ctx = _ctx(gpu_api, case)
    r = ctx.register_optimized(d["scan_xyzi"], d["prior"], gpu_api.motion(0.1, D0, [info] * 6), it, mf)
    T, D, its, H = _numpy_register(ctx, d["scan_xyzi"], d["prior"], D0, 0.1, info, it, mf, _a2(case))
    assert r.icp.n_iterations == len(its) > 1
    for k, (n_ok, steps, succ, term, ho, hr) in enumerate(its):
        assert (r.icp.iter_n_surf[k], r.icp.iter_lm_steps[k], r.icp.iter_lm_successful[k], r.icp.iter_lm_termination[k]) == (n_ok, steps, succ, term), k
    assert list(r.icp.hist_obs) == its[-1][4] and list(r.icp.hist_reject_plane) == its[-1][5]
    assert np.abs(np.array(r.icp.pose_opt) - T).max() < 1e-6
    assert np.abs(np.array(r.motion) - D).max() < 1e-6
    cov = _cov_T(H)
    assert np.abs(np.array(r.icp.cov).reshape(6, 6) - cov).max() <= 1e-6 * np.abs(cov).max()
    e = np.linalg.eigvalsh(cov[:3, :3])
    assert abs(r.icp.pos_err - math.sqrt(e[2])) <= 1e-6 * math.sqrt(e[2])


@pytest.mark.gpu
def test_stage_hook_series_branch(gpu_api):
    """0 < |phi| < 1e-2: the Taylor series of J_r(phi)^-1 and J_r(alpha phi) on the device (slow turns, the common case)"""
    d = _moving_case("cfg1", 1.5, 0.3)
    case = d["case"]
    ctx = _ctx(gpu_api, case)
    for rv in (np.array([0.0, 0.0, 4e-3]), np.array([1e-3, -2e-3, 6e-3]), np.array([3e-6, 0.0, -1e-5])):
        from superodom_b200 import synth
        D = np.r_[0.15, 0.01, 0.0, _unit(synth.quat_from_rotvec(rv))]
        H, g, cost = ctx.evaluate_optimized(d["scan_xyzi"], d["prior"], D, 0.1, 2000)
        prob, _ = _plane_rows(ctx, d["scan_xyzi"], d["prior"], D, 0.1, 2000, _a2(case))
        Hn, gn, cn = prob.normal_equations(np.asarray(d["prior"]), D)
        assert np.abs(H - Hn).max() <= 1e-10 * np.abs(Hn).max()
        assert np.abs(g - gn).max() <= 1e-10 * np.abs(gn).max() + 1e-12
        assert abs(cost - cn) <= 1e-10 * abs(cn)


# ------------------------------------------------------------------------------------------------------------------ live use
def _speed_change_trajectory(scene, speeds, yaw_rate):
    """VLP-16 scans along one arc, scan k swept at speeds[k] (constant within the sweep): starts, accelerations and stops"""
    from superodom_b200 import synth
    for seed in range(20):
        p = synth.random_sensor_pose(scene, 1400 + seed, 6.0)
        seq = []
        for k, v in enumerate(speeds):
            if not scene.free(p[:3]):
                break
            seq.append(synth.make_moving_scan(scene, "vlp16", p, v, yaw_rate if v else 0.0, 700 + k))
            p = seq[-1]["pose_next"]
        if len(seq) == len(speeds):
            return seq
    raise RuntimeError("no free arc")


@pytest.mark.gpu
def test_live_sequence_with_speed_changes(gpu_api):
    """50 scans (at rest, accelerating to 3 m/s, cruising, braking to rest): register with D0 from the previous registration, insert;
    every map equals the numpy insert of T(pose) * u(D_opt), and the end pose is within reach of the truth."""
    from oracle import oracle as O
    case = get_case("cfg1")
    speeds = [0.0] * 5 + [0.5 * k for k in range(1, 7)] + [3.0] * 20 + [3.0 - 0.5 * k for k in range(1, 7)] + [0.0] * 13
    seq = _speed_change_trajectory(case["scene"], speeds, 0.2)
    ctx = _ctx(gpu_api, case)
    om_points = case["map_xyzi"]
    prev = seq[0]["pose_prev"]
    for k, d in enumerate(seq):
        D0 = ON.compose(ON.inverse(prev), d["prior"])
        r = ctx.register_optimized(d["scan_xyzi"], d["prior"], gpu_api.motion(0.1, D0), 5, 2000)
        assert r.icp.status == 0, k
        pose = np.array(r.icp.pose)
        ctx.map_add_registered_scan(pose)
        u = np.concatenate([ON.warp_points(d["scan_xyzi"], np.array(r.motion), 0.1), d["scan_xyzi"][:, 3:]], 1)
        om_points = O.map_insert_numpy(om_points, O.transform_scan_numpy(u, pose), 0.2, origin=tuple(ctx.map_origin()))
        if k % 10 == 9 or k == len(seq) - 1:
            assert np.array_equal(ctx.map_download(0), om_points[O.cube_order(om_points, tuple(ctx.map_origin()))]), k
        prev = pose
    e = _err(pose, seq[-1]["pose_true"])
    assert e[0] < 0.05 and e[1] < 0.005, e


@pytest.mark.gpu
def test_sink_rows_equal_results(gpu_api):
    torch = pytest.importorskip("torch")
    ds = [_moving_case("cfg1", v, 0.3, k) for k, v in enumerate([1.5, 5.0, 3.0])]
    ctx = _ctx(gpu_api, ds[0]["case"], max_batch=3)
    sink = torch.full((8, 8), -7.0, dtype=torch.float64, device="cuda")
    ctx.set_pose_sink(sink.data_ptr(), 8, 1)
    ms = [gpu_api.motion(0.1) for _ in ds]
    rb = ctx.register_batch_optimized(np.concatenate([d["scan_xyzi"] for d in ds]), [len(d["scan_xyzi"]) for d in ds],
                                      np.stack([d["prior"] for d in ds]), ms, 5, 2000)
    ctx.evaluate_optimized(ds[0]["scan_xyzi"], ds[0]["prior"], IDENTITY, 0.1, 2000)        # a stage evaluation appends no row
    rs = ctx.register_optimized(ds[1]["scan_xyzi"], ds[1]["prior"], ms[1], 5, 2000)
    torch.cuda.synchronize()
    rows = sink.cpu().numpy()
    ctx.set_pose_sink(None)
    for k, r in enumerate(list(rb) + [rs]):
        assert np.array_equal(rows[1 + k, :7], np.array(r.icp.pose_opt)), k
        assert rows[1 + k, 7] == r.icp.status + 256 * r.icp.n_iterations, k
    assert (rows[0] == -7.0).all() and (rows[5:] == -7.0).all()


def _shim_exe(tmp_path):
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "optimized_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "optimized_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


def test_optimized_shim_compiles(tmp_path):
    assert os.path.exists(_shim_exe(tmp_path))


@pytest.mark.gpu
@pytest.mark.parametrize("info", [0.0, 0.01])
def test_shim_optimized_sequence_matches_abi(tmp_path, gpu_api, info):
    import struct
    exe = _shim_exe(tmp_path)
    seq = _speed_change_trajectory(get_case("tiny")["scene"], [0.0, 1.0, 2.0, 2.0, 1.0, 0.0], 0.3)
    scans = [d["scan_xyzi"] for d in seq]
    priors = [seq[0]["pose_true"]] + [d["prior"] for d in seq[1:]]
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiif", len(scans), 5, 0, 0.2))
        for s, p in zip(scans, priors):
            f.write(struct.pack("<i", len(s)))
            f.write(np.asarray(p, np.float64).tobytes())
            f.write(np.ascontiguousarray(s, np.float32).tobytes())
    out = subprocess.run([exe, str(path), repr(info)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows = [[float(v) for v in ln.split()] for ln in out.stdout.strip().splitlines()[:-1]]
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=1 << 17, plane_res=0.2, line_res=0.1)
    ctx.map_set_origin(priors[0][:3])
    ctx.map_add_scan(scans[0], priors[0])
    t_prev = 0.0
    for s in range(1, len(scans)):
        t = 0.1 * s                                               # the shim's timeLaserOdometry
        r = ctx.register_optimized(scans[s], priors[s], gpu_api.motion(t - t_prev, rows[s][16:23], [info] * 6), 5, 0)
        assert np.array_equal(np.array(r.icp.pose), np.array(rows[s][1:8])), s          # shim == ABI, bit for bit
        assert int(rows[s][8]) == r.icp.n_iterations
        assert np.array_equal(np.array(r.motion), np.array(rows[s][23:30])), s
        if r.icp.status == 1:
            continue
        ctx.map_add_registered_scan(np.array(r.icp.pose))
        assert int(rows[s][10]) == ctx.map_size()
        t_prev = t

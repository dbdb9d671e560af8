"""Within-scan motion compensation with an edge cloud: so_register_undistort_edges (APPROXIMATED), so_register_optimized_edges /
so_evaluate_optimized_edges (OPTIMIZED) and so_map_add_registered_edges.

CPU: the CPU oracle with all times zero == the oracle's plain registration with the same edge cloud; the numpy line row's 12 columns
== central differences; the new shim test compiles.
GPU: n_edge = 0 == so_register_undistort / so_register_optimized and mode 0 / all-zero times == so_register with the edge cloud, byte
for byte; the shipped flow (moving raw scan -> so_scan_extract_uniform + so_scan_extract_edges -> compensated registration) == the
CPU oracle on cfg1 / cfg2 at 1.5 and 5 m/s; the OPTIMIZED stage hook == numpy over so_correspond + so_correspond_edge, one OPTIMIZED
ICP iteration == the numpy two-block solve; the edge insert == so_map_add_edge of T(pose) * pInit_e / u_e(D_opt), and ==
so_map_add_scan_edge after so_register; its invalidation; argument errors before any device work; the shim's APPROXIMATED and
OPTIMIZED sequences with edge clouds == the C ABI bit for bit; the corridor at 5 and 10 m/s, where compensated edges (both modes)
beat uncompensated edges on every scan."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import optimized_edges_numpy as OEN
import optimized_numpy as ON
import undistort_edges_oracle as UEO
from conftest import get_case, quat_angle
from test_optimized_undistortion import IDENTITY, _a2, _plane_rows, _rand_pose, _unit
from test_undistortion import _res_equal
from test_undistortion_oracle import _assert_matches_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SKIP, BLOCK_RANGE = 2, 0.1              # so_scan_extract_uniform's skip_num / block_range for the surf clouds


def _compile_shim(tmp_path):
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "undistort_edges_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "undistort_edges_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("mf", [2000, 0])
def test_oracle_zero_times_equal_orc_register_full(mf):
    from superodom_b200 import synth
    from test_undistortion import _moving_case
    d = _moving_case("cfg1", 1.5, 0.3)
    case = d["case"]
    scan = d["scan_xyzi"].copy()
    scan[:, 3] = 0.0
    em = synth.make_edge_map(case["scene"], 0.1)
    edges = synth.make_edge_scan(em, d["pose_true"], 17)
    edges[:, 3] = 0.0
    om = UEO.UndistortEdgesOracleMap(case["map_xyzi"], em)
    ref = om.register_full(scan, edges, d["prior"], 0.2, 5, mf)
    assert ref.iter_n_edge[0] > 100
    for rot in (1, 0):
        om = UEO.UndistortEdgesOracleMap(case["map_xyzi"], em)
        r = om.register_undistort_edges(scan, edges, d["prior"], d["pose_prev"], 0.1, rot, 0.2, 5, mf)
        for f, _ in r._fields_:
            if not f.startswith("time"):
                a, b = getattr(r, f), getattr(ref, f)
                assert (bytes(a) == bytes(b)) if hasattr(a, "__len__") else a == b, f


@pytest.mark.parametrize("kind", ["plain", "alpha_outside", "linear_slerp", "negative_w"])
def test_line_row_jacobian_matches_central_differences(kind):
    """Both slerp branches: the regular one and Eigen's linear one (|q_D.w| >= 1 - eps)."""
    from test_ceres_restatement import _plus
    rng = np.random.default_rng(7 + len(kind))
    for trial in range(6):
        T = _rand_pose(rng)
        D = _rand_pose(rng, 0.5, 0.3)
        if kind == "linear_slerp":
            D[3:] = _unit(np.r_[rng.normal(0, 1e-9, 3), 1.0])
        if kind == "negative_w":
            D[3:] = -D[3:]
        n = 40
        P = rng.uniform(-30, 30, (n, 3))
        A = rng.uniform(-0.5, 1.5, n) if kind == "alpha_outside" else rng.uniform(0, 1, n)
        LA = rng.uniform(-30, 30, (n, 3))
        LB = LA + 0.2 * np.stack([_unit(v) for v in rng.normal(size=(n, 3))])
        J = OEN.line_jacobian(P, A, LA, LB, T, D)
        num = np.zeros_like(J)
        for k in range(12):
            h = 1e-6
            d = np.zeros(12)
            d[k] = h
            rp = OEN.line_residuals(P, A, LA, LB, _plus(T, d[:6]), _plus(D, d[6:]))
            rm = OEN.line_residuals(P, A, LA, LB, _plus(T, -d[:6]), _plus(D, -d[6:]))
            num[:, :, k] = (rp - rm) / (2 * h)
        scale = np.abs(J).max() + 1.0
        assert np.abs(J - num).max() < 2e-6 * scale, (kind, trial, np.abs(J - num).max())


def test_undistort_edges_shim_compiles(tmp_path):
    assert os.path.exists(_compile_shim(tmp_path))


# ------------------------------------------------------------------------------------------------------------------ GPU
_edge_maps = {}


def _edge_map(api, name):
    """Edge map of a case by extraction: ten static ring scans at random poses, inserted at their true poses (world frame)."""
    if name not in _edge_maps:
        from oracle import oracle as O
        from superodom_b200 import synth
        from test_edge_features import _edge_map_by_extraction
        case = get_case(name)
        ctx = api.Context(max_map_points=1 << 20, max_scan_points=262144, plane_res=0.2, line_res=0.1)
        poses = [synth.random_sensor_pose(case["scene"], 6100 + i, 12.0) for i in range(10)]
        _edge_maps[name] = _edge_map_by_extraction(ctx, O, case["scene"], case["cfg"]["sensor"], poses, 6200)
        ctx.close()
    return _edge_maps[name]


_flows = {}


def _flow(api, name, speed, yaw_rate, k=0):
    """The shipped flow on a moving raw scan: -> dict(surf, edges (both {x, y, z, time}), pose_true, pose_prev, prior, case)."""
    key = (name, speed, yaw_rate, k)
    if key not in _flows:
        from superodom_b200 import synth
        case = get_case(name)
        pose = synth.random_sensor_pose(case["scene"], 950 + k, 8.0)
        d = synth.make_moving_ring_scan(case["scene"], case["cfg"]["sensor"], pose, speed, yaw_rate, 60 + k)
        ctx = api.Context(max_map_points=1 << 20, max_scan_points=262144, plane_res=0.2, line_res=0.1)
        d["surf"] = ctx.scan_extract_uniform(d["points"], 5, SKIP, BLOCK_RANGE)
        d["edges"] = ctx.scan_extract_edges(d["points"])
        ctx.close()
        d["case"] = case
        _flows[key] = d
    return _flows[key]


def _ctx(api, name):
    case = get_case(name)
    ctx = api.Context(max_map_points=max(1 << 20, len(case["map_xyzi"]) * 2 + 1024), max_scan_points=262144,
                      plane_res=case["cfg"]["plane_res"], line_res=0.1)
    ctx.map_set_points(case["map_xyzi"])
    ctx.map_set_edge_points(_edge_map(api, name))
    return ctx


def _once(api, name, f):
    """f(ctx) on a fresh context of the case, closed afterwards"""
    ctx = _ctx(api, name)
    try:
        return f(ctx)
    finally:
        ctx.close()


def _iters(name):
    return (5, 2000) if name == "cfg1" else (20, 0)


@pytest.mark.gpu
def test_identity_cases(gpu_api):
    d = _flow(gpu_api, "cfg1", 1.5, 0.3)
    it, mf = _iters("cfg1")
    u = gpu_api.undistort(d["pose_prev"], 0.1)
    assert len(d["edges"]) > 200
    # no edge cloud: so_register_undistort
    a = _once(gpu_api, "cfg1", lambda c: c.register_undistort_edges(d["surf"], d["edges"][:0], d["prior"], u, it, mf))
    b = _once(gpu_api, "cfg1", lambda c: c.register_undistort(d["surf"], d["prior"], u, it, mf))
    assert a.n_iterations > 1
    _res_equal(a, b)
    m = gpu_api.motion(0.1)
    a = _once(gpu_api, "cfg1", lambda c: c.register_optimized_edges(d["surf"], d["edges"][:0], d["prior"], m, it, mf))
    b = _once(gpu_api, "cfg1", lambda c: c.register_optimized(d["surf"], d["prior"], m, it, mf))
    assert a.icp.n_iterations > 1
    _res_equal(a.icp, b.icp)
    assert bytes(a.motion) == bytes(b.motion) and bytes(a.pose_end) == bytes(b.pose_end)
    # mode 0, and all-zero times: so_register with the same edge cloud
    ref = _once(gpu_api, "cfg1", lambda c: c.register(d["surf"], d["prior"], it, mf, edge_xyzi=d["edges"]))
    assert ref.iter_n_edge[0] > 100
    u0 = gpu_api.undistort(d["pose_prev"], 0.1, mode=0)
    _res_equal(_once(gpu_api, "cfg1", lambda c: c.register_undistort_edges(d["surf"], d["edges"], d["prior"], u0, it, mf)), ref)
    s0, e0 = d["surf"].copy(), d["edges"].copy()
    s0[:, 3] = 0.0
    e0[:, 3] = 0.0
    ref0 = _once(gpu_api, "cfg1", lambda c: c.register(s0, d["prior"], it, mf, edge_xyzi=e0))
    for rot in (True, False):
        ur = gpu_api.undistort(d["pose_prev"], 0.1, rot)
        _res_equal(_once(gpu_api, "cfg1", lambda c: c.register_undistort_edges(s0, e0, d["prior"], ur, it, mf)), ref0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg1", "cfg2"])
def test_gpu_matches_oracle(gpu_api, name):
    it, mf = _iters(name)
    for speed, yaw in ((1.5, 0.3), (5.0, 0.5)):
        d = _flow(gpu_api, name, speed, yaw)
        ctx = _ctx(gpu_api, name)
        r = ctx.register_undistort_edges(d["surf"], d["edges"], d["prior"], gpu_api.undistort(d["pose_prev"], 0.1), it, mf)
        om = UEO.UndistortEdgesOracleMap(d["case"]["map_xyzi"], _edge_map(gpu_api, name))
        ro = om.register_undistort_edges(d["surf"], d["edges"], d["prior"], d["pose_prev"], 0.1, 1, d["case"]["cfg"]["plane_res"], it, mf,
                                         n_threads=16, line_res=0.1)
        assert r.n_iterations > 1 and r.iter_n_edge[0] > 100, (r.n_iterations, r.iter_n_edge[0])
        _assert_matches_oracle(r, ro)
        n = ro.n_iterations
        assert list(r.iter_n_edge[:n]) == list(ro.iter_n_edge[:n]) and list(r.hist_reject_line) == list(ro.hist_reject_line)
        ctx.close()


A2_LINE = float(np.sqrt(np.float32(3 * np.float32(0.1)))) ** 2          # TukeyLoss(sqrt(3 lineRes)), float sqrt (LidarSlam.cpp:263)


def _line_rows(ctx, edges, T, D, dt):
    """(P, alpha, a, b, w) of the lines so_correspond_edge fits at T on float(u_e(D)), and its rejection histogram"""
    ue = ON.warp_points(edges, D, dt)
    corr, hr = ctx.correspond_edge(np.concatenate([ue, edges[:, 3:4]], 1), T)
    ok = corr["w"] != 0.0
    return (edges[ok, :3].astype(np.float64), ON.alphas(edges[ok, 3], dt), corr["a"][ok], corr["b"][ok], corr["w"][ok]), hr


@pytest.mark.gpu
def test_optimized_stage_hook_matches_numpy(gpu_api):
    d = _flow(gpu_api, "cfg1", 5.0, 0.5)
    it, mf = _iters("cfg1")
    ctx = _ctx(gpu_api, "cfg1")
    motion_true = ON.compose(ON.inverse(d["pose_true"]), d["pose_next"])
    twisted = np.r_[0.3, -0.05, 0.01, -_unit(np.r_[0.01, -0.02, 0.05, 1.0])]
    for D in (motion_true, IDENTITY, twisted):
        H, g, cost = ctx.evaluate_optimized_edges(d["surf"], d["edges"], d["prior"], D, 0.1, mf)
        prob, n_ok = _plane_rows(ctx, d["surf"], d["prior"], D, 0.1, mf, _a2(d["case"]))
        rows, hr = _line_rows(ctx, d["edges"], d["prior"], D, 0.1)
        assert n_ok > 100 and hr[0] == len(rows[0]) > 100
        Hn, gn, cn = prob.normal_equations(np.asarray(d["prior"]), np.asarray(D))
        Hl, gl, cl = OEN.line_normal_equations(*rows, A2_LINE, np.asarray(d["prior"]), np.asarray(D))
        Hn, gn, cn = Hn + Hl, gn + gl, cn + cl
        assert np.abs(H - Hn).max() <= 1e-10 * np.abs(Hn).max()
        assert np.abs(g - gn).max() <= 1e-10 * np.abs(gn).max() + 1e-12
        assert abs(cost - cn) <= 1e-10 * abs(cn)
        # the line rows are there: the plane-only hook differs
        Hp, _, _ = ctx.evaluate_optimized(d["surf"], d["prior"], D, 0.1, mf)
        assert np.abs(H - Hp).max() > 1e-3 * np.abs(Hl).max()
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("speed,D0kind,info", [(5.0, "true", 0.0), (1.5, "identity", 0.0), (5.0, "identity", 0.01)])
def test_optimized_one_iteration_matches_numpy_solve(gpu_api, speed, D0kind, info):
    """max_icp_iters = 1: the device's solve on its own correspondences == the restatement's two-block solve on so_correspond's and
    so_correspond_edge's at (T0, D0), with the motion prior's multiplier counting planes plus lines."""
    d = _flow(gpu_api, "cfg1", speed, 0.3)
    D0 = ON.compose(ON.inverse(d["pose_true"]), d["pose_next"]) if D0kind == "true" else IDENTITY
    ctx = _ctx(gpu_api, "cfg1")
    lm = 4
    r = ctx.register_optimized_edges(d["surf"], d["edges"], d["prior"], gpu_api.motion(0.1, D0, [info] * 6), 1, 0, lm_max_iterations=lm)
    planes, n_ok = _plane_rows(ctx, d["surf"], d["prior"], D0, 0.1, 0, _a2(d["case"]))
    rows, hr = _line_rows(ctx, d["edges"], d["prior"], D0, 0.1)
    n_line = int(hr[0])
    prob = OEN.PlaneLineProblem(planes, *rows, A2_LINE)
    prob.D0 = np.r_[D0[:3], _unit(D0[3:])]
    prob.sqrt_info = np.sqrt((n_ok + n_line) * np.full(6, info))
    T, D, it, succ, unsucc, term = ON.solve(prob, d["prior"], D0, lm)
    assert (r.icp.iter_n_surf[0], r.icp.iter_n_edge[0]) == (n_ok, n_line) and n_line > 100
    assert list(r.icp.hist_reject_line) == list(hr)
    assert (r.icp.iter_lm_steps[0], r.icp.iter_lm_successful[0], r.icp.iter_lm_termination[0]) == (it, succ, term)
    assert np.abs(np.array(r.icp.pose_opt) - T).max() < 1e-8
    assert np.abs(np.array(r.motion) - D).max() < 1e-8
    ctx.close()


@pytest.mark.gpu
def test_registered_edges_insert(gpu_api):
    from oracle import oracle as O
    from superodom_b200.api import SuperOdomError
    d = _flow(gpu_api, "cfg1", 5.0, 0.5)
    it, mf = _iters("cfg1")
    u = gpu_api.undistort(d["pose_prev"], 0.1)
    # after so_register_undistort_edges: so_map_add_edge of T(pose) * pInit_e
    a, b = _ctx(gpu_api, "cfg1"), _ctx(gpu_api, "cfg1")
    ra = a.register_undistort_edges(d["surf"], d["edges"], d["prior"], u, it, mf)
    rb = b.register_undistort_edges(d["surf"], d["edges"], d["prior"], u, it, mf)
    pose = np.array(ra.pose)
    assert np.array_equal(pose, np.array(rb.pose))
    n0 = a.map_size()
    a.map_add_registered_edges(pose)
    pin = b.undistort_points(d["edges"], pose, u)
    b.map_add_edge(O.transform_scan_numpy(pin, pose))
    assert a.map_size() > n0 and np.array_equal(a.map_download(0), b.map_download(0))
    a.map_add_registered_scan(pose)                                # the surf record is untouched by the edge insert
    b.map_add_registered_scan(pose)
    assert np.array_equal(a.map_download(0), b.map_download(0))
    a.close(); b.close()
    # after so_register_optimized_edges: so_map_add_edge of T(pose) * u_e(D_opt)
    m = gpu_api.motion(0.1)
    a, b = _ctx(gpu_api, "cfg1"), _ctx(gpu_api, "cfg1")
    ra = a.register_optimized_edges(d["surf"], d["edges"], d["prior"], m, it, mf)
    rb = b.register_optimized_edges(d["surf"], d["edges"], d["prior"], m, it, mf)
    pose = np.array(ra.icp.pose)
    assert np.array_equal(pose, np.array(rb.icp.pose)) and ra.icp.iter_n_edge[0] > 100
    n0 = a.map_size()
    a.map_add_registered_edges(pose)
    uo = np.concatenate([ON.warp_points(d["edges"], np.array(ra.motion), 0.1), d["edges"][:, 3:4]], 1)
    b.map_add_edge(O.transform_scan_numpy(uo, pose))
    assert a.map_size() > n0 and np.array_equal(a.map_download(0), b.map_download(0))
    a.close(); b.close()
    pose = np.array(rb.icp.pose)
    # after so_register: so_map_add_scan_edge of the same cloud, bit for bit
    a, b = _ctx(gpu_api, "cfg1"), _ctx(gpu_api, "cfg1")
    ra = a.register(d["surf"], d["prior"], it, mf, edge_xyzi=d["edges"])
    b.register(d["surf"], d["prior"], it, mf, edge_xyzi=d["edges"])
    a.map_add_registered_edges(np.array(ra.pose))
    b.map_add_scan_edge(d["edges"], np.array(ra.pose))
    assert np.array_equal(a.map_download(0), b.map_download(0))
    # a scan-buffer call in between: SO_ERR_ARG; so_correspond_edge in between: SO_ERR_ARG for the edges only
    a.register_undistort_edges(d["surf"], d["edges"], d["prior"], u, it, mf)
    a.correspond(d["surf"], d["prior"], 0)
    with pytest.raises(SuperOdomError):
        a.map_add_registered_edges(pose)
    a.register_undistort_edges(d["surf"], d["edges"], d["prior"], u, it, mf)
    a.correspond_edge(d["edges"], d["prior"])
    with pytest.raises(SuperOdomError):
        a.map_add_registered_edges(pose)
    n0 = a.map_size()
    a.map_add_registered_scan(pose)
    assert a.map_size() > n0
    # a registration without an edge cloud: SO_OK, nothing inserted
    a.register_undistort(d["surf"], d["prior"], u, it, mf)
    n0 = a.map_size()
    a.map_add_registered_edges(pose)
    assert a.map_size() == n0
    a.close(); b.close()


@pytest.mark.gpu
def test_argument_errors_before_device_work(gpu_api):
    d = _flow(gpu_api, "cfg1", 1.5, 0.3)
    it, mf = _iters("cfg1")
    u = gpu_api.undistort(d["pose_prev"], 0.1)
    a, b = _ctx(gpu_api, "cfg1"), _ctx(gpu_api, "cfg1")
    ra = a.register_undistort_edges(d["surf"], d["edges"], d["prior"], u, it, mf)
    b.register_undistort_edges(d["surf"], d["edges"], d["prior"], u, it, mf)
    s = np.ascontiguousarray(d["surf"], np.float32)
    e = np.ascontiguousarray(d["edges"], np.float32)
    pose = np.ascontiguousarray(d["prior"], np.float64)
    o = a._opts(it, mf)
    r = gpu_api.IcpResult()
    P = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    call = a.L.so_register_undistort_edges
    n0 = a.kernel_launches()
    assert call(a.h, P(s), len(s), None, 5, 16, 12, 12, P(pose), C.byref(u), C.byref(o), C.byref(r)) == -1           # NULL edge cloud
    assert call(a.h, P(s), len(s), P(e), 262145, 16, 12, 12, P(pose), C.byref(u), C.byref(o), C.byref(r)) == -3      # n_edge > capacity
    assert call(a.h, P(s), len(s), P(e), len(e), 16, 12, 16, P(pose), C.byref(u), C.byref(o), C.byref(r)) == -1      # time outside the record
    bad = gpu_api.undistort(d["pose_prev"], -0.1)
    assert call(a.h, P(s), len(s), P(e), len(e), 16, 12, 12, P(pose), C.byref(bad), C.byref(o), C.byref(r)) == -1
    bad = gpu_api.undistort(d["pose_prev"], 0.1, mode=2)
    assert call(a.h, P(s), len(s), P(e), len(e), 16, 12, 12, P(pose), C.byref(bad), C.byref(o), C.byref(r)) == -1
    mo = gpu_api.motion(0.1)
    rm = gpu_api.MotionResult()
    call = a.L.so_register_optimized_edges
    assert call(a.h, P(s), len(s), None, 5, 16, 12, 12, P(pose), C.byref(mo), C.byref(o), C.byref(rm)) == -1
    assert call(a.h, P(s), len(s), P(e), 262145, 16, 12, 12, P(pose), C.byref(mo), C.byref(o), C.byref(rm)) == -3
    assert call(a.h, P(s), len(s), P(e), len(e), 16, 12, 12, P(pose), C.byref(gpu_api.motion(-0.1)), C.byref(o), C.byref(rm)) == -1
    op = a._opts(it, mf, pose_prior=(1.0, (0.1, 0.1, 0.1)))
    assert call(a.h, P(s), len(s), P(e), len(e), 16, 12, 12, P(pose), C.byref(mo), C.byref(op), C.byref(rm)) == -1
    H, g, cst = np.zeros(144), np.zeros(12), C.c_double()
    assert a.L.so_evaluate_optimized_edges(a.h, P(s), len(s), None, 5, 16, 12, 12, P(pose), P(np.array(IDENTITY)), 0.1, mf, P(H), P(g),
                                           C.byref(cst)) == -1
    assert a.kernel_launches() == n0
    # the registered scan and edge cloud are the ones of the first call
    for c in (a, b):
        c.map_add_registered_edges(np.array(ra.pose))
        c.map_add_registered_scan(np.array(ra.pose))
    assert np.array_equal(a.map_download(0), b.map_download(0))
    a.close(); b.close()


def _ring_trajectory(api, n, speed, yaw_rate):
    """n moving VLP-16 ring scans along one constant-velocity arc of cfg1's scene -> [(surf, edges, pose_true, prior)]."""
    from superodom_b200 import synth
    scene = get_case("cfg1")["scene"]
    ctx = api.Context(max_map_points=1 << 20, max_scan_points=262144, plane_res=0.2, line_res=0.1)
    for seed in range(20):
        p = synth.random_sensor_pose(scene, 1400 + seed, 6.0)
        seq = []
        for k in range(n):
            if not scene.free(p[:3]):
                break
            d = synth.make_moving_ring_scan(scene, "vlp16", p, speed, yaw_rate, 700 + k)
            seq.append((ctx.scan_extract_uniform(d["points"], 5, SKIP, BLOCK_RANGE), ctx.scan_extract_edges(d["points"]), d["pose_true"], d["prior"]))
            p = d["pose_next"]
        if len(seq) == n:
            ctx.close()
            return seq
    raise RuntimeError("no free arc")


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rotation", [(1, 1), (1, 0), (2, 1)])
def test_shim_undistorted_edge_sequence_matches_abi(tmp_path, gpu_api, mode, rotation):
    exe = _compile_shim(tmp_path)
    seq = _ring_trajectory(gpu_api, 5, 2.0, 0.3 if rotation else 0.0)
    priors = [seq[0][2]] + [s[3] for s in seq[1:]]
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiif", len(seq), 5, 0, 0.2))
        for (surf, edges, _, _), p in zip(seq, priors):
            f.write(np.asarray(p, np.float64).tobytes())
            for cloud in (surf, edges):
                f.write(struct.pack("<i", len(cloud)))
                f.write(np.ascontiguousarray(cloud, np.float32).tobytes())
    out = subprocess.run([exe, str(path), str(rotation), str(tmp_path / "map.bin"), str(mode)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows = [list(map(float, ln.split())) for ln in out.stdout.strip().splitlines()]
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=1 << 17, plane_res=0.2, line_res=0.1)
    ctx.map_set_origin(priors[0][:3])
    ctx.map_add_scan_edge(seq[0][1], priors[0])
    ctx.map_add_scan(seq[0][0], priors[0])
    prev, t_prev = np.asarray(priors[0]), 0.0
    n_edge_rows = 0
    for s in range(1, len(seq)):
        t = 0.1 * s
        if mode == 1:
            r = ctx.register_undistort_edges(seq[s][0], seq[s][1], priors[s], gpu_api.undistort(prev, t - t_prev, bool(rotation)), 5, 0)
        else:                                                     # the shim's motion prior D0 = prev^-1 * prior, information 0
            ro = ctx.register_optimized_edges(seq[s][0], seq[s][1], priors[s], gpu_api.motion(t - t_prev, rows[s][12:19], [0.0] * 6), 5, 0)
            assert np.array_equal(np.array(ro.motion), np.array(rows[s][19:26])), s
            r = ro.icp
        assert np.array_equal(np.array(r.pose), np.array(rows[s][1:8])), s          # shim == ABI, bit for bit
        assert int(rows[s][8]) == r.n_iterations
        if r.status == 1:
            continue
        n_edge_rows += r.iter_n_edge[r.n_iterations - 1]
        ctx.map_add_registered_edges(np.array(r.pose))
        ctx.map_add_registered_scan(np.array(r.pose))
        assert int(rows[s][9]) == ctx.map_size()
        prev, t_prev = np.array(r.pose), t
    assert n_edge_rows > 0
    shim_map = np.fromfile(tmp_path / "map.bin", np.float32).reshape(-1, 4)
    assert np.array_equal(shim_map, ctx.map_download(0))
    ctx.close()


def corridor_arms(api, speeds=(5.0, 10.0), n_scans=6, log=None, timing_repeat=0):
    """Moving OS1-128 ring scans in the corridor taken through extraction, registered four ways: (a) edges without compensation (the
    shim's path before the compensated edge registrations), (b) planes with APPROXIMATED, (c) edges with APPROXIMATED, (d) edges with
    OPTIMIZED (motion prior D0 = T_prev^-1 * prior, information 0, as the shim).  -> rows of position errors (m) and device times (ms)
    per arm; with timing_repeat > 0 also the median device time per arm over that many repeats of the last scan, on the same map."""
    from superodom_b200 import synth
    sc = synth.make_corridor_scene()
    raw = synth.sample_surfaces(sc, 0.2)
    surf_map = synth.voxel_filter_blocks(np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1), 0.2)
    ctx = api.Context(max_map_points=max(1 << 20, 2 * len(surf_map)), max_scan_points=262144, plane_res=0.2, line_res=0.1)
    ctx.map_set_points(surf_map)
    ctx.map_set_resolution(0.1, 0.2)
    for i, x in enumerate(np.arange(-40.0, 40.1, 8.0)):
        T = np.array([x + 0.7, 0.3 * ((i % 3) - 1), 0.1, 0.0, 0.0, 0.0, 1.0])
        ctx.map_add_scan_edge(ctx.scan_extract_edges(synth.make_ring_scan(sc, "os1_128", T, 8000 + i)), T)
    rng = np.random.default_rng(8400)
    rows = []
    for speed in speeds:
        for s in range(n_scans):
            yaw = rng.uniform(-0.2, 0.2)
            T = np.array([rng.uniform(-20, 20), rng.uniform(-0.8, 0.8), rng.uniform(-0.3, 0.3), 0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)])
            d = synth.make_moving_ring_scan(sc, "os1_128", T, speed, 0.3, 8500 + s)
            surf = ctx.scan_extract_uniform(d["points"], 5, SKIP, BLOCK_RANGE)
            edges = ctx.scan_extract_edges(d["points"])
            u = api.undistort(d["pose_prev"], 0.1)
            m = api.motion(0.1, ON.compose(ON.inverse(d["pose_prev"]), d["prior"]))
            arms = dict(a=lambda: ctx.register(surf, d["prior"], 20, 0, edge_xyzi=edges),
                        b=lambda: ctx.register_undistort(surf, d["prior"], u, 20, 0),
                        c=lambda: ctx.register_undistort_edges(surf, edges, d["prior"], u, 20, 0),
                        d=lambda: ctx.register_optimized_edges(surf, edges, d["prior"], m, 20, 0).icp)
            res = {k: f() for k, f in arms.items()}
            row = dict(speed=speed, n_surf=len(surf), n_edges=len(edges))
            for k, r in res.items():
                row["err_" + k] = float(np.linalg.norm(np.array(r.pose)[:3] - d["pose_true"][:3]))
                row["rot_" + k] = quat_angle(np.array(r.pose)[3:], d["pose_true"][3:])
                row["ms_" + k] = r.time_ms
                row["status_" + k] = r.status
            rows.append(row)
            if log:
                log(row)
    timing = {}
    if timing_repeat:
        for k, f in arms.items():
            f()
            t = [f() for _ in range(timing_repeat)]
            timing[k] = dict(device_ms=float(np.median([r.time_ms for r in t])), total_ms=float(np.median([r.time_total_ms for r in t])),
                             n_iterations=int(t[0].n_iterations))
        timing["n_surf"], timing["n_edges"] = len(surf), len(edges)
    ctx.close()
    return (rows, timing) if timing_repeat else rows


@pytest.mark.gpu
def test_corridor_compensated_edges_beat_uncompensated_edges(gpu_api):
    rows = corridor_arms(gpu_api, log=print)
    for r in rows:
        assert r["status_a"] == r["status_b"] == r["status_c"] == r["status_d"] == 0, r
        assert r["err_c"] < r["err_a"] and r["err_d"] < r["err_a"], r

"""Global localization against the prior map (so_localize_global): x/y/z voxel shifts x yaw steps of the scan scored against an
occupancy bitmap of the surf map, the best hypotheses refined by the ordinary batched registration.

CPU: the host-only size / argument checks, the struct layouts and the C++ shim build.
GPU: scores equal the numpy restatement element for element, recovery from metres and any heading away, the refinement is
so_register_batch bit for bit, determinism, no side effects, soft statuses, shim == C ABI."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import global_localization_numpy as GN
from conftest import get_case, quat_angle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO_ERR_ARG, SO_ERR_CAPACITY = -1, -3
SO_STATUS_NOT_ENOUGH_FEATURES, SO_STATUS_NO_CORRESPONDENCES = 1, 2
DEG = math.pi / 180.0


# --------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("region", [
    dict(),                                                                   # defaults: full circle, nothing shifted
    dict(half_x=10.0, half_y=10.0, yaw_half=math.pi),                         # the default search of the benchmark
    dict(half_x=1.0, half_y=1.0, half_z=0.25, yaw_half=4.0, yaw_step=15 * DEG, max_range=20.0),
    dict(half_x=2.0, half_y=0.6, yaw_half=20 * DEG),                          # partial yaw: 2 * 10 + 1 steps
    dict(half_x=0.3, half_y=3.3, half_z=1.0, yaw_half=5 * DEG, res=0.5, yaw_step=1 * DEG, max_range=12.3, dilate=2),
    dict(yaw_half=math.pi, yaw_step=7 * DEG),                                 # 360 / 7 rounds to 51 steps
])
def test_size_matches_the_formulas(region):
    from superodom_b200 import api
    dims, n_hyp, nbytes = api.localize_global_size(**region)
    P = GN.plan(**region)
    assert dims == (P["nx"], P["ny"], P["nz"], P["nyaw"])
    assert n_hyp == P["n_hyp"] == P["nx"] * P["ny"] * P["nz"] * P["nyaw"]
    assert nbytes == P["bitmap_bytes"]
    res = region.get("res", 0.25)
    I = math.floor(region.get("half_x", 0.0) / res)
    assert P["nx"] == 2 * I + 1
    if region.get("yaw_half", 0.0) >= math.pi:
        assert P["nyaw"] == round(2 * math.pi / region.get("yaw_step", 2 * DEG))
    else:
        assert P["nyaw"] == 2 * math.floor(region.get("yaw_half", 0.0) / region.get("yaw_step", 2 * DEG)) + 1


def test_default_search_size():
    from superodom_b200 import api
    dims, n_hyp, nbytes = api.localize_global_size(half_x=10.0, half_y=10.0, yaw_half=math.pi)
    assert dims == (81, 81, 1, 180) and n_hyp == 1_180_980
    assert nbytes == 4 * 13 * 401 * 321                    # 401 voxels per row in 13 words, 401 rows, 321 planes


@pytest.mark.parametrize("bad", [
    dict(half_x=-1.0), dict(half_y=-0.1), dict(half_z=-2.0), dict(half_x=float("nan")), dict(half_y=float("inf")),
    dict(yaw_half=-0.1), dict(res=-0.25), dict(yaw_step=-1.0), dict(max_range=-40.0), dict(res=float("nan")),
    dict(k=-1), dict(k=65), dict(score_points=-1), dict(score_points=4097), dict(dilate=-1), dict(dilate=9),
    dict(nms_xy=-1.0), dict(nms_yaw=float("nan")),
])
def test_size_rejects_invalid_arguments(bad):
    from superodom_b200 import api
    with pytest.raises(api.SuperOdomError) as ei:
        api.localize_global_size(**bad)
    assert ei.value.code == SO_ERR_ARG


def test_size_flags_capacity_limits():
    from superodom_b200 import api
    # 2^24 hypotheses: 4097 x 4097 shifts = 16.8 M > 2^24 with a single yaw
    with pytest.raises(api.SuperOdomError) as ei:
        api.localize_global_size(half_x=512.0, half_y=512.0, res=0.25)
    assert ei.value.code == SO_ERR_CAPACITY
    # 81 x 81 shifts x 2557 yaws = 16 776 477 <= 2^24 passes; one more yaw step does not
    dims, n, _ = api.localize_global_size(half_x=10.0, half_y=10.0, yaw_half=math.pi, yaw_step=2 * math.pi / 2557)
    assert dims == (81, 81, 1, 2557) and n == 16_776_477
    with pytest.raises(api.SuperOdomError) as ei:
        api.localize_global_size(half_x=10.0, half_y=10.0, yaw_half=math.pi, yaw_step=2 * math.pi / 2558)
    assert ei.value.code == SO_ERR_CAPACITY
    # bitmap above 2^32 bits: a 400 m reach at 5 cm
    with pytest.raises(api.SuperOdomError) as ei:
        api.localize_global_size(res=0.05, max_range=400.0)
    assert ei.value.code == SO_ERR_CAPACITY
    L = api.load_library()
    assert L.so_localize_global_size(None, None, None, None) == SO_ERR_ARG


def test_struct_layouts_match_header(tmp_path):
    from superodom_b200 import api
    f = tmp_path / "sz.c"
    f.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "superodom_b200.h"\n'
                 'int main(void){printf("%zu %zu %zu %zu %zu\\n", sizeof(so_global_opts), sizeof(so_global_candidate), '
                 'sizeof(so_global_result), offsetof(so_global_result, icp), offsetof(so_global_opts, nms_xy));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(f), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)]).split()))
    assert got == (C.sizeof(api.GlobalOpts), C.sizeof(api.GlobalCandidate), C.sizeof(api.GlobalResult),
                   api.GlobalResult.icp.offset, api.GlobalOpts.nms_xy.offset)


def _build_shim(tmp_path):
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "global_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "global_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


def test_shim_with_global_localize_compiles(tmp_path):
    assert os.path.exists(_build_shim(tmp_path))


# --------------------------------------------------------------------------------------------------------------- GPU
_TIME_FIELDS = ("time_ms", "time_total_ms")


def _icp_bits(r):
    from superodom_b200 import api
    c = api.IcpResult.from_buffer_copy(bytes(r))
    for f in _TIME_FIELDS:
        setattr(c, f, 0.0)
    return bytes(c)


def _global_bits(res, cands):
    from superodom_b200 import api
    r = api.GlobalResult.from_buffer_copy(bytes(res))
    for f in ("time_raster_ms", "time_dilate_ms", "time_score_ms", "time_sort_ms", "time_refine_ms", "time_total_ms"):
        setattr(r, f, 0.0)
    for f in _TIME_FIELDS:
        setattr(r.icp, f, 0.0)
    return bytes(r), [bytes(c) for c in cands]


def _yaw_quat(yaw):
    return np.array([0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2)])


def _with_rp(center, roll, pitch):
    """center with its rotation replaced by yaw(center) (x) roll/pitch."""
    from superodom_b200 import synth
    yaw = GN.tf2_yaw(center[3:])
    q = synth.quat_mul(_yaw_quat(yaw), synth.quat_mul(synth.quat_from_rotvec(np.array([roll, 0, 0])),
                                                       synth.quat_from_rotvec(np.array([0, pitch, 0]))))
    return np.r_[center[:3], q / np.linalg.norm(q)]


def _ctx(api, case, max_batch=16, **kw):
    ctx = api.Context(max_map_points=max(1 << 20, len(case["map_xyzi"]) + (1 << 18)), max_scan_points=262144,
                      plane_res=case["cfg"]["plane_res"], max_batch=max_batch, **kw)
    ctx.map_set_points(case["map_xyzi"])
    return ctx


def _check_scores(gpu_api, case, center, **region):
    ctx = _ctx(gpu_api, case, max_batch=1)
    g = gpu_api.global_opts(**region)
    got, n_pts = ctx.localize_scores(case["scan_xyzi"], center, g)
    want, n_want = GN.localize_scores_numpy(case["scan_xyzi"], center, ctx.map_download(0)[:, :3], **region)
    assert n_pts == n_want > 0
    assert got.shape == want.shape
    bad = np.argwhere(got != want)
    assert len(bad) == 0, (len(bad), bad[:5], got[tuple(bad[0])], want[tuple(bad[0])])
    assert got.max() > 0
    ctx.close()
    return got, n_pts


@pytest.mark.gpu
def test_scores_exact_cfg1_vlp16(gpu_api):
    """9 x 9 shifts, 3 z levels, 24 yaws (full circle at 15 deg), roll and pitch 3 / -2 deg; max_range 15 m cuts through the
    VLP-16 scan, so many score points sit at the edge of the bitmap box."""
    case = get_case("cfg1")
    center = _with_rp(case["pose_true"], 3 * DEG, -2 * DEG)
    center[:3] += [0.37, -0.21, 0.05]
    region = dict(half_x=1.0, half_y=1.0, half_z=0.25, yaw_half=math.pi, yaw_step=15 * DEG, max_range=15.0)
    scores, _ = _check_scores(gpu_api, case, center, **region)
    assert scores.shape == (24, 3, 9, 9)
    pts = GN.score_points(case["scan_xyzi"], 1024, 15.0)
    r = np.linalg.norm(pts[:, :3].astype(np.float64), axis=1)
    assert (r > 14.0).sum() > 20                                             # points reaching into the box's outermost voxels


@pytest.mark.gpu
def test_scores_exact_cfg2_block_face_and_yaw_wrap(gpu_api):
    """cfg2: a region straddling the x = 25 m block face, a yaw range wrapping through +-pi, dilation 2, 2048 score points."""
    case = get_case("cfg2")
    center = np.r_[24.6, -3.1, case["pose_true"][2], _yaw_quat(175 * DEG)]
    center = _with_rp(center, -1.5 * DEG, 2.5 * DEG)
    region = dict(half_x=2.0, half_y=1.5, yaw_half=20 * DEG, dilate=2, score_points=2048, max_range=30.0)
    scores, n = _check_scores(gpu_api, case, center, **region)
    assert scores.shape == (21, 1, 13, 17) and n > 1024


def _recovery_center(case, i):
    rng = np.random.default_rng(7100 + i)
    t = case["pose_true"]
    d = rng.uniform(-8.0, 8.0, 2)
    dyaw = rng.uniform(-math.pi, math.pi)
    from superodom_b200 import synth
    q = synth.quat_mul(_yaw_quat(dyaw), t[3:])
    return np.r_[t[0] + d[0], t[1] + d[1], t[2], q / np.linalg.norm(q)]


@pytest.mark.gpu
def test_recovery_cfg2_os1_128(gpu_api):
    """8 OS1-128 scans, centre up to 8 m and any heading away from the truth, default search (half 10 m, full circle): every pose
    within 5 cm / 0.5 deg.  Prints winner and runner-up SUCCESS counts (the aisles repeat every 5 m)."""
    case0 = get_case("cfg2")
    ctx = _ctx(gpu_api, case0)
    g = gpu_api.global_opts(half_x=10.0, half_y=10.0, yaw_half=math.pi)
    errors = []
    for i in range(8):
        case = get_case("cfg2", i)
        center = _recovery_center(case, i)
        pose, res, cands = ctx.localize_global(case["scan_xyzi"], center, 20, g)
        dt = float(np.linalg.norm(pose[:3] - case["pose_true"][:3]))
        da = float(quat_angle(pose[3:], case["pose_true"][3:])) / DEG
        ns = sorted((c.n_success for c in cands if c.status == 0), reverse=True)
        # the best candidate that converged somewhere else (> 0.5 m or > 5 deg from the winner): the margin against a wrong aisle
        other = [c.n_success for c in cands if c.status == 0 and (np.linalg.norm(np.array(c.pose)[:3] - pose[:3]) > 0.5 or
                                                                   quat_angle(np.array(c.pose)[3:], pose[3:]) > 5 * DEG)]
        print(f"recovery scan {i}: status {res.status} winner {res.winner} of {res.n_candidates} best score {res.best_score} of "
              f"{res.n_score_points}, err {dt:.4f} m {da:.4f} deg, SUCCESS winner {ns[0] if ns else 0} runner-up {ns[1] if len(ns) > 1 else 0} "
              f"best elsewhere {max(other) if other else 0}, offset {np.linalg.norm(center[:2] - case['pose_true'][:2]):.2f} m")
        errors.append((i, res.status, dt, da))
    ctx.close()
    for i, st, dt, da in errors:
        assert st == 0 and dt < 0.05 and da < 0.5, errors


@pytest.mark.gpu
def test_refinement_is_register_batch_and_deterministic(gpu_api):
    """The winner's so_icp_result == so_register_batch from the winning prior, bit for bit; two calls are bit-identical; a
    max_batch 1 context gives the same result and candidate list as a max_batch 16 one."""
    case = get_case("cfg2", 1)
    center = _recovery_center(case, 1)
    g = gpu_api.global_opts(half_x=10.0, half_y=10.0, yaw_half=math.pi)
    ctx = _ctx(gpu_api, case, max_batch=16)
    pose, res, cands = ctx.localize_global(case["scan_xyzi"], center, 20, g)
    assert res.status == 0 and res.n_candidates == len(cands) > 1 and res.winner >= 0
    prior = np.array(cands[res.winner].prior)
    rb = ctx.register_batch(np.ascontiguousarray(case["scan_xyzi"], np.float32), [len(case["scan_xyzi"])], prior[None], 20)
    assert _icp_bits(rb[0]) == _icp_bits(res.icp)
    assert np.array_equal(np.array(rb[0].pose), pose)
    _, res2, cands2 = ctx.localize_global(case["scan_xyzi"], center, 20, g)
    assert _global_bits(res, cands) == _global_bits(res2, cands2)
    ctx.close()
    ctx1 = _ctx(gpu_api, case, max_batch=1)
    _, res1, cands1 = ctx1.localize_global(case["scan_xyzi"], center, 20, g)
    assert _global_bits(res, cands) == _global_bits(res1, cands1)
    ctx1.close()


@pytest.mark.gpu
def test_no_side_effects(gpu_api):
    """Map unchanged, pose sink rows and cursor unchanged, a following so_register equals a fresh context's, and the registered-scan
    insert at the returned pose equals so_map_add_scan of the same cloud."""
    import torch
    case = get_case("cfg2", 2)
    scan = case["scan_xyzi"]
    center = _recovery_center(case, 2)
    g = gpu_api.global_opts(half_x=10.0, half_y=10.0, yaw_half=math.pi)
    ctx = _ctx(gpu_api, case)
    before = ctx.map_download(0).copy()
    sink = torch.full((8, 8), -7.0, dtype=torch.float64, device="cuda")
    ctx.set_pose_sink(sink.data_ptr(), 8, 3)
    pose, res, _ = ctx.localize_global(scan, center, 20, g)
    torch.cuda.synchronize()
    assert res.status == 0
    assert np.array_equal(ctx.map_download(0), before)
    assert bool((sink == -7.0).all())
    # the next registration appends at row 3: the cursor did not move
    prior = case["pose_prior"]
    r = ctx.register(scan, prior, 20)
    torch.cuda.synchronize()
    rows = sink.cpu().numpy()
    assert np.array_equal(rows[3, :7], np.array(r.pose_opt)) and (rows[4:] == -7.0).all() and (rows[:3] == -7.0).all()
    ctx.set_pose_sink(None)
    fresh = _ctx(gpu_api, case)
    rf = fresh.register(scan, prior, 20)
    assert _icp_bits(r) == _icp_bits(rf)
    fresh.close()
    # registered-scan insert after the global localization == so_map_add_scan of the same cloud
    ctx_a = _ctx(gpu_api, case)
    pose_a, res_a, _ = ctx_a.localize_global(scan, center, 20, g)
    assert np.array_equal(pose_a, pose)
    ctx_a.map_add_registered_scan(pose_a)
    ctx_b = _ctx(gpu_api, case)
    ctx_b.map_add_scan(scan, pose_a)
    assert np.array_equal(ctx_a.map_download(0), ctx_b.map_download(0))
    assert len(ctx_a.map_download(0)) > len(before)
    # ... and so_register_prefiltered refuses to run on the overwritten scan buffers
    ctx_a.scan_prefilter(scan, 0.1, 0.2, auto_voxel_size=False, download=False)
    ctx_a.localize_global(scan, center, 20, g)
    with pytest.raises(gpu_api.SuperOdomError):
        ctx_a.register_prefiltered(prior, 20)
    for c in (ctx, ctx_a, ctx_b):
        c.close()


@pytest.mark.gpu
def test_soft_statuses(gpu_api):
    """A region with no map: SO_STATUS_NO_CORRESPONDENCES and the centre pose.  An empty map does not fault.  A map too sparse
    for hasEnoughFeatures: SO_STATUS_NOT_ENOUGH_FEATURES."""
    case = get_case("cfg1")
    g = gpu_api.global_opts(half_x=2.0, half_y=2.0, yaw_half=math.pi, max_range=20.0)
    ctx = _ctx(gpu_api, case, max_batch=4)
    far = np.r_[400.0, -300.0, 0.0, _yaw_quat(0.3)]
    pose, res, cands = ctx.localize_global(case["scan_xyzi"], far, 5, g)
    assert res.status == SO_STATUS_NO_CORRESPONDENCES and res.best_score == 0 and res.n_candidates == 0 and res.winner == -1
    assert np.array_equal(pose, far)
    ctx.close()
    empty = gpu_api.Context(max_map_points=1 << 16, max_scan_points=1 << 17, plane_res=0.2)
    pose, res, _ = empty.localize_global(case["scan_xyzi"], case["pose_prior"], 5, g)
    assert res.status == SO_STATUS_NO_CORRESPONDENCES and np.array_equal(pose, case["pose_prior"])
    pose, res, _ = empty.localize_global(np.zeros((0, 4), np.float32), case["pose_prior"], 5, g)
    assert res.status == SO_STATUS_NO_CORRESPONDENCES
    # 40 map points: scores > 0, but every candidate fails hasEnoughFeatures (5x5 block neighbourhood holds <= 50 points)
    sparse = gpu_api.Context(max_map_points=1 << 16, max_scan_points=1 << 17, plane_res=0.2)
    sparse.map_set_points(case["map_xyzi"][::max(1, len(case["map_xyzi"]) // 40)][:40])
    pose, res, cands = sparse.localize_global(case["scan_xyzi"], case["pose_true"], 5, g)
    assert res.best_score > 0 and res.n_candidates > 0
    assert res.status == SO_STATUS_NOT_ENOUGH_FEATURES and all(c.status == SO_STATUS_NOT_ENOUGH_FEATURES for c in cands)
    assert np.array_equal(pose, case["pose_true"])
    # argument errors before any device work
    with pytest.raises(gpu_api.SuperOdomError):
        sparse.localize_global(case["scan_xyzi"], np.r_[np.nan, 0, 0, 0, 0, 0, 1.0], 5, g)
    with pytest.raises(gpu_api.SuperOdomError):
        sparse.localize_global(case["scan_xyzi"], case["pose_true"], 5, gpu_api.global_opts(k=65))
    empty.close()
    sparse.close()


@pytest.mark.gpu
def test_shim_global_localize_matches_abi(tmp_path, gpu_api):
    """LidarSLAM::globalLocalize (C++ shim) returns the C ABI's pose bit for bit and sets T_w_lidar and last_T_w_lidar."""
    exe = _build_shim(tmp_path)
    case = get_case("cfg1", 1)
    center = _recovery_center(case, 1)
    opts = gpu_api.global_opts(half_x=8.0, half_y=8.0, yaw_half=math.pi, max_range=30.0)
    m = np.ascontiguousarray(case["map_xyzi"], np.float32)
    s = np.ascontiguousarray(case["scan_xyzi"], np.float32)
    iters, cap = 5, 2000
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiiif", len(m), len(s), iters, cap, 0.2))
        f.write(np.asarray(center, np.float64).tobytes())
        f.write(bytes(opts))
        f.write(m.tobytes())
        f.write(s.tobytes())
    out = subprocess.run([exe, str(path)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    l1, l2 = out.stdout.strip().splitlines()
    rc, winner, *pose_s = l1.split()
    ctx = gpu_api.Context(max_map_points=1 << 22, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    ctx.map_add_surf(m)
    pose, res, _ = ctx.localize_global(s, center, iters, opts, max_surface_features=cap)
    assert int(rc) == res.status == 0 and int(winner) == res.winner
    assert np.array_equal(np.array([float(v) for v in pose_s]), pose)
    assert np.array_equal(np.array([float(v) for v in l2.split()]), pose)
    assert np.linalg.norm(pose[:3] - case["pose_true"][:3]) < 0.05
    ctx.close()

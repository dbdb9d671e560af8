"""Within-scan motion compensation (so_register_undistort*, mode APPROXIMATED).

CPU: the numpy restatement of pInit (undistort_numpy.py) on its own terms, the motion-distorted scan generator, the ABI layout.
GPU: the device pInit against the restatement bit for bit; undistorted registration against so_register where the two must
agree (all times zero, mode 0), batches against single calls, the undistorted map insert, the prefiltered path, argument errors,
and the accuracy gain on motion-distorted scans."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import undistort_numpy as UN
from conftest import get_case, quat_angle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rand_pose(rng, scale=1.0):
    from superodom_b200 import synth
    q = synth.quat_from_rotvec(rng.normal(0, scale, 3))
    return np.concatenate([rng.normal(0, 5 * scale, 3), q / np.linalg.norm(q)])


def _cases():
    """(cloud [n,4] x,y,z,time, pose, prev_pose, dt, rotation): alpha > 1, both rotation settings, a rotation small enough for
    slerp's linear branch, a negative quaternion dot, non-finite times."""
    from superodom_b200 import synth
    rng = np.random.default_rng(5)
    out = []
    for k in range(8):
        n = 5000
        pts = rng.uniform(-60, 60, (n, 3))
        t = rng.uniform(0.0, 0.1, n)
        if k % 4 == 1:
            t = rng.uniform(-0.05, 0.3, n)                        # alpha beyond [0, 1]: extrapolation
        cloud = np.concatenate([pts, t[:, None]], 1).astype(np.float32)
        if k == 3:
            cloud[:5, 3] = [np.nan, np.inf, -np.inf, 0.0, -0.0]
        prev = _rand_pose(rng)
        w = rng.normal(0, 0.2, 3)
        if k == 2:
            w = np.array([1e-9, -2e-9, 5e-10])                    # |q_D.w| >= 1 - eps: Eigen's linear branch
        qc = synth.quat_mul(prev[3:], synth.quat_from_rotvec(w))
        qc /= np.linalg.norm(qc)
        if k in (4, 5):
            qc = -qc                                              # same rotation, negative dot with the previous quaternion
        cur = np.concatenate([prev[:3] + rng.normal(0, 1.0, 3), qc])
        out.append((cloud, cur, prev, 0.1 if k != 6 else 0.05, k % 2 == 0 or k == 5))
    return out


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_numpy_zero_time_is_identity():
    for cloud, cur, prev, dt, rot in _cases():
        c = cloud.copy()
        c[:, 3] = 0.0
        p = UN.undistort_points(c, cur, prev, dt, rot)
        assert np.array_equal(p, c[:, :3])


def test_numpy_end_of_interval_is_the_relative_motion():
    """alpha = 1: pInit = D * p (T_prev^-1 T_cur), here checked against a rotation-matrix evaluation."""
    from superodom_b200 import synth
    for cloud, cur, prev, dt, rot in _cases():
        c = cloud.copy()
        c[:, 3] = np.float32(dt) if np.float32(dt) == dt else 0.0
        if not c[0, 3]:
            continue
        p = UN.undistort_points(c, cur, prev, dt, True)
        Rp, Rc = synth.quat_to_R(prev[3:]), synth.quat_to_R(cur[3:])
        ref = c[:, :3].astype(np.float64) @ (Rp.T @ Rc).T + Rp.T @ (cur[:3] - prev[:3])
        assert np.abs(p - ref).max() < 1e-4


def test_numpy_linear_branch_and_sign():
    cases = _cases()
    qD, _ = UN.delta(cases[2][2], cases[2][1])
    assert abs(qD[3]) >= 1.0 - UN.EPS
    qD, _ = UN.delta(cases[4][2], cases[4][1])
    assert qD[3] < 0.0


def test_moving_scan_translation_only_is_undone_exactly():
    """With no yaw rate the constant-velocity model is exact: T_true * pInit (D from the scan's own motion) puts every point where
    it was hit, up to float rounding -- the same world points as the per-column poses give."""
    from superodom_b200 import synth
    scene, _ = get_case("tiny")["scene"], None
    pose = synth.random_sensor_pose(scene, 901, 4.0)
    d = synth.make_moving_scan(scene, "vlp16", pose, 3.0, 0.0, 11, range_noise=0.0)
    s = d["scan_xyzi"]
    assert 0.0 <= s[:, 3].min() and s[:, 3].max() < 0.1
    p = UN.undistort_points(s, d["pose_true"], d["pose_prev"], 0.1, True)
    R = synth.quat_to_R(pose[3:])
    world = p.astype(np.float64) @ R.T + pose[:3]
    v = R @ np.array([3.0, 0.0, 0.0])
    truth = s[:, :3].astype(np.float64) @ R.T + pose[:3] + s[:, 3:4].astype(np.float64) * v
    assert np.abs(world - truth).max() < 1e-4
    raw = s[:, :3].astype(np.float64) @ R.T + pose[:3]
    assert np.linalg.norm(raw - truth, axis=1).max() > 0.25                       # the distortion being removed: up to v * sweep = 0.3 m


def test_undistort_struct_layout():
    from superodom_b200 import api
    assert C.sizeof(api.Undistort) == 72
    assert api.Undistort.dt.offset == 64 and api.Undistort.prev_pose.offset == 8


def test_undistort_struct_layout_in_c(tmp_path):
    src = tmp_path / "l.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "superodom_b200.h"\nint main(void){printf("%zu %zu %zu\\n", sizeof(so_undistort),'
                   ' offsetof(so_undistort, prev_pose), offsetof(so_undistort, dt)); return 0;}\n')
    exe = tmp_path / "l"
    subprocess.check_call(["cc", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)]).decode().split() == ["72", "8", "64"]


# ------------------------------------------------------------------------------------------------------------------ GPU
def _ctx(api, case, **kw):
    ctx = api.Context(max_map_points=max(1 << 20, len(case["map_xyzi"]) * 2 + 1024), max_scan_points=262144, plane_res=case["cfg"]["plane_res"], **kw)
    ctx.map_set_points(case["map_xyzi"])
    return ctx


_moving = {}


def _moving_case(name, speed, yaw_rate, k=0, imu=False):
    from superodom_b200 import synth
    key = (name, speed, yaw_rate, k, imu)
    if key not in _moving:
        case = get_case(name)
        pose = synth.random_sensor_pose(case["scene"], 950 + k, 8.0)
        d = synth.make_moving_scan(case["scene"], case["cfg"]["sensor"], pose, speed, yaw_rate, 60 + k, imu_deskewed=imu)
        d["case"] = case
        _moving[key] = d
    return _moving[key]


def _res_equal(a, b):
    for f, _ in a._fields_:
        if f.startswith("time"):
            continue
        va, vb = getattr(a, f), getattr(b, f)
        if hasattr(va, "__len__"):
            assert bytes(va) == bytes(vb), f
        else:
            assert va == vb or (isinstance(va, float) and math.isnan(va) and math.isnan(vb)), f


@pytest.mark.gpu
def test_device_pinit_matches_numpy_bits(gpu_api):
    ctx = gpu_api.Context(max_map_points=1 << 16, max_scan_points=1 << 14)
    flips = 0
    for cloud, cur, prev, dt, rot in _cases():
        got = ctx.undistort_points(cloud, cur, gpu_api.undistort(prev, dt, rot))
        ref = UN.undistort_points(cloud, cur, prev, dt, rot)
        assert np.array_equal(got[:, 3].view(np.uint32), cloud[:, 3].view(np.uint32))
        diff = got[:, :3].view(np.uint32) != ref.view(np.uint32)
        flips += int(diff.sum())
        # a flip needs the double within ~1e-16 of a float rounding boundary (device FP64 sin / acos vs libm): at most one ulp
        assert np.all(np.abs(got[:, :3].view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))[diff] <= 1)
    assert flips == 0, f"{flips} coordinates one float ulp apart from the numpy restatement"


@pytest.mark.gpu
@pytest.mark.parametrize("name,mf", [("cfg1", 2000), ("cfg1", 0), ("cfg2", 0)])
def test_zero_times_and_mode0_equal_so_register(gpu_api, name, mf):
    d = _moving_case(name, 1.5, 0.3)
    case = d["case"]
    scan = d["scan_xyzi"].copy()
    ctx = _ctx(gpu_api, case)
    it = case["cfg"]["max_iterations"]
    ref = ctx.register(scan, d["prior"], it, mf)
    zero = scan.copy()
    zero[:, 3] = 0.0
    for rot in (True, False):
        r = ctx.register_undistort(zero, d["prior"], gpu_api.undistort(d["pose_prev"], 0.1, rot), it, mf)
        ref0 = ctx.register(zero, d["prior"], it, mf)
        _res_equal(r, ref0)
    r = ctx.register_undistort(scan, d["prior"], gpu_api.undistort(d["pose_prev"], 0.1, True, mode=0), it, mf)
    _res_equal(r, ref)


@pytest.mark.gpu
def test_first_iteration_runs_on_pinit_at_the_prior(gpu_api):
    """One ICP iteration: the registration of the raw cloud with undistortion == so_register of the numpy pInit at the prior (the
    two order the scan differently, so the sums agree to rounding, not bits)."""
    d = _moving_case("cfg1", 5.0, 0.5)
    ctx = _ctx(gpu_api, d["case"])
    scan = d["scan_xyzi"]
    r = ctx.register_undistort(scan, d["prior"], gpu_api.undistort(d["pose_prev"], 0.1), 1, 0)
    p = UN.undistort_points(scan, d["prior"], d["pose_prev"], 0.1)
    ref = ctx.register(np.concatenate([p, scan[:, 3:]], 1), d["prior"], 1, 0)
    assert np.abs(np.array(r.pose_opt) - np.array(ref.pose_opt)).max() < 1e-6
    assert list(r.iter_n_surf) == list(ref.iter_n_surf) and list(r.hist_obs) == list(ref.hist_obs)


@pytest.mark.gpu
@pytest.mark.parametrize("mf", [2000, 0])
def test_batch_equals_single_calls(gpu_api, mf):
    ds = [_moving_case("cfg1", v, 0.3, k) for k, v in enumerate([0.0, 1.5, 5.0, 3.0, 5.0])]
    case = ds[0]["case"]
    us = [gpu_api.undistort(d["pose_prev"], 0.1, rotation=(k != 3), mode=0 if k == 2 else 1) for k, d in enumerate(ds)]
    single = _ctx(gpu_api, case)
    ref = [single.register_undistort(d["scan_xyzi"], d["prior"], u, 5, mf, skip_map_checks=True) for d, u in zip(ds, us)]
    for mb in (2, 5):
        ctx = _ctx(gpu_api, case, max_batch=mb)
        for f in range(0, len(ds), mb):
            sl = slice(f, f + mb)
            sub = ds[sl]
            res = ctx.register_batch_undistort(np.concatenate([d["scan_xyzi"] for d in sub]), [len(d["scan_xyzi"]) for d in sub],
                                               np.stack([d["prior"] for d in sub]), us[sl], 5, mf, skip_map_checks=True)
            for a, b in zip(res, ref[sl]):
                _res_equal(a, b)


@pytest.mark.gpu
def test_undistorted_insert_equals_insert_of_pinit(gpu_api):
    d = _moving_case("cfg1", 5.0, 0.5)
    u = gpu_api.undistort(d["pose_prev"], 0.1)
    a, b = _ctx(gpu_api, d["case"]), _ctx(gpu_api, d["case"])
    r = a.register_undistort(d["scan_xyzi"], d["prior"], u, 5, 2000)
    pose = np.array(r.pose)
    a.map_add_registered_scan(pose)
    p = b.undistort_points(d["scan_xyzi"], pose, u)
    assert np.array_equal(p[:, :3], UN.undistort_points(d["scan_xyzi"], pose, d["pose_prev"], 0.1))
    b.map_add_scan(p, pose)
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
    u = gpu_api.undistort(d["pose_prev"], 0.1)
    a, b = _ctx(gpu_api, case), _ctx(gpu_api, case)
    filt, _, _, _ = a.scan_prefilter(d["scan_xyzi"], 0.2, case["cfg"]["plane_res"], auto_voxel_size=False)
    ra = a.register_prefiltered_undistort(d["prior"], u, 10)
    rb = b.register_undistort(filt, d["prior"], u, 10)
    _res_equal(ra, rb)
    a.map_add_registered_scan(np.array(ra.pose))
    b.map_add_registered_scan(np.array(rb.pose))
    assert np.array_equal(a.map_download(), b.map_download())


@pytest.mark.gpu
def test_argument_errors_before_device_work(gpu_api):
    d = _moving_case("cfg1", 1.5, 0.3)
    ctx = _ctx(gpu_api, d["case"])
    ctx.kernel_launches(reset=True)
    bad = [gpu_api.undistort(d["pose_prev"], 0.1, mode=2), gpu_api.undistort(d["pose_prev"], 0.1, mode=3),
           gpu_api.undistort(d["pose_prev"], 0.0), gpu_api.undistort(d["pose_prev"], -0.1), gpu_api.undistort(d["pose_prev"], float("nan")),
           gpu_api.undistort(d["pose_prev"], float("inf")), gpu_api.undistort(np.r_[d["pose_prev"][:6], np.nan], 0.1),
           gpu_api.undistort(np.zeros(7), 0.1), gpu_api.undistort(d["pose_prev"], 0.1, rotation=2)]
    for u in bad:
        with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
            ctx.register_undistort(d["scan_xyzi"], d["prior"], u, 5, 2000)
        with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
            ctx.register_batch_undistort(d["scan_xyzi"], [len(d["scan_xyzi"])], d["prior"][None], [u], 5, 2000)
        with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
            ctx.undistort_points(d["scan_xyzi"], d["prior"], u)
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
        ctx.register_prefiltered_undistort(d["prior"], gpu_api.undistort(d["pose_prev"], 0.1), 5)
    assert ctx.kernel_launches() == 0


@pytest.mark.gpu
def test_profile_class_7(gpu_api):
    d = _moving_case("cfg1", 1.5, 0.3)
    ctx = _ctx(gpu_api, d["case"])
    ctx.profile_enable(True)
    r = ctx.register_undistort(d["scan_xyzi"], d["prior"], gpu_api.undistort(d["pose_prev"], 0.1), 5, 2000)
    ms, n = ctx.profile_get(7)
    assert n == r.n_iterations and ms > 0.0
    ctx.profile_enable(False)


def _err(pose, truth):
    return float(np.linalg.norm(np.asarray(pose[:3]) - truth[:3])), quat_angle(np.asarray(pose[3:]), truth[3:])


@pytest.mark.gpu
@pytest.mark.parametrize("name,mf", [("cfg1", 2000), ("cfg2", 0)])
@pytest.mark.parametrize("imu", [False, True])
def test_undistortion_reduces_error_at_speed(gpu_api, name, mf, imu):
    """Against the ground-truth start pose: standing still both modes land together; at 1.5 and 5 m/s APPROXIMATED is closer.
    imu: the cloud has its rotation removed (so_scan_deskew imu_only), so only the translation is interpolated."""
    it = CASES_ITERS[name]
    for speed, yaw_rate in ((0.0, 0.0), (1.5, 0.3), (5.0, 0.5)):
        d = _moving_case(name, speed, yaw_rate, imu=imu)
        ctx = _ctx(gpu_api, d["case"])
        rn = ctx.register(d["scan_xyzi"], d["prior"], it, mf)
        ra = ctx.register_undistort(d["scan_xyzi"], d["prior"], gpu_api.undistort(d["pose_prev"], 0.1, rotation=not imu), it, mf)
        en, ea = _err(rn.pose, d["pose_true"]), _err(ra.pose, d["pose_true"])
        if speed == 0.0:
            assert abs(en[0] - ea[0]) < 0.01
        else:                                                     # measured (DESIGN.md §4): 0.002-0.011 m against 0.07-0.30 m
            assert ea[0] < 0.03 and ea[1] < 0.002 and ea[0] < 0.25 * en[0], (name, imu, speed, en, ea)


CASES_ITERS = {"cfg1": 5, "cfg2": 20}

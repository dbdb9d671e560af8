"""The shim's degeneracy members (include/superodom_b200/LidarSlam.hpp): isDegenerate follows the reference's rule on the final
covariance after every registration and stays false with the default thresholds; DegeneracyAware registers through
so_register_degeneracy, bit for bit as the C ABI called directly."""
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exe(tmp_path):
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "degeneracy_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "degeneracy_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


def test_degeneracy_shim_compiles(tmp_path):
    assert os.path.exists(_exe(tmp_path))


def _sequence():
    from test_optimized_undistortion import _speed_change_trajectory
    from conftest import get_case
    seq = _speed_change_trajectory(get_case("tiny")["scene"], [0.0, 1.0, 2.0, 2.0, 1.0, 0.0], 0.3)
    scans = [np.ascontiguousarray(d["scan_xyzi"], np.float32) for d in seq]
    priors = [seq[0]["pose_true"]] + [d["prior"] for d in seq[1:]]
    return scans, priors


def _run(exe, tmp_path, scans, priors, pos, ori, aware):
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiif", len(scans), 5, 0, 0.2))
        for s, p in zip(scans, priors):
            f.write(struct.pack("<i", len(s)))
            f.write(np.asarray(p, np.float64).tobytes())
            f.write(s.tobytes())
    out = subprocess.run([exe, str(path), repr(pos), repr(ori), str(int(aware))], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    return [[float(v) for v in ln.split()] for ln in out.stdout.strip().splitlines()]


@pytest.mark.gpu
def test_is_degenerate_follows_the_rule(tmp_path, gpu_api):
    exe = _exe(tmp_path)
    scans, priors = _sequence()
    for pos, ori in ((0.0, 0.0), (0.5, 0.5), (0.9, 0.05)):
        rows = _run(exe, tmp_path, scans, priors, pos, ori, False)
        for r in rows[1:]:
            if int(r[11]) == 1:                                   # not enough features: nothing registered, nothing to judge
                continue
            expect = r[9] < np.float32(pos) or r[10] < np.float32(ori)
            assert int(r[8]) == int(expect), (pos, ori, r)
            if pos == 0.0 and ori == 0.0:
                assert int(r[8]) == 0, r                          # the default thresholds never set it
        print(pos, ori, [(int(r[8]), round(r[9], 3), round(r[10], 3)) for r in rows[1:]])


@pytest.mark.gpu
def test_degeneracy_aware_reaches_so_register_degeneracy(tmp_path, gpu_api):
    exe = _exe(tmp_path)
    scans, priors = _sequence()
    thr = 0.6
    rows = _run(exe, tmp_path, scans, priors, thr, thr, True)
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=1 << 17, plane_res=0.2, line_res=0.1)
    ctx.map_set_origin(priors[0][:3])
    ctx.map_add_scan(scans[0], priors[0])
    d = gpu_api.degeneracy(float(np.float32(thr)), float(np.float32(thr)), True)
    flagged = 0
    for s in range(1, len(scans)):
        r = ctx.register_degeneracy(scans[s], priors[s], d, 5, 0)
        assert np.array_equal(np.array(r.icp.pose), np.array(rows[s][1:8])), s          # shim == ABI, bit for bit
        assert np.array_equal(np.array(r.icp.pose_opt), np.array(rows[s][14:21])), s     # last_degeneracy is filled in
        assert (r.flags_pos, r.flags_ori) == (int(rows[s][12]), int(rows[s][13])), s
        flagged += r.flags_pos | r.flags_ori
        if r.icp.status == 1:
            continue
        ctx.map_add_registered_scan(np.array(r.icp.pose))
    ctx.close()
    assert flagged, "the threshold flags a direction in some scan"

"""Host side of so_loop_verify: so_loop_prior equals the restatement the loop tests use (test_loop_detection._loop_prior), the decision
rule header at its thresholds (tests/cpp/verify_rule_test.cpp), the option defaults, the entry points declared, exported and bound,
and the shim's new members compiling."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _random_poses(rng, n):
    from scipy.spatial.transform import Rotation
    out = []
    for _ in range(n):
        q = Rotation.from_euler("ZYX", [rng.uniform(-math.pi, math.pi), rng.normal(0, 0.1), rng.normal(0, 0.1)]).as_quat()
        out.append(np.r_[rng.uniform(-100, 100, 3), q])
    return out


def test_loop_prior_equals_the_restatement():
    from superodom_b200 import api
    from test_loop_detection import _loop_prior
    rng = np.random.default_rng(11)
    yaws = list(rng.uniform(-math.pi, math.pi, 200)) + [math.pi, -math.pi, math.pi - 1e-12, -math.pi + 1e-12, 0.0]
    worst = 0.0
    for k, yaw in enumerate(yaws):
        cand, query = _random_poses(rng, 2)
        got = api.loop_prior(cand, query, yaw)
        want = _loop_prior([query, cand], dict(query=0, id=1, yaw=yaw))
        if np.dot(got[3:], want[3:]) < 0:                                 # the same rotation, either sign
            want[3:] = -want[3:]
        worst = max(worst, float(np.abs(got - want).max()))
        assert np.array_equal(got[:3], cand[:3])
    print(f"so_loop_prior vs restatement: max difference {worst:.3g}")
    assert worst <= 1e-15


def test_decision_rule_at_its_thresholds(tmp_path):
    exe = tmp_path / "verify_rule_test"
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-ffp-contract=off",
                           os.path.join(ROOT, "tests", "cpp", "verify_rule_test.cpp"), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout


def test_option_defaults():
    from superodom_b200 import api
    o = api.loop_verify_opts()
    assert (o.half_window, o.id_begin, o.id_end, o.exclude_recent) == (2, 0, -1, 30)
    assert (o.icp.max_icp_iters, o.icp.max_surface_features, o.icp.lm_max_iterations, o.icp.yaw_ratio) == (20, 0, 4, 0.0)
    assert (o.icp.skip_map_checks, o.icp.use_pose_prior) == (0, 0)
    assert (o.inlier_dist, o.min_overlap, o.max_conflict) == (0.5, 0.5, 0.05)
    d = api.free_space()
    assert bytes(o.image) == bytes(d)
    v = api.loop_verify_opts(image=dict(el_res_deg=2.0, el_min_deg=-16.0, el_max_deg=16.0), icp=dict(max_icp_iters=10), min_overlap=0.3)
    assert (v.image.el_res_deg, v.image.el_min_deg, v.icp.max_icp_iters, v.min_overlap, v.max_conflict) == (2.0, -16.0, 10, 0.3, 0.05)
    with pytest.raises(TypeError):
        api.loop_verify_opts(no_such_field=1)
    # the Python default ICP options of the loop tests' manual alignment are the ones the defaults hold
    ref = api.Context._opts(20, 0)
    assert bytes(ref) == bytes(o.icp)


def test_entries_exported_and_bound(tmp_path):
    from superodom_b200 import api, build
    for name in ("so_loop_prior", "so_loop_verify_opts_defaults", "so_loop_verify"):
        assert name in api.EXPORTS
    lib = build.build()
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    for name in ("so_loop_prior", "so_loop_verify_opts_defaults", "so_loop_verify"):
        assert re.search(rf"\b{name}\b", syms), name
    L = api.load_library()
    assert len(L.so_loop_verify.argtypes) == 6 and len(L.so_loop_prior.argtypes) == 4
    # the ctypes layouts are the header's
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "superodom_b200.h"\nint main(void) { printf("%zu %zu %zu %zu\\n", '
                   'sizeof(so_loop_verify_opts), sizeof(so_loop_verify_result), offsetof(so_loop_verify_result, rel7), '
                   'offsetof(so_loop_verify_opts, image)); return 0; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "sizes")])
    got = [int(v) for v in subprocess.run([str(tmp_path / "sizes")], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(api.LoopVerifyOpts), C.sizeof(api.LoopVerifyResult), api.LoopVerifyResult.rel7.offset,
                   api.LoopVerifyOpts.image.offset]
    with open(os.path.join(ROOT, "include", "superodom_b200.h")) as f:
        hdr = f.read()
    assert re.search(r"int so_loop_verify\(so_ctx\* ctx, so_ctx\* scratch, const so_loop_candidate\* c, size_t n, "
                     r"const so_loop_verify_opts\* opts,\s+so_loop_verify_result\* out\);", hdr)


def test_shim_members_compile():
    subprocess.check_call(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "loop_verify_test.cpp")])

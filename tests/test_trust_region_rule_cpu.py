"""The trust-region rules every solve follows (so_trust_region_rule.h: the registration's device loop and the pose graph's host loop),
compiled on the CPU by tests/cpp/trust_region_rule_test.cpp: every exit test at its threshold, the step quality, the radius and
decrease-factor updates, when the diagonal is reused, the diagonal clamp, and exits 4 and 5, which no solve reaches
(tests/test_trust_region_cpu.py).  The header's constants equal those of the numpy restatement (tests/test_ceres_restatement.py) that
the GPU tests compare the solves against."""
import os
import subprocess

import test_ceres_restatement as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_rules_at_their_thresholds_and_constants(tmp_path):
    exe = tmp_path / "trust_region_rule_test"
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-ffp-contract=off",
                           os.path.join(ROOT, "tests", "cpp", "trust_region_rule_test.cpp"), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("ok\n"), out.stdout
    got = {name: float.fromhex(value) for name, value in (line.split() for line in out.stdout.splitlines()[1:])}
    want = {name: getattr(R, name) for name in ("FUNCTION_TOL", "GRADIENT_TOL", "PARAMETER_TOL", "MIN_REL_DECREASE", "MIN_LM_DIAG",
                                                "MAX_LM_DIAG", "MAX_RADIUS", "MIN_RADIUS")}
    assert got == want

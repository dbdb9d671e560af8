"""The two restatements of so_register_optimized's two-block solve -- optimized_numpy (test_ceres_restatement.solve_full over the pose7
blocks T and D, numpy's LAPACK least squares) and oracle/so_oracle.cpp (ceres_solve_t<12> on MotionEvaluator, Householder QR) --
agree on the families of tests/motion_solve_sets.py, which reach what the benign moving scans never do: rejected steps (one, and
several back to back), the radius recovering after a rejection, rejections with the motion prior rows in the system, and the
gradient-tolerance exit through Plus of both blocks.  The vectorised rows of optimized_numpy equal its former per-row form.

As in the six-column solve (tests/test_trust_region_cpu.py), termination 4 needs 15 rejections in a row, so at least 16 LM iterations,
and termination 5 a non-positive model cost change of a step from a positive definite damped system; the first is shown unreached at
16 iterations below, the second cannot occur away from underflow.
"""
import math

import numpy as np

import motion_solve_sets as MS
import optimized_numpy as ON
import trust_region_sets as TS


# ---- the per-row form optimized_numpy computed its rows with before they were vectorised
def _slerp_R_row(q, a):
    ad = abs(q[3])
    if ad >= 1.0 - ON.UN.EPS:
        s0, s1 = 1.0 - a, a
    else:
        th = math.acos(ad)
        s0, s1 = math.sin((1 - a) * th) / math.sin(th), math.sin(a * th) / math.sin(th)
    if q[3] < 0:
        s1 = -s1
    x, y, z, w = s1 * q[0], s1 * q[1], s1 * q[2], s0 + s1 * q[3]
    return np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


def _warp_rows(P, A, D):
    q = D[3:] / np.linalg.norm(D[3:])
    return np.stack([_slerp_R_row(q, a) @ p for p, a in zip(P, A)]) + A[:, None] * D[:3]


def _jacobian_rows(P, A, N, T, D):
    R = ON._rot(T[3:])
    q = D[3:] / np.linalg.norm(D[3:])
    phi = ON._log_q(q)
    jinv = np.linalg.inv(ON._jr(phi))
    out = np.zeros((len(P), 12))
    for i, (p, a, n, u) in enumerate(zip(P, A, N, _warp_rows(P, A, D))):
        av = R.T @ n
        b = _slerp_R_row(q, a).T @ av
        out[i, :3], out[i, 3:6], out[i, 6:9] = n, np.cross(u, av), a * av
        out[i, 9:] = a * (np.cross(p, b) @ ON._jr(a * phi) @ jinv)
    return out


def test_vectorised_rows_equal_the_per_row_form():
    rng = np.random.default_rng(4)
    for trial in range(80):
        n = int(rng.integers(1, 40))
        P = rng.uniform(-20, 20, (n, 3))
        N = np.linalg.qr(rng.normal(size=(3, 3)))[0][rng.integers(0, 3, n)]
        A = rng.uniform(-0.5, 1.5, n)
        A[: n // 4] = 0.0
        T = np.concatenate([rng.uniform(-5, 5, 3), TS._unit_quat(rng, rng.uniform(0, 1))])
        D = np.concatenate([rng.uniform(-1, 1, 3), TS._unit_quat(rng, [0.0, 1e-7, 5e-5, 5e-3, 0.3][trial % 5])])
        if trial % 3 == 2:
            D[3:] = -D[3:]                                   # q.w < 0: the same rotation, slerp's sign flip
        scale = max(1.0, np.abs(P).max())
        assert np.abs(ON.warp_double(P, A, D) - _warp_rows(P, A, D)).max() <= 1e-12 * scale, trial
        assert np.abs(ON.jacobian(P, A, N, T, D) - _jacobian_rows(P, A, N, T, D)).max() <= 1e-12 * scale, trial


def _agree(p, r):
    """numpy result r and the C++ restatement agree on the solve's trip counts, exit and result"""
    T, D, so = MS.oracle_solve(p)
    what = (p["family"], len(p["P"]), p["lm"], r["steps"])
    assert (so["iterations"], so["successful"], so["unsuccessful"], so["termination"]) == \
        (r["iterations"], r["successful"], r["unsuccessful"], r["termination"]), (what, so)
    assert np.abs(T - r["x"][:7]).max() <= 1e-9 and np.abs(D - r["x"][7:]).max() <= 1e-9, what
    assert abs(so["radius"] - r["radius"]) <= 1e-9 * r["radius"], (what, so["radius"], r["radius"])
    assert abs(so["decrease_factor"] - r["decrease_factor"]) <= 1e-9 * r["decrease_factor"], what
    return T, D, so


def test_numpy_and_cpp_restatements_agree_on_the_two_block_families():
    from oracle import oracle as O
    O.build()
    kept = MS.fair_sample(7, 36, row_counts=(1, 7, 255, 256, 257, 4096, 4097), lms=(12, 16, 4))
    kept += MS.fair_sample(8, 40, families=("strip", "lever", "prior"), row_counts=(7, 255, 257, 4096), lms=(12, 16))
    kept += MS.fair_sample(9, 2, families=("well", "strip", "static"), row_counts=(65536, 65537), lms=(12,))
    cover = dict(rejected=0, two_rejected=0, rejected_then_accepted=0, prior_rejected=0)
    terms = set()
    for p, r in kept:
        s = r["steps"]
        cover["rejected"] += "r" in s
        cover["two_rejected"] += "rr" in s
        cover["rejected_then_accepted"] += "ra" in s
        cover["prior_rejected"] += "r" in s and bool(p["info"].any())
        terms.add(r["termination"])
        assert s.count("r") == r["unsuccessful"] - 1 and s.count("a") == r["successful"]      # iteration 0 counts once
        T, D, so = _agree(p, r)
        if p["family"] == "zero":
            assert (r["gmax"], r["termination"], r["iterations"]) == (0.0, 1, 0) and so["gmax"] == 0.0
        if p["family"] == "static" and not p["info"].any():
            # the D columns and the prior rows are zero: the step never moves D's translation, and its quaternion only by Plus's
            # renormalisation
            assert np.array_equal(D[:3], p["motion"][:3]) and np.abs(D[3:] - p["motion"][3:]).max() <= 1e-15, D - p["motion"]
    print("coverage:", cover, "terminations:", sorted(terms), "of", len(kept))
    assert cover["rejected"] >= 20 and cover["two_rejected"] >= 5 and cover["rejected_then_accepted"] >= 5, cover
    assert cover["prior_rejected"] >= 1, cover
    assert {0, 1, 2, 3} <= terms, terms


def test_exact_zero_and_saturated_starts_end_at_the_gradient_tolerance():
    rng = np.random.default_rng(3)
    for n in (1, 7, 257, 4097):
        p = MS.make("zero", rng, n, 4)
        prob = MS.numpy_problem(p)
        assert not np.any(ON.residuals(prob.P, prob.A, prob.N, prob.Dd, p["start"], p["motion"]))
        r = MS.numpy_solve(p)
        assert (r["gmax"], r["termination"], r["iterations"], r["unsuccessful"]) == (0.0, 1, 0, 1)
        p = MS.make("saturated", rng, n, 4)
        p["info"] = np.zeros(6)                                # no prior rows: H = g = 0
        r = MS.numpy_solve(p)
        # gmax = |x - Plus(x, 0)| over both blocks: the rounding of Plus's renormalisation
        assert r["gmax"] <= 1e-15 and (r["termination"], r["iterations"]) == (1, 0), r


def test_sixteen_iterations_do_not_reach_the_radius_floor():
    """The families that reject steps at lm_max_iterations = 16 (the device's cap, and the least termination 4 needs): no solve ends
    at the radius floor; the longest run of rejections is far short of 15."""
    problems = MS.sample(5, 45, lms=(16,), families=("strip", "lever", "prior", "extrapolated"), row_counts=(7, 255, 4097))
    runs, terms = [], set()
    for p in problems:
        r = MS.numpy_solve(p)
        terms.add(r["termination"])
        runs.append(max((len(m) for m in r["steps"].split("a")), default=0))
    print("terminations:", sorted(terms), "longest run of rejections:", max(runs))
    assert 4 not in terms and max(runs) < 15

"""The device's two-block solve of so_register_optimized (m_begin_solve / m_lm_continue / m_after_eval / chol12_solve / m_gmax in
so_motion.cu, on one thread of k_motion_step, with k_motion_eval's partials summed in a fixed order and cov12_warp at the end) on given
correspondences, through so_solve_optimized, against both restatements (optimized_numpy.solve_full2 and oracle.solve_optimized) on the
families of tests/motion_solve_sets.py, and its batched forms against each other bit for bit.  Which exits stay unreached, and why, is
argued in tests/test_motion_solve_cpu.py."""
import numpy as np
import pytest

import motion_solve_sets as MS

pytestmark = pytest.mark.gpu

SO_STATUS_NO_CORRESPONDENCES = 2


def _pack(problems):
    from superodom_b200 import api
    n = sum(len(p["P"]) for p in problems)
    rows = np.zeros(n, api.SOLVE_ROW_DTYPE)
    times = np.zeros(n, np.float32)
    pr = np.zeros(len(problems), api.SOLVE_OPTIMIZED_PROBLEM_DTYPE)
    o = 0
    for b, p in enumerate(problems):
        k = len(p["P"])
        rows["p"][o:o + k], rows["n"][o:o + k], rows["d"][o:o + k], rows["w"][o:o + k] = p["P"], p["N"], p["D"], p["W"]
        times[o:o + k] = p["tau"]
        pr[b]["n_rows"], pr[b]["lm_max_iterations"], pr[b]["pose"], pr[b]["motion"] = k, p["lm"], p["start"], p["motion"]
        pr[b]["dt"], pr[b]["motion_prior"], pr[b]["motion_info"] = p["dt"], p["D0"], p["info"]
        o += k
    return rows, times, pr


def _solve(ctx, problems):
    return ctx.solve_optimized(*_pack(problems))


def _empty(rng):
    p = MS.make("well", rng, 1, 4)
    for k in ("P", "N", "D", "W", "tau"):
        p[k] = p[k][:0]
    p["family"] = "empty"
    return p


@pytest.fixture(scope="module")
def ctx():
    from superodom_b200 import api
    c = api.Context(max_scan_points=70000, max_batch=8, plane_res=MS.PLANE_RES)
    yield c
    c.close()


def _close(a, b, rel, scale=0.0):
    """a == b to rel relative; scale: the size of the terms b was summed from"""
    return abs(a - b) <= rel * abs(b) + 1e-15 * scale


def _cov_block(r, p):
    """T's 6x6 block of the pseudo-inverse of the numpy restatement's 12x12 H = J^T J at the final (T, D), with cov12_warp's cut:
    eigenvalues ascending, a direction cut when sqrt(w_k / w_max) < 1e-7, and every smaller one with it"""
    _, _, J = MS.numpy_problem(p).linearise(r["x"][:7], r["x"][7:])
    w, V = np.linalg.eigh(J.T @ J)
    inv = np.zeros(12)
    cut = False
    for k in range(11, -1, -1):
        cut = cut or not (w[k] > 0 and w[11] > 0 and np.sqrt(w[k] / w[11]) >= 1e-7)
        inv[k] = 0.0 if cut else 1.0 / w[k]
    return ((V * inv) @ V.T)[:6, :6]


def _sample():
    kept = MS.fair_sample(31, 18, row_counts=(1, 7, 255, 256, 257, 4096, 4097), lms=(12, 16, 4))
    kept += MS.fair_sample(32, 16, families=("strip", "lever", "prior"), row_counts=(7, 255, 4096, 4097), lms=(12, 16))
    kept += MS.fair_sample(33, 2, families=("well", "strip", "static", "saturated"), row_counts=(65536, 65537), lms=(12,))
    return kept


def _check(p, r, d):
    """the device's result d on problem p against the numpy result r and the C++ restatement; raises AssertionError"""
    s, res = d["solve"], r["steps"]
    what = (p["family"], len(p["P"]), p["lm"], res)
    assert s["status"] == 0, what
    assert (s["lm_iterations"], s["successful"], s["unsuccessful"], s["termination"]) == \
        (r["iterations"], r["successful"], r["unsuccessful"], r["termination"]), (what, s)
    dx = max(np.abs(s["pose"] - r["x"][:7]).max(), np.abs(d["motion"] - r["x"][7:]).max())
    assert dx <= 1e-9, (what, dx)
    assert _close(s["initial_cost"], r["initial_cost"], 1e-10) and _close(s["final_cost"], r["final_cost"], 1e-10, r["initial_cost"]), what
    # the device solves the normal equations by Cholesky: its steps, so the step qualities the radius follows, are known to cond^2 eps
    # where QR's are known to cond eps; the radius is compared to 1e-9 relative or to what that rounding can leave, if larger (measured:
    # up to 8e-9 relative on two prior problems at 16 iterations, whose estimate is 6e-7 and 1e-6)
    rad = max(1e-9, r["radius_error_normal"])
    assert _close(s["radius"], r["radius"], rad) and _close(s["decrease_factor"], r["decrease_factor"], 1e-9), (what, s["radius"], r["radius"])
    # gmax is the max-norm of g(x) = J^T r through Plus.  Near a minimiser it is small and moves by about H dx between two
    # minimisers dx apart (measured: 1.1e-9 relative on a 7-row well-posed problem, 3e-13 absolute on a 1-row one), and by the
    # rounding of Plus's renormalisation where g is 0; so it is compared to 1e-9 relative plus those two
    _, _, Jn = MS.numpy_problem(p).linearise(r["x"][:7], r["x"][7:])
    gerr = abs(s["gmax"] - r["gmax"])
    assert gerr <= 1e-9 * r["gmax"] + 2.0 * np.abs(Jn.T @ Jn).max() * dx + 1e-15, (what, s["gmax"], r["gmax"], dx)
    T, D, so = MS.oracle_solve(p)
    assert (s["lm_iterations"], s["successful"], s["unsuccessful"], s["termination"]) == \
        (so["iterations"], so["successful"], so["unsuccessful"], so["termination"]), (what, so)
    assert np.abs(s["pose"] - T).max() <= 1e-9 and np.abs(d["motion"] - D).max() <= 1e-9, what
    assert _close(s["final_cost"], so["final_cost"], 1e-10, so["initial_cost"]), what
    assert _close(s["radius"], so["radius"], rad) and _close(s["decrease_factor"], so["decrease_factor"], 1e-9), what
    # exact claims
    if p["family"] == "zero":
        assert (s["gmax"], s["termination"], s["lm_iterations"]) == (0.0, 1, 0), what
    if p["family"] == "static" and not p["info"].any():
        assert np.array_equal(d["motion"][:3], p["motion"][:3]) and np.abs(d["motion"][3:] - p["motion"][3:]).max() <= 1e-15, what
    if p["family"] == "saturated" and not p["info"].any():
        assert s["gmax"] <= 1e-15 and (s["termination"], s["lm_iterations"]) == (1, 0), what
    cov = np.asarray(d["cov"]).reshape(6, 6)
    ref = _cov_block(r, p)
    scale = np.abs(ref).max()
    err = np.abs(cov - ref).max() / scale if scale > 0 else np.abs(cov).max()
    assert err <= 1e-6, (what, err)
    return gerr / r["gmax"] if r["gmax"] > 0 else 0.0, err, abs(s["radius"] - r["radius"]) / r["radius"]


def test_device_solve_matches_both_restatements(ctx):
    kept = _sample()
    cover = dict(rejected=0, two_rejected=0, rejected_then_accepted=0, prior_rejected=0)
    regimes = set()
    worst_gmax = worst_cov = worst_radius = 0.0
    failures = []
    for p, r in kept:
        try:
            g, c, rd = _check(p, r, _solve(ctx, [p])[0])
            worst_gmax, worst_cov, worst_radius = max(worst_gmax, g), max(worst_cov, c), max(worst_radius, rd)
        except AssertionError as e:
            failures.append(str(e)[:300])
        res = r["steps"]
        cover["rejected"] += "r" in res
        cover["two_rejected"] += "rr" in res
        cover["rejected_then_accepted"] += "ra" in res
        cover["prior_rejected"] += "r" in res and bool(p["info"].any())
        regimes.add(1 if len(p["P"]) <= 4096 else (4 if len(p["P"]) <= 65536 else 16))
    print("device two-block solves:", cover, "eval_pts regimes:", sorted(regimes), "of", len(kept),
          "worst relative radius difference", worst_radius, "worst relative gmax difference", worst_gmax, "worst covariance error", worst_cov)
    assert not failures, f"{len(failures)} of {len(kept)} solves differ:\n" + "\n".join(failures)
    assert cover["rejected"] >= 5 and cover["two_rejected"] >= 5 and cover["rejected_then_accepted"] >= 5, cover
    assert cover["prior_rejected"] >= 1, cover
    assert regimes == {1, 4, 16}, regimes


def test_empty_problems_end_without_correspondences(ctx):
    rng = np.random.default_rng(2)
    empty = _empty(rng)
    alone = _solve(ctx, [empty])[0]                        # a batch whose every problem is empty: no evaluation CTA at all
    others = [MS.make("well", rng, n, 4) for n in (7, 257)]
    batch = _solve(ctx, [others[0], empty, others[1]])
    for d in (alone, batch[1]):
        s = d["solve"]
        assert (s["termination"], s["status"], s["lm_iterations"], s["successful"]) == (6, SO_STATUS_NO_CORRESPONDENCES, 0, 0)
        assert np.array_equal(s["pose"], empty["start"]) and np.abs(d["motion"] - empty["motion"]).max() <= 1e-15
    assert alone.tobytes() == batch[1:2].tobytes()
    for b, p in ((0, others[0]), (2, others[1])):
        assert batch[b]["solve"]["status"] == 0 and batch[b:b + 1].tobytes() == _solve(ctx, [p]).tobytes()


def test_batched_forms_agree_bit_for_bit(ctx):
    kept = _sample()
    # a batch of 8 of mixed sizes and families: one with a rejected step from each family that has one, then others, and an empty one
    batch = []
    for fam in dict.fromkeys(p["family"] for p, _ in kept):
        of_fam = [(p, r) for p, r in kept if p["family"] == fam]
        batch.append(next((p for p, r in of_fam if "r" in r["steps"]), of_fam[0][0]))
    batch = [p for p in batch if p["family"] in ("strip", "lever", "prior", "static", "zero", "well")][:6]
    batch += [p for p, r in kept if len(p["P"]) > 4096 and not any(p is q for q in batch)][:1]
    batch.append(_empty(np.random.default_rng(5)))
    assert len(batch) == 8 and len({len(p["P"]) for p in batch}) > 3, [(p["family"], len(p["P"])) for p in batch]
    together = _solve(ctx, batch)
    for b, p in enumerate(batch):
        assert _solve(ctx, [p]).tobytes() == together[b:b + 1].tobytes(), (p["family"], len(p["P"]))
    perm = np.random.default_rng(6).permutation(8)
    permuted = _solve(ctx, [batch[k] for k in perm])
    assert permuted.tobytes() == together[perm].tobytes()
    twice = _solve(ctx, [batch[0], batch[3], batch[0]])
    assert twice[0:1].tobytes() == twice[2:3].tobytes() == together[0:1].tobytes()
    assert twice[1:2].tobytes() == together[3:4].tobytes()


def test_argument_errors_come_first(ctx):
    """so_register_optimized's so_motion errors and the size errors are returned before any device work"""
    from superodom_b200 import api
    p = MS.make("well", np.random.default_rng(8), 7, 4)
    rows, times, pr = _pack([p])
    out = np.zeros(1, api.SOLVE_OPTIMIZED_RESULT_DTYPE)
    bad_prior = np.zeros(7)
    for field, value in (("dt", 0.0), ("dt", np.nan), ("lm_max_iterations", 17), ("n_rows", 70001), ("motion_prior", bad_prior),
                         ("motion_info", -np.ones(6)), ("motion", bad_prior)):
        bad = pr.copy()
        bad[0][field] = value
        ctx.kernel_launches(reset=True)
        assert ctx.L.so_solve_optimized(ctx.h, rows.ctypes.data, times.ctypes.data, bad.ctypes.data, 1, out.ctypes.data) < 0, field
        assert ctx.kernel_launches() == 0, field
    assert ctx.L.so_solve_optimized(ctx.h, rows.ctypes.data, None, pr.ctypes.data, 1, out.ctypes.data) < 0
    assert ctx.L.so_solve_optimized(ctx.h, rows.ctypes.data, times.ctypes.data, np.repeat(pr, 9).ctypes.data, 9, out.ctypes.data) < 0

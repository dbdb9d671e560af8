"""The two restatements of Ceres' trust-region solve (tests/test_ceres_restatement.py in numpy, oracle/so_oracle.cpp in C++) agree on
the problem families of tests/trust_region_sets.py, which reach what random well-posed problems never do: rejected steps (one, and
several back to back), the decrease factor doubling and its reset, the LM diagonal recomputed after the step that follows a
rejection, the radius recovering, the gradient-tolerance exit, and rejections with the SE3 prior rows and in the reduced solve.
Reusing the diagonal after a rejection and recomputing it there cannot be told apart: a rejected step leaves H and g as they were, so
the recomputed diagonal is the same bits.  Only the recompute after an accepted step is observable.

Two exits stay unreached, in every copy of the loop:
  * termination 4 (radius <= 1e-32): from 1e4 it takes 15 rejections in a row -- the radius falls by 2, 4, 8, ... -- so at least 16
    LM iterations, the device's cap.  Long before that the step is tiny and the parameter or function tolerance ends the solve:
    test_sixteen_iterations_do_not_reach_the_radius_floor runs the rejecting families at 16 iterations and finds no solve there.
  * termination 5 (five invalid steps in a row): a step is invalid when it is not finite or the model cost change is not positive.
    The damped system M = H + D / radius is positive definite (D >= 1e-6) for every finite input, so y = M^-1 g is finite, and the model
    cost change of the step -y is y'g - y'H y / 2 = y'H y / 2 + y'(D / radius) y, positive in exact arithmetic whenever g != 0; with
    g = 0 the gradient tolerance exits first.  Only rounding on a g at the edge of underflow could make it non-positive.
Whether Ceres 2.0's LevenbergMarquardtStrategy::StepIsInvalid halves the radius (as all three copies do) or divides it by the decrease
factor is not pinned: no copy of the loop can reach that branch to tell.
"""
import numpy as np

import trust_region_sets as TS


def _fair_sample(seed, per_family, row_counts):
    problems = TS.sample(seed, per_family, lms=(4, 12), row_counts=row_counts)
    results = [TS.numpy_solve(p) for p in problems]
    kept = [(p, r) for p, r in zip(problems, results) if TS.fair(r)]
    print(f"\n{len(problems) - len(kept)} of {len(problems)} problems dropped: a decision within 1e-6 of its threshold, or a radius "
          f"rounding can move by 1e-10")
    return kept


def test_numpy_and_cpp_restatements_agree_on_the_trust_region_families():
    from oracle import oracle as O
    O.build()
    kept = _fair_sample(7, 120, (1, 7, 255, 4097)) + _fair_sample(8, 1, (65537,))
    cover = dict(rejected=0, two_rejected=0, rejected_then_accepted=0, prior_rejected=0, reduced_rejected=0)
    terms = set()
    for p, r in kept:
        s = r["steps"]
        cover["rejected"] += "r" in s
        cover["two_rejected"] += "rr" in s
        cover["rejected_then_accepted"] += "ra" in s
        cover["prior_rejected"] += "r" in s and p["prior"] is not None
        cover["reduced_rejected"] += "r" in s and p["degen"] is not None and sum(r["n_flag"]) > 0
        terms.add(r["termination"])
        assert r["steps"].count("r") == r["unsuccessful"] - 1 and r["steps"].count("a") == r["successful"]      # iteration 0 counts once
        if p["family"] == "zero":
            assert (r["gmax"], r["termination"], r["iterations"]) == (0.0, 1, 0)
        if p["family"] == "saturated" and not np.any(np.abs(numpy_residuals(p)) <= TS.A):
            # g = 0; gmax = |x - Plus(x, 0)| is the rounding of Plus's renormalisation
            assert r["gmax"] <= 1e-15 and (r["termination"], r["iterations"]) == (1, 0)
        if p["degen"] is not None:
            continue                                   # the oracle has no reduced solve; the device test compares it with numpy
        xo, so = TS.oracle_solve(p)
        what = (p["family"], len(p["P"]), p["lm"], s)
        assert (so["iterations"], so["successful"], so["unsuccessful"], so["termination"]) == \
            (r["iterations"], r["successful"], r["unsuccessful"], r["termination"]), (what, so)
        assert np.abs(xo - r["x"]).max() <= 1e-9, what
        assert abs(so["radius"] - r["radius"]) <= 1e-9 * r["radius"], (what, so["radius"], r["radius"])
        assert abs(so["decrease_factor"] - r["decrease_factor"]) <= 1e-9 * r["decrease_factor"], what
    print("coverage:", cover, "terminations:", sorted(terms))
    assert cover["rejected"] >= 20 and cover["two_rejected"] >= 5 and cover["rejected_then_accepted"] >= 5, cover
    assert cover["prior_rejected"] >= 1 and cover["reduced_rejected"] >= 1, cover
    assert {0, 1, 2, 3} <= terms, terms


def numpy_residuals(p):
    return TS.numpy_problem(p)._residuals(p["start"])[0]


def test_exact_zero_and_saturated_starts_end_at_the_gradient_tolerance():
    rng = np.random.default_rng(3)
    for n in TS.ROW_COUNTS:
        p = TS.make("zero", rng, n, 4)
        assert not np.any(numpy_residuals(p))
        r = TS.numpy_solve(p)
        assert (r["gmax"], r["termination"], r["iterations"], r["unsuccessful"]) == (0.0, 1, 0, 1)
        p["D"] = p["D"] + 3.0 * TS.A                            # every row beyond the Tukey scale: H = g = 0
        r = TS.numpy_solve(p)
        assert (r["gmax"], r["termination"], r["iterations"]) == (0.0, 1, 0)


def test_sixteen_iterations_do_not_reach_the_radius_floor():
    """The families that reject steps, at lm_max_iterations = 16 (the device's cap, and the least that termination 4 needs): no solve
    ends at the radius floor; the longest run of rejections is far short of 15."""
    problems = TS.sample(5, 60, lms=(16,), families=("strip", "lever", "prior", "degen"), row_counts=(7, 255, 4097))
    runs, terms = [], set()
    for p in problems:
        r = TS.numpy_solve(p)
        terms.add(r["termination"])
        runs.append(max((len(m) for m in r["steps"].split("a")), default=0))
    print("terminations:", sorted(terms), "longest run of rejections:", max(runs))
    assert 4 not in terms and max(runs) < 15

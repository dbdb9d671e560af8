"""Seeded problem families for the trust-region solve on given correspondences (so_solve, tests/test_trust_region*.py).

Every family is a list of problems {P (float32 values), N, D, W, start, lm, prior, degen}; what the solve does on them is decided by
the restatements (test_ceres_restatement.solve_full, degeneracy_numpy.solve_reduced, oracle.solve), not assumed here.

  well      _random_problem: points on three planes, starts up to 2.5 m / 0.6 rad off (the baseline: steps are accepted)
  strip     a thin strip: points along a 20 m line, axis normals, starts up to 0.5 m / 1 rad off.  Rotation is nonlinear on it and the
            Gauss-Newton model over-predicts the decrease: steps are rejected
  lever     short lever arms: points within 0.6 m of the sensor, starts up to 0.3 m / 1 rad off
  prior     SE3 prior rows (measurement x0 apart from the start).  Half: a strong prior whose measurement is rotated 2-2.8 rad from the
            start, on a well-posed problem at its truth.  The Gauss-Newton step on 2 vec(q_m^* q) is -2 tan(theta / 2) along the axis,
            but Plus turns a tangent step d into the rotation 2 atan(|d| / 2) -- exactly theta -- so it does not overshoot and these
            solves accept their steps.  The other half: the thin strip below with a weak-to-moderate prior near the truth, where the
            rows' rotation nonlinearity rejects steps with the prior rows in the system
  zero      exact zero residuals at the start (axis normals, d = -p_k in double, identity start): g = 0, gmax = 0, termination 1 at once
  saturated every row beyond the Tukey scale (s > a^2: H = g = 0, termination 1); with `live` rows inside it, an ordinary solve
  degen     the thin strip through the degeneracy-aware solve, thresholds that flag its weak directions: reduced steps rejected
"""
import numpy as np

import test_ceres_restatement as CR

PLANE_RES = 0.2
A = float(np.sqrt(np.float32(3 * np.float32(PLANE_RES))))      # TukeyLoss(std::sqrt(3 * planeRes_)) in float (LidarSlam.cpp:271)
A2 = A * A
ROW_COUNTS = (1, 7, 255, 4097, 65537)
FAMILIES = ("well", "strip", "lever", "prior", "zero", "saturated", "degen")
DEGEN_THRESHOLDS = (0.05, 0.05)


def _unit_quat(rng, angle):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    return np.concatenate([ax * np.sin(angle / 2), [np.cos(angle / 2)]])


def _offset(rng, x, dt, dr):
    """x moved by up to dt metres per axis and rotated by an angle up to dr about a random axis."""
    q = CR._qmul(x[3:], _unit_quat(rng, rng.uniform(0, dr)))
    return np.concatenate([x[:3] + rng.uniform(-dt, dt, 3), q / np.linalg.norm(q)])


def _sensor_frame(rng, world, normals, noise=0.01):
    """A random truth pose and the rows {p (sensor frame, float32), n, d, w} of world points on planes with the given normals."""
    n = len(world)
    truth = np.concatenate([rng.uniform(-5, 5, 3), _unit_quat(rng, rng.uniform(0, 0.5))])
    R = CR._rot(truth[3:])
    P = ((world - truth[:3]) @ R).astype(np.float32).astype(np.float64)
    D = -(normals * world).sum(1) + rng.normal(0, noise, n)
    W = rng.uniform(0.5, 1.0, n)
    return truth, P, D, W


def _problem(family, P, N, D, W, start, lm, prior=None, degen=None):
    return dict(family=family, P=P, N=N, D=D, W=W, start=np.asarray(start, float), lm=int(lm), prior=prior, degen=degen)


def make(family, rng, n, lm):
    """One problem of `family` with n rows and lm_max_iterations = lm."""
    if family == "well" or (family == "prior" and rng.integers(0, 2)):
        truth, P, N, D, W = CR._random_problem(rng, n)
        P = P.astype(np.float32).astype(np.float64)
        if family == "well":
            dt, dr = [(0.08, 0.015), (0.6, 0.12), (2.5, 0.6)][rng.integers(0, 3)]
            return _problem(family, P, N, D, W, _offset(rng, truth, dt, dr), lm)
        x0 = CR._qmul(truth[3:], _unit_quat(rng, rng.uniform(2.0, 2.8)))
        x0 = np.concatenate([truth[:3] + rng.uniform(-0.05, 0.05, 3), x0 / np.linalg.norm(x0)])
        return _problem(family, P, N, D, W, truth, lm, prior=(x0, float(rng.choice([20.0, 100.0, 1000.0])), (0.1, 0.2, 0.3)))
    if family == "prior":                                          # the thin strip with a prior near the truth
        world = np.stack([rng.uniform(-10, 10, n), rng.uniform(-0.05, 0.05, n), rng.uniform(-0.05, 0.05, n)], 1)
        N = np.eye(3)[rng.choice(3, n, p=[0.1, 0.45, 0.45])] * rng.choice([-1.0, 1.0], (n, 1))
        truth, P, D, W = _sensor_frame(rng, world, N)
        x0 = _offset(rng, truth, 0.1, 0.05)
        return _problem(family, P, N, D, W, _offset(rng, truth, 0.5, 1.0), lm,
                        prior=(x0, float(rng.choice([0.05, 0.5, 2.0])), tuple(rng.uniform(0, 0.5, 3))))
    if family in ("strip", "degen"):
        world = np.stack([rng.uniform(-10, 10, n), rng.uniform(-0.05, 0.05, n), rng.uniform(-0.05, 0.05, n)], 1)
        N = np.eye(3)[rng.choice(3, n, p=[0.1, 0.45, 0.45])] * rng.choice([-1.0, 1.0], (n, 1))
        truth, P, D, W = _sensor_frame(rng, world, N)
        start = _offset(rng, truth, 0.5, 1.0)
        return _problem(family, P, N, D, W, start, lm, degen=DEGEN_THRESHOLDS if family == "degen" else None)
    if family == "lever":
        world = rng.uniform(-0.6, 0.6, (n, 3))
        N = np.linalg.qr(rng.normal(size=(3, 3)))[0][rng.integers(0, 3, n)] * rng.choice([-1.0, 1.0], (n, 1))
        truth, P, D, W = _sensor_frame(rng, world, N, noise=0.002)
        return _problem(family, P, N, D, W, _offset(rng, truth, 0.3, 1.0), lm)
    if family == "zero":
        P = rng.uniform(-20, 20, (n, 3)).astype(np.float32).astype(np.float64)
        k = rng.integers(0, 3, n)
        N = np.eye(3)[k]
        D = -P[np.arange(n), k]
        return _problem(family, P, N, D, rng.uniform(0.5, 1.0, n), [0, 0, 0, 0, 0, 0, 1.0], lm)
    if family == "saturated":
        truth, P, N, D, W = CR._random_problem(rng, n)
        P = P.astype(np.float32).astype(np.float64)
        live = int(rng.integers(0, 2)) * min(n, 5)                 # none, or a handful of rows inside the Tukey scale
        D = D + np.where(np.arange(n) < live, 0.0, rng.choice([-1.0, 1.0], n) * rng.uniform(2.0, 50.0, n) * A)
        return _problem(family, P, N, D, W, _offset(rng, truth, 0.01, 0.002), lm)
    raise ValueError(family)


def prior_rows(p):
    """(measurement, sqrt_info) of the problem's prior, as the solve computes it from its row count; None without one."""
    if p["prior"] is None:
        return None
    x0, vcf, unc = p["prior"]
    return x0, CR.prior_sqrt_info(len(p["P"]), unc, vcf)


def numpy_problem(p):
    return CR.Problem(p["P"], p["N"], p["D"], p["W"], A2, prior=prior_rows(p))


def analysis(p):
    """degeneracy_numpy.analysis of H = J^T J at the start (degen problems), with the relative margin of every flag decision."""
    import degeneracy_numpy as DN
    _, _, J = numpy_problem(p).linearise(p["start"])
    a = DN.analysis(J.T @ J, *p["degen"])
    # the information blocks are Schur complements: their small eigenvalues cancel, and are known only to rounding of the size of H
    # (not of themselves), so a flag's margin is measured against that scale too
    margins, floor = [], max(1e-8 * np.abs(J.T @ J).max(), np.finfo(float).tiny)
    for w, thr in ((a["pos_info"], p["degen"][0]), (a["ori_info"], p["degen"][1])):
        cut = thr * thr * max(w[2], 0.0)
        margins += [abs(wk - cut) / max(abs(cut), floor) for wk in w[:2]]
    a["margin"] = min(margins)
    return a


def numpy_solve(p):
    """test_ceres_restatement.solve_full (degen: degeneracy_numpy.solve_reduced on analysis()'s B) -> its dict, plus flag counts."""
    import degeneracy_numpy as DN
    prob = numpy_problem(p)
    if p["degen"] is None:
        r = CR.solve_full(prob, p["start"], p["lm"])
        r["n_flag"] = (0, 0)
        return r
    a = analysis(p)
    r = DN.solve_reduced(prob, p["start"], a["B"], p["lm"], full=True)
    r["n_flag"] = (bin(a["flags_pos"]).count("1"), bin(a["flags_ori"]).count("1"))
    r["margin"] = min(r["margin"], a["margin"])
    return r


def oracle_corr(p):
    from oracle import oracle as O
    corr = np.zeros(len(p["P"]), O.CORR_DTYPE)
    corr["p"], corr["n"], corr["d"], corr["w"], corr["status"] = p["P"], p["N"], p["D"], p["W"], 0
    return corr


def oracle_solve(p):
    """oracle.solve (the ambient solve: the oracle has no reduced one) -> (pose, summary dict)."""
    from oracle import oracle as O
    assert p["degen"] is None
    return O.solve(oracle_corr(p), p["start"], PLANE_RES, p["lm"], pose_prior=p["prior"])


def sample(seed, per_family, lms=(4, 12, 16), row_counts=ROW_COUNTS, families=FAMILIES, max_rows=None):
    """per_family problems of each family, row counts and lm_max_iterations cycling through row_counts and lms (row counts above
    max_rows skipped)."""
    rng = np.random.default_rng(seed)
    counts = [n for n in row_counts if max_rows is None or n <= max_rows]
    out = []
    for fam in families:
        for i in range(per_family):
            out.append(make(fam, rng, counts[i % len(counts)], lms[(i // len(counts)) % len(lms)]))
    return out


def fair(r, min_margin=1e-6, max_radius_error=1e-10):
    """Whether no decision of the solve (numpy result r) is within min_margin (relative) of its threshold and rounding cannot move
    its final radius by more than max_radius_error (see test_ceres_restatement.solve_full): only then are identical trip counts, and
    poses and radii equal to 1e-9, a fair demand of solvers that factor differently (Cholesky of the normal equations / Householder
    QR) and sum in different orders."""
    return r["margin"] > min_margin and r["radius_error"] < max_radius_error

"""Seeded problem families for the two-block solve of so_register_optimized on given correspondences (so_solve_optimized,
tests/test_motion_solve*.py), in the style of trust_region_sets.py.

Every problem is {P (float32 values), tau (float32), N, D, W, start (T), motion (D at the start), dt, D0, info, lm}; the rows are plane
rows on u(D) (optimized_numpy), the prior rows SE3AbsolutatePoseFactor on D with multiplier sqrt(n_rows * info_k).  What the solve
does on them is decided by the restatements (optimized_numpy.solve_full2, oracle.solve_optimized), not assumed here.

  well         points on three planes, tau over [0, dt], a true motion of about 1 m and 0.05 rad, starts up to 0.6 m / 0.12 rad off
               (the baseline: steps are accepted)
  strip        a thin strip along a 20 m line with axis normals, T starts up to 0.5 m / 1.5 rad off: rotation is nonlinear on it, the
               Gauss-Newton model over-predicts the decrease and steps are rejected
  lever        points within 0.6 m of the sensor, T starts up to 0.3 m / 1 rad off
  prior        half: a strong motion_info with D0 1-3 m and 1-2 rad from the start, on a well-posed problem at its truth; half: the
               thin strip with a moderate prior near the true motion, so that steps are rejected with the prior rows in the system
  static       every tau 0, NaN or +-inf (alpha = 0): the D columns are exactly zero, and with info = 0 the solve never moves D's
               translation
  extrapolated alpha in [-0.5, 1.5]
  branches     a start D with q.w < 0, one with 0 < |phi| < 1e-2 (the series branch of J_r), and D exactly the identity (Eigen's linear
               slerp branch)
  zero         tau = 0, T, D and D0 the identity, axis normals and d = -p_k: every residual and the prior's are exactly zero, gmax = 0,
               termination 1 at once
  saturated    every row beyond the Tukey scale (H = g = 0 in the plane rows), with and without prior rows
"""
import math

import numpy as np

import optimized_numpy as ON
import test_ceres_restatement as CR
import trust_region_sets as TS

PLANE_RES = TS.PLANE_RES
A2 = TS.A2
DT = 0.1
IDENTITY = np.array([0.0, 0, 0, 0, 0, 0, 1.0])
ROW_COUNTS = (1, 7, 255, 256, 257, 4096, 4097, 65536, 65537)
LMS = (4, 12, 16)
FAMILIES = ("well", "strip", "lever", "prior", "static", "extrapolated", "branches", "zero", "saturated")


def _unit(x):
    """pose7 with its quaternion normalised in the order the device's make_state normalises D0"""
    x = np.array(x, float)
    x[3:] = x[3:] / math.sqrt(x[3] * x[3] + x[4] * x[4] + x[5] * x[5] + x[6] * x[6])
    return x


def _motion(rng, trans=1.0, rot=0.05):
    return np.concatenate([rng.uniform(-trans, trans, 3), TS._unit_quat(rng, rng.uniform(0, rot))])


def _rows(rng, world, normals, T, Dm, tau, noise=0.01):
    """Sensor-frame raw points (float32 values) whose u(Dm) lies on world at pose T, the planes' d and the weights"""
    A = ON.alphas(tau, DT)
    u = (world - T[:3]) @ CR._rot(T[3:])                                  # R(q_T)^T (x - t_T)
    Ra = ON._slerp_Rs(Dm[3:] / np.linalg.norm(Dm[3:]), A)
    P = np.einsum("nji,nj->ni", Ra, u - A[:, None] * Dm[:3]).astype(np.float32).astype(np.float64)
    D = -(normals * world).sum(1) + rng.normal(0, noise, len(world))
    return P, D, rng.uniform(0.5, 1.0, len(world))


def _problem(family, rng, world, N, tau, start, motion, D0, info, lm, noise=0.01, T=None, Dm=None):
    T = np.concatenate([rng.uniform(-5, 5, 3), TS._unit_quat(rng, rng.uniform(0, 0.5))]) if T is None else T
    Dm = _motion(rng) if Dm is None else Dm
    P, D, W = _rows(rng, world, N, T, Dm, tau, noise)
    return dict(family=family, P=P, tau=np.asarray(tau, np.float32), N=N, D=D, W=W, dt=DT, lm=int(lm), truth=(T, Dm),
                start=np.asarray(start(T), float), motion=_unit(motion(Dm)), D0=_unit(D0(Dm)), info=np.asarray(info, float))


def _strip(rng, n):
    world = np.stack([rng.uniform(-10, 10, n), rng.uniform(-0.05, 0.05, n), rng.uniform(-0.05, 0.05, n)], 1)
    return world, np.eye(3)[rng.choice(3, n, p=[0.1, 0.45, 0.45])] * rng.choice([-1.0, 1.0], (n, 1))


def _planes(rng, n):
    """points on three planes n.x = offs of random orientation"""
    normals = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    k = rng.integers(0, 3, n)
    N = normals[k] * rng.choice([-1.0, 1.0], n)[:, None]
    world = rng.uniform(-20, 20, (n, 3))
    offs = rng.uniform(2, 15, 3)[k]
    return world - ((world * N).sum(1) - offs)[:, None] * N, N


def make(family, rng, n, lm):
    """One problem of `family` with n rows and lm_max_iterations = lm."""
    tau = rng.uniform(0, DT, n).astype(np.float32)
    off = lambda dt, dr: (lambda x: TS._offset(rng, x, dt, dr))         # noqa: E731
    same = lambda x: x                                                   # noqa: E731
    no_info = np.zeros(6)
    small_info = lambda: rng.choice([0.0, 0.01, 0.5]) * np.ones(6)       # noqa: E731
    if family == "well":
        world, N = _planes(rng, n)
        return _problem(family, rng, world, N, tau, off(0.6, 0.12), off(0.6, 0.12), off(0.1, 0.02), small_info(), lm)
    if family == "strip":
        world, N = _strip(rng, n)
        return _problem(family, rng, world, N, tau, off(0.5, 1.5), off(0.2, 0.1), off(0.1, 0.02), small_info(), lm)
    if family == "lever":
        world = rng.uniform(-0.6, 0.6, (n, 3))
        N = np.linalg.qr(rng.normal(size=(3, 3)))[0][rng.integers(0, 3, n)] * rng.choice([-1.0, 1.0], (n, 1))
        return _problem(family, rng, world, N, tau, off(0.3, 1.0), off(0.2, 0.1), off(0.1, 0.02), small_info(), lm, noise=0.002)
    if family == "prior":
        if rng.integers(0, 2):                                           # strong prior far from the start
            world, N = _planes(rng, n)
            far = lambda x: _unit(np.concatenate([x[:3] + rng.uniform(1, 3, 3) * rng.choice([-1, 1], 3),   # noqa: E731
                                                  CR._qmul(x[3:], TS._unit_quat(rng, rng.uniform(1.0, 2.0)))]))
            return _problem(family, rng, world, N, tau, same, same, far, rng.choice([10.0, 100.0, 1000.0]) * np.ones(6), lm)
        world, N = _strip(rng, n)
        return _problem(family, rng, world, N, tau, off(0.5, 1.5), off(0.2, 0.1), off(0.1, 0.05),
                        rng.choice([0.05, 0.5, 2.0]) * rng.uniform(0.2, 1.0, 6), lm)
    if family == "static":
        tau = rng.choice(np.array([0.0, np.nan, np.inf, -np.inf], np.float32), n)
        world, N = _planes(rng, n)
        info = no_info if rng.integers(0, 2) else small_info()
        return _problem(family, rng, world, N, tau, off(0.6, 0.12), off(0.6, 0.12), off(0.1, 0.02), info, lm)
    if family == "extrapolated":
        tau = rng.uniform(-0.5 * DT, 1.5 * DT, n).astype(np.float32)
        world, N = _planes(rng, n)
        return _problem(family, rng, world, N, tau, off(0.6, 0.12), off(0.6, 0.12), off(0.1, 0.02), small_info(), lm)
    if family == "branches":
        world, N = _planes(rng, n)
        kind = rng.integers(0, 3)
        if kind == 0:                                                    # the same rotation with q.w < 0
            start_d = lambda x: np.concatenate([x[:3], -TS._offset(rng, x, 0.3, 0.05)[3:]])       # noqa: E731
        elif kind == 1:                                                  # 0 < |phi| < 1e-2
            start_d = lambda x: np.concatenate([x[:3] + rng.uniform(-0.3, 0.3, 3), TS._unit_quat(rng, rng.uniform(1e-5, 9e-3))])  # noqa: E731
        else:
            start_d = lambda x: IDENTITY.copy()                          # noqa: E731
        return _problem(family, rng, world, N, tau, off(0.3, 0.05), start_d, off(0.1, 0.02), small_info(), lm)
    if family == "zero":
        P = rng.uniform(-20, 20, (n, 3)).astype(np.float32).astype(np.float64)
        k = rng.integers(0, 3, n)
        return dict(family=family, P=P, tau=np.zeros(n, np.float32), N=np.eye(3)[k], D=-P[np.arange(n), k], W=rng.uniform(0.5, 1.0, n),
                    dt=DT, lm=int(lm), truth=(IDENTITY, IDENTITY), start=IDENTITY.copy(), motion=IDENTITY.copy(), D0=IDENTITY.copy(),
                    info=small_info())
    if family == "saturated":
        world, N = _planes(rng, n)
        p = _problem(family, rng, world, N, tau, off(0.01, 0.002), off(0.01, 0.002), off(0.3, 0.1), small_info(), lm)
        p["D"] = p["D"] + rng.choice([-1.0, 1.0], n) * rng.uniform(2.0, 50.0, n) * TS.A
        return p
    raise ValueError(family)


def numpy_problem(p):
    return ON.Problem(p["P"], ON.alphas(p["tau"], p["dt"]), p["N"], p["D"], p["W"], A2, p["D0"], p["info"])


def numpy_solve(p):
    """optimized_numpy.solve_full2 -> its dict (x = [T, D], steps, margin, radius_error, ...)"""
    return ON.solve_full2(numpy_problem(p), p["start"], p["motion"], p["lm"])


def oracle_solve(p):
    """oracle.solve_optimized -> (T, D, summary dict)"""
    from oracle import oracle as O
    return O.solve_optimized(p["P"], p["tau"], p["N"], p["D"], p["W"], p["start"], p["motion"], p["dt"], p["D0"], p["info"], PLANE_RES,
                             p["lm"])


def sample(seed, per_family, lms=LMS, row_counts=ROW_COUNTS, families=FAMILIES):
    """per_family problems of each family, row counts and lm_max_iterations cycling through row_counts and lms."""
    rng = np.random.default_rng(seed)
    out = []
    for fam in families:
        for i in range(per_family):
            out.append(make(fam, rng, row_counts[i % len(row_counts)], lms[(i // len(row_counts)) % len(lms)]))
    return out


def fair_sample(seed, per_family, **kw):
    """sample(), keeping the problems trust_region_sets.fair accepts (with their numpy results); prints how many were dropped"""
    problems = sample(seed, per_family, **kw)
    results = [numpy_solve(p) for p in problems]
    kept = [(p, r) for p, r in zip(problems, results) if TS.fair(r)]
    print(f"\n{len(problems) - len(kept)} of {len(problems)} two-block problems dropped: a decision within 1e-6 of its threshold, or a "
          f"radius rounding can move by 1e-10")
    return kept

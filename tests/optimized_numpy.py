"""numpy restatement of so_register_optimized's solve (so_motion.cu): the warp u(D), the plane rows over two pose7 blocks (T, D), their
12-column Jacobian, the motion prior rows and the two-block trust-region loop.

Written apart from the device code: rotation matrices instead of quaternion rotations, the D rotation columns as
alpha (p x b)^T J_r(alpha phi) J_r(phi)^-1 with J_r built as 3x3 matrices, numpy's LAPACK least squares for the step.  The warp
(float(u(D)), what every ICP iteration searches with) restates the device's bits through undistort_numpy."""
from __future__ import annotations

import math

import numpy as np

import undistort_numpy as UN
from test_ceres_restatement import (FUNCTION_TOL, GRADIENT_TOL, MAX_LM_DIAG, MAX_RADIUS, MIN_LM_DIAG, MIN_RADIUS, MIN_REL_DECREASE,
                                    PARAMETER_TOL, _plus, _qmul, _rot)


def warp_points(xyz_time: np.ndarray, D, dt: float) -> np.ndarray:
    """float(u(D)) [n, 3] float32: undistort_numpy's pInit with (q_D, t_D) taken from D instead of T_prev^-1 T_cur."""
    # with prev = the identity at the origin, undistort_numpy's D = prev^-1 * cur is cur exactly (products with 1 and 0), normalised
    # in the device's operation order
    return UN.undistort_points(xyz_time, np.asarray(D, np.float64), np.array([0.0, 0, 0, 0, 0, 0, 1.0]), dt, True)


def alphas(times, dt):
    t = np.asarray(times, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        return np.where(np.isfinite(t), t / float(dt), 0.0)


def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def _log_q(q):
    """rotation vector of a unit quaternion on the shortest path"""
    q = np.asarray(q, np.float64) / np.linalg.norm(q)
    if q[3] < 0:
        q = -q
    vn = np.linalg.norm(q[:3])
    if vn == 0.0:
        return np.zeros(3)
    return q[:3] * (2.0 * math.atan2(vn, q[3]) / vn)


def _jr(v):
    th = np.linalg.norm(v)
    K = _skew(v)
    if th < 1e-4:
        return np.eye(3) - 0.5 * K + K @ K / 6.0
    return np.eye(3) - (1 - math.cos(th)) / th ** 2 * K + (th - math.sin(th)) / th ** 3 * K @ K


def _slerp_R(q, a):
    """R(slerp(identity, q, a)) with Eigen's branches (linear for |q.w| >= 1 - eps: not unit, as Eigen leaves it)"""
    q = np.asarray(q, np.float64)
    ad = abs(q[3])
    if ad >= 1.0 - UN.EPS:
        s0, s1 = 1.0 - a, a
    else:
        th = math.acos(ad)
        s0, s1 = math.sin((1 - a) * th) / math.sin(th), math.sin(a * th) / math.sin(th)
    if q[3] < 0:
        s1 = -s1
    qa = np.array([s1 * q[0], s1 * q[1], s1 * q[2], s0 + s1 * q[3]])
    x, y, z, w = qa                                                      # qrot of a possibly non-unit quaternion, as a matrix
    return np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


def warp_double(P, A, D):
    """u_i(D) in double [n, 3]"""
    D = np.asarray(D, np.float64)
    q = D[3:] / np.linalg.norm(D[3:])
    return np.stack([_slerp_R(q, a) @ p for p, a in zip(P, A)]) + A[:, None] * D[:3]


def residuals(P, A, N, Dd, T, D):
    return (N * (warp_double(P, A, D) @ _rot(T[3:]).T + T[:3])).sum(1) + Dd


def jacobian(P, A, N, T, D):
    """[n, 12] local Jacobian of residuals() in (dt_T, dtheta_T, dt_D, dtheta_D) under PoseLocalParameterization"""
    R = _rot(T[3:])
    q = np.asarray(D[3:], np.float64) / np.linalg.norm(D[3:])
    phi = _log_q(q)
    jinv = np.linalg.inv(_jr(phi))
    U = warp_double(P, A, D)
    out = np.zeros((len(P), 12))
    for i, (p, a, n, u) in enumerate(zip(P, A, N, U)):
        av = R.T @ n
        b = _slerp_R(q, a).T @ av
        out[i, :3] = n
        out[i, 3:6] = np.cross(u, av)
        out[i, 6:9] = a * av
        out[i, 9:] = a * (np.cross(p, b) @ _jr(a * phi) @ jinv)
    return out


class Problem:
    """Plane rows {p, alpha, n, d, w} under ScaledLoss(TukeyLoss(a), w) over (T, D), and the motion prior rows on D."""

    def __init__(self, P, A, N, Dd, W, a2, D0, info):
        self.P, self.A, self.N, self.Dd, self.W, self.a2 = P, A, N, Dd, W, a2
        self.D0 = np.asarray(D0, np.float64)
        self.sqrt_info = np.sqrt(len(P) * np.asarray(info, np.float64))

    def _rho(self, s):
        inside = s <= self.a2
        v = np.where(inside, 1.0 - s / self.a2, 0.0)
        return (np.where(inside, self.a2 / 6.0 * (1.0 - v ** 3), self.a2 / 6.0) * self.W, np.where(inside, 0.5 * v * v, 0.0) * self.W)

    def _prior(self, D):
        e = _qmul(np.array([-self.D0[3], -self.D0[4], -self.D0[5], self.D0[6]]), D[3:])
        r = np.concatenate([D[:3] - self.D0[:3], 2.0 * e[:3]])
        J = np.zeros((6, 12))
        J[:3, 6:9] = np.eye(3)
        J[3:, 9:] = e[3] * np.eye(3) + _skew(e[:3])
        return r * self.sqrt_info, J * self.sqrt_info[:, None]

    def cost(self, T, D):
        r = residuals(self.P, self.A, self.N, self.Dd, T, D)
        rp, _ = self._prior(D)
        return 0.5 * self._rho(r * r)[0].sum() + 0.5 * (rp * rp).sum()

    def linearise(self, T, D):
        r = residuals(self.P, self.A, self.N, self.Dd, T, D)
        rho0, rho1 = self._rho(r * r)
        sc = np.sqrt(rho1)
        J = jacobian(self.P, self.A, self.N, T, D) * sc[:, None]
        rp, Jp = self._prior(D)
        return 0.5 * rho0.sum() + 0.5 * (rp * rp).sum(), np.concatenate([r * sc, rp]), np.concatenate([J, Jp])

    def normal_equations(self, T, D):
        """plane rows only: H, g, cost (so_evaluate_optimized)"""
        r = residuals(self.P, self.A, self.N, self.Dd, T, D)
        rho0, rho1 = self._rho(r * r)
        J = jacobian(self.P, self.A, self.N, T, D)
        return (J * rho1[:, None]).T @ J, J.T @ (rho1 * r), 0.5 * rho0.sum()


def solve(prob, T0, D0, max_iterations=4):
    """-> (T, D, iterations, successful_steps, unsuccessful_steps, termination), the codes of so_icp_result.iter_lm_termination"""
    T, D = np.array(T0, float), np.array(D0, float)
    D[3:] /= np.linalg.norm(D[3:])
    cost, res, J = prob.linearise(T, D)
    scale = 1.0 / (1.0 + np.linalg.norm(J, axis=0))

    def gmax_of(T, D, g):
        return max(np.abs(T - _plus(T, -g[:6])).max(), np.abs(D - _plus(D, -g[6:])).max())
    gmax = gmax_of(T, D, J.T @ res)
    Js = J * scale
    radius, decrease, reuse, diag = 1e4, 2.0, False, None
    it = succ = unsucc = invalid = 0
    step_ok = False
    while True:
        if step_ok:
            succ += 1
        else:
            unsucc += 1
        if it >= max_iterations:
            return T, D, it, succ, unsucc, 0
        if gmax <= GRADIENT_TOL:
            return T, D, it, succ, unsucc, 1
        if radius <= MIN_RADIUS:
            return T, D, it, succ, unsucc, 4
        it += 1
        step_ok = False
        if not reuse:
            diag = np.clip((Js * Js).sum(0), MIN_LM_DIAG, MAX_LM_DIAG)
        reuse = True
        y = np.linalg.lstsq(np.concatenate([Js, np.diag(np.sqrt(diag / radius))]), np.concatenate([res, np.zeros(12)]), rcond=None)[0]
        step = -y
        mr = Js @ step
        model_change = -(mr * (res + mr / 2.0)).sum()
        if not (np.isfinite(step).all() and model_change > 0.0):
            invalid += 1
            if invalid >= 5:
                return T, D, it, succ, unsucc, 5
            radius *= 0.5
            continue
        invalid = 0
        d = step * scale
        Tc, Dc = _plus(T, d[:6]), _plus(D, d[6:])
        cand_cost = prob.cost(Tc, Dc)
        if math.sqrt(((T - Tc) ** 2).sum() + ((D - Dc) ** 2).sum()) <= PARAMETER_TOL * (math.sqrt((T * T).sum() + (D * D).sum()) + PARAMETER_TOL):
            return T, D, it, succ, unsucc, 2
        change = cost - cand_cost
        if abs(change) <= FUNCTION_TOL * cost:
            return T, D, it, succ, unsucc, 3
        rel = change / model_change
        if rel > MIN_REL_DECREASE:
            T, D = Tc, Dc
            cost, res, J = prob.linearise(T, D)
            Js = J * scale
            gmax = gmax_of(T, D, J.T @ res)
            step_ok = True
            radius = min(MAX_RADIUS, radius / max(1.0 / 3.0, 1.0 - (2.0 * rel - 1.0) ** 3))
            decrease, reuse = 2.0, False
        else:
            radius /= decrease
            decrease *= 2.0
            reuse = True


def compose(T, D):
    """T * D as pose7"""
    return np.concatenate([T[:3] + _rot(T[3:]) @ D[:3], _qmul(T[3:], D[3:])])


def inverse(T):
    qc = np.array([-T[3], -T[4], -T[5], T[6]])
    return np.concatenate([-(_rot(qc) @ T[:3]), qc])

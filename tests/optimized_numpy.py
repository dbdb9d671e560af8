"""numpy restatement of so_register_optimized's solve (so_motion.cu): the warp u(D), the plane rows over two pose7 blocks (T, D), their
12-column Jacobian and the motion prior rows; the two-block trust-region loop is test_ceres_restatement.solve_full over the two pose7
blocks (T, D).

Written apart from the device code: rotation matrices instead of quaternion rotations, the D rotation columns as
alpha (p x b)^T J_r(alpha phi) J_r(phi)^-1 with J_r(phi)^-1 a 3x3 matrix inverse, numpy's LAPACK least squares for the step.  The warp
(float(u(D)), what every ICP iteration searches with) restates the device's bits through undistort_numpy."""
from __future__ import annotations

import math

import numpy as np

import undistort_numpy as UN
from test_ceres_restatement import _plus, _qmul, _rot, solve_full


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


def _slerp_coeffs(q, A):
    """s0, s1 [n] of Eigen's slerp(identity, q, alpha) for unit q: linear for |q.w| >= 1 - eps (not unit then, as Eigen leaves it)"""
    A = np.asarray(A, np.float64)
    ad = abs(q[3])
    if ad >= 1.0 - UN.EPS:
        s0, s1 = 1.0 - A, A.copy()
    else:
        th = math.acos(ad)
        s0, s1 = np.sin((1 - A) * th) / math.sin(th), np.sin(A * th) / math.sin(th)
    return s0, (-s1 if q[3] < 0 else s1)


def _slerp_Rs(q, A):
    """R(slerp(identity, q, alpha)) [n, 3, 3] for every alpha: the rotation of a possibly non-unit quaternion, as a matrix"""
    s0, s1 = _slerp_coeffs(np.asarray(q, np.float64), A)
    x, y, z, w = s1 * q[0], s1 * q[1], s1 * q[2], s0 + s1 * q[3]
    return np.stack([np.stack([w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z], -1)], -2)


def warp_double(P, A, D):
    """u_i(D) in double [n, 3]"""
    D = np.asarray(D, np.float64)
    q = D[3:] / np.linalg.norm(D[3:])
    return np.einsum("nij,nj->ni", _slerp_Rs(q, A), P) + A[:, None] * D[:3]


def residuals(P, A, N, Dd, T, D):
    return (N * (warp_double(P, A, D) @ _rot(T[3:]).T + T[:3])).sum(1) + Dd


def jacobian(P, A, N, T, D):
    """[n, 12] local Jacobian of residuals() in (dt_T, dtheta_T, dt_D, dtheta_D) under PoseLocalParameterization"""
    R = _rot(T[3:])
    q = np.asarray(D[3:], np.float64) / np.linalg.norm(D[3:])
    phi = _log_q(q)
    jinv = np.linalg.inv(_jr(phi))
    Ra = _slerp_Rs(q, A)
    U = np.einsum("nij,nj->ni", Ra, P) + A[:, None] * np.asarray(D[:3], np.float64)
    av = N @ R                                                           # rows: R^T n
    b = np.einsum("nji,nj->ni", Ra, av)                                  # R(q_alpha)^T R^T n
    w = np.cross(P, b)
    # w^T J_r(v), v = alpha phi: w^T [v]x = w x v, so w^T J_r(v) = w - c1 (w x v) + c2 (w x v) x v
    V = A[:, None] * phi
    th = np.abs(A) * np.linalg.norm(phi)
    small = th < 1e-4
    ths = np.where(small, 1.0, th)
    c1 = np.where(small, 0.5, (1 - np.cos(ths)) / ths ** 2)
    c2 = np.where(small, 1.0 / 6.0, (ths - np.sin(ths)) / ths ** 3)
    wv = np.cross(w, V)
    wj = w - c1[:, None] * wv + c2[:, None] * np.cross(wv, V)
    return np.concatenate([N, np.cross(U, av), A[:, None] * av, A[:, None] * (wj @ jinv)], 1)


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


class _Stacked:
    """A (T, D) problem as solve_full sees it: one vector of the two pose7 blocks"""

    def __init__(self, prob):
        self.prob = prob

    def cost(self, x):
        return self.prob.cost(x[:7], x[7:])

    def linearise(self, x):
        return self.prob.linearise(x[:7], x[7:])


def solve_full2(prob, T0, D0, max_iterations=4):
    """solve_full over (T, D) from T0 and D0 (its quaternion normalised): its dict, with x = [T, D]"""
    D = np.array(D0, float)
    D[3:] /= np.linalg.norm(D[3:])
    return solve_full(_Stacked(prob), np.concatenate([np.asarray(T0, float), D]), max_iterations)


def solve(prob, T0, D0, max_iterations=4):
    """-> (T, D, iterations, successful_steps, unsuccessful_steps, termination), the codes of so_icp_result.iter_lm_termination"""
    r = solve_full2(prob, T0, D0, max_iterations)
    return r["x"][:7], r["x"][7:], r["iterations"], r["successful"], r["unsuccessful"], r["termination"]


def compose(T, D):
    """T * D as pose7"""
    return np.concatenate([T[:3] + _rot(T[3:]) @ D[:3], _qmul(T[3:], D[3:])])


def inverse(T):
    qc = np.array([-T[3], -T[4], -T[5], T[6]])
    return np.concatenate([-(_rot(qc) @ T[:3]), qc])

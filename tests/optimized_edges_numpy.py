"""numpy restatement of so_register_optimized_edges' line rows (so_motion.cu, k_motion_eval_edge): EdgeAnalyticCostFunction at
lp = R(q) u(D) + t over the two pose7 blocks (T, D).

r = (lp - a) x (lp - b) / |a - b|, dr/dlp = skew(b - a) / |a - b|; row k of the 12-column Jacobian is optimized_numpy's plane row
with n replaced by the k-th row of that matrix.  Loss: ScaledLoss(TukeyLoss) over the 3-vector, rho' scaling both J^T J and J^T r."""
from __future__ import annotations

import numpy as np

import optimized_numpy as ON


def _dlp(LA, LB):
    """[n, 3, 3] skew(b - a) / |a - b| per correspondence"""
    e = LB - LA
    K = np.zeros((len(e), 3, 3))
    K[:, 0, 1], K[:, 0, 2] = -e[:, 2], e[:, 1]
    K[:, 1, 0], K[:, 1, 2] = e[:, 2], -e[:, 0]
    K[:, 2, 0], K[:, 2, 1] = -e[:, 1], e[:, 0]
    return K / np.linalg.norm(e, axis=1)[:, None, None]


def line_residuals(P, A, LA, LB, T, D):
    """[n, 3]"""
    lp = ON.warp_double(P, A, D) @ ON._rot(T[3:]).T + T[:3]
    return np.cross(lp - LA, lp - LB) / np.linalg.norm(LA - LB, axis=1)[:, None]


def line_jacobian(P, A, LA, LB, T, D):
    """[n, 3, 12] local Jacobian of line_residuals() in (dt_T, dtheta_T, dt_D, dtheta_D)"""
    M = _dlp(LA, LB)
    return np.stack([ON.jacobian(P, A, M[:, k, :], T, D) for k in range(3)], 1)


def line_normal_equations(P, A, LA, LB, W, a2, T, D):
    """(H [12, 12], g [12], cost) of the line rows under ScaledLoss(TukeyLoss(a), w)"""
    r = line_residuals(P, A, LA, LB, T, D)
    s = (r * r).sum(1)
    inside = s <= a2
    v = np.where(inside, 1.0 - s / a2, 0.0)
    rho0 = np.where(inside, a2 / 6.0 * (1.0 - v ** 3), a2 / 6.0) * W
    rho1 = np.where(inside, 0.5 * v * v, 0.0) * W
    J = line_jacobian(P, A, LA, LB, T, D)
    H = np.einsum("n,nki,nkj->ij", rho1, J, J)
    g = np.einsum("n,nki,nk->i", rho1, J, r)
    return H, g, 0.5 * rho0.sum()


class PlaneLineProblem(ON.Problem):
    """optimized_numpy's Problem plus line rows {p, alpha, a, b, w} under ScaledLoss(TukeyLoss(a_line), w): the two-block solve of
    so_register_optimized_edges (set sqrt_info with n = planes + lines, the multiplier's count)."""

    def __init__(self, planes: ON.Problem, P, A, LA, LB, W, a2_line):
        self.__dict__.update(planes.__dict__)
        self.LP, self.LA_, self.LA, self.LB, self.LW, self.a2_line = P, A, LA, LB, W, a2_line

    def _line(self, T, D):
        r = line_residuals(self.LP, self.LA_, self.LA, self.LB, T, D)
        s = (r * r).sum(1)
        inside = s <= self.a2_line
        v = np.where(inside, 1.0 - s / self.a2_line, 0.0)
        return r, np.where(inside, self.a2_line / 6.0 * (1.0 - v ** 3), self.a2_line / 6.0) * self.LW, np.where(inside, 0.5 * v * v, 0.0) * self.LW

    def cost(self, T, D):
        return super().cost(T, D) + 0.5 * self._line(T, D)[1].sum()

    def linearise(self, T, D):
        c, res, J = super().linearise(T, D)
        r, rho0, rho1 = self._line(T, D)
        sc = np.sqrt(rho1)
        Jl = line_jacobian(self.LP, self.LA_, self.LA, self.LB, T, D) * sc[:, None, None]
        return c + 0.5 * rho0.sum(), np.concatenate([res, (r * sc[:, None]).ravel()]), np.concatenate([J, Jl.reshape(-1, 12)])

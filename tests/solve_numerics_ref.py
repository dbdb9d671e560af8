"""Plain high-precision restatements of the end of the solve, independent of oracle/so_oracle.cpp:

line_rows / line_normal_equations
    EdgeAnalyticCostFunction (lidarOptimization.cpp:12-47) per row -- r = ((lp - a) x (lp - b)) / |a - b| with lp = R p + t,
    J = skew(b - a) [I, -R [p]x] / |a - b| on the tangent (dt, dtheta) of PoseLocalParameterization::Plus -- under Ceres 2.0's
    ScaledLoss(TukeyLoss(a), w) and its Corrector (rho'' <= 0: residual and Jacobian scaled by sqrt(rho')).  H = sum rho' J^T J,
    g = sum rho' J^T r and cost = 1/2 sum rho are summed exactly (math.fsum per entry) over float64 per-row terms.

covariance_reference
    ceres::Covariance's pseudo-inverse on a symmetric H in mpmath (50 digits): eigen-decomposition, directions with
    sqrt(w_i / w_max) < 1e-7 cut together with every smaller one, V diag(1/w) V^T; then EstimateRegistrationError's 3x3 analyses
    (LidarSlam.cpp:873-884) of the position and orientation blocks, again in mpmath."""
import math

import mpmath
import numpy as np

CUT = 1e-7                      # sqrt(min_reciprocal_condition_number = 1e-14) of ceres::Covariance::Options


def tukey_a2(res):
    """a^2 of TukeyLoss(std::sqrt(3 * res)) with res a float: float product, float sqrt, squared in double."""
    a = float(np.sqrt(np.float32(3) * np.float32(res)))
    return a * a


def quat_to_R(q):
    x, y, z, w = (float(v) for v in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def pose_plus(x, d):
    """PoseLocalParameterization::Plus: t += dt, q <- normalize(q * [dtheta / 2, 1])"""
    x = np.asarray(x, np.float64)
    t = x[:3] + d[:3]
    qa, qb = x[3:], np.array([d[3] / 2, d[4] / 2, d[5] / 2, 1.0])
    q = np.array([qa[3] * qb[0] + qa[0] * qb[3] + qa[1] * qb[2] - qa[2] * qb[1],
                  qa[3] * qb[1] + qa[1] * qb[3] + qa[2] * qb[0] - qa[0] * qb[2],
                  qa[3] * qb[2] + qa[2] * qb[3] + qa[0] * qb[1] - qa[1] * qb[0],
                  qa[3] * qb[3] - qa[0] * qb[0] - qa[1] * qb[1] - qa[2] * qb[2]])
    return np.concatenate([t, q / np.linalg.norm(q)])


def _skew(v):
    z = np.zeros(v.shape[:-1])
    return np.stack([np.stack([z, -v[..., 2], v[..., 1]], -1), np.stack([v[..., 2], z, -v[..., 0]], -1),
                     np.stack([-v[..., 1], v[..., 0], z], -1)], -2)


def line_residual(p, a, b, pose):
    """r [n, 3] of the line rows at pose7 (p: sensor-frame points [n, 3], a, b: line points [n, 3])"""
    p, a, b = (np.asarray(v, np.float64).reshape(-1, 3) for v in (p, a, b))
    lp = p @ quat_to_R(pose[3:]).T + np.asarray(pose[:3], np.float64)
    den = np.linalg.norm(a - b, axis=1)[:, None]
    return np.cross(lp - a, lp - b) / den


def line_rows(p, a, b, w, pose, a2):
    """-> r [n, 3], J [n, 3, 6], rho0 [n], rho1 [n] (the ScaledLoss values w * rho, w * rho')"""
    p, a, b = (np.asarray(v, np.float64).reshape(-1, 3) for v in (p, a, b))
    w = np.asarray(w, np.float64)
    R = quat_to_R(pose[3:])
    r = line_residual(p, a, b, pose)
    den = np.linalg.norm(a - b, axis=1)[:, None, None]
    K = _skew(b - a)
    J = np.concatenate([K, K @ (-(R @ _skew(p)))], 2) / den
    s = (r * r).sum(1)
    inside = s <= a2
    t = np.where(inside, 1.0 - s / a2, 0.0)
    rho0 = np.where(inside, a2 / 6.0 * (1.0 - t ** 3), a2 / 6.0) * w
    rho1 = np.where(inside, 0.5 * t * t, 0.0) * w
    return r, J, rho0, rho1


def line_normal_equations(p, a, b, w, pose, a2):
    """-> H [6, 6], g [6], cost, and the number of rows inside the Tukey core (s <= a^2)"""
    r, J, rho0, rho1 = line_rows(p, a, b, w, pose, a2)
    Ht = rho1[:, None, None] * np.einsum("nki,nkj->nij", J, J)
    gt = rho1[:, None] * np.einsum("nki,nk->ni", J, r)
    H = np.array([[math.fsum(Ht[:, i, j]) for j in range(6)] for i in range(6)])
    g = np.array([math.fsum(gt[:, i]) for i in range(6)])
    cost = math.fsum(0.5 * rho0)
    return H, g, cost, int(((r * r).sum(1) <= a2).sum())


def _mp_eigsy(M, dps):
    with mpmath.workdps(dps):
        w, V = mpmath.eigsy(mpmath.matrix(M.tolist()))
        order = sorted(range(len(w)), key=lambda i: w[i])
        return [w[i] for i in order], [[V[r, i] for i in order] for r in range(V.rows)]


def covariance_reference(H, dps=50):
    """-> dict(cov [6, 6] (T's block), keep [n] bool (ascending eigenvalue order), ratio [n] = sqrt(w_i / w_max),
    w [n], pos_err, pos_dir, pos_inv_cond, pos_gap, ori_err_deg, ori_dir, ori_inv_cond, ori_gap) of the exactly-read double H."""
    H = np.asarray(H, np.float64)
    n = H.shape[0]
    with mpmath.workdps(dps):
        w, V = _mp_eigsy(H, dps)
        wmax = w[-1]
        ratio = [mpmath.sqrt(x / wmax) if (x > 0 and wmax > 0) else mpmath.mpf(0) for x in w]
        keep = [True] * n
        cut = False
        for i in range(n - 1, -1, -1):                  # descending: a cut direction cuts every smaller one
            cut = cut or ratio[i] < CUT
            keep[i] = not cut
        C = mpmath.matrix(6, 6)
        for i in range(6):
            for j in range(6):
                C[i, j] = mpmath.fsum(V[i][k] * V[j][k] / w[k] for k in range(n) if keep[k])
        out = dict(cov=np.array([[float(C[i, j]) for j in range(6)] for i in range(6)]), keep=np.array(keep),
                   ratio=np.array([float(x) for x in ratio]), w=np.array([float(x) for x in w]))
        for name, o, scale in (("pos", 0, 1.0), ("ori", 3, 180.0 / math.pi)):
            B = np.array([[C[o + i, o + j] for j in range(3)] for i in range(3)], dtype=object)
            e, E = _mp_eigsy(B, dps)
            e = [max(x, mpmath.mpf(0)) for x in e]       # the block is positive semi-definite: its zero stays zero
            err = mpmath.sqrt(e[2])
            key = "pos_err" if name == "pos" else "ori_err_deg"
            out[key] = float(err * scale)
            out[name + "_dir"] = np.array([float(E[r][2]) for r in range(3)])
            out[name + "_inv_cond"] = float(mpmath.sqrt(e[0]) / err) if err > 0 else float("nan")
            out[name + "_gap"] = float((e[2] - e[1]) / e[2]) if e[2] > 0 else 0.0
            out[name + "_eig"] = np.array([float(x) for x in e])
    return out

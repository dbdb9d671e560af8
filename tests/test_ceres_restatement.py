"""A second, independent restatement of the Ceres solve the registration runs per ICP iteration (LidarSlam.cpp:213-240), in numpy,
cross-checked against oracle/so_oracle.cpp on random problems.

Ceres is not installable here, so the oracle's trust-region loop is a restatement of Ceres 2.0.0's published algorithm
(trust_region_minimizer.cc, levenberg_marquardt_strategy.cc, trust_region_step_evaluator.cc, corrector.cc, loss_function.cc) and so
is this file -- written separately, with numpy's LAPACK least squares instead of the oracle's hand-written Householder QR, its own
quaternion algebra and its own loop structure.  Two restatements that agree on the CONTROL FLOW (LM iterations, successful steps,
termination reason: what drives the outer ICP loop through `summary.num_successful_steps == 1`, LidarSlam.cpp:141) and on the
minimiser to 1e-9 on a hundred random problems shrink the room for a transcription slip in either; they do not replace a golden
vector from Ceres itself, which the reference does not ship ("parity unpinned" for this part, DESIGN.md section 3).
"""
import numpy as np

FUNCTION_TOL, GRADIENT_TOL, PARAMETER_TOL = 1e-6, 1e-10, 1e-8
MIN_REL_DECREASE, MIN_LM_DIAG, MAX_LM_DIAG = 1e-3, 1e-6, 1e32
MAX_RADIUS, MIN_RADIUS = 1e16, 1e-32


def _qmul(a, b):              # xyzw, Hamilton
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def _rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _plus(x, d):              # PoseLocalParameterization::Plus (pose_local_parameterization.cpp:7-22)
    q = _qmul(x[3:], np.array([d[3] / 2, d[4] / 2, d[5] / 2, 1.0]))
    return np.concatenate([x[:3] + d[:3], q / np.linalg.norm(q)])


def _plus_blocks(x, d):       # Plus of each pose7 block of x by its 6 tangent values in d
    return np.concatenate([_plus(x[7 * k:7 * k + 7], d[6 * k:6 * k + 6]) for k in range(len(x) // 7)])


class Problem:
    """n point-to-plane blocks {p, n, d, w} under ScaledLoss(TukeyLoss(a), w) (LidarSlam.cpp:268-274), and optionally the 6 rows of
    SE3AbsolutatePoseFactor (factor/SE3AbsolutatePoseFactor.cpp: [p - p_m ; 2 vec(q_m^* q)] times a diagonal sqrt-information, no
    loss), prior = (measurement pose7, sqrt_info[6]) as prior_sqrt_info gives it."""

    def __init__(self, P, N, D, W, a2, prior=None):
        self.P, self.N, self.D, self.W, self.a2 = P, N, D, W, a2
        self.prior = prior

    def _residuals(self, x):
        R = _rot(x[3:])
        return (self.N * (self.P @ R.T + x[:3])).sum(1) + self.D, R

    def _rho(self, s):
        inside = s <= self.a2
        v = np.where(inside, 1.0 - s / self.a2, 0.0)
        rho0 = np.where(inside, self.a2 / 6.0 * (1.0 - v ** 3), self.a2 / 6.0) * self.W
        rho1 = np.where(inside, 0.5 * v * v, 0.0) * self.W
        return rho0, rho1

    def _prior_rows(self, x):
        """residual [6] and local Jacobian [6, 6] of the prior rows: d(2 vec(e))/d(dtheta) = w I + [v]x of e = q_m^* q
        (Utility::Qleft's bottom-right block)."""
        meas, si = self.prior
        qm = np.array([-meas[3], -meas[4], -meas[5], meas[6]])
        e = _qmul(qm, x[3:])
        r = np.concatenate([x[:3] - meas[:3], 2.0 * e[:3]])
        ex, ey, ez, ew = e
        J = np.zeros((6, 6))
        J[:3, :3] = np.eye(3)
        J[3:, 3:] = [[ew, -ez, ey], [ez, ew, -ex], [-ey, ex, ew]]
        return r * si, J * si[:, None]

    def cost(self, x):
        r, _ = self._residuals(x)
        c = 0.5 * self._rho(r * r)[0].sum()
        if self.prior is not None:
            c += 0.5 * (self._prior_rows(x)[0] ** 2).sum()
        return c

    def linearise(self, x):
        """cost, corrected residuals, corrected local Jacobian [n, 6] (Corrector with rho'' <= 0: both scaled by sqrt(rho'))."""
        r, R = self._residuals(x)
        rho0, rho1 = self._rho(r * r)
        a = self.N @ R                                     # rows: R^T n
        J = np.concatenate([self.N, np.cross(self.P, a)], 1)      # [n^T, -n^T R [p]x] = [n, p x (R^T n)]
        sc = np.sqrt(rho1)
        cost, res, J = 0.5 * rho0.sum(), r * sc, J * sc[:, None]
        if self.prior is not None:
            rp, Jp = self._prior_rows(x)
            cost, res, J = cost + 0.5 * (rp * rp).sum(), np.concatenate([res, rp]), np.concatenate([J, Jp])
        return cost, res, J


def prior_sqrt_info(n_ok, prior_uncertainty, visual_confidence_factor):
    """addAbsolutePoseConstraints' information diagonal (LidarSlam.cpp:287-294) from the number of accepted correspondences, with the
    float inputs widened as the device widens them, and its square root by Eigen's unblocked LLT: the first non-positive pivot and
    everything after it stay as they are (the yaw weight is 0, so yaw is never square-rooted)."""
    vcf = float(np.float32(visual_confidence_factor))
    m1, m2 = max(50, int(n_ok * 0.1)), max(10, int(n_ok * 0.01))
    info = [(1 - float(np.float32(u))) * m1 * vcf for u in prior_uncertainty] + [m2 * vcf, m2 * vcf, max(5, int(n_ok * 0.001)) * 0]
    out, failed = np.zeros(6), False
    for k in range(6):
        failed = failed or info[k] <= 0.0
        out[k] = info[k] if failed else np.sqrt(info[k])
    return out


def _rel_margin(value, threshold):
    """How far a decision `value <= threshold` (or `>`) is from flipping, relative to the threshold."""
    return abs(value - threshold) / abs(threshold) if threshold != 0.0 else (np.inf if value != 0.0 else 0.0)


def solve_full(prob, x0, max_iterations=4, B=None):
    """Ceres' trust-region LM on prob from x0, a vector of k pose7 blocks (prob.linearise(x) gives the Jacobian over their 6k tangent
    columns, block by block; Plus, the gradient max-norm, x_norm and the step norm run over all blocks); B (6k x m, optional): the
    solve on B's columns, local parameterisation x [+] B y (Jacobian J B, Jacobi scaling and LM diagonal over the m columns, gradient
    max-norm through Plus(x, -B B^T g); x_norm and the parameter / function tolerances ambient).  -> dict: x, iterations, successful, unsuccessful, termination (codes as
    oracle/so_oracle.cpp), initial_cost, final_cost, and the trust-region state the solve ends in (radius, decrease_factor, gmax);
    steps: 'a' accepted / 'r' rejected / 'i' invalid per LM iteration; margin: the smallest relative distance of any decision the
    solve took from its threshold (gradient, radius, parameter and function tolerances, step quality, model cost change);
    radius_error: an estimate of the relative error of the final radius that rounding alone leaves; radius_error_normal: the same for a
    solver that forms the normal equations (the device's Cholesky), whose step is known only to cond^2 x machine epsilon.  A step is only known to about
    cond x machine epsilon (cond: of the damped least-squares system it is solved from), and so is the model cost change; the cost
    change is a difference of sums rounded at the scale of the initial cost.  Both carry into the step quality rd, and every accepted
    step multiplies the radius by 1 / max(1/3, 1 - (2 rd - 1)^3), whose relative sensitivity to rd is summed over the steps."""
    x = np.array(x0, float)
    B = np.eye(6 * (len(x) // 7)) if B is None else np.asarray(B, float)
    m = B.shape[1]
    cost, res, J = prob.linearise(x)
    initial_cost = cost
    Jr = J @ B
    scale = 1.0 / (1.0 + np.linalg.norm(Jr, axis=0))       # Jacobi scaling, fixed at iteration 0
    Js = Jr * scale

    def gmax_of(xx, JJ, rr):
        return np.abs(xx - _plus_blocks(xx, -(B @ (B.T @ (JJ.T @ rr))))).max()
    gmax = gmax_of(x, J, res)
    radius, decrease, reuse = 1e4, 2.0, False
    diag = None
    it = succ = unsucc = invalid = 0
    step_ok = False
    steps, margins = [], []
    eps, radius_error, radius_error_normal = np.finfo(float).eps, 0.0, 0.0

    def done(term):
        return dict(x=x, iterations=it, successful=succ, unsuccessful=unsucc, termination=term, initial_cost=initial_cost,
                    final_cost=cost, radius=radius, decrease_factor=decrease, gmax=gmax, steps="".join(steps),
                    margin=min(margins) if margins else np.inf, radius_error=radius_error, radius_error_normal=radius_error_normal)
    while True:
        if step_ok:
            succ += 1
        else:
            unsucc += 1
        if it >= max_iterations:
            return done(0)
        margins.append(_rel_margin(gmax, GRADIENT_TOL))
        if gmax <= GRADIENT_TOL:
            return done(1)
        margins.append(_rel_margin(radius, MIN_RADIUS))
        if radius <= MIN_RADIUS:
            return done(4)
        it += 1
        step_ok = False
        if not reuse:
            diag = np.clip((Js * Js).sum(0), MIN_LM_DIAG, MAX_LM_DIAG)
        reuse = True
        A = np.concatenate([Js, np.diag(np.sqrt(diag / radius))], 0)
        b = np.concatenate([res, np.zeros(m)])
        step = -np.linalg.lstsq(A, b, rcond=None)[0]
        cond = np.linalg.cond(A)
        mr = Js @ step
        model_change = -(mr * (res + mr / 2.0)).sum()
        if np.isfinite(step).all():
            margins.append(abs(model_change) / max(abs(mr * res).sum() + 0.5 * (mr * mr).sum(), np.finfo(float).tiny))
        if not (np.isfinite(step).all() and model_change > 0.0):
            steps.append("i")
            invalid += 1
            if invalid >= 5:
                return done(5)
            radius *= 0.5
            continue
        invalid = 0
        cand = _plus_blocks(x, B @ (step * scale))
        cand_cost = prob.cost(cand)
        sn, tol = np.linalg.norm(x - cand), PARAMETER_TOL * (np.linalg.norm(x) + PARAMETER_TOL)
        margins.append(_rel_margin(sn, tol))
        if sn <= tol:
            return done(2)
        change = cost - cand_cost
        margins.append(_rel_margin(abs(change), FUNCTION_TOL * cost))
        if abs(change) <= FUNCTION_TOL * cost:
            return done(3)
        rel = change / model_change
        margins.append(_rel_margin(rel, MIN_REL_DECREASE))
        if rel > MIN_REL_DECREASE:
            steps.append("a")
            t = 2.0 * rel - 1.0
            if 1.0 - t ** 3 > 1.0 / 3.0 and radius / (1.0 - t ** 3) < MAX_RADIUS:      # d ln(factor) / d ln(rd), 0 where capped
                radius_error += abs(6.0 * t * t * rel / (1.0 - t ** 3)) * (cond * eps + eps * initial_cost / abs(change))
                radius_error_normal += abs(6.0 * t * t * rel / (1.0 - t ** 3)) * (cond * cond * eps + eps * initial_cost / abs(change))
            x = cand
            cost, res, J = prob.linearise(x)
            Js = (J @ B) * scale
            gmax = gmax_of(x, J, res)
            step_ok = True
            radius = min(MAX_RADIUS, radius / max(1.0 / 3.0, 1.0 - (2.0 * rel - 1.0) ** 3))
            decrease, reuse = 2.0, False
        else:
            steps.append("r")
            radius /= decrease
            decrease *= 2.0
            reuse = True


def solve(prob, x0, max_iterations=4):
    """-> (x, iterations, successful_steps, unsuccessful_steps, termination)  termination codes as oracle/so_oracle.cpp."""
    r = solve_full(prob, x0, max_iterations)
    return r["x"], r["iterations"], r["successful"], r["unsuccessful"], r["termination"]


def _random_problem(rng, n):
    """Points on a few planes seen from a sensor, a ground-truth pose, and correspondences {p (sensor frame), n, d, w}."""
    truth = np.concatenate([rng.uniform(-5, 5, 3), (lambda q: q / np.linalg.norm(q))(np.concatenate([rng.normal(0, 0.15, 3), [1.0]]))])
    R = _rot(truth[3:])
    normals = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    k = rng.integers(0, 3, n)
    Nrm = normals[k] * rng.choice([-1.0, 1.0], n)[:, None]
    world = rng.uniform(-20, 20, (n, 3))
    offs = rng.uniform(2, 15, 3)[k]
    world -= ((world * Nrm).sum(1) - offs)[:, None] * Nrm                 # onto the plane n.x = offs
    D = -offs + rng.normal(0, 0.01, n)                                     # a little plane noise
    P = (world - truth[:3]) @ R                                            # sensor frame: R^T (x - t)
    W = rng.uniform(0.5, 1.0, n)
    return truth, P, Nrm, D, W


def test_numpy_and_cpp_restatements_of_the_ceres_solve_agree():
    from oracle import oracle as O
    O.build()
    rng = np.random.default_rng(42)
    plane_res = 0.2
    a = float(np.sqrt(np.float32(3 * np.float32(plane_res))))             # TukeyLoss(std::sqrt(3 * planeRes_)): float sqrt (LidarSlam.cpp:271)
    a2 = a * a
    seen_terms, seen_unsucc = set(), 0
    for trial in range(100):
        n = int(rng.integers(40, 400))
        truth, P, Nrm, D, W = _random_problem(rng, n)
        # every fourth start is far off, every fifth very far (Tukey saturation, rejected steps, radius shrinking)
        dt, dr = (2.5, 0.6) if trial % 5 == 4 else ((0.6, 0.12) if trial % 4 == 3 else (0.08, 0.015))
        start = _plus(truth, np.concatenate([rng.uniform(-1, 1, 3) * dt, rng.uniform(-1, 1, 3) * dr]))
        corr = np.zeros(n, O.CORR_DTYPE)
        corr["p"], corr["n"], corr["d"], corr["w"], corr["status"] = P, Nrm, D, W, 0
        for lm in (1, 2, 4, 12):
            xo, so = O.solve(corr, start, plane_res, lm)
            xn, it, succ, unsucc, term = solve(Problem(P, Nrm, D, W, a2), start, lm)
            assert (it, succ, unsucc, term) == (so["iterations"], so["successful"], so["unsuccessful"], so["termination"]), (trial, lm, (it, succ, unsucc, term), so)
            assert np.abs(xn - xo).max() <= 1e-9, (trial, lm, np.abs(xn - xo).max())
            seen_terms.add(term)
            seen_unsucc += unsucc > 1
    # the sample exercises the max-iterations exit and the function / parameter tolerance exits (rejected steps do not occur with this
    # bounded loss from these starts; tests/test_trust_region_cpu.py runs the rejection branch on problem families that reach it)
    assert {0, 2, 3} <= seen_terms, (seen_terms, seen_unsucc)

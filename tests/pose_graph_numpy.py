"""The pose-graph problem of so_pose_graph_solve (include/superodom_b200.h; DESIGN.md section 4, "Pose graph") restated in numpy.

PoseGraph is a `prob` for test_ceres_restatement.solve_full over the free nodes' pose7 blocks (the fixed node is held inside the
problem, so x_norm, the step norm and the gradient cover the free nodes only, as Ceres' reduced program does).  solve_sparse runs the
same trust-region rules with the exact step from a sparse factorisation of the normal equations (scipy.sparse), for graphs too large
for the dense restatement; solve_chain the same with a banded factorisation, for graphs whose edges all join k and k +- 1.  Edges are
a POSE_EDGE_DTYPE array (superodom_b200.api).

The row helpers below (_rots, _qmul_rows, plus_blocks) are the row forms of test_ceres_restatement's _rot, _qmul and _plus with the
same elementwise operations in the same order, so their results are bit-identical to the per-row calls
(tests/test_pose_graph_edges_cpu.py)."""
import numpy as np

import test_ceres_restatement as CR


def _skew(v):
    """[v]x of every row of v [m, 3] -> [m, 3, 3]"""
    z = np.zeros(len(v))
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1),
                     np.stack([-v[:, 1], v[:, 0], z], 1)], 1)


def _rots(q):
    """CR._rot of every row of q [m, 4] -> [m, 3, 3]"""
    x, y, z, w = np.asarray(q, float).T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], 1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], 1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1)], 1)


def _qmul_rows(a, b):
    """CR._qmul of every row pair of a, b [m, 4] -> [m, 4]"""
    ax, ay, az, aw = np.asarray(a, float).T
    bx, by, bz, bw = np.asarray(b, float).T
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], 1)


def plus_blocks(x, d):
    """CR._plus_blocks: Plus of each pose7 block of x by its 6 tangent values in d.  np.vecdot runs the dot product np.linalg.norm
    runs on one row, so the norms are the per-row ones bit for bit."""
    X, D = np.asarray(x, float).reshape(-1, 7), np.asarray(d, float).reshape(-1, 6)
    h = np.stack([D[:, 3] / 2, D[:, 4] / 2, D[:, 5] / 2, np.ones(len(D))], 1)
    q = _qmul_rows(X[:, 3:], h)
    return np.concatenate([X[:, :3] + D[:, :3], q / np.sqrt(np.vecdot(q, q))[:, None]], 1).ravel()


def _jrinv_coeff(th):
    th = np.asarray(th, float)
    t2 = th * th
    with np.errstate(divide="ignore", invalid="ignore"):
        closed = 1.0 / t2 - 1.0 / (2.0 * th * np.tan(0.5 * th))
    return np.where(th < 1e-2, 1.0 / 12.0 + t2 / 720.0 + t2 * t2 / 30240.0, closed)


def edge_terms(X, E):
    """Per edge at node poses X [n, 7]: raw residual [m, 6] (t_E, Log R_E), raw Jacobians Ji, Jj [m, 6, 6] in the tangent of Plus."""
    i, j = E["i"], E["j"]
    z = E["z"]
    zq = z[:, 3:] / np.linalg.norm(z[:, 3:], axis=1, keepdims=True)
    qi, qj = X[i, 3:], X[j, 3:]
    conj = np.array([-1.0, -1.0, -1.0, 1.0])
    qE = _qmul_rows(_qmul_rows(zq * conj, qi * conj), qj)
    Rz, Ri, Rj = _rots(zq), _rots(qi), _rots(qj)
    a = np.einsum("mki,mk->mi", Ri, X[j, :3] - X[i, :3])                  # R_i^T (t_j - t_i)
    tE = np.einsum("mki,mk->mi", Rz, a - z[:, :3])
    sg = np.where(qE[:, 3] < 0.0, -1.0, 1.0)
    vn = np.linalg.norm(qE[:, :3], axis=1)
    th = 2.0 * np.arctan2(vn, sg * qE[:, 3])
    f = np.where(vn > 0.0, sg * th / np.where(vn > 0.0, vn, 1.0), 0.0)
    phi = f[:, None] * qE[:, :3]
    P = _skew(phi)
    Jinv = np.eye(3)[None] + 0.5 * P + _jrinv_coeff(th)[:, None, None] * (P @ P)
    RzRi = np.transpose(Rz, (0, 2, 1)) @ np.transpose(Ri, (0, 2, 1))
    m = len(E)
    Ji, Jj = np.zeros((m, 6, 6)), np.zeros((m, 6, 6))
    Ji[:, :3, :3] = -RzRi
    Ji[:, :3, 3:] = np.transpose(Rz, (0, 2, 1)) @ _skew(a)
    Ji[:, 3:, 3:] = -Jinv @ np.transpose(Rj, (0, 2, 1)) @ Ri
    Jj[:, :3, :3] = RzRi
    Jj[:, 3:, 3:] = Jinv
    return np.concatenate([tE, phi], 1), Ji, Jj


def robust(E, r):
    """rho (s = |S r|^2) and rho' per edge: identity for c = 0, ceres::CauchyLoss(c) for c > 0."""
    S = E["sqrt_info"].reshape(-1, 6, 6)
    res = np.einsum("mij,mj->mi", S, r)
    s = (res * res).sum(1)
    c = E["cauchy"]
    b = np.where(c > 0, c * c, 1.0)
    rho = np.where(c > 0, b * np.log(1.0 + s * (1.0 / b)), s)
    rho1 = np.where(c > 0, np.maximum(np.finfo(float).tiny, 1.0 / (1.0 + s * (1.0 / b))), 1.0)
    return res, rho, rho1


class PoseGraph:
    """prob for solve_full: x is the free nodes' pose7 blocks in node order, node `fixed` held at init[fixed]."""

    def __init__(self, init, edges, fixed=0):
        self.init = np.array(init, float)
        self.init[:, 3:] /= np.linalg.norm(self.init[:, 3:], axis=1, keepdims=True)
        self.E, self.fixed = edges, int(fixed)
        self.n = len(self.init)
        self.free = np.array([k for k in range(self.n) if k != self.fixed])
        self.col = np.full(self.n, -1)
        self.col[self.free] = np.arange(len(self.free))

    def x0(self):
        return self.init[self.free].ravel()

    def nodes(self, x):
        X = self.init.copy()
        X[self.free] = np.asarray(x).reshape(-1, 7)
        return X

    def cost(self, x):
        r, _, _ = edge_terms(self.nodes(x), self.E)
        return 0.5 * robust(self.E, r)[1].sum()

    def weights(self, x):
        r, _, _ = edge_terms(self.nodes(x), self.E)
        return robust(self.E, r)[2]

    def blocks(self, x):
        """cost, corrected residuals [m, 6] and corrected S J blocks [m, 6, 6] of both nodes."""
        r, Ji, Jj = edge_terms(self.nodes(x), self.E)
        res, rho, rho1 = robust(self.E, r)
        S = self.E["sqrt_info"].reshape(-1, 6, 6)
        sc = np.sqrt(rho1)[:, None]
        return 0.5 * rho.sum(), res * sc, (S @ Ji) * sc[:, :, None], (S @ Jj) * sc[:, :, None]

    def linearise(self, x):
        cost, res, Ji, Jj = self.blocks(x)
        m, k = len(self.E), len(self.free)
        J = np.zeros((6 * m, 6 * k))
        for e in range(m):
            for node, B in ((self.E["i"][e], Ji[e]), (self.E["j"][e], Jj[e])):
                c = self.col[node]
                if c >= 0:
                    J[6 * e:6 * e + 6, 6 * c:6 * c + 6] = B
        return cost, res.ravel(), J

    def sparse_jacobian(self, x):
        import scipy.sparse as sp
        cost, res, Ji, Jj = self.blocks(x)
        rows, cols, vals = [], [], []
        rr, cc = np.meshgrid(np.arange(6), np.arange(6), indexing="ij")
        for node, B in ((self.E["i"], Ji), (self.E["j"], Jj)):
            keep = self.col[node] >= 0
            e = np.nonzero(keep)[0]
            rows.append((6 * e[:, None, None] + rr[None]).ravel())
            cols.append((6 * self.col[node][keep][:, None, None] + cc[None]).ravel())
            vals.append(B[keep].ravel())
        J = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                          shape=(6 * len(self.E), 6 * len(self.free)))
        return cost, res.ravel(), J


class _SparseStep:
    """The step of solve_sparse: the global Jacobian in scipy.sparse and a sparse direct solve (spsolve)."""

    def __init__(self, prob):
        self.prob = prob

    def linearise(self, x):
        cost, self.res, self.J = self.prob.sparse_jacobian(x)
        return cost, self.res

    def column_norms2(self):
        return np.asarray(self.J.multiply(self.J).sum(0)).ravel()

    def gradient(self):
        return self.J.T @ self.res

    def system(self, scale):
        """Hs = Js'Js and gs = Js'r of the scaled Jacobian Js = J diag(scale) -> the diagonal of Hs."""
        import scipy.sparse as sp
        self.Js = (self.J @ sp.diags(scale)).tocsc()
        self.Hs = (self.Js.T @ self.Js).tocsc()
        self.gs = self.Js.T @ self.res
        return self.Hs.diagonal()

    def solve(self, d):
        """y of (Hs + diag(d)) y = gs"""
        import scipy.sparse as sp
        import scipy.sparse.linalg as spl
        return spl.spsolve((self.Hs + sp.diags(d)).tocsc(), self.gs)

    def model(self, step):
        return self.Js @ step


class _ChainStep:
    """The step of solve_chain: per-edge blocks and a banded Cholesky solve (scipy.linalg.solveh_banded).  Every edge joins k and
    k +- 1, so the free nodes' columns couple only to the next free node's and Hs + D^2 has 11 sub-diagonals; no global Jacobian is
    formed, and a step costs O(n b^2)."""

    def __init__(self, prob):
        self.prob = prob
        i, j = prob.E["i"].astype(np.int64), prob.E["j"].astype(np.int64)
        assert (np.abs(i - j) == 1).all(), "solve_chain: an edge that does not join k and k +- 1"
        self.ci, self.cj = prob.col[i], prob.col[j]                     # -1: a constant node
        self.F = len(prob.free)
        both = (self.ci >= 0) & (self.cj >= 0)
        # edge-to-column sums as sparse products: P[c, e] = 1 where column block c is the edge's i (j) end; low[c], the block of
        # rows c + 1 and columns c, takes the edges from c to c + 1 (fwd) and from c + 1 to c (rev)
        self.Pi, self.Pj = self._scatter(self.ci, self.ci >= 0), self._scatter(self.cj, self.cj >= 0)
        self.Pf, self.Pr = self._scatter(self.ci, both & (self.cj == self.ci + 1)), self._scatter(self.cj, both & (self.ci == self.cj + 1))

    def _scatter(self, c, keep):
        import scipy.sparse as sp
        e = np.nonzero(keep)[0]
        return sp.csr_matrix((np.ones(len(e)), (c[e], e)), shape=(self.F, len(c)))

    def _sum(self, fi, fj, Pi=None, Pj=None):
        """per free column block: the sum of fi over the edges' i ends and of fj over their j ends -> [F, ...]"""
        Pi, Pj = (self.Pi, self.Pj) if Pi is None else (Pi, Pj)
        m = len(fi)
        return (Pi @ fi.reshape(m, -1) + Pj @ fj.reshape(m, -1)).reshape((self.F,) + fi.shape[1:])

    def linearise(self, x):
        cost, res, self.Ji, self.Jj = self.prob.blocks(x)
        self.r = res
        return cost, res.ravel()

    def column_norms2(self):
        return self._sum((self.Ji * self.Ji).sum(1), (self.Jj * self.Jj).sum(1)).ravel()

    def gradient(self):
        return self._sum(np.einsum("mki,mk->mi", self.Ji, self.r), np.einsum("mki,mk->mi", self.Jj, self.r)).ravel()

    def system(self, scale):
        s = np.vstack([scale.reshape(-1, 6), np.zeros((1, 6))])        # row -1: a constant node's columns are zero
        self.Si, self.Sj = self.Ji * s[self.ci][:, None, :], self.Jj * s[self.cj][:, None, :]
        tr = lambda A: np.transpose(A, (0, 2, 1))
        D = self._sum(tr(self.Si) @ self.Si, tr(self.Sj) @ self.Sj)
        self.gs = self._sum(np.einsum("mki,mk->mi", self.Si, self.r), np.einsum("mki,mk->mi", self.Sj, self.r)).ravel()
        low = self._sum(tr(self.Sj) @ self.Si, tr(self.Si) @ self.Sj, self.Pf, self.Pr)
        ab = np.zeros((12, 6 * self.F))                                 # lower band: ab[row - col, col]
        for r in range(6):
            for c in range(6):
                if r >= c:
                    ab[r - c, c::6] = D[:, r, c]
                ab[6 + r - c, c:6 * (self.F - 1):6] = low[:-1, r, c]
        self.ab = ab
        return np.diagonal(D, axis1=1, axis2=2).ravel().copy()

    def solve(self, d):
        from scipy.linalg import solveh_banded
        ab = self.ab.copy()
        ab[0] += d
        return solveh_banded(ab, self.gs, lower=True)

    def model(self, step):
        st = np.vstack([step.reshape(-1, 6), np.zeros((1, 6))])
        return (np.einsum("mij,mj->mi", self.Si, st[self.ci]) + np.einsum("mij,mj->mi", self.Sj, st[self.cj])).ravel()


def _solve_exact(lin, x0, max_iterations):
    """solve_full's rules with the exact step of the linear algebra lin (_SparseStep or _ChainStep)."""
    x = np.array(x0, float)
    cost, res = lin.linearise(x)
    initial_cost = cost
    scale = 1.0 / (1.0 + np.sqrt(lin.column_norms2()))
    gmax = np.abs(x - plus_blocks(x, -lin.gradient())).max()
    radius, decrease, reuse, diag = 1e4, 2.0, False, None
    it = succ = unsucc = invalid = 0
    step_ok, steps, margins = False, [], []

    def done(term):
        return dict(x=x, iterations=it, successful=succ, unsuccessful=unsucc, termination=term, initial_cost=initial_cost,
                    final_cost=cost, radius=radius, decrease_factor=decrease, gmax=gmax, steps="".join(steps),
                    margin=min(margins) if margins else np.inf, radius_error=0.0)
    while True:
        if step_ok:
            succ += 1
        else:
            unsucc += 1
        if it >= max_iterations:
            return done(0)
        margins.append(CR._rel_margin(gmax, CR.GRADIENT_TOL))
        if gmax <= CR.GRADIENT_TOL:
            return done(1)
        margins.append(CR._rel_margin(radius, CR.MIN_RADIUS))
        if radius <= CR.MIN_RADIUS:
            return done(4)
        it += 1
        step_ok = False
        hs_diag = lin.system(scale)
        if not reuse:
            diag = np.clip(hs_diag, CR.MIN_LM_DIAG, CR.MAX_LM_DIAG)
        reuse = True
        step = -lin.solve(diag / radius)
        mr = lin.model(step)
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
        cand = plus_blocks(x, step * scale)
        cand_cost = lin.prob.cost(cand)
        sn, tol = np.linalg.norm(x - cand), CR.PARAMETER_TOL * (np.linalg.norm(x) + CR.PARAMETER_TOL)
        margins.append(CR._rel_margin(sn, tol))
        if sn <= tol:
            return done(2)
        change = cost - cand_cost
        margins.append(CR._rel_margin(abs(change), CR.FUNCTION_TOL * cost))
        if abs(change) <= CR.FUNCTION_TOL * cost:
            return done(3)
        rel = change / model_change
        margins.append(CR._rel_margin(rel, CR.MIN_REL_DECREASE))
        if rel > CR.MIN_REL_DECREASE:
            steps.append("a")
            x = cand
            cost, res = lin.linearise(x)
            gmax = np.abs(x - plus_blocks(x, -lin.gradient())).max()
            step_ok = True
            radius = min(CR.MAX_RADIUS, radius / max(1.0 / 3.0, 1.0 - (2.0 * rel - 1.0) ** 3))
            decrease, reuse = 2.0, False
        else:
            steps.append("r")
            radius /= decrease
            decrease *= 2.0
            reuse = True


def solve_sparse(prob, x0, max_iterations=50):
    """solve_full's rules with the exact step from a sparse direct solve (scipy.sparse.linalg.spsolve) of
    (Hs + D^2) y = gs.  -> dict as solve_full (margin over the same decisions; radius_error not estimated: 0)."""
    return _solve_exact(_SparseStep(prob), x0, max_iterations)


def solve_chain(prob, x0, max_iterations=50):
    """solve_sparse for a graph whose edges all join k and k +- 1 (parallel and reversed edges, constant nodes anywhere), with the
    exact step from the banded Cholesky factorisation of Hs + D^2 (11 sub-diagonals), assembled from the per-edge blocks."""
    return _solve_exact(_ChainStep(prob), x0, max_iterations)


# ------------------------------------------------------------------------------------------------------------------ problem families
def _unit(q):
    return q / np.linalg.norm(q)


def rand_pose(rng, t_scale=1.0, r_scale=0.3):
    return np.r_[rng.normal(0, t_scale, 3), _unit(np.r_[rng.normal(0, r_scale, 3), 1.0])]


def compose(a, b):
    return np.r_[a[:3] + CR._rot(a[3:]) @ b[:3], CR._qmul(a[3:], b[3:])]


def inverse(a):
    qc = np.r_[-a[3:6], a[6]]
    return np.r_[-(CR._rot(qc) @ a[:3]), qc]


def edge(i, j, z, sqrt_info, cauchy=0.0):
    s = np.asarray(sqrt_info, float)
    return (int(i), int(j), np.asarray(z, float), np.diag(s) if s.shape == (6,) else s.reshape(6, 6), float(cauchy))


def to_array(edges):
    from superodom_b200.api import POSE_EDGE_DTYPE
    out = np.zeros(len(edges), POSE_EDGE_DTYPE)
    for k, (i, j, z, S, c) in enumerate(edges):
        out[k]["i"], out[k]["j"], out[k]["z"], out[k]["sqrt_info"], out[k]["cauchy"] = i, j, z, S.ravel(), c
    return out


def rotation(axis, angle):
    """pose7 of a rotation by angle about axis"""
    a = _unit(np.asarray(axis, float))
    return np.r_[0.0, 0.0, 0.0, a * np.sin(angle / 2), np.cos(angle / 2)]


def reversed_edge(e):
    """(i, j, Z, S, c) stored as (j, i, Z^-1, S'): E' = Z X_j^-1 X_i = Z E^-1 Z^-1, whose residual is about -blkdiag(R_Z, R_Z) r, so
    S' = S blkdiag(R_Z^T, R_Z^T) weighs it as S weighs r to first order (the references take any (i, j), exact or not)."""
    i, j, z, S, c = e
    Rt = CR._rot(z[3:]).T
    B = np.zeros((6, 6))
    B[:3, :3], B[3:, 3:] = Rt, Rt
    return (j, i, inverse(z), S @ B, c)


def drifted(rng, n, loops=0, step=1.0, noise=(0.02, 0.005), drift=(0.01, 0.003), sqrt_info=None, full_info=False, cauchy=0.0,
            false_loops=0, dup=False, rank_def=False, reverse=0.0, both_ways=False, angles=None, max_span=None):
    """A random walk of n poses (truth), odometry edges measured with noise, `loops` revisit edges between random non-adjacent pairs
    measured from the truth, `false_loops` wrong Z between unrelated nodes, and the start: the odometry chained with drift.
    dup: a second forward odometry edge at every third k; both_ways: a reversed one (reversed_edge of a second measurement) at every
    third k; reverse: each edge stored reversed with this probability; angles: odometry edge k's measurement rotated by angles[k %
    len(angles)] about a random axis, and the start chained from the true increments, so the start's residual rotations have these
    angles (plus the drift); max_span: loop edges join nodes at most this far apart.  -> (init [n, 7], edges list, truth)."""
    truth = [np.r_[0, 0, 0, 0, 0, 0, 1.0]]
    for _ in range(n - 1):
        inc = np.r_[rng.normal(0, step, 3) * [1, 1, 0.2], _unit(np.r_[rng.normal(0, 0.15, 3), 1.0])]
        truth.append(compose(truth[-1], inc))
    truth = np.array(truth)
    si = np.r_[np.full(3, 1 / noise[0]), np.full(3, 1 / noise[1])] if sqrt_info is None else np.asarray(sqrt_info, float)

    def info():
        if full_info:
            A = rng.normal(0, 0.2, (6, 6)) + np.diag(si)
            if rank_def:
                A[5] = 0.0
            return A
        return si

    def meas(i, j, sd):
        z = compose(inverse(truth[i]), truth[j])
        return compose(z, np.r_[rng.normal(0, sd[0], 3), _unit(np.r_[rng.normal(0, sd[1] / 2, 3), 1.0])])
    edges = []
    odo = []
    for k in range(n - 1):
        z = meas(k, k + 1, noise)
        if angles is not None:
            z = compose(z, rotation(rng.normal(size=3), angles[k % len(angles)]))
            odo.append(compose(inverse(truth[k]), truth[k + 1]))
        else:
            odo.append(z)
        edges.append(edge(k, k + 1, z, info()))
        if dup and k % 3 == 0:
            edges.append(edge(k, k + 1, meas(k, k + 1, noise), info()))
        if both_ways and k % 3 == 1:
            edges.append(reversed_edge(edge(k, k + 1, meas(k, k + 1, noise), info())))
    for _ in range(loops):
        if max_span is None:
            i, j = sorted(rng.choice(n, 2, replace=False))
        else:
            i = int(rng.integers(0, n - 2))
            j = min(n - 1, i + int(rng.integers(2, max_span + 1)))
        if j - i < 2:
            j = min(n - 1, i + 2)
            if j - i < 2:
                continue
        edges.append(edge(i, j, meas(i, j, noise), info(), cauchy))
    for _ in range(false_loops):
        i, j = sorted(rng.choice(n, 2, replace=False))
        edges.append(edge(i, j, rand_pose(rng, 3.0, 0.3), info(), cauchy))
    if reverse > 0.0:
        flip = rng.random(len(edges)) < reverse
        edges = [reversed_edge(e) if f else e for e, f in zip(edges, flip)]
    init = [truth[0]]
    for k in range(n - 1):
        d = np.r_[rng.normal(0, drift[0], 3), _unit(np.r_[rng.normal(0, drift[1] / 2, 3), 1.0])]
        init.append(compose(init[-1], compose(odo[k], d)))
    return np.array(init), edges, truth

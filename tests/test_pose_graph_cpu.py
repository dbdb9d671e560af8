"""The pose-graph problem without a GPU: the restatement's analytic Jacobians against central differences, its objective against the
scipy helper of tests/test_keyframes.py, so_pose_graph_check on every input it rejects, and the ctypes structs against the header."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import pose_graph_numpy as PG
import test_ceres_restatement as CR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _plus_node(X, k, d):
    Y = X.copy()
    Y[k] = CR._plus(X[k], d)
    return Y


@pytest.mark.parametrize("angle", [0.0, 1e-7, 1e-3, 0.5, 2.0, np.pi - 1e-3, np.pi - 1e-6])
@pytest.mark.parametrize("cauchy", [0.0, 0.5])
def test_jacobians_against_central_differences(angle, cauchy):
    """The corrected S J blocks of both nodes against central differences of the corrected residual through Plus, at relative rotation
    angles from 0 to just below pi (the series branch of J_r^-1 below 1e-2, the closed form above)."""
    rng = np.random.default_rng(int(angle * 1e3) + int(cauchy * 10))
    X = np.array([PG.rand_pose(rng), PG.rand_pose(rng)])
    ax = PG._unit(rng.normal(size=3))
    dq = np.r_[ax * np.sin(angle / 2), np.cos(angle / 2)]
    rel = PG.compose(PG.inverse(X[0]), X[1])
    z = PG.compose(rel, np.r_[rng.normal(0, 0.3, 3), CR._qmul(np.r_[-dq[:3], dq[3]], [0, 0, 0, 1.0])])   # E's rotation: dq
    S = rng.normal(0, 0.3, (6, 6)) + np.diag(rng.uniform(1, 3, 6))
    E = PG.to_array([PG.edge(0, 1, z, S, cauchy)])
    prob = PG.PoseGraph(X, E, fixed=0)
    _, res, Ji, Jj = prob.blocks(X[1:].ravel())
    r0, _, _ = PG.edge_terms(X, E)
    th = np.linalg.norm(r0[0, 3:])
    assert abs(th - angle) < 1e-6 + 1e-9 * angle, (th, angle)

    def corrected(Y):
        r, _, _ = PG.edge_terms(Y, E)
        rr, _, rho1 = PG.robust(E, r)
        return (rr * np.sqrt(rho1)[:, None])[0]
    # the Corrector scales J by sqrt(rho') without the rho'' term: differentiate S r, then scale by sqrt(rho')
    _, _, rho1 = PG.robust(E, r0)
    for node, B in ((0, Ji[0]), (1, Jj[0])):
        num = np.zeros((6, 6))
        h = 1e-6
        for c in range(6):
            d = np.zeros(6)
            d[c] = h
            sp = PG.robust(E, PG.edge_terms(_plus_node(X, node, d), E)[0])[0][0]
            sm = PG.robust(E, PG.edge_terms(_plus_node(X, node, -d), E)[0])[0][0]
            num[:, c] = (sp - sm) / (2 * h) * np.sqrt(rho1[0])
        err = np.abs(num - B).max() / max(np.abs(B).max(), 1.0)
        assert err < 1e-6, (node, angle, err)
    assert np.allclose(res[0], corrected(X))


def _keyframes_helper():
    import test_keyframes as TK
    return TK


def test_restatement_states_the_objective_of_the_scipy_helper():
    """Diagonal S, no loss: at the scipy helper's solution the restatement's cost equals the helper's 1/2 |r|^2 to 1e-12 relative and
    its gradient is at rounding level.  The helper stops at ftol = xtol = 1e-12 and Ceres' rules at a function
    tolerance of 1e-6, so the two solutions are compared to the tolerance measured on these graphs (largest difference 2e-5 m /
    2e-6 in a quaternion component; bound 1e-3)."""
    TK = _keyframes_helper()
    rng = np.random.default_rng(3)
    for n, loops in ((6, 1), (12, 3), (25, 6)):
        init, edges, truth = PG.drifted(rng, n, loops=loops, drift=(0.05, 0.01))
        helper_edges = [(i, j, z, np.diag(S)) for i, j, z, S, c in edges]
        sol = TK._pose_graph(init, helper_edges)
        E = PG.to_array(edges)
        prob = PG.PoseGraph(sol, E)
        r = []
        for i, j, z, w in helper_edges:
            Ez = TK._compose(TK._inverse(z), TK._compose(TK._inverse(sol[i]), sol[j]))
            from scipy.spatial.transform import Rotation
            r.append(w * np.r_[Ez[:3], Rotation.from_quat(Ez[3:]).as_rotvec()])
        half = 0.5 * (np.concatenate(r) ** 2).sum()
        cost, res, J = prob.linearise(prob.x0())
        assert abs(cost - half) <= 1e-12 * half, (cost, half)
        # the gradient at rounding level, measured where it matters: the cost decrease a Newton step from the helper's solution
        # would give (1/2 g'H^-1 g), relative to the cost, is rounding of the cost (measured 3e-16 to 2e-15)
        g = J.T @ res
        decrement = 0.5 * g @ np.linalg.solve(J.T @ J, g)
        assert decrement <= 1e-14 * cost, (decrement, cost)
        out = CR.solve_full(PG.PoseGraph(init, E), PG.PoseGraph(init, E).x0(), 50)
        X = PG.PoseGraph(init, E).nodes(out["x"])
        d = np.abs(X - sol)
        d[:, 3:] = np.minimum(d[:, 3:], np.abs(X[:, 3:] + sol[:, 3:]))
        print(f"n={n}: restatement vs scipy helper: max pose difference {d.max():.2e}, termination {out['termination']}")
        assert d.max() < 1e-3


def test_sparse_step_equals_the_dense_restatement():
    """solve_sparse (the exact step by a sparse direct solve) takes solve_full's decisions on graphs both can run."""
    rng = np.random.default_rng(11)
    for n, loops, c in ((5, 1, 0.0), (20, 4, 0.0), (30, 6, 1.0)):
        init, edges, _ = PG.drifted(rng, n, loops=loops, cauchy=c, drift=(0.1, 0.02))
        prob = PG.PoseGraph(init, PG.to_array(edges))
        a = CR.solve_full(prob, prob.x0(), 50)
        b = PG.solve_sparse(prob, prob.x0(), 50)
        assert (a["iterations"], a["successful"], a["unsuccessful"], a["termination"]) == \
            (b["iterations"], b["successful"], b["unsuccessful"], b["termination"])
        assert np.abs(a["x"] - b["x"]).max() < 1e-9


# ------------------------------------------------------------------------------------------------------------------ argument checks
def _code(fn):
    from superodom_b200 import api
    with pytest.raises(api.SuperOdomError) as e:
        fn()
    return e.value.code, str(e.value)


def _good(n=4):
    return [PG.edge(k, k + 1, [0.1, 0, 0, 0, 0, 0, 1.0], np.ones(6)) for k in range(n - 1)]


@pytest.mark.parametrize("case, needle", [
    ("n1", "two nodes"), ("id", "out of range"), ("neg", "out of range"), ("self", "i == j"), ("zq", "quaternion"),
    ("nanz", "not finite"), ("nans", "sqrt_info"), ("negc", "cauchy"), ("nanc", "cauchy"), ("fixed", "fixed node"),
    ("fixedneg", "fixed node"), ("iters", "max_iterations"), ("disc", "not connected"),
])
def test_check_rejects(case, needle):
    from superodom_b200 import api
    api.load_library()
    n, e, fixed, iters = 4, PG.to_array(_good()), 0, 50
    if case == "n1":
        n, e = 1, e[:0]
    elif case == "id":
        e[1]["j"] = 4
    elif case == "neg":
        e[0]["i"] = -1
    elif case == "self":
        e[2]["j"] = e[2]["i"]
    elif case == "zq":
        e[0]["z"][3:] = 0.0
    elif case == "nanz":
        e[0]["z"][1] = np.nan
    elif case == "nans":
        e[1]["sqrt_info"][7] = np.inf
    elif case == "negc":
        e[1]["cauchy"] = -1.0
    elif case == "nanc":
        e[1]["cauchy"] = np.nan
    elif case == "fixed":
        fixed = 4
    elif case == "fixedneg":
        fixed = -1
    elif case == "iters":
        iters = -1
    elif case == "disc":
        e = e[[0, 2]]                                                  # nodes {0, 1} and {2, 3}
    code, msg = _code(lambda: api.pose_graph_check(n, e, fixed, iters))
    assert code == -1 and needle in msg, msg


def test_check_accepts_edge_cases():
    """Duplicate edges, an interior fixed node, reversed edges, a non-unit z quaternion, rank-deficient S and max_iterations 0."""
    from superodom_b200 import api
    e = _good(5) + [PG.edge(1, 2, [0.1, 0, 0, 0, 0, 0, 3.0], np.zeros(6)), PG.edge(4, 0, [0, 0, 0, 0, 0, 0, 1.0], np.ones(6), 2.0)]
    api.pose_graph_check(5, PG.to_array(e), fixed=2, max_iterations=0)
    api.pose_graph_check(2, PG.to_array(_good(2)))


def test_struct_layouts_match_header(tmp_path):
    from superodom_b200 import api
    f = tmp_path / "s.c"
    f.write_text('#include <stdio.h>\n#include "superodom_b200.h"\nint main(void){printf("%zu %zu %zu\\n", sizeof(so_pose_edge), '
                 'sizeof(so_pose_graph_opts), sizeof(so_pose_graph_result));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(f), "-o", str(exe)])
    a, b, c = (int(v) for v in subprocess.check_output([str(exe)]).split())
    assert (a, b, c) == (api.POSE_EDGE_DTYPE.itemsize, C.sizeof(api.PoseGraphOpts), C.sizeof(api.PoseGraphResult))

"""The pose-graph restatement's large-graph helpers and the loss-scale rule, without a GPU: the row forms of _rot, _qmul and Plus
bit-identical to test_ceres_restatement's per-row ones, solve_chain against solve_sparse, the reversed and both-ways edges of
pose_graph_numpy.drifted, and so_pose_graph_check / so_pose_graph_check_constant on Cauchy scales whose square is not a finite
normal double."""
import numpy as np
import pytest

import pose_graph_numpy as PG
import sessions_numpy as SN
import test_ceres_restatement as CR

SO_ERR_ARG = -1
TINY = np.finfo(float).tiny                                             # DBL_MIN
C_LO = 1.4916681462400413e-154                                          # the smallest c with c * c >= DBL_MIN
C_HI = 1.3407807929942596e+154                                          # the largest c with c * c finite


def _rows(rng, m):
    """m random quaternion rows: unit, non-unit, w < 0, near the identity and near a half turn"""
    q = rng.normal(size=(m, 4)) * rng.uniform(1e-3, 1e3, (m, 1))
    q[: m // 4, 3] = -np.abs(q[: m // 4, 3])
    q[m // 4: m // 2] = np.c_[rng.normal(0, 1e-9, (m // 4, 3)), np.ones(m // 4)]
    q[m // 2: 3 * m // 4] = np.c_[rng.normal(size=(m // 4, 3)), rng.normal(0, 1e-9, m // 4)]
    return q


def test_row_helpers_are_bit_identical_to_the_per_row_forms():
    rng = np.random.default_rng(1)
    m = 4000
    a, b = _rows(rng, m), _rows(rng, m)[::-1].copy()
    assert PG._rots(a).tobytes() == np.stack([CR._rot(r) for r in a]).tobytes()
    assert PG._qmul_rows(a, b).tobytes() == np.stack([CR._qmul(x, y) for x, y in zip(a, b)]).tobytes()
    x = np.c_[rng.normal(0, 100, (m, 3)), a / np.linalg.norm(a, axis=1, keepdims=True)]
    x[: m // 8, 3:] = -x[: m // 8, 3:]                                  # the same rotations with w < 0
    d = np.r_[rng.normal(0, 1.0, (m // 2, 6)), rng.normal(0, 1e-8, (m - m // 2, 6))]
    d[: m // 16, 3:] = rng.normal(0, 5.0, (m // 16, 3))                 # past a half turn
    assert (x[:, 6] < 0).sum() > m // 8
    assert PG.plus_blocks(x.ravel(), d.ravel()).tobytes() == CR._plus_blocks(x.ravel(), d.ravel()).tobytes()


@pytest.mark.parametrize("n, mask", [(50, None), (64, "first"), (97, "ends"), (150, "middle"), (200, "alternate")])
def test_chain_step_equals_the_sparse_step(n, mask):
    """solve_chain (banded Cholesky of the per-edge blocks) takes solve_sparse's decisions on chains with reversed, parallel and
    both-ways edges, Cauchy on some edges and constant nodes anywhere; poses, costs and the radius within rounding."""
    rng = np.random.default_rng(n)
    init, edges, _ = PG.drifted(rng, n, dup=True, both_ways=True, reverse=0.5, drift=(0.1, 0.03))
    edges = [(i, j, z, S, 1.0 if k % 5 == 0 else 0.0) for k, (i, j, z, S, c) in enumerate(edges)]
    E = PG.to_array(edges)
    assert (E["i"] > E["j"]).sum() > n // 4 and (E["i"] < E["j"]).sum() > n // 4
    if mask is None:
        prob = PG.PoseGraph(init, E, fixed=n // 3)
    else:
        c = np.zeros(n, bool)
        c[{"first": [0], "ends": [0, 1, n - 2, n - 1], "middle": list(range(n // 2, n // 2 + 5))}.get(mask, slice(0, n, 2))] = True
        prob = SN.ConstantPoseGraph(init, E, c)
    a = PG.solve_sparse(prob, prob.x0(), 50)
    b = PG.solve_chain(prob, prob.x0(), 50)
    assert a["steps"] == b["steps"] and (a["iterations"], a["successful"], a["unsuccessful"], a["termination"]) == \
        (b["iterations"], b["successful"], b["unsuccessful"], b["termination"])
    d = {k: abs(a[k] - b[k]) / abs(a[k]) for k in ("initial_cost", "final_cost", "gmax", "radius")}
    print(f"n={n} {mask}: {a['steps']}, poses {np.abs(a['x'] - b['x']).max():.2e}, " + ", ".join(f"{k} {v:.2e}" for k, v in d.items()))
    # three times the largest measured over these chains: poses 3.9e-14, costs 2.0e-15 relative, radius 5.4e-13 (the radius update
    # cubes the step quality); gmax, the gradient at the last iterate, is a small difference of large terms (1.0e-10 relative)
    assert np.abs(a["x"] - b["x"]).max() <= 1.2e-13
    assert max(d["initial_cost"], d["final_cost"]) <= 6e-15 and d["radius"] <= 1.6e-12 and d["gmax"] <= 3e-10


def test_chain_step_rejects_a_loop_edge():
    rng = np.random.default_rng(3)
    init, edges, _ = PG.drifted(rng, 10, loops=1)
    prob = PG.PoseGraph(init, PG.to_array(edges))
    with pytest.raises(AssertionError, match="k \\+- 1"):
        PG.solve_chain(prob, prob.x0(), 5)


def test_reversed_edges_state_the_same_measurement():
    """A reversed edge (j, i, Z^-1, S') of an edge (i, j, Z, S): at any poses its residual rotation has the same angle, and at the
    truth of exact measurements both residuals vanish."""
    rng = np.random.default_rng(4)
    init, edges, truth = PG.drifted(rng, 6, loops=2, drift=(0.05, 0.01), full_info=True)
    fwd = PG.to_array(edges)
    rev = PG.to_array([PG.reversed_edge(e) for e in edges])
    assert (rev["i"] == fwd["j"]).all() and (rev["j"] == fwd["i"]).all()
    r0, _, _ = PG.edge_terms(init, fwd)
    r1, _, _ = PG.edge_terms(init, rev)
    assert np.allclose(np.linalg.norm(r0[:, 3:], axis=1), np.linalg.norm(r1[:, 3:], axis=1), rtol=1e-12, atol=1e-15)
    _, edges, truth = PG.drifted(rng, 6, loops=2, noise=(0.0, 0.0), sqrt_info=np.ones(6))
    r1, _, _ = PG.edge_terms(truth, PG.to_array([PG.reversed_edge(e) for e in edges]))
    assert np.abs(r1).max() < 1e-12
    init2, edges2, _ = PG.drifted(np.random.default_rng(5), 30, reverse=1.0)
    assert all(i == j + 1 for i, j, *_ in edges2)


def test_angles_set_the_start_residual_rotation():
    angles = [0.0, 1e-8, 0.5, 2.0, np.pi - 1e-3]
    init, edges, _ = PG.drifted(np.random.default_rng(6), len(angles) + 1, angles=angles, noise=(0.0, 0.0),
                                drift=(0.0, 0.0), sqrt_info=np.ones(6))
    r, _, _ = PG.edge_terms(init, PG.to_array(edges))
    assert np.allclose(np.linalg.norm(r[:, 3:], axis=1), angles, rtol=1e-9, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------------ the loss scale
def _check(api, n, e, form):
    if form == "fixed":
        api.pose_graph_check(n, e, 0)
    else:
        c = np.zeros(n, np.uint8)
        c[0] = 1
        api.pose_graph_check_constant(n, e, c)


def _graph(c):
    e = PG.to_array([PG.edge(k, k + 1, [0.1, 0, 0, 0, 0, 0, 1.0], np.ones(6)) for k in range(3)])
    e[1]["cauchy"] = c
    return e


def test_loss_scale_boundaries():
    assert C_LO * C_LO >= TINY and np.nextafter(C_LO, 0) ** 2 < TINY
    with np.errstate(over="ignore"):
        assert np.isfinite(C_HI * C_HI) and not np.isfinite(np.nextafter(C_HI, np.inf) ** 2)


@pytest.mark.parametrize("form", ["fixed", "constant"])
@pytest.mark.parametrize("c", [C_LO, np.nextafter(C_LO, 1.0), 1e-100, 1.0, 1e100, np.nextafter(C_HI, 0.0), C_HI, 0.0])
def test_check_accepts_loss_scales_the_loss_can_evaluate(form, c):
    from superodom_b200 import api
    _check(api, 4, _graph(c), form)


@pytest.mark.parametrize("form", ["fixed", "constant"])
@pytest.mark.parametrize("c, why", [(1e200, "overflows"), (np.nextafter(C_HI, np.inf), "overflows"), (1e-200, "below DBL_MIN"),
                                    (1e-160, "below DBL_MIN"), (np.nextafter(C_LO, 0.0), "below DBL_MIN"), (5e-324, "below DBL_MIN")])
def test_check_rejects_loss_scales_the_loss_cannot_evaluate(form, c, why):
    from superodom_b200 import api
    with pytest.raises(api.SuperOdomError) as e:
        _check(api, 4, _graph(c), form)
    assert e.value.code == SO_ERR_ARG and "cauchy out of range" in str(e.value) and why in str(e.value) and "(edge 1)" in str(e.value)


def test_restated_loss_fails_outside_the_boundaries():
    """CauchyLoss's arithmetic (b = c^2, 1 / b, b log(1 + s / b)), which k_pg_edges runs too: NaN at 1e200 (b = inf, inf * log(1)) and
    1e-200 (b = 0, 0 * inf), inf at 1e-160 (1 / b overflows from a subnormal b): a solve would return garbage as success."""
    with np.errstate(all="ignore"):
        rho = [PG.robust(_graph(c)[1:2], np.full((1, 6), 0.1))[1][0] for c in (1e200, 1e-200, 1e-160)]
    assert np.isnan(rho[0]) and np.isnan(rho[1]) and rho[2] == np.inf


@pytest.mark.parametrize("c", [C_LO, C_HI])
def test_restated_loss_is_finite_at_the_accepted_boundaries(c):
    """rho and rho' are finite at both boundaries for s from 0 to 4 (at C_LO, s / c^2 overflows past s = DBL_MAX c^2, about 4)."""
    for s in (0.0, 1e-300, 1e-10, 1.0, 3.9):
        E = _graph(c)[1:2]
        E["sqrt_info"] = np.eye(6).ravel()
        with np.errstate(under="ignore"):                               # 1 / c^2 is subnormal at C_HI
            _, rho, rho1 = PG.robust(E, np.r_[np.sqrt(s), 0, 0, 0, 0, 0][None])
        assert np.isfinite(rho[0]) and np.isfinite(rho1[0]) and 0.0 < rho1[0] <= 1.0, (c, s, rho, rho1)

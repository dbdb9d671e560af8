"""so_pose_graph_solve and so_pose_graph_solve_constant at their edges, against the restatements of pose_graph_numpy.py:
reversed and parallel edges next to constant nodes of every arrangement (the reversed-edge chain block of k_pg_nodes), the
linearisation of k_pg_edges at its numerical edges (Log near 0 and pi, q and -q, unnormalised quaternions, general and
rank-deficient S, the Cauchy weight down to its DBL_MIN floor), the accepted loss-scale boundaries, graphs larger than one
co-resident grid of k_pg_trial (the grid-stride loops' later passes) and one context reused across sizes and forms.

Every bound is three times the value measured on an H100 80GB HBM3, and the comparisons of decisions skip, and count, the solves
trust_region_sets.fair finds within rounding of a threshold."""
import time

import numpy as np
import pytest

import pose_graph_numpy as PG
import sessions_numpy as SN
import test_ceres_restatement as CR
import trust_region_sets as TRS
from test_sessions import _normalised

C_LO, C_HI = 1.4916681462400413e-154, 1.3407807929942596e+154      # the loss-scale boundaries (test_pose_graph_edges_cpu.py)
SI = np.r_[np.full(3, 1 / 0.02), np.full(3, 1 / 0.005)]


def _ctx(api):
    return api.Context(max_map_points=1 << 20, max_scan_points=1 << 16)


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stats():
    return dict(n=0, unfair=0, cost=0.0, gmax=0.0, pose=0.0, radius=0.0, weight=0.0, terms=set(), rejected=0)


def _report(st, what):
    print(f"{what}: {st['n']} solves compared ({st['unfair']} near a threshold skipped), exits {sorted(st['terms'])}, with a rejected "
          f"step {st['rejected']}; max relative cost {st['cost']:.2e}, gmax {st['gmax']:.2e}, radius {st['radius']:.2e}, weight "
          f"{st['weight']:.2e}; max pose difference {st['pose']:.2e}")


def _rel(a, b, floor):
    return abs(a - b) / max(abs(b), floor)


def _prob(init, E, fixed, constant):
    return PG.PoseGraph(init, E, fixed) if constant is None else SN.ConstantPoseGraph(init, E, constant)


def _solve(ctx, init, E, fixed, constant, iters, weights=True):
    if constant is None:
        return ctx.pose_graph_solve(init, E, fixed=fixed, max_iterations=iters, weights=weights)
    return ctx.pose_graph_solve(init, E, max_iterations=iters, weights=weights, constant=constant)


def _compare(ctx, init, E, fixed, constant, iters, ref_fn, st, max_radius_error=1e-10):
    """the device solve against ref_fn (CR.solve_full, PG.solve_sparse or PG.solve_chain): identical decisions; the differences
    into st.  -> (device out, ref) or None when the reference is within rounding of a threshold."""
    prob = _prob(init, E, fixed, constant)
    t0 = time.perf_counter()
    ref = ref_fn(prob, prob.x0(), iters)
    st.setdefault("ref_s", 0.0)
    st["ref_s"] += time.perf_counter() - t0
    if not TRS.fair(ref, max_radius_error=max_radius_error):
        st["unfair"] += 1
        return None
    out = _solve(ctx, init, E, fixed, constant, iters)
    X, r, w = out
    assert (r["iterations"], r["successful"], r["unsuccessful"], r["termination"]) == \
        (ref["iterations"], ref["successful"], ref["unsuccessful"], ref["termination"]), (r, ref["steps"])
    Xr = prob.nodes(ref["x"])
    wr = prob.weights(ref["x"])
    st["cost"] = max(st["cost"], _rel(r["final_cost"], ref["final_cost"], 1e-12), _rel(r["initial_cost"], ref["initial_cost"], 1e-12))
    st["gmax"] = max(st["gmax"], _rel(r["gmax"], ref["gmax"], 1e-9))
    st["radius"] = max(st["radius"], _rel(r["radius"], ref["radius"], 0.0))
    st["weight"] = max(st["weight"], float(np.max(np.abs(w - wr) / wr)) if len(wr) else 0.0)
    st["pose"] = max(st["pose"], np.abs(X - Xr).max())
    st["terms"].add(r["termination"])
    st["rejected"] += "r" in ref["steps"]
    st["n"] += 1
    return out, ref


# ------------------------------------------------------------------------------------------------------------- 1. orientation
def _reverse_where(edges, pick):
    return [PG.reversed_edge(e) if pick(e) else e for e in edges]


def _family(rng, name, n):
    if name == "rev_chain":                                             # every chain edge (k + 1, k)
        return PG.drifted(rng, n, reverse=1.0, drift=(0.05, 0.01))
    if name == "rev_half":
        return PG.drifted(rng, n, loops=1, reverse=0.5, drift=(0.05, 0.01))
    if name == "rev_loops":                                             # loop edges (j, i), j > i + 1
        init, edges, truth = PG.drifted(rng, n, loops=max(2, n // 3), drift=(0.1, 0.03))
        return init, _reverse_where(edges, lambda e: abs(e[0] - e[1]) > 1), truth
    if name == "parallel":                                              # (k, k + 1) twice and (k + 1, k) beside them
        return PG.drifted(rng, n, dup=True, both_ways=True, reverse=0.3, drift=(0.05, 0.01))
    if name == "parallel_loops":                                        # each loop edge also stated reversed
        init, edges, truth = PG.drifted(rng, n, loops=max(2, n // 3), full_info=True, cauchy=2.0, drift=(0.1, 0.03))
        return init, edges + [PG.reversed_edge(e) for e in edges if abs(e[0] - e[1]) > 1], truth
    raise ValueError(name)


ORIENT = ("rev_chain", "rev_half", "rev_loops", "parallel", "parallel_loops")


def _edge_masks(n):
    """constant sets beyond test_sessions._masks: first, last, a middle run, runs at both ends, one free node between two
    constants, every node but one"""
    out = {}
    for name, ids in (("first", [0]), ("last", [n - 1]), ("middle", range(n // 3, max(n // 3 + 1, 2 * n // 3))),
                      ("ends", [0, 1, n - 2, n - 1] if n > 4 else [0, n - 1]),
                      ("one_free_between", [k for k in range(n) if k != n // 2] if n < 4 else [n // 2 - 1, n // 2 + 1]),
                      ("all_but_one", [k for k in range(n) if k != (n - 1) // 2])):
        m = np.zeros(n, np.uint8)
        m[list(ids)] = 1
        if m.sum() < n:
            out[name] = m
    return out


def _reverse_next_to(edges, mask):
    """chain edges touching a constant node stored reversed"""
    return _reverse_where(edges, lambda e: abs(e[0] - e[1]) == 1 and e[0] < e[1] and (mask[e[0]] or mask[e[1]]))


@pytest.mark.gpu
def test_orientation_and_multiplicity_against_the_dense_restatement(gpu_api):
    ctx = _ctx(gpu_api)
    st = _stats()
    rng = np.random.default_rng(31)
    for fam in ORIENT:
        for n in (2, 3, 4, 5, 7, 8, 9):
            for iters in (50, 3):
                init, edges, _ = _family(rng, fam, n)
                fixed = int(rng.integers(0, n))
                _compare(ctx, init, PG.to_array(edges), fixed, None, iters, CR.solve_full, st)
                for name, mask in _edge_masks(n).items():
                    _compare(ctx, init, PG.to_array(_reverse_next_to(edges, mask)), 0, mask, iters, CR.solve_full, st)
    _report(st, "orientation")
    # measured: 474 solves compared, 6 skipped, exits 0, 2 and 3
    assert st["n"] > 400 and {0, 2, 3} <= st["terms"]
    # three times the measured: cost 5.4e-9 relative, poses 3.8e-12, radius 0 (identical), weights 1.8e-10 relative; gmax 1.1e-3 (the
    # gradient at the last iterate, a small difference of large terms, as in test_pose_graph.py)
    assert st["cost"] <= 1.7e-8 and st["pose"] <= 1.2e-11 and st["radius"] == 0.0 and st["weight"] <= 5.4e-10 and st["gmax"] <= 3.4e-3
    ctx.close()


@pytest.mark.gpu
def test_chains_take_one_pcg_iteration_per_trial(gpu_api):
    """On a graph of chain edges alone, reversed and parallel ones included, the block-tridiagonal preconditioner is the whole system
    with any constant set: PCG ends after one iteration in every trial.  A wrong chain block (the transpose of a reversed edge's
    A_ij) leaves the solve correct but slower, which only this count sees."""
    ctx = _ctx(gpu_api)
    rng = np.random.default_rng(32)
    solves = 0
    for n in (2, 3, 4, 5, 8, 9, 16, 17):
        for rev, both in ((1.0, False), (0.5, True), (0.0, True)):
            init, edges, _ = PG.drifted(rng, n, dup=True, both_ways=both, reverse=rev, drift=(0.1, 0.03))
            E = PG.to_array(edges)
            _, r, _ = _solve(ctx, init, E, int(rng.integers(0, n)), None, 50)
            assert r["iterations"] > 0 and r["pcg_iterations"] == r["iterations"], (n, rev, r)
            solves += 1
            for name, mask in _edge_masks(n).items():
                _, r, _ = _solve(ctx, init, PG.to_array(_reverse_next_to(edges, mask)), 0, mask, 50)
                assert r["pcg_iterations"] == r["iterations"], (n, rev, name, r)
                solves += 1
    print(f"chains: {solves} solves, one PCG iteration per trial in each")
    ctx.close()


# ------------------------------------------------------------------------------------------------------------- 2. linearisation
ANGLES = (0.0, 1e-8, 1e-2 * (1 - 1e-7), 1e-2 * (1 + 1e-7), 0.5, 2.0, np.pi - 1e-3, np.pi - 1e-6)


def _band(angle):
    return "small" if angle < 0.1 else ("mid" if angle < 3.0 else ("pi-1e-3" if angle < np.pi - 1e-5 else "pi-1e-6"))


def _probe_graph(rng, angle, form):
    """two nodes, one edge whose residual rotation at the start has this angle about a random axis"""
    S = SI.copy()
    if form == "S_full":
        S = rng.normal(0, 5.0, (6, 6)) + np.diag(SI)
    elif form == "S_rankdef":
        S = rng.normal(0, 5.0, (6, 6)) + np.diag(SI)
        S[4] = 0.7 * S[1] - 0.2 * S[5]
    init, edges, _ = PG.drifted(rng, 2, angles=[angle], noise=(0.02, 0.0), drift=(0.0, 0.0), sqrt_info=np.ones(6))
    init = init.copy()
    i, j, z, _, c = edges[0]
    z = z.copy()
    if form == "neg_node":
        init[1, 3:] = -init[1, 3:]
    elif form == "neg_z":
        z[3:] = -z[3:]
    elif form == "neg_both":
        init[0, 3:], z[3:] = -init[0, 3:], -z[3:]
    elif form == "small_q":
        init[:, 3:] *= 1e-3
        z[3:] *= 1e-3
    elif form == "big_q":
        init[:, 3:] *= 1e3
        z[3:] *= 1e3
    return init, [PG.edge(i, j, z, S, c)]


FORMS = ("plain", "neg_node", "neg_z", "neg_both", "small_q", "big_q", "S_full", "S_rankdef")


@pytest.mark.gpu
def test_linearisation_at_its_numerical_edges(gpu_api):
    """max_iterations = 0 evaluates one linearisation: initial_cost == final_cost, gmax and rho' at the start of a two-node graph
    are one edge's 1/2 rho, its gradient max-norm through Plus and its weight.  max_iterations = 1 adds the first step."""
    ctx = _ctx(gpu_api)
    rng = np.random.default_rng(33)
    worst = {}
    unfair = 0
    for angle in ANGLES:
        for form in FORMS:
            for rep in range(2):
                init, edges = _probe_graph(rng, angle, form)
                E = PG.to_array(edges)
                prob = PG.PoseGraph(init, E)
                X, r, w = ctx.pose_graph_solve(init, E, max_iterations=0, weights=True)
                assert r["initial_cost"] == r["final_cost"] and r["iterations"] == 0 and r["termination"] == 0
                ref = CR.solve_full(prob, prob.x0(), 0)
                b = worst.setdefault(_band(angle), dict(cost=0.0, gmax=0.0, weight=0.0, pose=0.0, n=0))
                b["cost"] = max(b["cost"], _rel(r["initial_cost"], ref["initial_cost"], 1e-300))
                b["gmax"] = max(b["gmax"], _rel(r["gmax"], ref["gmax"], 1e-300))
                b["weight"] = max(b["weight"], abs(w[0] - prob.weights(prob.x0())[0]))
                ref1 = CR.solve_full(prob, prob.x0(), 1)
                if not TRS.fair(ref1):
                    unfair += 1
                    continue
                X1, r1 = ctx.pose_graph_solve(init, E, max_iterations=1)
                assert (r1["iterations"], r1["successful"], r1["termination"]) == (ref1["iterations"], ref1["successful"], ref1["termination"])
                b["pose"] = max(b["pose"], np.abs(X1 - prob.nodes(ref1["x"])).max())
                b["n"] += 1
    print(f"linearisation: {unfair} first steps near a threshold skipped")
    for k, b in worst.items():
        print(f"linearisation, angle band {k}: {b['n']} first steps compared; max relative cost {b['cost']:.2e}, gmax {b['gmax']:.2e}, "
              f"weight {b['weight']:.2e}, first-step pose {b['pose']:.2e}")
    # three times the measured per band (relative cost, relative gmax, first-step pose): below 0.1 rad 1.1e-14, 2.0e-15, 8.7e-14; 0.1
    # to 3 rad 7.3e-16, 6.0e-16, 6.7e-13; pi - 1e-3 5.9e-16, 1.5e-15, 4.9e-12; pi - 1e-6 4.4e-16, 9.7e-16, 5.6e-13.  Near pi the Log
    # is ill-conditioned (the axis is a vector part near 0 over its norm), so each band has its own bounds; rho' is 1 without a loss
    BOUNDS = {"small": (3.4e-14, 6e-15, 2.6e-13), "mid": (2.2e-15, 1.8e-15, 2e-12), "pi-1e-3": (1.8e-15, 4.4e-15, 1.5e-11),
              "pi-1e-6": (1.3e-15, 2.9e-15, 1.7e-12)}
    for k, (c, g, p) in BOUNDS.items():
        assert worst[k]["cost"] <= c and worst[k]["gmax"] <= g and worst[k]["pose"] <= p and worst[k]["weight"] == 0.0, (k, worst[k])
    ctx.close()


@pytest.mark.gpu
def test_cauchy_weight_down_to_its_floor(gpu_api):
    """One edge under Cauchy scales from s << c^2 to s >> c^2, down to rho' = DBL_MIN, its floor (c = 1.49e-154, s = 3): the
    weight, 1/2 rho and gmax of the start against the restatement, and a first step."""
    ctx = _ctx(gpu_api)
    rng = np.random.default_rng(34)
    worst_w = worst_c = 0.0
    floor_seen = False
    for angle in (0.3, 2.5):
        init, edges = _probe_graph(rng, angle, "S_full")
        i, j, z, S, _ = edges[0]
        s = PG.robust(PG.to_array(edges), PG.edge_terms(init, PG.to_array(edges))[0])[1][0]
        cs = [np.sqrt(s / q) for q in (1e-8, 1e-2, 1.0, 1e2, 1e8, 1e100, 1e300)]
        for c in cs + ["floor"]:
            if c == "floor":                                            # s = 3 at c = C_LO: s / c^2 = 1.35e308, 1 / that < DBL_MIN
                E = PG.to_array([PG.edge(i, j, z, S * np.sqrt(3.0 / s), C_LO)])
            else:
                E = PG.to_array([PG.edge(i, j, z, S, c)])
            prob = PG.PoseGraph(init, E)
            X, r, w = ctx.pose_graph_solve(init, E, max_iterations=0, weights=True)
            wr = prob.weights(prob.x0())[0]
            ref = CR.solve_full(prob, prob.x0(), 0)
            worst_w = max(worst_w, abs(w[0] - wr) / wr)
            worst_c = max(worst_c, _rel(r["initial_cost"], ref["initial_cost"], 1e-300))
            floor_seen |= bool(w[0] == np.finfo(float).tiny)
            if c == "floor":
                assert w[0] == np.finfo(float).tiny == wr and np.isfinite(r["initial_cost"]) and r["initial_cost"] > 0.0
    print(f"cauchy sweep: max relative weight {worst_w:.2e}, cost {worst_c:.2e}; the DBL_MIN floor reached {floor_seen}")
    # measured: weights and costs identical to the restatement's
    assert floor_seen and worst_w == 0.0 and worst_c == 0.0
    ctx.close()


# ------------------------------------------------------------------------------------------------------------- 3. loss scale
@pytest.mark.gpu
@pytest.mark.parametrize("c", [C_LO, C_HI])
def test_solves_at_the_accepted_loss_scale_boundaries(gpu_api, c):
    """A loop edge with c at a boundary the argument check accepts: the solve ends with a finite cost and finite poses.  At C_LO the
    edge's whitened s stays below DBL_MAX c^2 (about 4), where s / c^2 would overflow."""
    ctx = _ctx(gpu_api)
    init, edges, _ = PG.drifted(np.random.default_rng(35), 9, loops=0, drift=(0.05, 0.01))
    loop = PG.edge(0, 8, PG.compose(PG.inverse(init[0]), init[8]), np.full(6, 0.5), c)
    for fixed in (0, 4):
        X, r, w = ctx.pose_graph_solve(init, edges + [loop], fixed=fixed, weights=True)
        print(f"loss scale {c:.4g}: {r['iterations']} iterations, termination {r['termination']}, final cost {r['final_cost']:.6g}, "
              f"loop edge rho' {w[-1]:.3g}")
        assert np.isfinite(r["final_cost"]) and np.isfinite(r["initial_cost"]) and np.isfinite(X).all() and np.isfinite(w).all()
        assert r["iterations"] > 0 and r["termination"] in (1, 2, 3)
    ctx.close()


# ------------------------------------------------------------------------------------------------------------- 4. large graphs
def _walk(rng, n, loops=0, max_span=200, false_loops=0, cauchy=0.0, reverse=0.0, both_ways=False):
    """PG.drifted's problem built with whole-array operations, for n in the hundreds of thousands: a walk (truth), odometry edges
    measured with noise, loop edges between nodes at most max_span apart, false loops between random nodes, edges stored reversed
    with probability `reverse`, a reversed parallel edge at every third k with both_ways, and a start whose error grows along the
    walk.  -> (init [n, 7], POSE_EDGE_DTYPE array)"""
    from superodom_b200.api import POSE_EDGE_DTYPE

    def unit(q):
        return q / np.linalg.norm(q, axis=1, keepdims=True)

    def small_q(m, sd):
        return unit(np.c_[rng.normal(0, sd / 2, (m, 3)), np.ones(m)])

    def rel(a, b):                                                      # X_a^-1 X_b
        qa = a[:, 3:] * [-1, -1, -1, 1]
        return np.c_[np.einsum("mki,mk->mi", PG._rots(a[:, 3:]), b[:, :3] - a[:, :3]), PG._qmul_rows(qa, b[:, 3:])]

    def noisy(z, sd):
        return np.c_[z[:, :3] + np.einsum("mij,mj->mi", PG._rots(z[:, 3:]), rng.normal(0, sd[0], (len(z), 3))),
                     PG._qmul_rows(z[:, 3:], small_q(len(z), sd[1]))]
    yaw = np.cumsum(rng.normal(0, 0.15, n))
    q = unit(np.c_[rng.normal(0, 0.02, (n, 2)), np.sin(yaw / 2), np.cos(yaw / 2)])
    t = np.cumsum(rng.normal(0, 1.0, (n, 3)) * [1, 1, 0.2], 0)
    truth = np.c_[t, q]
    noise = (0.02, 0.005)
    ii, jj = [np.arange(n - 1)], [np.arange(1, n)]
    if both_ways:
        k = np.arange(1, n - 1, 3)
        ii.append(k + 1)
        jj.append(k)
    if loops:
        a = rng.integers(0, n - 2, loops)
        ii.append(a)
        jj.append(np.minimum(n - 1, a + rng.integers(2, max_span + 1, loops)))
    ii, jj = np.concatenate(ii), np.concatenate(jj)
    z = noisy(rel(truth[ii], truth[jj]), noise)
    c = np.where(np.abs(ii - jj) > 1, cauchy, 0.0)
    if false_loops:
        a, b = rng.integers(0, n, false_loops), rng.integers(0, n, false_loops)
        keep = a != b
        ii, jj = np.r_[ii, a[keep]], np.r_[jj, b[keep]]
        z = np.r_[z, np.c_[rng.normal(0, 3.0, (keep.sum(), 3)), small_q(keep.sum(), 0.6)]]
        c = np.r_[c, np.full(keep.sum(), cauchy)]
    m = len(ii)
    S = np.zeros((m, 6, 6))
    S[:, np.arange(6), np.arange(6)] = SI
    flip = rng.random(m) < reverse
    if flip.any():                                                      # PG.reversed_edge on every flipped edge
        R = PG._rots(z[flip, 3:])
        B = np.zeros((flip.sum(), 6, 6))
        B[:, :3, :3], B[:, 3:, 3:] = np.transpose(R, (0, 2, 1)), np.transpose(R, (0, 2, 1))
        zf = z[flip]
        zq = zf[:, 3:] * [-1, -1, -1, 1]
        z[flip] = np.c_[-np.einsum("mij,mj->mi", PG._rots(zq), zf[:, :3]), zq]
        S[flip] = S[flip] @ B
        ii[flip], jj[flip] = jj[flip], ii[flip]
    E = np.zeros(m, POSE_EDGE_DTYPE)
    E["i"], E["j"], E["z"], E["sqrt_info"], E["cauchy"] = ii, jj, z, S.reshape(m, 36), c
    drift_q = unit(np.c_[np.zeros((n, 2)), np.sin(np.cumsum(rng.normal(0, 0.003, n)) / 2), np.cos(np.cumsum(rng.normal(0, 0.003, n)) / 2)])
    init = np.c_[t + np.cumsum(rng.normal(0, 0.01, (n, 3)), 0), PG._qmul_rows(q, drift_q)]
    init[0] = truth[0]
    return init, E


def _runs_mask(n, run):
    """constant runs at both ends and in the middle"""
    m = np.zeros(n, np.uint8)
    m[:run], m[n - run:], m[n // 2 - run // 2: n // 2 + run // 2 + 1] = 1, 1, 1
    return m


def _twice_identical(ctx, init, E, fixed, constant, iters, first):
    again = _solve(ctx, init, E, fixed, constant, iters)
    assert first[0].tobytes() == again[0].tobytes() and first[2].tobytes() == again[2].tobytes()
    assert {k: v for k, v in first[1].items() if k != "time_ms"} == {k: v for k, v in again[1].items() if k != "time_ms"}


@pytest.mark.gpu
def test_chain_past_the_co_resident_grid(gpu_api):
    """k_pg_trial runs one thread per node on at most the co-resident CTAs.  With 255 registers at 256 threads (DESIGN.md section
    4) one CTA fits on an SM, so the grid is capped at SMs CTAs from n = 256 SMs + 1 on, and the 2 * gstride() loops of the cyclic
    reduction take a second pass from n = 512 SMs + 1.  n = 2 * 2048 SMs + 1 (540 673 on 132 SMs) strides twice even at 8 CTAs per
    SM, so this graph reaches those passes whatever the occupancy.  Reversed and parallel chain edges, constant runs at both ends
    and in the middle, against the exact banded step."""
    sms = _sms()
    n = 2 * sms * 2048 + 1
    rng = np.random.default_rng(41)
    t0 = time.perf_counter()
    init, E = _walk(rng, n, reverse=0.5, both_ways=True)
    mask = _runs_mask(n, 1000)
    print(f"chain n={n} ({sms} SMs), {len(E)} edges: built in {time.perf_counter() - t0:.1f} s")
    ctx = _ctx(gpu_api)
    st = _stats()
    t0 = time.perf_counter()
    got = _compare(ctx, init, E, 0, mask, 6, PG.solve_chain, st, max_radius_error=np.inf)
    assert got is not None
    out, ref = got
    r = out[1]
    print(f"chain n={n}: {r['iterations']} trials, {r['pcg_iterations']} PCG iterations, device {r['time_ms']:.0f} ms, reference "
          f"{st['ref_s']:.1f} s, steps {ref['steps']}")
    _report(st, f"chain n={n}")
    assert r["iterations"] <= r["pcg_iterations"] <= 2 * r["iterations"]
    assert out[0][mask == 1].tobytes() == _normalised(init)[mask == 1].tobytes()
    # three times the measured: cost 3.2e-15 relative, poses 1.7e-11, radius 6.2e-14, weights identical (no loss); one PCG iteration
    # per trial (6 over 6)
    assert st["cost"] <= 1e-14 and st["pose"] <= 5.2e-11 and st["radius"] <= 1.9e-13 and st["weight"] == 0.0
    _twice_identical(ctx, init, E, 0, mask, 6, out)
    ctx.close()


@pytest.mark.gpu
def test_graphs_with_loops_past_the_co_resident_grid(gpu_api):
    """Walks with 1 % loop edges (a third of them reversed), a few false loops, Cauchy on every loop edge, at SMs * 256 nodes (a full
    grid), one node more (one thread of a second pass), 2 SMs 256 + 1 and 4 SMs 256 + 1, against the exact sparse step; one solve
    with the fixed node in the last grid stride, one with a constant set."""
    sms = _sms()
    ctx = _ctx(gpu_api)
    st = _stats()
    rng = np.random.default_rng(42)
    for n, form in ((sms * 256, "fixed"), (sms * 256 + 1, "fixed_last"), (2 * sms * 256 + 1, "constant"),
                    (4 * sms * 256 + 1, "fixed_last")):
        init, E = _walk(rng, n, loops=n // 100, max_span=60, false_loops=5, cauchy=1.0, reverse=0.33)
        fixed = n - 1 if form == "fixed_last" else int(rng.integers(0, n))         # n - 1: alone in the grid's last stride
        mask = _runs_mask(n, 50) if form == "constant" else None
        ref_before = st.get("ref_s", 0.0)
        got = _compare(ctx, init, E, 0 if mask is not None else fixed, mask, 6, PG.solve_sparse, st, max_radius_error=np.inf)
        if got is None:
            print(f"loops n={n}: near a threshold, skipped")
            continue
        out, ref = got
        r = out[1]
        print(f"loops n={n} ({form}), {len(E)} edges: {r['iterations']} trials, {r['pcg_iterations']} PCG iterations, device "
              f"{r['time_ms']:.0f} ms, reference {st['ref_s'] - ref_before:.1f} s, steps {ref['steps']}")
        _twice_identical(ctx, init, E, 0 if mask is not None else fixed, mask, 6, out)
    _report(st, "loops past the grid")
    assert st["n"] == 4
    # PCG's step differs from the exact one by up to its tolerance (about 400 iterations per trial here): three times the measured
    # cost 1.3e-8 relative, poses 2.1e-6, radius 8.3e-8, weights 1.2e-6, gmax 6.3e-7
    assert st["cost"] <= 3.8e-8 and st["pose"] <= 6.2e-6 and st["radius"] <= 2.5e-7 and st["weight"] <= 3.5e-6 and st["gmax"] <= 1.9e-6
    ctx.close()


# ------------------------------------------------------------------------------------------------------------- 5. one context
@pytest.mark.gpu
def test_one_context_across_sizes_and_forms(gpu_api):
    """One context through graphs of falling and rising size, fixed and constant-set: every output bit-identical to the same call
    on a fresh context, so no phase reads a grow-only buffer past n or a stale constant mask or reduction partial."""
    sms = _sms()
    rng = np.random.default_rng(51)
    init9, edges9, _ = PG.drifted(rng, 9, loops=2, reverse=0.5, drift=(0.05, 0.01))
    init2, edges2, _ = PG.drifted(rng, 2, reverse=1.0, drift=(0.05, 0.01))
    big = sms * 256 + 1
    initb, Eb = _walk(rng, big, loops=big // 100, max_span=60, cauchy=1.0, reverse=0.3)
    init3, E3 = _walk(rng, 300, loops=3, reverse=0.5, both_ways=True)
    seq = [(init9, PG.to_array(edges9), 4, None), (initb, Eb, 0, _runs_mask(big, 40)), (init9, PG.to_array(edges9), 4, None),
           (init2, PG.to_array(edges2), 1, None), (init3, E3, 0, _runs_mask(300, 5)), (init9, PG.to_array(edges9), 4, None)]
    shared = _ctx(gpu_api)
    for k, (init, E, fixed, mask) in enumerate(seq):
        a = _solve(shared, init, E, fixed, mask, 8)
        fresh = _ctx(gpu_api)
        b = _solve(fresh, init, E, fixed, mask, 8)
        fresh.close()
        assert a[0].tobytes() == b[0].tobytes() and a[2].tobytes() == b[2].tobytes(), k
        assert {x: v for x, v in a[1].items() if x != "time_ms"} == {x: v for x, v in b[1].items() if x != "time_ms"}, k
        print(f"one context, step {k + 1}: n={len(init)}, {a[1]['iterations']} iterations, bit-identical to a fresh context")
    shared.close()

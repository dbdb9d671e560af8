"""The end of the solve against exact references (tests/solve_numerics_ref.py): the line rows' normal equations, a registration
that meets a NaN-weighted line row, and the covariance step at prescribed spectra through the so_covariance stage hook."""
import numpy as np
import pytest

import degenerate_sets as D
import solve_numerics_ref as R
from conftest import get_case

EPS = np.finfo(np.float64).eps
LINE_RES = 0.1
# Bound constant of the covariance comparisons, |cov - cov_ref| <= C_COV eps kappa |cov_ref|.  The Jacobi eigen-decomposition is
# backward stable: its rotations (FP64 angle t, c = rsqrt(1 + t^2), s = t c) are orthogonal to an ulp and zero their pair to an
# ulp, each rounds the entries it touches once, and the sweeps stop when the off-diagonal mass is 1e-33 of the diagonal's, so the computed
# pairs belong to H + E with |E| a small multiple of eps |H| (about sqrt(number of rotations touching an entry) ~ 4-6).  First-order
# perturbation then moves 1/w_i by |E| / w_i and the eigenvectors by |E| / gap, so the pseudo-inverse moves by about
# |E| / w_min_kept = c eps kappa relative, kappa = w_max / w_min_kept.  C_COV = 16 is that with a factor of ~3 to spare.
C_COV = 16.0


def _ctx(api, **kw):
    return api.Context(max_map_points=1 << 20, max_scan_points=262144, plane_res=0.2, line_res=LINE_RES, **kw)


# ---------------------------------------------------------------------------------------------------------- CPU-side checks
def test_line_rows_jacobian_matches_central_differences():
    """The restated line-row Jacobian is the derivative of its own residual along PoseLocalParameterization::Plus."""
    rng = np.random.default_rng(3)
    n = 40
    p = rng.uniform(-8, 8, size=(n, 3))
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    m = rng.uniform(-8, 8, size=(n, 3))
    a, b = m + 0.1 * d, m - 0.1 * d
    q = rng.normal(size=4)
    pose = np.concatenate([rng.uniform(-3, 3, 3), q / np.linalg.norm(q)])
    r, J, _, _ = R.line_rows(p, a, b, np.ones(n), pose, 1.0)
    h = 1e-6
    for j in range(6):
        e = np.zeros(6)
        e[j] = h
        num = (R.line_residual(p, a, b, R.pose_plus(pose, e)) - R.line_residual(p, a, b, R.pose_plus(pose, -e))) / (2 * h)
        assert np.abs(num - J[:, :, j]).max() <= 1e-7 * max(1.0, np.abs(J).max()), j


def test_covariance_reference_matches_numpy_on_well_conditioned_h():
    rng = np.random.default_rng(4)
    for n in (6, 12):
        for _ in range(3):
            V = np.linalg.qr(rng.normal(size=(n, n)))[0]
            H = (V * rng.uniform(1.0, 50.0, n)) @ V.T
            H = 0.5 * (H + H.T)
            ref = R.covariance_reference(H)
            w, U = np.linalg.eigh(H)
            cov = ((U / w) @ U.T)[:6, :6]
            assert ref["keep"].all() and np.abs(ref["cov"] - cov).max() <= 1e-12 * np.abs(cov).max()
            e, E = np.linalg.eigh(cov[:3, :3])
            assert abs(ref["pos_err"] - np.sqrt(e[2])) <= 1e-12 * np.sqrt(e[2])
            assert abs(ref["pos_inv_cond"] - np.sqrt(e[0] / e[2])) <= 1e-10
            assert abs(abs(ref["pos_dir"] @ E[:, 2]) - 1) <= 1e-10


def test_covariance_reference_cut_rule():
    """A zero eigenvalue and one below 1e-7 in sqrt(w / w_max) are cut, one above is kept."""
    w = np.array([0.0, 1e-15, 1e-13, 1.0, 2.0, 4.0])                # sqrt(w / 4): 0, 1.6e-8, 1.6e-7, ...
    ref = R.covariance_reference(np.diag(w[[3, 0, 4, 1, 5, 2]]))
    assert list(ref["keep"]) == [False, False, True, True, True, True]
    w = np.array([1e-10, 4.0, 4.0, 4.0, 4.0, 4.0])
    assert R.covariance_reference(np.diag(w))["keep"].all()


# ---------------------------------------------------------------------------------------------------------- A: line rows
def _edge_inputs(kind):
    """(surf map case, edge map, edge cloud) for the line-row comparisons."""
    from superodom_b200 import synth
    case = get_case("cfg1")
    em = synth.make_edge_map(case["scene"], LINE_RES)
    if kind == "synthetic":
        es = synth.make_edge_scan(em, case["pose_true"], 5000)
    else:
        es = None                              # extracted on the device from a ring scan (below)
    return case, em, es


def _line_poses(case):
    prior, true = np.asarray(case["pose_prior"], np.float64), np.asarray(case["pose_true"], np.float64)
    both = true.copy()
    both[:3] += [0.45, 0.35, 0.3]               # moves the residuals across sqrt(a^2) = 0.55 m
    far = true.copy()
    far[:3] += [3.0, -2.0, 1.5]                 # >= 2.5 m from every axis-aligned line: every row saturates
    return dict(prior=prior, true=true, both=both, far=far)


def _check_line_rows(ctx, om, es, pose_corr, case, min_ok):
    gc, ghr = ctx.correspond_edge(es, pose_corr)
    oc, ohr = om.correspond_edge(es, pose_corr, LINE_RES)
    assert np.array_equal(ghr, ohr) and np.array_equal(gc["status"].astype(np.int32), oc["status"])
    ok = oc["status"] == 0
    assert ok.sum() >= min_ok
    # (a, b) match the oracle's up to the swap the sign of an eigenvector allows
    same = np.abs(gc["a"][ok] - oc["a"][ok]).max(1) + np.abs(gc["b"][ok] - oc["b"][ok]).max(1) if ok.any() else np.zeros(0)
    swap = np.abs(gc["a"][ok] - oc["b"][ok]).max(1) + np.abs(gc["b"][ok] - oc["a"][ok]).max(1) if ok.any() else np.zeros(0)
    assert (np.minimum(same, swap) < 1e-7).all()
    a2 = R.tukey_a2(LINE_RES)
    p = es[:, :3].astype(np.float64)[ok]
    out = {}
    for name, pose in _line_poses(case).items():
        H, g, cost = ctx.evaluate(pose)
        rH, rg, rcost, inside = R.line_normal_equations(p, gc["a"][ok], gc["b"][ok], gc["w"][ok], pose, a2)
        if inside == 0:
            assert (H == 0).all() and (g == 0).all(), name
        else:
            assert np.abs(H - rH).max() <= 1e-10 * np.abs(rH).max(), name
            assert np.abs(g - rg).max() <= 1e-10 * max(np.abs(rg).max(), 1e-3 * np.abs(rH).max()), name
        assert abs(cost - rcost) <= 1e-10 * rcost, name
        out[name] = (inside, int(ok.sum()))
    return out


@pytest.mark.gpu
def test_line_rows_normal_equations_synthetic(gpu_api, oracle_mod):
    """so_correspond_edge + so_evaluate (edge rows only) against the restated line rows, at the prior, the truth, a pose with rows
    on both sides of the Tukey threshold and a far pose where every row saturates (H = g = 0, cost = 1/2 sum w a^2 / 6)."""
    case, em, es = _edge_inputs("synthetic")
    ctx = _ctx(gpu_api)
    ctx.map_set_points(case["map_xyzi"])
    ctx.map_set_resolution(LINE_RES, 0.2)
    ctx.map_set_edge_points(em)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    om.set_edge_points(em)
    for pose in (case["pose_prior"], case["pose_true"]):
        out = _check_line_rows(ctx, om, es, pose, case, 1000)
        inside, n = out["both"]
        assert 0.1 * n <= inside <= 0.9 * n, out
        assert out["far"][0] == 0
    # CTA partial boundaries of the edge kernels: 1, 255, 256, 257 rows
    for k in (1, 255, 256, 257):
        sub = np.ascontiguousarray(es[:k])
        _check_line_rows(ctx, om, sub, case["pose_prior"], case, 1 if k == 1 else k // 2)
    ctx.close()


@pytest.mark.gpu
def test_line_rows_normal_equations_extracted_edges(gpu_api, oracle_mod):
    """The same on edges so_scan_extract_edges takes from a cfg1 ring scan."""
    from superodom_b200 import synth
    case, em, _ = _edge_inputs("extracted")
    ctx = _ctx(gpu_api)
    ctx.map_set_points(case["map_xyzi"])
    ctx.map_set_resolution(LINE_RES, 0.2)
    ctx.map_set_edge_points(em)
    es = ctx.scan_extract_edges(synth.make_ring_scan(case["scene"], case["cfg"]["sensor"], case["pose_true"], 6300))
    assert len(es) > 200
    om = oracle_mod.OracleMap(case["map_xyzi"])
    om.set_edge_points(em)
    out = _check_line_rows(ctx, om, es, case["pose_prior"], case, 100)
    assert out["both"][0] > 0
    ctx.close()


# ---------------------------------------------------------------------------------------------------------- B: NaN-weighted line rows
@pytest.mark.gpu
def test_nan_weight_line_row_stops_registration_like_the_oracle(gpu_api, oracle_mod):
    """An exactly collinear 10-point cluster in the edge map, reached by one edge point: its fit weight 1 - sqrt(msd / 3 lineRes)
    reads rounding noise of either sign and comes out NaN.  Ceres 2.0 CHECK-fails on that row (ceres::Corrector); this library
    and the oracle stop the registration with SO_STATUS_INVALID_EVALUATION (3) at the first evaluation that holds the row: the
    pose the ICP iteration started from (here the prior), iter_cost NaN, no LM step, no covariance."""
    case, em, es = _edge_inputs("synthetic")
    e = D.edge_sets()
    col = np.flatnonzero(e["label"] == "collinear_10")
    clusters = e["map_xyzi"].reshape(-1, 10, 4)[col].reshape(-1, 4)
    em2 = np.ascontiguousarray(np.concatenate([em, clusters]))
    prior = np.asarray(case["pose_prior"], np.float64)
    Rp = R.quat_to_R(prior[3:])
    qw = e["scan_xyzi"][col, :3].astype(np.float64)
    qs = np.concatenate([((qw - prior[:3]) @ Rp).astype(np.float32), np.ones((len(col), 1), np.float32)], 1)
    ctx = _ctx(gpu_api)
    ctx.map_set_points(case["map_xyzi"])
    ctx.map_set_resolution(LINE_RES, 0.2)
    ctx.map_set_edge_points(em2)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    om.set_edge_points(em2)
    gc, _ = ctx.correspond_edge(qs, prior)
    oc, _ = om.correspond_edge(qs, prior, LINE_RES)
    both = np.flatnonzero((gc["status"] == 0) & (oc["status"] == 0) & np.isnan(gc["w"]) & np.isnan(oc["w"]))
    assert len(both) > 0, (np.isnan(gc["w"]).sum(), np.isnan(oc["w"]).sum())
    es2 = np.ascontiguousarray(np.concatenate([es, qs[both[:1]]]))
    cfg = case["cfg"]
    for cap in (2000, 0):
        r = ctx.register(case["scan_xyzi"], prior, cfg["max_iterations"], cap, edge_xyzi=es2)
        ro = om.register(case["scan_xyzi"], prior, 0.2, cfg["max_iterations"], cap, knn_mode=0, edge_xyzi=es2, line_res=LINE_RES)
        assert r.status == ro.status == 3
        n = ro.n_iterations
        assert r.n_iterations == n == 1
        assert list(r.iter_n_surf[:n]) == list(ro.iter_n_surf[:n]) and list(r.iter_n_edge[:n]) == list(ro.iter_n_edge[:n])
        assert list(r.iter_lm_steps[:n]) == list(ro.iter_lm_steps[:n]) == [0]
        assert list(r.iter_lm_successful[:n]) == list(ro.iter_lm_successful[:n])
        assert list(r.iter_lm_termination[:n]) == list(ro.iter_lm_termination[:n])
        assert np.isnan(r.iter_cost[0]) and np.isnan(ro.iter_cost[0])
        assert np.array_equal(np.array(r.pose_opt), prior) and np.array_equal(np.array(ro.pose_opt), prior)
        assert not np.array(r.cov).any()
    # without the NaN row the same registration runs to the end
    r = ctx.register(case["scan_xyzi"], prior, cfg["max_iterations"], 2000, edge_xyzi=es)
    assert r.status == 0
    ctx.close()


# ---------------------------------------------------------------------------------------------------------- C: covariance step
def _spectrum_cases():
    """(label, H) symmetric test matrices, seeded."""
    rng = np.random.default_rng(11)
    out = []

    def rot(n):
        return np.linalg.qr(rng.normal(size=(n, n)))[0]

    def sym(H):
        return 0.5 * (H + H.T)
    base = np.array([9e6, 1e6, 2.5e5, 4e4, 2.5e3, 1.0])
    for ratio in (1e-2, 1e-3, 1e-4, 1e-5, 1e-6, 5e-7, 3e-7, 1.5e-7, 7e-8, 3e-8, 1e-8, 1e-9):
        w = base.copy()
        w[-1] = (ratio * 3e3) ** 2                       # s_min / s_max = ratio
        w[:-1] = np.sort(rng.uniform(4e4, 9e6, 5))[::-1]
        w[0] = 9e6
        out.append((f"axis_{ratio:.0e}", np.diag(w[rng.permutation(6)])))
        V = rot(6)
        out.append((f"rot_{ratio:.0e}", sym((V * w) @ V.T)))
    for k in (1e1, 1e2, 1e3, 1e4):                       # translation / rotation column scales k apart
        A = sym((lambda V: (V * rng.uniform(1, 20, 6)) @ V.T)(rot(6)))
        Dg = np.diag([1, 1, 1, k, k, k])
        out.append((f"scale_{k:.0e}", sym(Dg @ A @ Dg)))
    for i in (0, 4):                                      # an exactly zero row / column
        A = sym((lambda V: (V * rng.uniform(1, 20, 6)) @ V.T)(rot(6)))
        A[i, :] = 0
        A[:, i] = 0
        out.append((f"zero_{i}", A))
    w = np.array([0.0, 3.0, 5.0, 7.0, 11.0, 13.0])
    out.append(("rot_exact_null", sym((lambda V: (V * w) @ V.T)(rot(6)))))
    out.append(("repeated_full", sym((lambda V: (V * np.array([2.0, 2.0, 2.0, 5.0, 5.0, 5.0])) @ V.T)(rot(6)))))
    out.append(("repeated_blocks", np.diag([4.0, 4.0, 4.0, 9.0, 9.0, 1.0])))
    out.append(("diagonal", np.diag([3.0, 7.0, 1.0, 0.5, 11.0, 2.0])))
    for n12 in range(3):                                  # the 12-column form (mode OPTIMIZED)
        w = rng.uniform(1, 50, 12)
        if n12 == 1:
            w[3] = 1e-9
        if n12 == 2:
            w[2] = 0.0
        out.append((f"h12_{n12}", sym((lambda V: (V * w) @ V.T)(rot(12)))))
    return out


def _assert_covariance(label, r, ref, H):
    cov = np.array(r.cov).reshape(6, 6)
    w = ref["w"]
    wmax = w[-1]
    clear = np.abs(w - R.CUT ** 2 * wmax) > C_COV * EPS * wmax   # cut decisions outside the band rounding can move
    kept = ref["keep"]
    kmin = w[kept].min() if kept.any() else wmax
    kappa = wmax / kmin
    tol = C_COV * EPS * kappa
    scale = np.abs(ref["cov"]).max()
    if clear.all():
        assert np.abs(cov - ref["cov"]).max() <= tol * scale, (label, np.abs(cov - ref["cov"]).max() / scale, tol)
        if kappa <= 1e9:
            assert np.abs(cov - ref["cov"]).max() <= 1e-6 * scale, label
        for f, key in (("pos_err", "pos_err"), ("ori_err_deg", "ori_err_deg")):
            assert abs(getattr(r, f) - ref[key]) <= tol * max(ref[key], 1e-300), (label, f)
        for f in ("pos", "ori"):
            got, want = getattr(r, f + "_inv_cond"), ref[f + "_inv_cond"]
            assert np.isfinite(got) == np.isfinite(want), (label, f, got, want)
            if np.isfinite(want):
                # an absolute error tol e_max in the block's smallest eigenvalue moves sqrt(e_min / e_max) by at most sqrt(tol)
                assert 0.0 <= got <= 1.0 and abs(got - want) <= np.sqrt(tol) + tol, (label, f, got, want)
            d = np.array(getattr(r, f + "_dir"))
            gap = ref[f + "_gap"]
            if gap > 1e-6:
                assert 1 - abs(d @ ref[f + "_dir"]) <= max(1e-12, (8 * tol / gap) ** 2 + 8 * tol / gap), (label, f, d, ref[f + "_dir"])
            else:                                         # direction not defined: a unit eigenvector of the largest eigenvalue
                o = 0 if f == "pos" else 3
                B = ref["cov"][o:o + 3, o:o + 3]
                assert abs(np.linalg.norm(d) - 1) <= 1e-12
                assert np.linalg.norm(B @ d - ref[f + "_eig"][2] * d) <= 1e-9 * np.abs(B).max(), (label, f)
    else:
        # a direction inside the band: the cut may go either way; the result is one of the two pseudo-inverses
        pass


@pytest.mark.gpu
def test_covariance_at_prescribed_spectra(gpu_api):
    """so_covariance against the mpmath pseudo-inverse on swept condition numbers (weak direction axis-aligned and rotated),
    column scales 1e4 apart, exact cuts, repeated eigenvalues, a diagonal H and the 12-column form."""
    ctx = _ctx(gpu_api)
    seen = set()
    for label, H in _spectrum_cases():
        r = ctx.covariance(H)
        ref = R.covariance_reference(H)
        _assert_covariance(label, r, ref, H)
        if label.startswith(("zero", "rot_exact", "h12_2")):
            assert not ref["keep"].all()
            for f in ("pos_inv_cond", "ori_inv_cond"):
                v = getattr(r, f)
                assert np.isfinite(v) and 0.0 <= v <= 1.0, (label, f, v)
        if label == "diagonal":
            assert np.abs(np.array(r.cov).reshape(6, 6) - ref["cov"]).max() <= 2 * EPS * np.abs(ref["cov"]).max()
        seen.add(label.split("_")[0])
    assert {"axis", "rot", "scale", "zero", "repeated", "diagonal", "h12"} <= seen
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny", "cfg1"])
def test_covariance_of_registration_normal_equations(gpu_api, name):
    """Well-conditioned H from real scenes: the plane rows' normal equations at the truth."""
    case = get_case(name)
    ctx = gpu_api.Context(max_map_points=max(1 << 20, len(case["map_xyzi"]) + 1024), max_scan_points=262144,
                          plane_res=case["cfg"]["plane_res"])
    ctx.map_set_points(case["map_xyzi"])
    ctx.correspond(case["scan_xyzi"], case["pose_true"], 0)
    H, _, _ = ctx.evaluate(case["pose_true"])
    r = ctx.covariance(H)
    ref = R.covariance_reference(H)
    assert ref["keep"].all()
    _assert_covariance(name, r, ref, H)
    ctx.close()

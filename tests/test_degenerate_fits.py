"""Plane and line fits on crafted degenerate neighbourhoods (tests/degenerate_sets.py): coincident, exactly collinear and
coplanar points, repeated eigenvalues, gate quantities a hair either side of their thresholds, planes through the origin,
coordinates at the edge of the block grid, lattice neighbourhoods.  First the CPU oracle against a plain numpy statement of the
gates, then the device fits against the oracle."""
from collections import Counter

import numpy as np
import pytest

import degenerate_sets as D
from conftest import get_case, quat_angle

IDENTITY = np.array([0, 0, 0, 0, 0, 0, 1.0])


def _mismatch_report(label, mask):
    return dict(Counter(label[mask].tolist()))


def test_oracle_plane_gates_match_numpy(oracle_mod):
    """The oracle's status on every crafted set equals the numpy classification (eigvalsh gates, then the lstsq plane and its
    point distances), for every set outside a 1e-9 relative band around a threshold -- which here is every set."""
    d = D.plane_sets()
    om = oracle_mod.OracleMap(d["map_xyzi"])
    oc, _, ohr = om.correspond(d["scan_xyzi"], IDENTITY, D.PLANE_RES, 0, 0)
    n = len(d["sets"])
    own = np.arange(n)[:, None] * 5 + np.arange(5)[None, :]
    assert np.array_equal(np.sort(oc["nn"], 1), own)                        # each query's 5-NN is exactly its own cluster
    exp, clear = D.classify(d)
    assert clear.all()
    bad = oc["status"] != exp
    assert not bad.any(), _mismatch_report(d["label"], bad)
    # the eigenvalues the gates read agree with LAPACK's to rounding
    scale = np.maximum(d["lam2"], 1e-30)
    for j, k in enumerate(("lam0", "lam1", "lam2")):
        assert (np.abs(oc["eigval"][:, j] - d[k]) <= 1e-13 * scale + 1e-25).all(), k
    # every class reaches the gate it was built for
    for lab, st in (("lam0_+1e-07", 0), ("lam0_-1e-07", 3), ("ratio_+1e-07", 0), ("ratio_-1e-07", 3),
                    ("plane_dist_+1e-05", 5), ("plane_dist_-1e-05", 0), ("coincident_5", 3), ("collinear_diag", 3)):
        assert (oc["status"][d["label"] == lab] == st).all(), lab
    assert ohr[0] > 300 and ohr[3] > 500 and ohr[5] > 100


@pytest.mark.gpu
@pytest.mark.parametrize("coop", [True, False])
def test_degenerate_plane_fits_match_oracle(gpu_api, oracle_mod, monkeypatch, coop):
    """so_correspond (k-NN + k_fit) on the crafted sets against the oracle: identical status and neighbours everywhere, the
    plane within the tolerances of test_correspondences_and_normal_equations.  coop=False searches one query per thread
    (SO_NO_COOP_KNN) instead of one warp per query."""
    if not coop:
        monkeypatch.setenv("SO_NO_COOP_KNN", "1")
    d = D.plane_sets()
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=65536, plane_res=D.PLANE_RES)
    ctx.map_set_points(d["map_xyzi"])
    gc, gho, ghr = ctx.correspond(d["scan_xyzi"], IDENTITY, 0)
    ctx.close()
    om = oracle_mod.OracleMap(d["map_xyzi"])
    oc, oho, ohr = om.correspond(d["scan_xyzi"], IDENTITY, D.PLANE_RES, 0, 0)
    _, clear = D.classify(d)
    gst, ost = gc["status"].astype(np.int64), oc["status"].astype(np.int64)
    bad = clear & (gst != ost)
    assert not bad.any(), ("status differs", _mismatch_report(d["label"], bad))
    assert np.array_equal(ghr, ohr)
    assert np.array_equal(gc["nn"].astype(np.int64), oc["nn"]) and np.array_equal(gc["nn_d2"], oc["nn_d2"])
    ok = ost == 0
    assert ok.sum() > 300
    assert np.allclose(gc["n"][ok], oc["n"][ok], rtol=0, atol=1e-8)
    assert np.allclose(gc["d"][ok], oc["d"][ok], rtol=1e-10, atol=0)
    assert np.allclose(gc["w"][ok], oc["w"][ok], rtol=1e-10, atol=0)
    assert (gc["w"][~ok] == 0).all() and (gc["n"][~ok] == 0).all()
    # Observability labels are read off the PCA normal, the eigenvector of the smallest eigenvalue.  Where that eigenvalue is
    # repeated (the square-plus-apex sets) the eigenvector is any vector of a plane, in the reference as well, so the labels are
    # compared only where the eigengap (lam1 - lam0) / lam2 leaves the vector defined.
    defined = ok & (d["gap"] > 1e-6)
    assert defined.sum() > 300
    bad = defined & (gc["obs"] != oc["obs"].astype(np.uint8)).any(1)
    assert not bad.any(), ("obs differs", _mismatch_report(d["label"], bad))


@pytest.mark.gpu
def test_degenerate_line_fits_match_oracle(gpu_api, oracle_mod):
    """so_correspond_edge (10-NN, best-line selection, line PCA) on 10 coincident points, 10 exactly collinear points and two
    distinct points repeated five times each, against the oracle."""
    e = D.edge_sets()
    p = D.plane_sets()
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=65536, plane_res=D.PLANE_RES, line_res=D.LINE_RES)
    ctx.map_set_points(p["map_xyzi"])
    ctx.map_set_edge_points(e["map_xyzi"])
    gc, ghr = ctx.correspond_edge(e["scan_xyzi"], IDENTITY)
    ctx.close()
    om = oracle_mod.OracleMap(p["map_xyzi"])
    om.set_edge_points(e["map_xyzi"])
    oc, ohr = om.correspond_edge(e["scan_xyzi"], IDENTITY, D.LINE_RES)
    own = np.arange(len(e["sets"]))[:, None] * 10 + np.arange(10)[None, :]
    assert np.array_equal(np.sort(oc["nn"], 1), own)
    bad = gc["status"].astype(np.int32) != oc["status"]
    assert not bad.any(), _mismatch_report(e["label"], bad)
    assert np.array_equal(ghr, ohr)
    assert np.array_equal(gc["nn"].astype(np.int64), oc["nn"])
    omask = np.zeros(len(oc), np.uint32)
    for j in range(10):
        omask |= np.where(np.arange(10)[None, :] < oc["n_sel"][:, None], (oc["sel"] == j), False).any(1).astype(np.uint32) << np.uint32(j)
    assert np.array_equal(gc["selected_mask"], omask)
    ok = oc["status"] == 0
    assert ok.sum() > 0
    same = np.abs(gc["a"][ok] - oc["a"][ok]).max(1) + np.abs(gc["b"][ok] - oc["b"][ok]).max(1)
    swap = np.abs(gc["a"][ok] - oc["b"][ok]).max(1) + np.abs(gc["b"][ok] - oc["a"][ok]).max(1)
    assert (np.minimum(same, swap) < 1e-7).all(), _mismatch_report(e["label"][ok], np.minimum(same, swap) >= 1e-7)
    # The fit weight 1 - sqrt(msd / 3 lineRes) reads the mean squared distance to the line, which is exactly zero for every one of
    # these sets: both implementations compute it as rounding noise of either sign (~1e-17), so w comes out within ~1e-8 of 1, or
    # NaN from the square root of a negative, in the oracle as on the device.  Only that much is defined, and asserted.
    for w in (gc["w"][ok], oc["w"][ok]):
        assert (np.isnan(w) | (np.abs(w - 1) < 1e-6)).all()


@pytest.mark.gpu
def test_duplicated_map_points_register_like_the_oracle(gpu_api, oracle_mod):
    """A prior map with repeated points (overlapping tiles, an unfiltered export): 300 points of the tiny map, each the nearest
    map point of a scan point at the prior, appear five times.  Those scan points see five coincident neighbours, which the
    reference rejects (BAD_PCA_STRUCTURE); the registration must follow it trip for trip."""
    case = get_case("tiny")
    cfg = case["cfg"]
    m, s = case["map_xyzi"], case["scan_xyzi"]
    q = oracle_mod.transform_scan_numpy(s, case["pose_prior"])[:, :3]
    idx, _, found = oracle_mod.OracleMap(m).knn(q, 1, 0)
    dup = np.unique(idx[found, 0])
    dup = np.random.default_rng(5).choice(dup, size=300, replace=False)
    m2 = np.ascontiguousarray(np.concatenate([m] + [m[dup]] * 4, 0))
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=65536, plane_res=cfg["plane_res"])
    ctx.map_set_points(m2)
    r = ctx.register(s, case["pose_prior"], cfg["max_iterations"], 0)
    ctx.close()
    om = oracle_mod.OracleMap(m2)
    ro = om.register(s, case["pose_prior"], cfg["plane_res"], cfg["max_iterations"], 0, knn_mode=0)
    ro0 = oracle_mod.OracleMap(m).register(s, case["pose_prior"], cfg["plane_res"], cfg["max_iterations"], 0, knn_mode=0)
    assert ro.hist_reject_plane[3] >= ro0.hist_reject_plane[3] + 100                 # the duplicates are reached and rejected
    assert r.status == 0 and ro.status == 0
    n = ro.n_iterations
    assert r.n_iterations == n
    assert list(r.iter_n_surf[:n]) == list(ro.iter_n_surf[:n])
    assert list(r.hist_reject_plane) == list(ro.hist_reject_plane) and list(r.hist_obs) == list(ro.hist_obs)
    assert list(r.iter_lm_steps[:n]) == list(ro.iter_lm_steps[:n])
    assert list(r.iter_lm_successful[:n]) == list(ro.iter_lm_successful[:n])
    assert list(r.iter_lm_termination[:n]) == list(ro.iter_lm_termination[:n])
    assert np.allclose(r.iter_cost[:n], ro.iter_cost[:n], rtol=1e-9)
    pg, po = np.array(r.pose), np.array(ro.pose)
    assert np.abs(pg[:3] - po[:3]).max() <= 1e-4 and quat_angle(pg[3:], po[3:]) <= 1e-4
    cg, co = np.array(r.cov).reshape(6, 6), np.array(ro.cov).reshape(6, 6)
    assert np.abs(cg - co).max() <= 1e-6 * np.abs(co).max()

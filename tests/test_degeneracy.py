"""Degeneracy-aware registration (so_register_degeneracy*, DESIGN.md section 3).

The analysis is held against its numpy restatement (tests/degeneracy_numpy.py) at prescribed spectra; with nothing constrained the
registration is so_register's bit for bit; in a corridor without poles the flagged direction is the corridor axis and the
constrained solve does not slide along it."""
import numpy as np
import pytest

import degeneracy_numpy as DN
from conftest import get_case

_TIME = ("time_ms", "time_total_ms")


def _icp_bits(r):
    from superodom_b200 import api
    c = api.IcpResult.from_buffer_copy(bytes(r))
    for f in _TIME:
        setattr(c, f, 0.0)
    return bytes(c)


def _deg_bits(r):
    """the degeneracy report of a so_degeneracy_result (everything after icp)"""
    from superodom_b200 import api
    return bytes(r)[api.DegeneracyResult.iter_n_flag_pos.offset:]


# --------------------------------------------------------------------------------------------------------------- CPU
def test_restatement_information_is_the_inverse_covariance_block():
    """For an invertible H the Schur complements are the inverses of the covariance blocks EstimateRegistrationError analyses."""
    rng = np.random.default_rng(1)
    for _ in range(20):
        J = rng.standard_normal((40, 6)) * rng.uniform(0.1, 10.0, 6)
        H = J.T @ J
        a = DN.analysis(H, 0.1, 0.1)
        cov = np.linalg.inv(H)
        assert np.allclose(a["I_t"], np.linalg.inv(cov[:3, :3]), rtol=1e-9, atol=1e-9 * np.abs(H).max())
        assert np.allclose(a["I_r"], np.linalg.inv(cov[3:, 3:]), rtol=1e-9, atol=1e-9 * np.abs(H).max())
        w = np.linalg.eigvalsh(cov[:3, :3])
        assert np.isclose(np.sqrt(a["pos_info"][0] / a["pos_info"][2]), np.sqrt(w[0] / w[2]), rtol=1e-9)


def test_restatement_flags_and_columns():
    rng = np.random.default_rng(2)
    H = DN.with_spectrum(rng, [1e-3, 40.0, 90.0], [20.0, 50.0, 70.0], rot_t=np.eye(3), rot_r=np.eye(3))
    a = DN.analysis(H, 0.1, 0.1)
    assert a["flags_pos"] == 1 and a["flags_ori"] == 0 and a["B"].shape == (6, 5)
    assert abs(abs(a["pos_axes"][0][0]) - 1.0) < 1e-12
    assert np.allclose(a["B"].T @ a["B"], np.eye(5), atol=1e-12)
    assert np.allclose(a["B"][:, 0:2].T @ np.array([1.0, 0, 0, 0, 0, 0]), 0.0, atol=1e-12)
    assert DN.analysis(H, 0.1, 0.1, constrain=0)["B"].shape == (6, 6)
    Z = np.zeros((6, 6))
    z = DN.analysis(Z, 0.1, 0.1)
    assert z["flags_pos"] == 7 and z["flags_ori"] == 7 and z["B"].shape == (6, 0)


# --------------------------------------------------------------------------------------------------------------- GPU
def _spectra_cases():
    rng = np.random.default_rng(7)
    I3 = np.eye(3)
    cases = []
    # weak x translation, axis-aligned
    cases.append(("axis", DN.with_spectrum(rng, [2e-3, 40.0, 90.0], [20.0, 55.0, 70.0], rot_t=I3, rot_r=I3), 0.05, 0.05))
    # weak translation and weak rotation along rotated axes
    cases.append(("rotated", DN.with_spectrum(rng, [0.5, 300.0, 900.0], [0.02, 45.0, 80.0]), 0.1, 0.1))
    # weak translation coupled to rotation
    cases.append(("coupled", DN.with_spectrum(rng, [0.3, 120.0, 400.0], [30.0, 60.0, 150.0], coupling=20.0), 0.1, 0.1))
    # singular H_rr: the pseudo-inverse cuts a direction; I_r has a (numerically) zero eigenvalue
    cases.append(("singular_rr", DN.with_spectrum(rng, [5.0, 120.0, 400.0], [0.0, 60.0, 150.0], coupling=3.0), 0.05, 0.05))
    # exactly singular H: no information on x nor on yaw
    J = rng.standard_normal((30, 6))
    J[:, 0] = 0.0
    J[:, 5] = 0.0
    cases.append(("singular", J.T @ J, 0.05, 0.05))
    # columns 1e4 apart in scale
    D = np.diag([1e2, 1e2, 1e2, 1e-2, 1e-2, 1e-2])
    cases.append(("scaled", D @ DN.with_spectrum(rng, [0.01, 30.0, 70.0], [5.0, 40.0, 90.0], coupling=2.0) @ D, 0.05, 0.1))
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["axis", "rotated", "coupled", "singular_rr", "singular", "scaled"])
def test_analysis_matches_restatement(gpu_api, name):
    H, tp, tr = {c[0]: c[1:] for c in _spectra_cases()}[name]
    ref = DN.analysis(H, tp, tr)
    for info, thr in ((ref["pos_info"], tp), (ref["ori_info"], tr)):      # thresholds kept away from the ratios
        for v in info:
            ratio = np.sqrt(max(v, 0.0) / info[2]) if info[2] > 0 else 0.0
            assert ratio < 0.5 * thr or ratio > 2.0 * thr, (name, ratio, thr)
    ctx = gpu_api.Context(max_map_points=1 << 16, max_scan_points=4096)
    r = ctx.degeneracy_analysis(H, gpu_api.degeneracy(tp, tr))
    ctx.close()
    assert (r.flags_pos, r.flags_ori) == (ref["flags_pos"], ref["flags_ori"]), name
    assert ref["flags_pos"] | ref["flags_ori"], name                                   # every case flags something
    for dev_i, dev_a, ri, ra in ((r.pos_info, r.pos_axes, ref["pos_info"], ref["pos_axes"]), (r.ori_info, r.ori_axes, ref["ori_info"], ref["ori_axes"])):
        di, da = np.array(dev_i), np.array(dev_a).reshape(3, 3)
        scale = max(abs(ri[2]), 1e-300)
        assert np.abs(di - ri).max() <= 1e-8 * scale, (name, di, ri)
        for k in range(3):
            gap = min([abs(ri[k] - ri[j]) for j in range(3) if j != k])
            if gap > 1e-6 * scale:                                                         # a repeated eigenvalue has no unique axis
                assert min(np.abs(da[k] - ra[k]).max(), np.abs(da[k] + ra[k]).max()) <= 1e-8, (name, k, da[k], ra[k])


@pytest.mark.gpu
def test_argument_errors(gpu_api):
    c = get_case("tiny")
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=65536, plane_res=0.2)
    ctx.map_set_points(c["map_xyzi"])
    for d in (gpu_api.degeneracy(float("nan"), 0.1), gpu_api.degeneracy(-0.1, 0.1), gpu_api.degeneracy(0.1, 1.0),
              gpu_api.Degeneracy(0.1, 0.1, 2, 0)):
        with pytest.raises(gpu_api.SuperOdomError):
            ctx.register_degeneracy(c["scan_xyzi"], c["pose_prior"], d, 5)
        with pytest.raises(gpu_api.SuperOdomError):
            ctx.degeneracy_analysis(np.eye(6), d)
    ctx.close()


def _ctx(api, case, max_batch=1, edges=False):
    ctx = api.Context(max_map_points=max(1 << 20, 2 * len(case["map_xyzi"])), max_scan_points=262144, max_batch=max_batch,
                      plane_res=case["cfg"]["plane_res"] if "plane_res" in case["cfg"] else 0.2)
    ctx.map_set_points(case["map_xyzi"])
    if edges:
        ctx.map_set_edge_points(np.ascontiguousarray(case["map_xyzi"][::3]))
    return ctx


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["report_only", "zero_thresholds", "edges", "pose_prior"])
def test_nothing_constrained_is_so_register(gpu_api, mode):
    """constrain = 0 with any thresholds, or constrain = 1 with both thresholds 0: so_register's result bit for bit, and the
    analysis is still reported; repeated runs give the same bits."""
    case = get_case("cfg1", 0)
    ctx = _ctx(gpu_api, case, edges=mode == "edges")
    kw = dict(pose_prior=(0.5, (0.2, 0.1, 0.3))) if mode == "pose_prior" else {}
    edge = np.ascontiguousarray(case["scan_xyzi"][::9]) if mode == "edges" else None
    d = gpu_api.degeneracy(0.0, 0.0, True) if mode == "zero_thresholds" else gpu_api.degeneracy(0.6, 0.9, False)
    ref = ctx.register(case["scan_xyzi"], case["pose_prior"], 10, 2000, edge_xyzi=edge, **kw)
    runs = [ctx.register_degeneracy(case["scan_xyzi"], case["pose_prior"], d, 10, 2000, edge_xyzi=edge, **kw) for _ in range(2)]
    ctx.close()
    for r in runs:
        assert _icp_bits(r.icp) == _icp_bits(ref), mode
        assert r.pos_info[2] > 0 and r.ori_info[2] > 0
    assert _deg_bits(runs[0]) == _deg_bits(runs[1])
    if mode == "report_only":      # high thresholds flag directions; only reported
        assert sum(runs[0].iter_n_flag_pos[: ref.n_iterations]) + sum(runs[0].iter_n_flag_ori[: ref.n_iterations]) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name,cap", [("cfg1", 2000), ("cfg1", 0), ("cfg2", 0)])
def test_well_constrained_scans_are_so_register(gpu_api, name, cap):
    """Default-size thresholds on scans that constrain every direction: nothing is flagged, the result is so_register's."""
    case = get_case(name, 0)
    ctx = _ctx(gpu_api, case)
    ref = ctx.register(case["scan_xyzi"], case["pose_prior"], 10, cap)
    r = ctx.register_degeneracy(case["scan_xyzi"], case["pose_prior"], gpu_api.degeneracy(0.05, 0.05), 10, cap)
    ctx.close()
    assert ref.status == 0
    assert sum(r.iter_n_flag_pos) == 0 and sum(r.iter_n_flag_ori) == 0, (list(r.pos_info), list(r.ori_info))
    assert _icp_bits(r.icp) == _icp_bits(ref)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "edges", "pose_prior"])
def test_batch_equals_single_calls(gpu_api, mode):
    """A batch of four cfg2 scans, two of them constrained with a threshold that flags: every scan's pose, solve record and
    degeneracy report equal the single call's; with constrain = 0 the batch equals so_register_batch bit for bit."""
    edges = mode == "edges"
    pkw = dict(pose_prior=(0.5, (0.2, 0.1, 0.3))) if mode == "pose_prior" else {}
    cases = [get_case("cfg2", i) for i in range(4)]
    ctx = _ctx(gpu_api, cases[0], max_batch=4, edges=edges)
    scans = np.ascontiguousarray(np.concatenate([c["scan_xyzi"] for c in cases]))
    n = [len(c["scan_xyzi"]) for c in cases]
    poses = np.array([c["pose_prior"] for c in cases])
    ecl = [np.ascontiguousarray(c["scan_xyzi"][::11]) for c in cases] if edges else None
    ekw = dict(edges_xyzi=np.ascontiguousarray(np.concatenate(ecl)), n_edge=[len(e) for e in ecl]) if edges else {}
    ds = [gpu_api.degeneracy(0.9, 0.9, s % 2 == 0) for s in range(4)]
    res = ctx.register_batch_degeneracy(scans, n, poses, ds, 10, 0, skip_map_checks=True, **ekw, **pkw)
    for s in (0, 2):                                                  # the constrained scans do run the reduced solve
        assert sum(res[s].iter_n_flag_pos) + sum(res[s].iter_n_flag_ori) > 0, s
    for s in range(4):
        single = ctx.register_degeneracy(cases[s]["scan_xyzi"], poses[s], ds[s], 10, 0, edge_xyzi=ecl[s] if edges else None,
                                         skip_map_checks=True, **pkw)
        a, b = res[s], single
        assert bytes(a.icp.pose_opt) == bytes(b.icp.pose_opt) and bytes(a.icp.cov) == bytes(b.icp.cov), s
        assert bytes(a.icp.iter_lm_steps) == bytes(b.icp.iter_lm_steps) and bytes(a.icp.iter_cost) == bytes(b.icp.iter_cost), s
        assert _deg_bits(a) == _deg_bits(b), s
    off = [gpu_api.degeneracy(0.9, 0.9, False)] * 4
    r0 = ctx.register_batch_degeneracy(scans, n, poses, off, 10, 0, skip_map_checks=True, **ekw, **pkw)
    if edges:
        rb = ctx.register_batch_edges(scans, n, ekw["edges_xyzi"], ekw["n_edge"], poses, 10, 0, skip_map_checks=True)
    else:
        rb = ctx.register_batch(scans, n, poses, 10, 0, skip_map_checks=True, **pkw)
    ctx.close()
    for s in range(4):
        assert _icp_bits(r0[s].icp) == _icp_bits(rb[s]), s


@pytest.mark.gpu
def test_registered_scan_inserts_after_it(gpu_api):
    case = get_case("cfg1", 0)
    maps = []
    for deg in (False, True):
        ctx = _ctx(gpu_api, case)
        if deg:
            r = ctx.register_degeneracy(case["scan_xyzi"], case["pose_prior"], gpu_api.degeneracy(0.3, 0.3, False), 10, 2000).icp
        else:
            r = ctx.register(case["scan_xyzi"], case["pose_prior"], 10, 2000)
        ctx.map_add_registered_scan(r.pose)
        maps.append(ctx.map_download())
        ctx.close()
    assert len(maps[0]) > len(case["map_xyzi"]) and maps[0].tobytes() == maps[1].tobytes()


# --------------------------------------------------------------------------------------------------------------- corridor
def _corridor(api, n_scans, offset):
    """The corridor WITHOUT poles as a map, and seeded OS1-128 scans in it: (ctx, [(scan, pose_true, prior, yaw)]), the priors
    offset by `offset` on top of the usual perturbation."""
    from superodom_b200 import synth
    sc = synth.make_corridor_scene(poles=False)
    raw = synth.sample_surfaces(sc, 0.2)
    surf = synth.voxel_filter_blocks(np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1), 0.2)
    ctx = api.Context(max_map_points=max(1 << 20, 2 * len(surf)), max_scan_points=262144, plane_res=0.2)
    ctx.map_set_points(surf)
    rng = np.random.default_rng(9100)
    scans = []
    for s in range(n_scans):
        yaw = rng.uniform(-0.2, 0.2)
        T = np.array([rng.uniform(-20, 20), rng.uniform(-0.8, 0.8), rng.uniform(-0.3, 0.3), 0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)])
        rec = synth.make_ring_scan(sc, "os1_128", T, 9200 + s)
        scan = np.ascontiguousarray(np.concatenate([rec[:, :3], rec[:, 5:6]], 1))
        prior = synth.perturb_pose(T, 9300 + s)
        prior[:3] += np.asarray(offset)
        scans.append((scan, T, prior, yaw))
    return ctx, scans


def corridor_rows(api, n_scans=6, offset=(0.15, 0.0, 0.0), thr=0.3, log=None):
    """Seeded OS1-128 scans in the corridor WITHOUT poles (nothing constrains x), priors offset by `offset` plus the usual
    perturbation, registered by so_register and by so_register_degeneracy (constrain = 1).  -> one dict per scan."""
    ctx, scans = _corridor(api, n_scans, offset)
    rows = []
    for scan, T, prior, yaw in scans:
        ru = ctx.register(scan, prior, 20, 0)
        rc = ctx.register_degeneracy(scan, prior, api.degeneracy(thr, thr), 20, 0)
        ax = np.array(rc.pos_axes[0:3])
        def yawerr(p):
            return abs(2 * np.arctan2(p[5], p[6]) - yaw)
        row = dict(status=(ru.status, rc.icp.status), flags=(rc.flags_pos, rc.flags_ori),
                   ratio_x=float(np.sqrt(max(rc.pos_info[0], 0.0) / rc.pos_info[2])),
                   axis_deg=float(np.degrees(np.arccos(min(1.0, abs(ax[0]))))),
                   move_u=float(abs(np.dot(np.array(ru.pose_opt[:3]) - prior[:3], ax))),
                   move_c=float(abs(np.dot(np.array(rc.icp.pose_opt[:3]) - prior[:3], ax))),
                   err_u=np.abs(np.array(ru.pose[:3]) - T[:3]).tolist(), err_c=np.abs(np.array(rc.icp.pose[:3]) - T[:3]).tolist(),
                   yaw_u=float(yawerr(ru.pose)), yaw_c=float(yawerr(rc.icp.pose)),
                   n_flag=(list(rc.iter_n_flag_pos[: rc.icp.n_iterations]), list(rc.iter_n_flag_ori[: rc.icp.n_iterations])))
        if log:
            log(row)
        rows.append(row)
    ctx.close()
    return rows


@pytest.mark.gpu
def test_corridor_without_poles_is_held_along_its_axis(gpu_api):
    """Measured on six seeded scans (H100 80GB HBM3, 700 W power limit): sqrt(i_x / i_max) of I_t is 0.11-0.20, so threshold 0.3 flags x; the flagged
    axis is 0.1-3.0 degrees off x; along it the constrained pose moves 0.01-0.24 mm from the prior, the unconstrained one 1.3-11 mm;
    y / z errors grow by at most 7 mm and yaw by 3e-5 rad."""
    rows = corridor_rows(gpu_api, log=print)
    for r in rows:
        assert r["status"] == (0, 0), r
        assert r["flags"][0] & 1, r                                  # the weakest translation direction is flagged ...
        assert r["axis_deg"] < 3.0, r                                # ... and it is the corridor axis
        assert r["move_c"] < 5e-4 < r["move_u"], r                   # the constrained solve stays put along it, the ambient one slides
        for k in (1, 2):                                             # across the corridor and vertically no worse
            assert r["err_c"][k] <= r["err_u"][k] + 0.01, r
        assert r["yaw_c"] <= r["yaw_u"] + 2e-3, r


# --------------------------------------------------------------------------------------------------------------- reduced solve
def test_reduced_solve_restatement_reduces_to_the_ambient_one():
    """B = I is the ambient solve exactly; a B without the x column never moves x."""
    import test_ceres_restatement as CR
    rng = np.random.default_rng(11)
    a2 = _a2()
    for k in range(20):
        truth, P, Nrm, D, W = CR._random_problem(rng, int(rng.integers(40, 400)))
        prob = CR.Problem(P, Nrm, D, W, a2)
        x0 = CR._plus(truth, np.concatenate([rng.uniform(-1, 1, 3) * 0.3, rng.uniform(-1, 1, 3) * 0.05]))
        a = CR.solve(prob, x0)
        b = DN.solve_reduced(prob, x0, np.eye(6))
        assert np.array_equal(a[0], b[0]) and a[1:] == b[1:], k
        c = DN.solve_reduced(prob, x0, np.eye(6)[:, 1:])
        assert c[0][0] == x0[0] and c[1] >= 1, k


def _a2(plane_res=0.2):
    a = float(np.sqrt(np.float32(3 * np.float32(plane_res))))
    return a * a


@pytest.mark.gpu
@pytest.mark.parametrize("scene,offset,thr", [("corridor", (0.15, 0.0, 0.0), 0.3), ("corridor", (-0.1, 0.05, 0.03), 0.3),
                                              ("cfg1", None, 0.9)])
def test_icp_loop_matches_numpy(gpu_api, scene, offset, thr):
    """The whole degeneracy-aware registration against the numpy ICP loop on the device's own search and fit: per ICP iteration the
    accepted correspondences, LM steps, successful steps, termination and flagged directions are identical, and the final pose
    agrees within 1e-8."""
    if scene == "corridor":
        ctx, scans = _corridor(gpu_api, 1, offset)
        scan, _, prior, _ = scans[0]
        iters, mf = 20, 0
    else:
        case = get_case(scene, 0)
        ctx = _ctx(gpu_api, case)
        scan, prior, iters, mf = case["scan_xyzi"], case["pose_prior"], 5, 2000
    r = ctx.register_degeneracy(scan, prior, gpu_api.degeneracy(thr, thr), iters, mf, skip_map_checks=True)
    x, its = DN.register(ctx, scan, prior, thr, thr, iters, mf, _a2())
    ctx.close()
    got = [(r.icp.iter_n_surf[k], r.icp.iter_lm_steps[k], r.icp.iter_lm_successful[k], r.icp.iter_lm_termination[k],
            r.iter_n_flag_pos[k], r.iter_n_flag_ori[k]) for k in range(r.icp.n_iterations)]
    print(scene, offset, got)
    assert r.icp.status == 0 and got == its
    assert sum(k[4] + k[5] for k in its) > 0                         # the reduced solve ran
    assert np.abs(np.array(r.icp.pose_opt) - x).max() < 1e-8

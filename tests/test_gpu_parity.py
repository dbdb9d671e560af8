"""GPU parity tests: the sm_90a path, called through the C ABI, against the CPU oracle on identical inputs.

Bars (task section 3): bit-exact for integer / index work (neighbour ids, float d2, status codes, histograms,
iteration counts); FP64 quantities within the stated tolerances (normal equations 1e-10 relative, pose 1e-4 m /
1e-4 rad per BASELINE.json north_star -- observed ~1e-15)."""
import ctypes as C

import numpy as np
import pytest

import ref_octree_golden
import solve_numerics_ref
from conftest import get_case, quat_angle

pytestmark = pytest.mark.gpu

POSE_TOL_M = 1e-4       # north_star
POSE_TOL_RAD = 1e-4


def _ctx(api, case, **kw):
    ctx = api.Context(max_map_points=max(1 << 20, len(case["map_xyzi"]) + 1024), max_scan_points=262144,
                      plane_res=case["cfg"]["plane_res"], **kw)
    ctx.map_set_points(case["map_xyzi"])
    return ctx


def _gi(idx):
    g = idx.astype(np.int64)
    g[idx == 0xFFFFFFFF] = -1
    return g


def _assert_pose_close(pg, po, tol_m=POSE_TOL_M, tol_r=POSE_TOL_RAD):
    assert np.abs(pg[:3] - po[:3]).max() <= tol_m, (pg, po)
    assert quat_angle(pg[3:], po[3:]) <= tol_r, (pg, po)


def _cell_faces(plane_res, lo, hi):
    """float32 coordinates in [lo, hi) of the k-NN grid's cell faces (cell edge 50 / nb, nb = min(192, floor(100 / sqrt(3 planeRes)))
    cells per 50 m block, DESIGN section 2), with the float32 neighbours on either side of each."""
    nb = min(192, int(100.0 / np.sqrt(3.0 * np.float64(np.float32(plane_res)))))
    j = np.arange(int(np.floor((lo + 25.0) * nb / 50.0)), int(np.ceil((hi + 25.0) * nb / 50.0)) + 1)
    f = (-25.0 + j * (50.0 / nb)).astype(np.float32)
    f = f[(f >= lo) & (f < hi)]
    return f, np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))


def _knn_case(name):
    """(map_xyzi, plane_res, queries) for test_knn_bit_exact.  lattice: voxel centres at planeRes spacing, a second lattice
    whose planes lie on the grid's cell faces (and one float32 step either side), exact distance ties everywhere; queries on lattice
    points, midpoints, faces and at random.  dense: clusters of 6-64 coincident or nearly coincident points, so that far more than
    the 24 candidates the search buffers fall inside its bound."""
    rng = np.random.default_rng(0)
    if name not in ("lattice", "dense"):
        case = get_case(name)
        base = case["map_xyzi"][::7, :3]
        q = base + rng.normal(0, 0.12, size=base.shape).astype(np.float32)
        q = np.concatenate([q, rng.uniform(-30, 30, size=(500, 3)).astype(np.float32) + q.mean(0)])     # incl. far-away queries
        return case["map_xyzi"], case["cfg"]["plane_res"], q
    pr = 0.2
    if name == "lattice":
        g = (np.arange(-30, 30) + 0.5) * pr
        a = np.stack(np.meshgrid(g, g, (np.arange(-3, 3) + 0.5) * pr, indexing="ij"), -1).reshape(-1, 3)
        fx, fxm, fxp = _cell_faces(pr, 8.0, 12.0)
        fz, fzm, fzp = _cell_faces(pr, -1.0, 1.0)
        xs = np.concatenate([fx, fxm[::3], fxp[1::3]])
        zs = np.concatenate([fz, fzm[::2], fzp[1::2]])
        b = np.stack(np.meshgrid(xs, np.float32(fx - 20.0), zs, indexing="ij"), -1).reshape(-1, 3)
        pts = np.concatenate([a.astype(np.float32), b.astype(np.float32)])
        q = np.concatenate([pts[rng.choice(len(pts), 3000, replace=False)],
                            (pts[rng.choice(len(a), 2000)] + np.float32(pr / 2) * rng.integers(0, 2, size=(2000, 3))).astype(np.float32),
                            np.stack([rng.choice(fx, 2000), rng.uniform(-6, 6, 2000), rng.choice(fz, 2000)], 1).astype(np.float32),
                            np.stack([rng.uniform(8, 12, 2000), rng.choice(np.float32(fx - 20.0), 2000), rng.uniform(-1, 1, 2000)], 1).astype(np.float32),
                            rng.uniform(-7, 13, size=(2000, 3)).astype(np.float32) * np.float32([1, 1, 0.2])])
    else:
        cen = rng.uniform(-5, 5, size=(600, 3)) * [1, 1, 0.3]
        pts = []
        for i, c in enumerate(cen):
            n = int(rng.integers(6, 65))
            jit = [0.0, 1e-6, 1e-4, 1e-2][i % 4]
            pts.append(c + rng.normal(0, jit, size=(n, 3)) if jit else np.repeat(c[None], n, 0))
        pts = np.concatenate(pts).astype(np.float32)
        q = np.concatenate([cen.astype(np.float32), (cen + rng.normal(0, 0.1, size=cen.shape)).astype(np.float32),
                            ((cen[:-1] + cen[1:]) / 2).astype(np.float32), rng.uniform(-6, 6, size=(2000, 3)).astype(np.float32) * np.float32([1, 1, 0.3])])
    xyzi = np.concatenate([pts, np.ones((len(pts), 1), np.float32)], 1)
    return xyzi, pr, q


@pytest.mark.parametrize("name", ["tiny", "cfg1", "hall", "lattice", "dense"])
def test_knn_bit_exact(gpu_api, oracle_mod, name):
    map_xyzi, pr, q = _knn_case(name)
    ctx = gpu_api.Context(max_map_points=max(1 << 20, len(map_xyzi) + 1024), max_scan_points=262144, plane_res=pr)
    ctx.map_set_points(map_xyzi)
    om = oracle_mod.OracleMap(map_xyzi)
    gi, gd = ctx.knn(q, 5, 0.0)                           # exact, unbounded
    oi, od, of = om.knn(q, 5, 0)
    assert np.array_equal(_gi(gi)[of], oi[of]) and np.array_equal(gd[of], od[of])
    assert (gi[~of] == 0xFFFFFFFF).all()
    bound = np.float32(3 * np.float32(pr))
    gi, gd = ctx.knn(q, 5, float(bound))                  # radius-bounded: same neighbours up to the bound
    keep = od <= bound
    assert np.array_equal(_gi(gi)[keep & of[:, None]], oi[keep & of[:, None]])
    assert (gi[~keep | ~of[:, None]] == 0xFFFFFFFF).all()
    import torch
    qs = q if name in ("lattice", "dense") else q[:2000]
    for k in range(1, 9):
        gi, gd = ctx.knn(qs, k, 0.0)
        oi, od, of = om.knn(qs, k, 0)
        assert np.array_equal(_gi(gi)[of], oi[of]) and np.array_equal(gd[of], od[of]), k
        if name in ("lattice", "dense"):
            assert of.all()
            gi, gd = ctx.knn(qs, k, float(bound))
            keep = od <= bound
            assert np.array_equal(_gi(gi)[keep], oi[keep]) and np.array_equal(gd[keep], od[keep]) and (gi[~keep] == 0xFFFFFFFF).all(), k
        # so_knn_device (device-resident queries and results) returns the same bits as so_knn
        for b in (0.0, float(bound)):
            hi, hd = ctx.knn(qs, k, b)
            dq = torch.from_numpy(np.concatenate([qs, np.ones((len(qs), 1), np.float32)], 1)).cuda()      # float4 queries
            di = torch.empty((len(qs), k), dtype=torch.int32, device="cuda")
            dd = torch.empty((len(qs), k), dtype=torch.float32, device="cuda")
            ctx.knn_device(dq.data_ptr(), len(qs), k, b, di.data_ptr(), dd.data_ptr())
            torch.cuda.synchronize()
            assert np.array_equal(di.cpu().numpy().view(np.uint32), hi) and np.array_equal(dd.cpu().numpy(), hd), (k, b)
    if name == "dense":                # the search buffers 24 candidates inside its bound and inserts the rest directly: reached here
        _, od5, _ = om.knn(q[:600], 5, 0)
        inside = ((map_xyzi[None, :, :3].astype(np.float64) - q[:600, None, :]) ** 2).sum(-1) <= od5[:, 4:5] * 1.001
        assert (inside.sum(1) > 24).sum() > 100
    if name == "hall":                                    # reference's own octree (verbatim, stored output) agrees here
        ri, rd = ref_octree_golden.knn(om, "hall", q[:-500])
        gi, gd = ctx.knn(q[:-500], 5, 0.0)
        assert np.array_equal(_gi(gi), ri) and np.array_equal(gd, rd)
    ctx.close()


@pytest.mark.parametrize("name,cap", [("tiny", 0), ("cfg1", 2000), ("cfg1", 0), ("hall", 0)])
def test_correspondences_and_normal_equations(gpu_api, oracle_mod, name, cap):
    case = get_case(name)
    pr = case["cfg"]["plane_res"]
    ctx = _ctx(gpu_api, case)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    gc, gho, ghr = ctx.correspond(case["scan_xyzi"], case["pose_prior"], cap)
    oc, oho, ohr = om.correspond(case["scan_xyzi"], case["pose_prior"], pr, cap, 0)
    ost = oc["status"].astype(np.int64)
    ost[ost < 0] = 255
    assert np.array_equal(gc["status"].astype(np.int64), ost)                  # every accept/reject gate agrees
    assert np.array_equal(gho, oho) and np.array_equal(ghr, ohr)
    ok = ost == 0
    assert ok.sum() > 100
    searched = (ost != 255) & (ost != 1)
    found5 = searched & (ost != 2)
    assert np.array_equal(gc["nn"][found5].astype(np.int64), oc["nn"][found5])
    assert np.array_equal(gc["nn_d2"][found5], oc["nn_d2"][found5])
    assert np.array_equal(gc["obs"][ok], oc["obs"][ok].astype(np.uint8))
    assert np.allclose(gc["n"][ok], oc["n"][ok], rtol=0, atol=1e-8)
    assert np.allclose(gc["d"][ok], oc["d"][ok], rtol=1e-10, atol=0)
    assert np.allclose(gc["w"][ok], oc["w"][ok], rtol=1e-10, atol=0)
    assert (gc["w"][~ok] == 0).all() and (gc["n"][~ok] == 0).all()
    for pose in (case["pose_prior"], case["pose_true"]):
        H, g, cost = ctx.evaluate(pose)
        oH, og, ocost, nok = oracle_mod.evaluate(oc, pose, pr)
        assert np.abs(H - oH).max() <= 1e-10 * np.abs(oH).max()
        assert np.abs(g - og).max() <= 1e-10 * max(np.abs(og).max(), 1e-3 * np.abs(oH).max())
        assert abs(cost - ocost) <= 1e-10 * ocost
    ctx.close()


@pytest.mark.parametrize("name,cap", [("tiny", 0), ("cfg1", 2000), ("cfg1", 0), ("hall", 0)])
def test_register_pose_parity(gpu_api, oracle_mod, name, cap):
    case = get_case(name)
    cfg = case["cfg"]
    ctx = _ctx(gpu_api, case)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    r = ctx.register(case["scan_xyzi"], case["pose_prior"], cfg["max_iterations"], cap)
    ro = om.register(case["scan_xyzi"], case["pose_prior"], cfg["plane_res"], cfg["max_iterations"], cap, knn_mode=0)
    assert r.status == 0 and ro.status == 0
    _assert_pose_close(np.array(r.pose), np.array(ro.pose))
    _assert_pose_close(np.array(r.pose_opt), np.array(ro.pose_opt))
    n = ro.n_iterations
    assert r.n_iterations == n                                                    # same ICP trip count
    assert list(r.iter_n_surf[:n]) == list(ro.iter_n_surf[:n])
    assert list(r.iter_lm_steps[:n]) == list(ro.iter_lm_steps[:n])              # same Ceres control flow
    assert list(r.iter_lm_successful[:n]) == list(ro.iter_lm_successful[:n])
    assert list(r.iter_lm_termination[:n]) == list(ro.iter_lm_termination[:n])
    assert np.allclose(r.iter_cost[:n], ro.iter_cost[:n], rtol=1e-9)
    assert np.allclose(r.iter_dtrans[:n], ro.iter_dtrans[:n], atol=1e-9) and np.allclose(r.iter_drot[:n], ro.iter_drot[:n], atol=1e-9)
    assert list(r.hist_obs) == list(ro.hist_obs) and list(r.hist_reject_plane) == list(ro.hist_reject_plane)
    cg, co = np.array(r.cov).reshape(6, 6), np.array(ro.cov).reshape(6, 6)
    assert np.abs(cg - co).max() <= 1e-6 * np.abs(co).max()                      # SURVEY 8d: ||dC||/||C|| <= 1e-6
    for f in ("pos_err", "pos_inv_cond", "ori_err_deg", "ori_inv_cond", "total_translation", "total_rotation"):
        assert abs(getattr(r, f) - getattr(ro, f)) <= 1e-6 * abs(getattr(ro, f)) + 1e-12, f
    assert abs(abs(np.dot(r.pos_dir, ro.pos_dir)) - 1) < 1e-6 and abs(abs(np.dot(r.ori_dir, ro.ori_dir)) - 1) < 1e-6
    assert r.map_surf_5x5 == ro.map_surf_5x5 and list(r.pos_in_localmap) == list(ro.pos_in_localmap)
    # truth is recovered (the oracle is, too) and the run is bit-reproducible
    assert np.linalg.norm(np.array(r.pose)[:3] - case["pose_true"][:3]) < 0.02
    r2 = ctx.register(case["scan_xyzi"], case["pose_prior"], cfg["max_iterations"], cap)
    assert np.array_equal(np.array(r.pose), np.array(r2.pose)) and np.array_equal(np.array(r.cov), np.array(r2.cov))
    if name == "hall":
        # the reference's own (verbatim) octree in the loop (stored result): same pose, because on this layout the octree is exact
        g = ref_octree_golden.load()
        _assert_pose_close(np.array(r.pose), g["hall.pose"])
        assert int(g["hall.n_iterations"]) == r.n_iterations
    ctx.close()


def test_golden_fixture_through_the_abi(gpu_api):
    import os
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_case.npz"))
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=65536, plane_res=float(G["plane_res"]))
    ctx.map_set_points(G["map_xyzi"])
    gc, gho, ghr = ctx.correspond(G["scan_xyzi"], G["pose_prior"], 0)
    assert np.array_equal(gc["status"].astype(np.int32), G["status"])
    ok = G["status"] == 0
    assert np.array_equal(gc["nn"][ok].astype(np.int64), G["nn"][ok])
    assert np.array_equal(gho, G["hist_obs"]) and np.array_equal(ghr, G["hist_rej"])
    H, g, cost = ctx.evaluate(G["pose_prior"])
    assert np.allclose(H, G["H"], rtol=1e-9) and abs(cost - G["cost"]) < 1e-9 * G["cost"]
    r = ctx.register(G["scan_xyzi"], G["pose_prior"], int(G["max_iterations"]), 0)
    _assert_pose_close(np.array(r.pose), G["pose_exact"])
    assert r.n_iterations == int(G["n_iterations_exact"])
    ctx.close()


def test_pcl_point_layout_and_stride(gpu_api):
    """pcl::PointXYZI layout: 32-byte stride, intensity at byte 16 -- what the C++ shim passes (points.data())."""
    case = get_case("tiny")
    ctx = _ctx(gpu_api, case)
    s = case["scan_xyzi"]
    r0 = ctx.register(s, case["pose_prior"], 5)
    pcl = np.zeros((len(s), 8), np.float32)
    pcl[:, :3] = s[:, :3]
    pcl[:, 3] = 1.0
    pcl[:, 4] = s[:, 3]
    o = ctx._opts(5)
    r1 = gpu_api.IcpResult()
    pose = np.ascontiguousarray(case["pose_prior"])
    rc = ctx.L.so_register(ctx.h, pcl.ctypes.data_as(C.c_void_p), len(s), None, 0, 32, 16, pose.ctypes.data_as(C.c_void_p), C.byref(o), C.byref(r1))
    assert rc == 0 and np.array_equal(np.array(r0.pose), np.array(r1.pose))
    ctx.close()


def test_soft_statuses_and_edge_cases(gpu_api):
    case = get_case("tiny")
    api = gpu_api
    # map with too few points: hasEnoughFeatures false -> status 1, pose = prior (LidarSlam.cpp:113-116)
    ctx = api.Context(max_map_points=1 << 16, max_scan_points=65536, plane_res=0.2)
    ctx.map_set_points(case["map_xyzi"][:40])
    r = ctx.register(case["scan_xyzi"], case["pose_prior"], 5)
    assert r.status == 1 and np.array_equal(np.array(r.pose), case["pose_prior"])
    # empty map
    ctx.map_set_points(np.zeros((0, 4), np.float32))
    r = ctx.register(case["scan_xyzi"], case["pose_prior"], 5)
    assert r.status == 1
    ctx.close()
    ctx = _ctx(api, case)
    # scan nowhere near the map -> every point rejected -> status 2, pose = prior
    far = case["scan_xyzi"].copy()
    far[:, :3] += 400.0
    r = ctx.register(far, case["pose_prior"], 5, skip_map_checks=True)
    assert r.status == 2 and np.allclose(np.array(r.pose_opt), case["pose_prior"])
    assert r.hist_reject_plane[1] + r.hist_reject_plane[2] == len(far)
    # empty scan
    r = ctx.register(np.zeros((0, 4), np.float32), case["pose_prior"], 5)
    assert r.status == 2
    # ragged tiny scans (1, 31, 257 points) run and match the full-scan machinery
    for n in (1, 31, 257):
        r = ctx.register(case["scan_xyzi"][:n], case["pose_true"], 5)
        assert r.status in (0, 2)
    # argument errors are reported, not thrown
    assert ctx.L.so_register(ctx.h, None, 10, None, 0, 16, 12, None, None, None) < 0
    assert b"bad args" in ctx.L.so_last_error()
    with pytest.raises(api.SuperOdomError):
        ctx.register(np.zeros((300000, 4), np.float32), case["pose_prior"], 5)       # over max_scan_points
    ctx.close()


def test_block_boundary_restriction(gpu_api, oracle_mod):
    """Neighbours come only from the query's own 50 m block (LocalMap.h:488-525): straddle x = 25."""
    rng = np.random.default_rng(4)
    n = 60000
    p = np.stack([rng.uniform(20, 30, n), rng.uniform(-5, 5, n), rng.uniform(-1, 1, n) * 0.02 - 1.5], 1).astype(np.float32)
    xyzi = np.concatenate([p, np.ones((n, 1), np.float32)], 1)
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=65536, plane_res=0.2)
    ctx.map_set_points(xyzi)
    om = oracle_mod.OracleMap(xyzi)
    q = np.stack([rng.uniform(24.5, 25.5, 4000), rng.uniform(-4, 4, 4000), np.full(4000, -1.5)], 1).astype(np.float32)
    q[:8, 0] = np.float32([25.0, 24.999998, 25.000002, 24.99, 25.01, 25.0, 25.0, 25.0])
    gi, gd = ctx.knn(q, 5, 0.0)
    oi, od, of = om.knn(q, 5, 0)
    assert np.array_equal(_gi(gi), oi) and np.array_equal(gd, od)
    side_q = q[:, 0].astype(np.float64) + 25.0 >= 50.0
    side_n = p[gi.astype(np.int64), 0].astype(np.float64) + 25.0 >= 50.0
    assert (side_n == side_q[:, None]).all()
    ctx.close()


def test_map_shift_and_counts(gpu_api, oracle_mod):
    case = get_case("tiny")
    ctx = _ctx(gpu_api, case)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    assert list(ctx.map_origin()) == [10, 10, 5]
    for t in ([0, 0, 0], [-400.0, 0, 0], [30.0, 460.0, 0.0]):
        assert list(ctx.map_shift(t)) == list(om.shift(t))
        assert list(ctx.map_origin()) == list(om.origin())
        ijk = ctx.map_shift(t)
        assert ctx.map_counts_5x5(ijk) == om.counts_5x5(ijk)
    assert ctx.map_size() == len(case["map_xyzi"])
    r = ctx.register(case["scan_xyzi"], case["pose_prior"], 5)        # still registers after the rolls
    ro = om.register(case["scan_xyzi"], case["pose_prior"], 0.2, 5)
    _assert_pose_close(np.array(r.pose), np.array(ro.pose))
    ijk = ctx.map_shift([900.0, 0, 0])                                # far away: the map's block rolls off the grid
    assert ctx.map_size() == 0 and list(ijk) == list(om.shift([900.0, 0, 0]))
    back = ctx.map_download(0)
    assert len(back) == 0
    ctx.close()


def test_batch_equals_singles(gpu_api):
    case0 = get_case("tiny", 0)
    scans, poses = [], []
    for i in range(5):
        c = get_case("tiny", i)
        s = c["scan_xyzi"][: len(c["scan_xyzi"]) - 37 * i]           # ragged lengths
        scans.append(s)
        poses.append(c["pose_prior"])
    ctx = _ctx(gpu_api, case0, max_batch=8)
    singles = [ctx.register(s, p, 5, skip_map_checks=True) for s, p in zip(scans, poses)]
    flat = np.ascontiguousarray(np.concatenate(scans, 0))
    res = ctx.register_batch(flat, [len(s) for s in scans], np.stack(poses), 5, skip_map_checks=True)
    for a, b in zip(singles, res):
        assert np.array_equal(np.array(a.pose), np.array(b.pose)) and a.n_iterations == b.n_iterations
        assert np.array_equal(np.array(a.cov), np.array(b.cov))
    import torch
    d = torch.from_numpy(flat).cuda()
    res2 = ctx.register_batch_device(d.data_ptr(), [len(s) for s in scans], np.stack(poses), 5, skip_map_checks=True)
    for a, b in zip(singles, res2):
        assert np.array_equal(np.array(a.pose), np.array(b.pose))
    ctx.close()


# Scan sizes of the boundary-size batch: 1 / 4 / 16 points per evaluation thread switch at 4 096 / 65 536 points, a TMA ring stage
# is refilled above 4 096 points per CTA, and a scan whose first point sits at an odd offset takes the generic-load fallback.
# Eighteen scans form two chunks of nine, so both chunks evaluate through the TMA ring, while a single registration takes the fused
# plain-load kernel.  Offsets alternate in parity; 65 536 and 100 001 sit behind odd-sized scans at odd offsets; one scan is empty.
_BATCH_SIZES = [1, 4097, 256, 65537, 255, 4096, 257, 65536, 0, 4095, 3, 100001, 2, 65535, 1000, 7, 131072, 511]


def _result_bits(r):
    """pose, pose_opt, cov, status, iteration count, the per-iteration arrays and the histograms as raw bytes (NaN-safe)"""
    return np.array(list(r.pose) + list(r.pose_opt) + list(r.cov) + [r.status, r.n_iterations] + list(r.iter_n_surf) + list(r.iter_dtrans)
                    + list(r.iter_drot) + list(r.iter_lm_steps) + list(r.iter_lm_successful) + list(r.iter_lm_termination)
                    + list(r.iter_cost) + list(r.hist_obs) + list(r.hist_reject_plane), np.float64).tobytes()


def test_batch_equals_singles_at_boundary_sizes(gpu_api, oracle_mod, monkeypatch):
    """test_batch_equals_singles at every evaluation granularity: 18 scans cut from the cfg2 scan (_BATCH_SIZES), each bit-equal to
    its single so_register in every recorded field -- host batch, device batch, repeated calls, a fresh context, one stream."""
    case0 = get_case("cfg2")
    full = case0["scan_xyzi"]
    scans, poses = [], []
    for i, n in enumerate(_BATCH_SIZES):
        start = (i * 7919) % (len(full) - n + 1)
        scans.append(full[start:start + n])
        poses.append(case0["pose_prior"])
    offs = np.cumsum([0] + _BATCH_SIZES[:-1])
    big = np.array(_BATCH_SIZES) > 4096
    assert (offs[big] % 2 == 1).any() and (offs[big] % 2 == 0).any()
    ctx = _ctx(gpu_api, case0, max_batch=len(scans))
    singles = [ctx.register(s, p, 5, skip_map_checks=True) for s, p in zip(scans, poses)]
    want = [_result_bits(a) for a in singles]
    assert sum(a.status == 0 for a in singles) >= 8
    flat = np.ascontiguousarray(np.concatenate(scans, 0))
    res = ctx.register_batch(flat, [len(s) for s in scans], np.stack(poses), 5, skip_map_checks=True)
    for i, b in enumerate(res):
        assert _result_bits(b) == want[i], ("host batch", i, _BATCH_SIZES[i])
    import torch
    d = torch.from_numpy(flat).cuda()
    res2 = ctx.register_batch_device(d.data_ptr(), [len(s) for s in scans], np.stack(poses), 5, skip_map_checks=True)
    for i, b in enumerate(res2):
        assert _result_bits(b) == want[i], ("device batch", i, _BATCH_SIZES[i])
    for rep in range(2):
        res3 = ctx.register_batch(flat, [len(s) for s in scans], np.stack(poses), 5, skip_map_checks=True)
        assert [_result_bits(b) for b in res3] == want, ("repeat", rep)
    # the single-scan normal equations at the ring's boundary sizes against the oracle
    om = oracle_mod.OracleMap(case0["map_xyzi"], ref_octree=False)
    pr = case0["cfg"]["plane_res"]
    for i in (_BATCH_SIZES.index(4097), _BATCH_SIZES.index(65537), _BATCH_SIZES.index(131072)):
        ctx.correspond(scans[i], poses[i], 0)
        H, g, cost = ctx.evaluate(poses[i])
        oc, _, _ = om.correspond(scans[i], poses[i], pr, 0, 0, n_threads=8)
        oH, og, ocost, _ = oracle_mod.evaluate(oc, poses[i], pr)
        assert np.abs(H - oH).max() <= 1e-10 * np.abs(oH).max(), _BATCH_SIZES[i]
        assert np.abs(g - og).max() <= 1e-10 * max(np.abs(og).max(), 1e-3 * np.abs(oH).max()), _BATCH_SIZES[i]
        assert abs(cost - ocost) <= 1e-10 * ocost, _BATCH_SIZES[i]
    ctx.close()
    for env in (None, "SO_SINGLE_STREAM"):              # a fresh context, then a fresh one scheduling both chunks on one stream
        if env:
            monkeypatch.setenv(env, "1")
        ctx = _ctx(gpu_api, case0, max_batch=len(scans))
        res4 = ctx.register_batch(flat, [len(s) for s in scans], np.stack(poses), 5, skip_map_checks=True)
        ctx.close()
        assert [_result_bits(b) for b in res4] == want, env
        if env:
            monkeypatch.delenv(env)


def test_full_size_properties_cfg2(gpu_api, oracle_mod):
    """BASELINE cfg2 (131 072-pt scan vs 1 M-pt map, 20 ICP iterations): size-independent properties, plus direct
    oracle parity for the first ICP iteration's correspondences (one oracle pass is ~1 s)."""
    case = get_case("cfg2")
    cfg = case["cfg"]
    ctx = api_ctx = _ctx(gpu_api, case)
    r = ctx.register(case["scan_xyzi"], case["pose_prior"], cfg["max_iterations"], 0)
    pose = np.array(r.pose)
    assert r.status == 0
    assert np.linalg.norm(pose[:3] - case["pose_true"][:3]) < 0.01 and quat_angle(pose[3:], case["pose_true"][3:]) < 2e-3
    # idempotence: registering again from the converged pose moves < 1 mm
    r2 = ctx.register(case["scan_xyzi"], pose, cfg["max_iterations"], 0)
    assert np.linalg.norm(np.array(r2.pose)[:3] - pose[:3]) < 1e-3
    # histogram bookkeeping: every processed point lands in exactly one rejection bin; 3 obs labels per accepted point
    assert sum(r.hist_reject_plane) == len(case["scan_xyzi"]) and sum(r.hist_obs) == 3 * r.hist_reject_plane[0]
    assert r.iter_n_surf[r.n_iterations - 1] == r.hist_reject_plane[0]
    # rigid-motion equivariance is NOT exact for this algorithm (block grid, float rounding), but a different prior must
    # land on the same optimum to well under the tolerance
    from superodom_b200 import synth
    r3 = ctx.register(case["scan_xyzi"], synth.perturb_pose(case["pose_true"], 4242), cfg["max_iterations"], 0)
    assert np.linalg.norm(np.array(r3.pose)[:3] - pose[:3]) < 2e-3
    # one oracle pass at full size
    om = oracle_mod.OracleMap(case["map_xyzi"], ref_octree=False)
    gc, gho, ghr = ctx.correspond(case["scan_xyzi"], case["pose_prior"], 0)
    oc, oho, ohr = om.correspond(case["scan_xyzi"], case["pose_prior"], cfg["plane_res"], 0, 0, n_threads=8)
    assert np.array_equal(gc["status"].astype(np.int64), oc["status"].astype(np.int64))
    assert np.array_equal(gho, oho) and np.array_equal(ghr, ohr)
    ok = oc["status"] == 0
    assert np.array_equal(gc["nn"][ok].astype(np.int64), oc["nn"][ok])
    H, g, cost = ctx.evaluate(case["pose_prior"])
    oH, og, ocost, _ = oracle_mod.evaluate(oc, case["pose_prior"], cfg["plane_res"])
    assert np.abs(H - oH).max() <= 1e-10 * np.abs(oH).max() and abs(cost - ocost) <= 1e-10 * ocost
    # and the whole registration against the oracle (about 10 s of CPU)
    ro = om.register(case["scan_xyzi"], case["pose_prior"], cfg["plane_res"], cfg["max_iterations"], 0, knn_mode=0, n_threads=8)
    _assert_pose_close(pose, np.array(ro.pose))
    assert r.n_iterations == ro.n_iterations
    api_ctx.close()


def test_cfg3_mid360_with_covariance(gpu_api, oracle_mod):
    """BASELINE cfg3: 240 000-pt Mid-360 scan vs 2 M-pt map at planeRes 0.1, covariance / eigen outputs checked."""
    case = get_case("cfg3")
    cfg = case["cfg"]
    ctx = gpu_api.Context(max_map_points=len(case["map_xyzi"]) + 1024, max_scan_points=262144, plane_res=cfg["plane_res"])
    ctx.map_set_points(case["map_xyzi"])
    r = ctx.register(case["scan_xyzi"], case["pose_prior"], cfg["max_iterations"], 0)
    om = oracle_mod.OracleMap(case["map_xyzi"], ref_octree=False)
    ro = om.register(case["scan_xyzi"], case["pose_prior"], cfg["plane_res"], cfg["max_iterations"], 0, knn_mode=0, n_threads=8)
    assert r.status == 0 and ro.status == 0
    _assert_pose_close(np.array(r.pose), np.array(ro.pose))
    assert r.n_iterations == ro.n_iterations
    cg, co = np.array(r.cov).reshape(6, 6), np.array(ro.cov).reshape(6, 6)
    assert np.abs(cg - co).max() <= 1e-6 * np.abs(co).max()
    for f in ("pos_err", "pos_inv_cond", "ori_err_deg", "ori_inv_cond"):
        assert abs(getattr(r, f) - getattr(ro, f)) <= 1e-6 * abs(getattr(ro, f))
    assert np.linalg.norm(np.array(r.pose)[:3] - case["pose_true"][:3]) < 0.01
    ctx.close()


def test_map_insert_voxel_filter_bit_exact(gpu_api, oracle_mod):
    """LocalMap::addSurfPointCloud (LocalMap.h:591-645) on the device vs the numpy restatement: fresh map, a second insert
    that touches only some blocks (untouched blocks must stay as they are, even after planeRes changed), off-grid points."""
    from superodom_b200 import synth
    rng = np.random.default_rng(9)
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=65536, plane_res=0.2)
    a = np.concatenate([rng.uniform(-60, 60, size=(200000, 2)), rng.uniform(-2, 6, size=(200000, 1)), rng.uniform(0, 255, size=(200000, 1))], 1).astype(np.float32)
    a[:100, 0] += 5000.0                                     # off-grid: dropped
    ctx.map_add_surf(a)
    ref = oracle_mod.map_insert_numpy(np.zeros((0, 4), np.float32), a, 0.2)
    got = ctx.map_download(0)
    assert got.shape == ref.shape and np.array_equal(got, ref)
    # second insert, coarser leaf (auto_voxel_size switches planeRes per scan, laserMapping.cpp:624-633), one block only
    ctx.map_set_resolution(0.2, 0.4)
    b = np.concatenate([rng.uniform(-20, 20, size=(50000, 2)), rng.uniform(-2, 6, size=(50000, 1)), rng.uniform(0, 255, size=(50000, 1))], 1).astype(np.float32)
    ctx.map_add_surf(b)
    ref2 = oracle_mod.map_insert_numpy(ref, b, 0.4)
    got2 = ctx.map_download(0)                                # emitted cube by cube (getAllLocalMap order)
    ref2_cubes = ref2[oracle_mod.cube_order(ref2)]
    assert got2.shape == ref2.shape and np.array_equal(got2, ref2_cubes)
    lin_before = synth.block_linear(synth.block_of(ref[:, :3]))
    lin_after = synth.block_linear(synth.block_of(got2[:, :3]))
    centre = 10 + 21 * 10 + 21 * 21 * 5
    for cube in np.unique(lin_before[lin_before != centre]):   # cubes the second cloud did not reach keep their clouds verbatim
        assert np.array_equal(got2[lin_after == cube], ref[lin_before == cube])
    # the index over the new map answers k-NN exactly
    om = oracle_mod.OracleMap(ref2)
    q = ref2[::50, :3] + rng.normal(0, 0.05, size=ref2[::50, :3].shape).astype(np.float32)
    gi, gd = ctx.knn(q, 5, 0.0)
    oi, od, of = om.knn(q, 5, 0)
    assert np.array_equal(_gi(gi)[of], oi[of]) and np.array_equal(gd[of], od[of])
    # 5x5x3 download is a subset in the same order
    near = ctx.map_download(1, [10, 10, 5])
    assert len(near) == len(got2)                             # everything lies within +-2 blocks of the centre here
    ctx.close()


def test_resolution_change_rebuilds_index(gpu_api, oracle_mod):
    """planeRes drives the gates AND the search radius; switching it (adjustVoxelSize, laserMapping.cpp:600-651) must keep parity."""
    case = get_case("tiny")
    ctx = _ctx(gpu_api, case)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    for pr in (0.4, 0.1, 0.2):
        ctx.map_set_resolution(0.1, pr)
        gc, gho, ghr = ctx.correspond(case["scan_xyzi"], case["pose_prior"], 0)
        oc, oho, ohr = om.correspond(case["scan_xyzi"], case["pose_prior"], pr, 0, 0)
        assert np.array_equal(gho, oho) and np.array_equal(ghr, ohr), pr
        r = ctx.register(case["scan_xyzi"], case["pose_prior"], 5)
        ro = om.register(case["scan_xyzi"], case["pose_prior"], pr, 5)
        _assert_pose_close(np.array(r.pose), np.array(ro.pose))
        assert r.n_iterations == ro.n_iterations
    ctx.close()


@pytest.mark.parametrize("prior", [(1.0, (0.2, 0.5, 0.9)), (100.0, (0.0, 0.0, 0.0)), (2.0, (1.0, 0.3, 0.3)), (0.5, (0.3, 1.0, 0.2))])
def test_absolute_pose_prior_factor(gpu_api, oracle_mod, prior):
    """SE3AbsolutatePoseFactor rows (LidarSlam.cpp:281-298; dormant upstream because isDegenerate is never set): the 6 extra
    residuals, their sqrt-information (including Eigen's LLT quirk when an uncertainty saturates at 1 -> information 0)."""
    case = get_case("tiny")
    ctx = _ctx(gpu_api, case)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    r = ctx.register(case["scan_xyzi"], case["pose_prior"], 5, 0, pose_prior=prior)
    ro = om.register(case["scan_xyzi"], case["pose_prior"], 0.2, 5, 0, knn_mode=0, pose_prior=prior)
    r0 = ctx.register(case["scan_xyzi"], case["pose_prior"], 5, 0)
    _assert_pose_close(np.array(r.pose), np.array(ro.pose))
    n = ro.n_iterations
    assert r.n_iterations == n and list(r.iter_lm_steps[:n]) == list(ro.iter_lm_steps[:n])
    assert list(r.iter_lm_successful[:n]) == list(ro.iter_lm_successful[:n])
    assert np.allclose(r.iter_cost[:n], ro.iter_cost[:n], rtol=1e-9)
    cg, co = np.array(r.cov).reshape(6, 6), np.array(ro.cov).reshape(6, 6)
    assert np.abs(cg - co).max() <= 1e-6 * np.abs(co).max()
    assert r.prediction_source == 1 and r0.prediction_source == 0
    # the prior pulls towards the initial guess
    d_with = np.linalg.norm(np.array(r.pose)[:3] - case["pose_prior"][:3])
    d_without = np.linalg.norm(np.array(r0.pose)[:3] - case["pose_prior"][:3])
    assert d_with <= d_without + 1e-9
    ctx.close()


def test_scan_prefilter_adjust_voxel_size(gpu_api, oracle_mod):
    """laserMapping::adjustVoxelSize (laserMapping.cpp:600-651): leaf selection + pcl::VoxelGrid on the scan, bit-exact."""
    case = get_case("cfg1")
    ctx = _ctx(gpu_api, case)
    rng = np.random.default_rng(12)
    for scale, expect in ((0.3, (0.1, 0.2)), (0.75, (0.2, 0.4)), (1.0, (0.4, 0.8))):       # statistic 3 / 47 / 112 vs thresholds 25, 65
        s = case["scan_xyzi"].copy()
        s[:, :3] *= np.float32(scale)
        out, lr, pr, avg = ctx.scan_prefilter(s, 0.2, 0.4, True)
        ref, rlr, rpr, ravg = oracle_mod.adjust_voxel_size_numpy(s, 0.2, 0.4, True)
        assert abs(avg - ravg) <= 1e-6 * ravg and (np.float32(lr), np.float32(pr)) == (np.float32(rlr), np.float32(rpr))
        if expect:
            assert (np.float32(lr), np.float32(pr)) == (np.float32(expect[0]), np.float32(expect[1]))
        assert out.shape == ref.shape and np.array_equal(out, ref)
    s = case["scan_xyzi"].copy()
    s[::1000, 0] = np.nan                                        # non-finite points are skipped by the VoxelGrid
    out, lr, pr, avg = ctx.scan_prefilter(s, 0.2, 0.4, False)                                  # fixed leaf
    ref, _, _, _ = oracle_mod.adjust_voxel_size_numpy(s, 0.2, 0.4, False)
    assert np.array_equal(out, ref) and (lr, pr) == (np.float32(0.2), np.float32(0.4))
    # the filtered scan registers
    r = ctx.register(out, case["pose_prior"], 5, 2000)
    assert r.status == 0 and np.linalg.norm(np.array(r.pose)[:3] - case["pose_true"][:3]) < 0.05
    # ... and registering it straight from the device (no download + second upload) is the same registration, bit for bit; the
    # registered-scan insert that follows puts that cloud into the map
    m, _, _, _ = ctx.scan_prefilter(s, 0.2, 0.4, False, download=False)
    assert m == len(out)
    r2 = ctx.register_prefiltered(case["pose_prior"], 5, 2000)
    assert np.array_equal(np.array(r2.pose), np.array(r.pose)) and r2.n_iterations == r.n_iterations and np.array_equal(np.array(r2.cov), np.array(r.cov))
    with pytest.raises(gpu_api.SuperOdomError):
        ctx.register_prefiltered(case["pose_prior"], 5, 2000)                                  # consumed: needs a new so_scan_prefilter
    ref = gpu_api.Context(max_map_points=max(1 << 20, len(case["map_xyzi"]) + 1024), max_scan_points=262144, plane_res=case["cfg"]["plane_res"])
    ref.map_set_points(case["map_xyzi"])
    ref.map_set_resolution(0.2, 0.4)                                                           # what the prefilter call set (laserMapping.cpp:648-649)
    ref.map_add_scan(out, np.array(r2.pose))
    ctx.map_add_registered_scan(np.array(r2.pose))
    assert np.array_equal(ctx.map_download(0), ref.map_download(0))
    ref.close()
    # returns beyond the 13-bit voxel range of the narrow sort key (+-4096 voxels) take the wide-key path: same result as numpy
    far = s.copy()
    far[5::997, :3] *= np.float32(400.0)
    out2, _, _, _ = ctx.scan_prefilter(far, 0.2, 0.2, False)
    ref2, _, _, _ = oracle_mod.adjust_voxel_size_numpy(far, 0.2, 0.2, False)
    assert np.abs(far[np.isfinite(far).all(1), :3]).max() > 4096 * 0.2 and np.array_equal(out2, ref2)
    ctx.close()


def _edge_case(name="cfg1"):
    from superodom_b200 import synth
    case = get_case(name)
    em = synth.make_edge_map(case["scene"], 0.1)
    es = synth.make_edge_scan(em, case["pose_true"], 5000)
    return case, em, es


def test_edge_line_branch_correspondences(gpu_api, oracle_mod):
    """a19: processEdgeFeatures / ComputeLineDistanceParameters (LidarSlam.cpp:310-321,402-493) -- 10-NN in the edge map,
    best-line-by-inliers selection, line PCA gates -- against the oracle, per edge point."""
    case, em, es = _edge_case()
    ctx = _ctx(gpu_api, case)
    ctx.map_set_resolution(0.1, 0.2)
    ctx.map_set_edge_points(em)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    om.set_edge_points(em)
    assert ctx.map_counts_5x5([10, 10, 5], with_edge=True) == (len(em), len(case["map_xyzi"]))
    gc, ghr = ctx.correspond_edge(es, case["pose_prior"])
    oc, ohr = om.correspond_edge(es, case["pose_prior"], 0.1)
    assert np.array_equal(ghr, ohr) and ohr[0] > 1000
    assert np.array_equal(gc["status"].astype(np.int32), oc["status"])
    searched = oc["nn"][:, 0] >= 0
    assert np.array_equal(gc["nn"][searched].astype(np.int64), oc["nn"][searched])                # exact 10-NN, same order
    omask = np.zeros(len(oc), np.uint32)
    for j in range(10):
        omask |= np.where(np.arange(10)[None, :] < oc["n_sel"][:, None], (oc["sel"] == j), False).any(1).astype(np.uint32) << np.uint32(j)
    assert np.array_equal(gc["selected_mask"][searched], omask[searched])                          # same inlier selection
    ok = oc["status"] == 0
    # the line direction is an eigenvector: its sign is arbitrary, so (a, b) may come out swapped (the residual's J^T J, J^T r,
    # |r|^2 are invariant under the swap)
    same = np.abs(gc["a"][ok] - oc["a"][ok]).max(1) + np.abs(gc["b"][ok] - oc["b"][ok]).max(1)
    swap = np.abs(gc["a"][ok] - oc["b"][ok]).max(1) + np.abs(gc["b"][ok] - oc["a"][ok]).max(1)
    assert (np.minimum(same, swap) < 1e-7).all()          # eigenvector of a 2-10 point scatter: conditioning-limited
    assert np.allclose(gc["w"][ok], oc["w"][ok], rtol=1e-9)
    # normal equations of the edge rows alone, against the restated line rows on the device's own (a, b, w)
    # (tests/test_solve_numerics.py covers more poses and inputs)
    a2 = solve_numerics_ref.tukey_a2(0.1)
    for pose in (case["pose_prior"], case["pose_true"]):
        H, g, cost = ctx.evaluate(pose)
        rH, rg, rcost, _ = solve_numerics_ref.line_normal_equations(es[ok, :3].astype(np.float64), gc["a"][ok], gc["b"][ok], gc["w"][ok], pose, a2)
        assert np.abs(H - rH).max() <= 1e-10 * np.abs(rH).max()
        assert np.abs(g - rg).max() <= 1e-10 * max(np.abs(rg).max(), 1e-3 * np.abs(rH).max())
        assert abs(cost - rcost) <= 1e-10 * rcost
    ctx.close()


@pytest.mark.parametrize("cap", [2000, 0])
def test_edge_line_branch_registration(gpu_api, oracle_mod, cap):
    """Full registration with both feature kinds (3 residual rows per edge + 1 per plane in one LM problem)."""
    case, em, es = _edge_case()
    cfg = case["cfg"]
    ctx = _ctx(gpu_api, case)
    ctx.map_set_resolution(0.1, 0.2)
    ctx.map_set_edge_points(em)
    om = oracle_mod.OracleMap(case["map_xyzi"])
    om.set_edge_points(em)
    r = ctx.register(case["scan_xyzi"], case["pose_prior"], cfg["max_iterations"], cap, edge_xyzi=es)
    ro = om.register(case["scan_xyzi"], case["pose_prior"], 0.2, cfg["max_iterations"], cap, knn_mode=0, edge_xyzi=es, line_res=0.1)
    _assert_pose_close(np.array(r.pose), np.array(ro.pose))
    n = ro.n_iterations
    assert r.n_iterations == n
    assert list(r.iter_n_surf[:n]) == list(ro.iter_n_surf[:n]) and list(r.iter_n_edge[:n]) == list(ro.iter_n_edge[:n])
    assert list(r.iter_lm_steps[:n]) == list(ro.iter_lm_steps[:n]) and list(r.iter_lm_successful[:n]) == list(ro.iter_lm_successful[:n])
    assert list(r.hist_reject_line) == list(ro.hist_reject_line) and r.iter_n_edge[0] > 1000
    assert np.allclose(r.iter_cost[:n], ro.iter_cost[:n], rtol=1e-9)
    cg, co = np.array(r.cov).reshape(6, 6), np.array(ro.cov).reshape(6, 6)
    assert np.abs(cg - co).max() <= 1e-6 * np.abs(co).max()
    assert r.map_edge_5x5 == ro.map_edge_5x5 == len(em) and r.scan_edge_num == len(es)
    r0 = ctx.register(case["scan_xyzi"], case["pose_prior"], cfg["max_iterations"], cap)           # edge branch idle again
    assert list(r0.hist_reject_line) == [0] * 7 and r0.iter_n_edge[0] == 0
    e_with = np.linalg.norm(np.array(r.pose)[:3] - case["pose_true"][:3])
    assert e_with < 0.01
    ctx.close()


def test_edge_clouds_in_batched_replay(gpu_api):
    """so_register_batch_edges: every scan of a batch carries its own edge cloud (a19 in replay).  Each scan's result must be
    BIT-equal to the single-scan so_register of the same (scan, edge cloud, prior) -- whose parity against the oracle is the test
    above -- including a scan with no edge points and scans of different sizes in one batch (spread over both chunk streams)."""
    from superodom_b200 import synth
    case, em, es = _edge_case()
    ctx = _ctx(gpu_api, case, max_batch=16)
    ctx.map_set_resolution(0.1, 0.2)
    ctx.map_set_edge_points(em)
    B = 16
    scans, edges, priors = [], [], []
    for i in range(B):
        T = synth.perturb_pose(case["pose_true"], 7100 + i, dt=0.3, dth_deg=2.0)
        scans.append(synth.make_scan(case["scene"], "vlp16", T, 7200 + i))
        edges.append(np.zeros((0, 4), np.float32) if i == 3 else synth.make_edge_scan(em, T, 3000 + i, keep_every=2 + i % 3))
        priors.append(synth.perturb_pose(T, 7300 + i, dt=0.05, dth_deg=0.5))
    singles = [ctx.register(scans[i], priors[i], 5, 0, edge_xyzi=edges[i] if len(edges[i]) else None) for i in range(B)]
    res = ctx.register_batch_edges(np.concatenate(scans), [len(x) for x in scans], np.concatenate(edges), [len(e) for e in edges], np.array(priors), 5, 0)
    for i in range(B):
        a, b = singles[i], res[i]
        assert a.status == b.status == 0 and np.array_equal(np.array(a.pose), np.array(b.pose)), i
        assert a.n_iterations == b.n_iterations and list(a.iter_n_edge) == list(b.iter_n_edge) and list(a.hist_reject_line) == list(b.hist_reject_line), i
        assert np.array_equal(np.array(a.cov), np.array(b.cov)) and b.scan_edge_num == len(edges[i]), i
        assert (b.iter_n_edge[0] > 500) == (i != 3), (i, b.iter_n_edge[0])
    # an edge-less batch afterwards runs with the branch idle
    r0 = ctx.register_batch(np.concatenate(scans), [len(x) for x in scans], np.array(priors), 5, 0)
    assert all(r.iter_n_edge[0] == 0 and r.status == 0 for r in r0)
    ctx.close()


def test_edge_map_insert_and_download_order(gpu_api, oracle_mod):
    """addEdgePointCloud (LocalMap.h:529-589) = the surf insert at leaf lineRes; getAllLocalMap returns each cube's edge cloud
    followed by its surf cloud, cubes in index order (LocalMap.h:647-658)."""
    from superodom_b200 import synth
    case, em, es = _edge_case("tiny")
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=65536, plane_res=0.2, line_res=0.1)
    raw = synth.sample_edges(case["scene"], 0.1)
    raw4 = np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1)
    ctx.map_add_edge(raw4)
    ctx.map_add_surf(case["map_xyzi"])
    ref_e = oracle_mod.map_insert_numpy(np.zeros((0, 4), np.float32), raw4, 0.1)
    ref_s = oracle_mod.map_insert_numpy(np.zeros((0, 4), np.float32), case["map_xyzi"], 0.2)
    allm = ctx.map_download(0)
    assert len(allm) == len(ref_e) + len(ref_s)
    assert np.array_equal(allm[: len(ref_e)], ref_e) and np.array_equal(allm[len(ref_e):], ref_s)     # one cube: edge cloud, then surf cloud
    ctx.map_add_scan_edge(es, case["pose_true"])
    ref_e2 = oracle_mod.map_insert_numpy(ref_e, oracle_mod.transform_scan_numpy(es, case["pose_true"]), 0.1)
    assert np.array_equal(ctx.map_download(0)[: len(ref_e2)], ref_e2)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# scan preparation in front of the path (SURVEY 8f row 2): so_scan_deskew / so_scan_extract_uniform
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("imu_only", [False, True])
def test_scan_deskew_matches_oracle(gpu_api, oracle_mod, imu_only):
    """removePointDistortion: FP64 rigid motions rounded to float32.  The device composes the same motions as quaternion
    products and uses CUDA's acos/sin, so the pre-rounding values differ from the oracle's by ~1e-15 relative.  Tolerance
    (written here, as the task asks): every coordinate within ONE float32 ulp at the point's largest coordinate of the
    oracle's, and >= 99.9 % of the coordinates bit-identical."""
    from superodom_b200 import synth
    d = synth.make_raw_sweep(131_072, seed=4100)
    pts, st, sp, t0 = d["points"], d["sample_times"], d["sample_poses"], d["start_time"]
    exp, exp_start, exp_past = oracle_mod.deskew(pts, 5, t0, st, sp, imu_only=imu_only, T_i_l=d["T_i_l"])
    ctx = gpu_api.Context(max_map_points=1024, max_scan_points=len(pts), plane_res=0.2)
    got = pts.copy()
    start, past = ctx.scan_deskew(got, 5, t0, st, sp, imu_only=imu_only, T_i_l=d["T_i_l"])
    assert past == exp_past == 0
    assert np.abs(start[:3] - exp_start[:3]).max() < 1e-12
    assert min(np.abs(start[3:] - exp_start[3:]).max(), np.abs(start[3:] + exp_start[3:]).max()) < 1e-12
    assert np.array_equal(got[:, 3:], pts[:, 3:])                                         # intensity / time / ring bytes untouched
    bad = ~np.isfinite(pts[:, :3]).all(1)
    assert bad.sum() == 8 and np.array_equal(got[bad, :3], pts[bad, :3], equal_nan=True)
    g, e = got[~bad, :3], exp[~bad, :3]
    assert np.abs(g - pts[~bad, :3]).max() > 0.05                                         # the sweep really moved points
    assert (np.abs(g - e) <= np.spacing(np.abs(e).max(axis=1, keepdims=True))).all()
    assert (g == e).mean() >= 0.999, (g == e).mean()


def test_scan_deskew_buffer_edges(gpu_api, oracle_mod):
    from superodom_b200 import synth
    d = synth.make_raw_sweep(2000, seed=4101, with_defects=False)
    pts, st, sp, t0 = d["points"], d["sample_times"], d["sample_poses"], d["start_time"]
    ctx = gpu_api.Context(max_map_points=1024, max_scan_points=4096, plane_res=0.2)
    for args in ((t0, st + 10.0, sp), (t0, st[:12], sp[:12]), (-0.032, st - st[0] - 0.05, sp)):      # before-first / past-end / rewind
        exp, exp_start, exp_past = oracle_mod.deskew(pts, 5, *args)
        got = pts.copy()
        start, past = ctx.scan_deskew(got, 5, *args)
        assert past == exp_past
        assert np.abs(start - exp_start).max() < 1e-12
        assert (np.abs(got[:, :3] - exp[:, :3]) <= np.spacing(np.abs(exp[:, :3]).max(axis=1, keepdims=True))).all()
    with pytest.raises(gpu_api.SuperOdomError):
        ctx.scan_deskew(pts.copy(), 5, t0, st[::-1].copy(), sp)                                     # std::map keys are ascending


@pytest.mark.parametrize("skip,block_range", [(1, 0.2), (3, 0.2), (4, 1.5), (7, 0.0)])
def test_scan_extract_uniform_bit_exact(gpu_api, oracle_mod, skip, block_range):
    from superodom_b200 import synth
    pts = synth.make_raw_sweep(131_072, seed=4102)["points"]
    ctx = gpu_api.Context(max_map_points=1024, max_scan_points=len(pts), plane_res=0.2)
    for int_abs in (False, True):
        exp = oracle_mod.extract_uniform(pts, 5, skip, block_range, int_abs=int_abs)
        got = ctx.scan_extract_uniform(pts, 5, skip, block_range, int_abs=int_abs)
        assert got.shape == exp.shape and 0 < len(got) < len(pts)
        assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))                             # bit-exact, NaN payloads included
    assert len(ctx.scan_extract_uniform(pts[:1], 5, skip, block_range)) == 0                        # the loop starts at index 1
    with pytest.raises(gpu_api.SuperOdomError):
        ctx.scan_extract_uniform(pts, 5, 0, block_range)


def test_scan_chain_deskew_extract_register(gpu_api, oracle_mod):
    """Driver cloud -> deskew -> uniform extraction -> registration, GPU chain against the oracle chain."""
    from superodom_b200 import synth
    case = get_case("cfg1")
    scan = case["scan_xyzi"]
    n = len(scan)
    raw = np.zeros((n, 8), np.float32)
    raw[:, :3] = scan[:, :3]
    raw[:, 5] = np.linspace(0, 0.1, n)
    t0 = 50.0
    st = t0 - 0.02 + np.arange(40) * 0.005
    sp = np.zeros((40, 7)); sp[:, 6] = 1.0                                   # static sensor: deskew must be the identity
    ctx = _ctx(gpu_api, case)
    got = raw.copy()
    ctx.scan_deskew(got, 5, t0, st, sp)
    assert np.array_equal(got, raw)
    feat = ctx.scan_extract_uniform(got, 5, 1, 0.2)
    exp_feat = oracle_mod.extract_uniform(raw, 5, 1, 0.2)
    assert np.array_equal(feat, exp_feat) and len(feat) >= n - 2
    cfg = case["cfg"]
    rg = ctx.register(feat, case["pose_prior"], cfg["max_iterations"], cfg["max_surface_features"])
    om = oracle_mod.OracleMap(case["map_xyzi"])
    ro = om.register(exp_feat, case["pose_prior"], cfg["plane_res"], cfg["max_iterations"], cfg["max_surface_features"])
    assert rg.status == ro.status == 0 and rg.n_iterations == ro.n_iterations
    _assert_pose_close(np.array(rg.pose), np.array(ro.pose))


def test_scan_order_key_paths_and_stream_modes_agree(gpu_api, monkeypatch):
    """The scan-order keys (32-bit when cell + scan bits fit, else 64-bit) and the chunk scheduling (two streams, one stream,
    conditional graph or unrolled) are execution details: a batch must come out bit-identical under all of them."""
    case = get_case("cfg1")
    scans = [get_case("cfg1", i)["scan_xyzi"] for i in range(16)]
    priors = np.stack([get_case("cfg1", i)["pose_prior"] for i in range(16)])
    n_points = np.array([len(s) for s in scans], np.uint32)
    flat = np.ascontiguousarray(np.concatenate(scans, 0))

    def run():
        ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=int(n_points.max()), max_batch=16, plane_res=0.2)
        ctx.map_set_points(case["map_xyzi"])
        res = ctx.register_batch(flat, n_points, priors, 5, 2000)
        out = np.array([list(r.pose) + [r.n_iterations] + list(r.hist_obs) for r in res])
        ctx.close()
        return out
    base = run()
    # ... and so are the one-CTA scan preparation of small registrations (these capped scans keep <= 2001 points each) against the
    # device-wide ordering, and the optimiser step folded into the evaluation kernel against the two-kernel form
    for env in ("SO_FORCE_KEY64", "SO_SINGLE_STREAM", "SO_NO_COND_GRAPH", "SO_NO_SMALL_PREPARE", "SO_NO_FUSED_LM"):
        monkeypatch.setenv(env, "1")
        assert np.array_equal(run(), base), env
        monkeypatch.delenv(env)
    # the batch equals its scans registered one by one (small path, fused optimiser step), bit for bit
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=int(n_points.max()), max_batch=1, plane_res=0.2)
    ctx.map_set_points(case["map_xyzi"])
    for i in (0, 7, 15):
        r = ctx.register(scans[i], priors[i], 5, 2000, skip_map_checks=True)
        assert np.array_equal(np.array(list(r.pose) + [r.n_iterations] + list(r.hist_obs)), base[i]), i
    ctx.close()
    # a single small registration searches with one WARP per query (k_knn_scan_coop); the batch above used one thread per query:
    # equal results already say the two searches agree -- here also against the single registration with the warp search off,
    # and on the neighbour ids themselves (stage call, decimated scan)
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=int(n_points.max()), max_batch=1, plane_res=0.2)
    ctx.map_set_points(case["map_xyzi"])
    corr_coop = ctx.correspond(scans[3][::4], priors[3], 2000)[0]          # 7 200 points: small enough for the warp search
    ctx.close()
    monkeypatch.setenv("SO_NO_COOP_KNN", "1")
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=int(n_points.max()), max_batch=1, plane_res=0.2)
    ctx.map_set_points(case["map_xyzi"])
    for i in (0, 7, 15):
        r = ctx.register(scans[i], priors[i], 5, 2000, skip_map_checks=True)
        assert np.array_equal(np.array(list(r.pose) + [r.n_iterations] + list(r.hist_obs)), base[i]), i
    corr_lane = ctx.correspond(scans[3][::4], priors[3], 2000)[0]
    ctx.close()
    monkeypatch.delenv("SO_NO_COOP_KNN")
    assert (corr_coop["status"] == 0).sum() > 1000
    for f in ("status", "nn", "nn_d2", "n", "d", "w"):
        assert np.array_equal(corr_coop[f], corr_lane[f]), f


@pytest.mark.gpu
def test_decimated_upload_equals_whole_upload(gpu_api, monkeypatch):
    """so_register of a capped scan uploads only the points shouldProcessPoint keeps ahead of the registration and the whole
    cloud beside it: the result must equal the whole-cloud-first path bit for bit (packed and pcl::PointXYZI layouts), and the
    cloud so_map_add_registered_scan inserts afterwards must be the whole scan, not the kept points."""
    case = get_case("cfg1")
    s, prior = case["scan_xyzi"], np.ascontiguousarray(case["pose_prior"])
    pcl = np.zeros((len(s), 8), np.float32)
    pcl[:, :3] = s[:, :3]
    pcl[:, 4] = s[:, 3]

    def run(strided):
        ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=len(s), max_batch=1, plane_res=0.2)
        ctx.map_set_points(case["map_xyzi"])
        outs = []
        for _ in range(2):                                    # second call: cached index list, staging buffer reuse
            if strided:
                o, r = ctx._opts(5, 2000), gpu_api.IcpResult()
                rc = ctx.L.so_register(ctx.h, pcl.ctypes.data_as(C.c_void_p), len(s), None, 0, 32, 16, prior.ctypes.data_as(C.c_void_p), C.byref(o), C.byref(r))
                assert rc == 0
            else:
                r = ctx.register(s, prior, 5, 2000)
            assert r.status == 0 and r.scan_surf_num == len(s)
            outs.append(list(r.pose) + list(r.pose_opt) + list(r.cov) + [r.n_iterations] + list(r.hist_obs) + list(r.hist_reject_plane) + list(r.iter_n_surf))
        assert outs[0] == outs[1]
        n0 = ctx.map_size()
        ctx.map_add_registered_scan(np.array(r.pose))
        m = ctx.map_download(0)
        ctx.close()
        return np.array(outs[0]), n0, m
    base, n0, m_base = run(False)
    pcl_out, _, m_pcl = run(True)
    assert np.array_equal(base, pcl_out) and np.array_equal(m_base, m_pcl)
    monkeypatch.setenv("SO_NO_DEC_UPLOAD", "1")
    whole, _, m_whole = run(False)
    monkeypatch.delenv("SO_NO_DEC_UPLOAD")
    assert np.array_equal(base, whole)
    assert np.array_equal(m_base, m_whole) and len(m_base) > n0 + 2001       # the insert saw the whole 28 800-point scan

"""Keyframes on the device (so_keyframe_*), the map rebuilt from them (so_map_from_keyframes) and keyframes registered against a
submap (so_register_keyframes).

GPU: a kept keyframe is, bit for bit, the tail the registered-scan inserts place (four registration forms, edge clouds included); the
store's argument and capacity errors; the rebuild against the restatement in keyframe_map_numpy.py on cfg1- and cfg2-sized sequences,
both stores, archive on and off (window in id order, the whole map, a registration on it, a capacity failure); small leaves; a
submap registration against so_register of the downloaded keyframe; and a loop closed end to end in a synth scene with injected
odometry drift, corrected by a numpy / scipy pose graph and the rebuild."""
import numpy as np
import pytest

import keyframe_map_numpy as KM
from conftest import get_case

SO_ERR_ARG, SO_ERR_CAPACITY = -1, -3


def _err(api, fn):
    with pytest.raises(api.SuperOdomError) as e:
        fn()
    return int(str(e.value).split("(")[1].split(")")[0])


def _ctx(api, **kw):
    a = dict(max_map_points=1 << 21, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    a.update(kw)
    return api.Context(**a)


def _timed(scan, seed):
    """The scan with a per-point time in [0, 0.1) s in its intensity column (the shipped pipeline stores the time there)."""
    s = scan.copy()
    s[:, 3] = np.random.default_rng(seed).uniform(0.0, 0.1, len(s)).astype(np.float32)
    return s


def _merged(edge, surf, origin):
    """so_map_download(0) of a window holding edge and surf: per block (cube order) the edge cloud, then the surf cloud."""
    from superodom_b200 import synth
    pts = np.concatenate([edge, surf], 0)
    kind = np.r_[np.zeros(len(edge)), np.ones(len(surf))]
    lin = synth.block_linear(synth.block_of(pts[:, :3], tuple(origin)))
    order = np.lexsort((kind, lin))
    return pts[order]


def _rows(a):
    a = np.ascontiguousarray(a, np.float32)
    v = a.view(np.uint32)
    return a[np.lexsort(v.T[::-1])]


def _pose_bits_equal(a, b):
    return np.array(a.pose).tobytes() == np.array(b.pose).tobytes()


# --------------------------------------------------------------------------------------------------------- 1. the store
@pytest.mark.gpu
def test_store_equals_the_insert_tail(gpu_api):
    from superodom_b200 import synth
    case = get_case("cfg1", 0)
    em = synth.make_edge_map(case["scene"], 0.1)
    scan = _timed(case["scan_xyzi"], 1)
    edges = _timed(synth.make_edge_scan(em, case["pose_true"], 17), 2)
    prior = case["pose_prior"]
    prev = synth.perturb_pose(prior, 5, 0.3, 1.0)
    forms = {
        "register": lambda c: c.register(scan, prior, 5, 2000, edge_xyzi=edges),
        "prefiltered": lambda c: (c.scan_prefilter(scan, 0.1, 0.2, auto_voxel_size=False, download=False), c.register_prefiltered(prior, 5, 2000))[1],
        "undistort_edges": lambda c: c.register_undistort_edges(scan, edges, prior, gpu_api.undistort(prev, 0.1), 5, 2000),
        "optimized_edges": lambda c: c.register_optimized_edges(scan, edges, prior, gpu_api.motion(0.1), 5, 2000).icp,
    }
    for name, reg in forms.items():
        ctx = _ctx(gpu_api)
        ctx.map_set_points(case["map_xyzi"])
        ctx.map_set_edge_points(em)
        assert _err(gpu_api, lambda: ctx.keyframe_add_registered(prior)) == SO_ERR_ARG           # no store
        ctx.keyframe_reserve(1 << 17, 4)
        assert _err(gpu_api, lambda: ctx.keyframe_add_registered(prior)) == SO_ERR_ARG           # no registration yet
        r = reg(ctx)
        pose = np.array(r.pose)
        before = ctx.map_download(0)
        assert ctx.keyframe_add_registered(pose) == 0
        assert np.array_equal(ctx.map_download(0), before)                                      # the map is not touched
        n_edge = len(edges) if "edges" in name or name == "register" else 0
        f, n_s, n_e = ctx.keyframe_info()
        assert f == 1 and n_s > 0 and n_e == n_edge, (name, n_s, n_e)
        kf_s, kf_e = ctx.keyframe_download(0, 0), ctx.keyframe_download(0, 1)
        # way 1: the registered-scan inserts into the emptied map; way 2: the kept clouds inserted as host scans at the same pose
        ctx.map_set_points(np.zeros((0, 4), np.float32))
        ctx.map_set_edge_points(np.zeros((0, 4), np.float32))
        ctx.map_add_registered_scan(pose)
        ctx.map_add_registered_edges(pose)
        b = _ctx(gpu_api)
        b.map_add_scan(kf_s, pose)
        if len(kf_e):
            b.map_add_scan_edge(kf_e, pose)
        assert np.array_equal(ctx.map_origin(), b.map_origin())
        a_map, b_map = ctx.map_download(0), b.map_download(0)
        assert len(a_map) > 1000 and a_map.tobytes() == b_map.tobytes(), name
        # the world-frame download is so_map_add_scan's transform: at a leaf no two points share, the map is the transformed scan
        w = ctx.keyframe_download(0, 0, pose)
        c2 = _ctx(gpu_api, plane_res=1e-3)
        c2.map_add_scan(kf_s, pose)
        assert len(w) == len(kf_s) and _rows(c2.map_download(0)).tobytes() == _rows(w).tobytes()
        # capacity: the frame table, then the pool
        for _ in range(3):
            ctx.keyframe_add_registered(pose)
        assert _err(gpu_api, lambda: ctx.keyframe_add_registered(pose)) == SO_ERR_CAPACITY
        assert ctx.keyframe_info()[0] == 4
        assert _err(gpu_api, lambda: ctx.keyframe_reserve(n_s, 3)) == SO_ERR_ARG                # below what is held
        ctx.keyframe_reserve(5 * n_s + 1, 8)
        assert ctx.keyframe_download(3, 0).tobytes() == kf_s.tobytes()                          # kept across the resize
        ctx.keyframe_add_registered(pose)
        assert _err(gpu_api, lambda: ctx.keyframe_add_registered(pose)) == SO_ERR_CAPACITY      # 6 * n_s > cap
        assert ctx.keyframe_info()[:2] == (5, 5 * n_s)
        assert np.allclose(ctx.keyframe_poses(), pose)
        ctx.keyframe_reserve(0, 0)
        assert ctx.keyframe_info() == (0, 0, 0)
        for c in (ctx, b, c2):
            c.close()


# ---------------------------------------------------------------------------------------------- 2. rebuild == definition
def _keyframes(api, name, n, mf):
    """A context with n keyframes of `name` (surf and edge clouds), registered on the case map; -> (ctx, case, edge map)"""
    from superodom_b200 import synth
    case = get_case(name, 0)
    em = synth.make_edge_map(case["scene"], 0.1)
    ctx = _ctx(api, max_map_points=1 << 22)
    ctx.map_set_points(case["map_xyzi"])
    ctx.map_set_edge_points(em)
    ctx.keyframe_reserve(n << 18, n)
    for i in range(n):
        c = get_case(name, i)
        e = synth.make_edge_scan(em, c["pose_true"], 30 + i)
        r = ctx.register(c["scan_xyzi"], c["pose_prior"], 5, mf, edge_xyzi=e)
        ctx.keyframe_add_registered(np.array(r.pose))
    return ctx, case, em


def _general_poses(n, seed, reach):
    from superodom_b200 import synth
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        t = rng.uniform(-reach, reach, 3) * np.array([1.0, 1.0, 0.05])
        q = synth.quat_from_rotvec(rng.normal(0, [0.05, 0.05, 1.5]))
        out.append(np.r_[t, q / np.linalg.norm(q)])
    return np.array(out)


def _reference(src, ids, poses, store, leaf, origin, archive):
    clouds = [src.keyframe_download(i, store, p) for i, p in zip(ids, poses)]
    return KM.map_from_keyframes(clouds, leaf, origin, archive)


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,mf", [("cfg1", 8, 2000), ("cfg2", 4, 0)])
@pytest.mark.parametrize("archive", [False, True])
def test_rebuild_equals_the_definition(gpu_api, name, n, mf, archive):
    src, case, em = _keyframes(gpu_api, name, n, mf)
    ids = np.array([3, 0, 2, 1] + list(range(4, n)), np.int32)
    reach = 800.0 if archive else 30.0                                   # archive on: a trajectory that leaves the window
    poses = _general_poses(n, 7, reach)
    for same in (False, True):
        dst = src if same else _ctx(gpu_api, max_map_points=1 << 22)
        if archive:
            dst.map_archive(1 << 22)
        dst.map_from_keyframes(src, ids, poses, 3)
        origin = dst.map_origin()
        ws, arcs = _reference(src, ids, poses, 0, 0.2, tuple(origin), archive)
        we, arce = _reference(src, ids, poses, 1, 0.1, tuple(origin), archive)
        assert len(ws) > 1000 and len(we) > 100
        if archive:
            assert len(arcs) > 0 and len(arce) > 0
        assert dst.map_download(0).tobytes() == _merged(we, ws, origin).tobytes()                # window, block by block, id order
        for store, (w, a) in enumerate(((ws, arcs), (we, arce))):
            assert _rows(dst.map_download_all(store)).tobytes() == _rows(KM.download_all(w, a)).tobytes()
            assert dst.map_archive_info(store)[0] == sum(len(b) for b in a.values())
        if same:
            assert np.array_equal(src.keyframe_poses(), poses[np.argsort(ids)])
        # a registration on the rebuilt map == on the restatement loaded as a prior map (the whole map: the registration may shift)
        from superodom_b200 import synth
        ref = _ctx(gpu_api, max_map_points=1 << 22)
        if archive:
            ref.map_archive(1 << 22)
        ref.map_set_points(KM.download_all(ws, arcs))
        ref.map_set_edge_points(KM.download_all(we, arce))
        assert np.array_equal(ref.map_origin(), origin)
        scan = src.keyframe_download(0, 0)
        prior = synth.perturb_pose(poses[list(ids).index(0)], 11, 0.1, 1.0)
        r1 = dst.register(scan, prior, 5, mf)
        r2 = ref.register(scan, prior, 5, mf)
        assert r1.status == 0 and r1.n_iterations > 0 and _pose_bits_equal(r1, r2)
        ref.close()
        # a capacity failure leaves both stores as they were
        t = _ctx(gpu_api, max_map_points=len(ws) - 1)
        if archive:
            t.map_archive(1 << 22)
        t.map_from_keyframes(src, ids[:1], poses[:1], 3)
        before = (t.map_download(0), t.map_download_all(0), t.map_download_all(1))
        assert _err(gpu_api, lambda: t.map_from_keyframes(src, ids, poses, 3)) == SO_ERR_CAPACITY
        after = (t.map_download(0), t.map_download_all(0), t.map_download_all(1))
        assert all(x.tobytes() == y.tobytes() for x, y in zip(before, after))
        t.close()
        if not same:
            dst.close()
    src.close()


@pytest.mark.gpu
def test_rebuild_capacity_of_the_archive_leaves_both_stores(gpu_api):
    src, _, _ = _keyframes(gpu_api, "cfg1", 3, 2000)
    ids = np.arange(3, dtype=np.int32)
    poses = _general_poses(3, 9, 800.0)
    dst = _ctx(gpu_api)
    dst.map_archive(1 << 20)
    dst.map_from_keyframes(src, ids[:1], poses[:1], 3)
    before = (dst.map_download(0), dst.map_download_all(0), dst.map_download_all(1))
    n_arc = sum(dst.map_archive_info(s)[0] for s in (0, 1))
    _, arcs = _reference(src, ids, poses, 0, 0.2, tuple(dst.map_origin()), True)
    need = sum(len(b) for b in arcs.values())
    assert need > 0
    dst.map_archive(max(need - 1, dst.map_archive_info(0)[0], dst.map_archive_info(1)[0], 1))
    assert _err(gpu_api, lambda: dst.map_from_keyframes(src, ids, poses, 3)) == SO_ERR_CAPACITY
    after = (dst.map_download(0), dst.map_download_all(0), dst.map_download_all(1))
    assert all(x.tobytes() == y.tobytes() for x, y in zip(before, after))
    assert sum(dst.map_archive_info(s)[0] for s in (0, 1)) == n_arc
    # argument errors
    assert _err(gpu_api, lambda: dst.map_from_keyframes(src, [3], poses[:1], 1)) == SO_ERR_ARG
    assert _err(gpu_api, lambda: dst.map_from_keyframes(src, [0], poses[:1], 0)) == SO_ERR_ARG
    assert _err(gpu_api, lambda: dst.map_from_keyframes(src, [0], np.full((1, 7), np.nan), 1)) == SO_ERR_ARG
    dst.map_from_keyframes(src, [], np.zeros((0, 7)), 3)                                            # empty ids: empty stores
    assert dst.map_size() == 0 and dst.map_archive_info(0)[0] == 0
    dst.close()
    src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("leaf", [0.02, 0.2])
def test_single_keyframe_equals_the_insert(gpu_api, leaf):
    """One keyframe into an empty map == so_map_add_scan of it, bit for bit, also below 0.04 m where the per-block filter takes the
    absolute voxel index as the insert does."""
    src, _, _ = _keyframes(gpu_api, "cfg1", 1, 2000)
    pose = _general_poses(1, 3, 10.0)[0]
    a, b = _ctx(gpu_api, plane_res=leaf), _ctx(gpu_api, plane_res=leaf)
    a.map_from_keyframes(src, [0], [pose], 1)
    b.map_add_scan(src.keyframe_download(0, 0), pose)
    assert a.map_size() > 1000 and a.map_download(0).tobytes() == b.map_download(0).tobytes()
    for x in (a, b, src):
        x.close()


# ---------------------------------------------------------------------------------------------- 3. submap and alignment
@pytest.mark.gpu
@pytest.mark.parametrize("mf", [0, 2000])
def test_register_keyframes_equals_register(gpu_api, mf):
    from superodom_b200 import synth
    src, case, _ = _keyframes(gpu_api, "cfg1", 4, 2000)
    poses = src.keyframe_poses()
    sub = _ctx(gpu_api, max_batch=4)
    sub.map_from_keyframes(src, [0, 1], poses[:2], 1)
    for i in (2, 3):
        prior = synth.perturb_pose(poses[i], 40 + i, 0.1, 1.0)
        a = sub.register_keyframes(src, [i], [prior], 5, mf)[0]
        b = sub.register(src.keyframe_download(i, 0), prior, 5, mf)
        assert a.status == 0 and a.n_iterations > 0 and _pose_bits_equal(a, b)
        assert np.array(a.cov).tobytes() == np.array(b.cov).tobytes()
    # several keyframes in one call, out of order (a gather) and in order (read in place)
    for ids in ([3, 2], [2, 3]):
        priors = [synth.perturb_pose(poses[i], 40 + i, 0.1, 1.0) for i in ids]
        rs = sub.register_keyframes(src, ids, priors, 5, mf)
        for i, p, r in zip(ids, priors, rs):
            one = sub.register_keyframes(src, [i], [p], 5, mf)[0]
            assert np.allclose(np.array(r.pose), np.array(one.pose), atol=1e-9)
    assert _err(gpu_api, lambda: sub.register_keyframes(src, [9], [poses[0]], 5, mf)) == SO_ERR_ARG
    sub.close()
    src.close()


# ---------------------------------------------------------------------------------------------- 4. loop closure end to end
def _se3(p):
    from scipy.spatial.transform import Rotation
    return np.asarray(p[:3], np.float64), Rotation.from_quat(p[3:])


def _compose(a, b):
    ta, Ra = _se3(a)
    tb, Rb = _se3(b)
    return np.r_[ta + Ra.apply(tb), (Ra * Rb).as_quat()]


def _inverse(a):
    t, R = _se3(a)
    Ri = R.inv()
    return np.r_[-Ri.apply(t), Ri.as_quat()]


def _pose_graph(init, edges, fixed=0):
    """Least-squares SE(3) pose graph (test helper): nodes init [n, 7]; edges (i, j, Z_ij, sqrt_info[6]) with residual
    log(Z_ij^-1 X_i^-1 X_j) as (translation, rotation vector); node `fixed` held."""
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    n = len(init)
    free = [k for k in range(n) if k != fixed]

    def nodes(x):
        out = init.copy()
        for m, k in enumerate(free):
            d = x[6 * m: 6 * m + 6]
            t, R = _se3(init[k])
            out[k] = np.r_[t + d[:3], (Rotation.from_rotvec(d[3:]) * R).as_quat()]
        return out

    def res(x):
        X = nodes(x)
        r = []
        for i, j, Z, w in edges:
            E = _compose(_inverse(Z), _compose(_inverse(X[i]), X[j]))
            r.append(w * np.r_[E[:3], Rotation.from_quat(E[3:]).as_rotvec()])
        return np.concatenate(r)

    sol = least_squares(res, np.zeros(6 * len(free)), method="lm", xtol=1e-12, ftol=1e-12)
    return nodes(sol.x)


def _loop_poses(scene, n, radius):
    from superodom_b200 import synth
    out = []
    for i in range(n):
        a = 2 * np.pi * i / (n - 1)
        for dr in (0.0, 0.7, -0.7, 1.4, -1.4, 2.1, -2.1):
            p = np.array([(radius + dr) * np.cos(a), (radius + dr) * np.sin(a), 0.0])
            if scene.free(p):
                break
        q = synth.quat_from_rotvec(np.array([0.0, 0.0, a + np.pi / 2]))
        out.append(np.r_[p, q])
    out[-1][:3] += np.array([0.8, 0.4, 0.0])                    # the return is near, not at, the start
    return np.array(out)


def _share_far(pts, ref, d):
    from scipy.spatial import cKDTree
    dist, _ = cKDTree(ref[:, :3]).query(pts[:, :3])
    return float(np.mean(dist > d))


@pytest.mark.gpu
def test_loop_closure_end_to_end(gpu_api):
    """A loop of VLP-16 scans (20 m range) around the cfg2 hall, each registered pose pushed 2.2 cm in the world frame before it is
    inserted and kept.  The live pass stops at the first keyframe back within 6 m of the start (the loop candidate): a submap of the
    first three keyframes and so_register_keyframes give the loop factor, a numpy / scipy pose graph moves the keyframes, and
    so_map_from_keyframes rebuilds the map.  Measured values and bounds: DESIGN.md, "Keyframes and loop closure"."""
    from superodom_b200 import synth
    scene = get_case("cfg2", 0)["scene"]
    n_max, mf = 60, 0
    truth = _loop_poses(scene, n_max, 16.0)
    drift = np.r_[0.02, 0.01, 0.0, 0.0, 0.0, 0.0, 1.0]             # per step: 2.2 cm of world-frame translation, composed on the left
    ctx = _ctx(gpu_api)
    ctx.map_set_origin(truth[0][:3])
    ctx.keyframe_reserve(n_max << 15, n_max)
    est = [truth[0]]
    ctx.register(synth.make_scan(scene, "vlp16", truth[0], 5000, rmax=20.0), truth[0], 10, mf)    # empty map: the pose stays the prior
    ctx.keyframe_add_registered(truth[0])
    ctx.map_add_registered_scan(truth[0])
    n = n_max
    for i in range(1, n_max):
        prior = _compose(est[-1], _compose(_inverse(truth[i - 1]), truth[i]))        # odometry prior: the true increment
        r = ctx.register(synth.make_scan(scene, "vlp16", truth[i], 5000 + i, rmax=20.0), prior, 10, mf)
        assert r.status == 0, (i, r.status)
        p = _compose(drift, np.array(r.pose))
        est.append(p)
        ctx.keyframe_add_registered(p)
        ctx.map_add_registered_scan(p)
        if i > n_max // 2 and np.linalg.norm(p[:3] - est[0][:3]) < 6.0:             # the loop candidate: back near the start
            n = i + 1
            break
    est = np.array(est)
    truth = truth[:n]
    err_before = np.linalg.norm(est[:, :3] - truth[:, :3], axis=1)
    print(f"loop: {n} keyframes, final keyframe error {err_before[-1]:.3f} m, max {err_before.max():.3f} m")
    assert n < n_max and err_before[-1] > 0.2
    live_map = ctx.map_download(0)
    # loop factor: the last keyframe against a submap of the first three
    sub = _ctx(gpu_api)
    sub.map_set_origin(truth[0][:3])
    sub.map_from_keyframes(ctx, [0, 1, 2], est[:3], 1)
    loop = sub.register_keyframes(ctx, [n - 1], [est[n - 1]], 20, mf)[0]
    assert loop.status == 0
    t_loop = np.array(loop.pose)
    loop_err = np.linalg.norm(t_loop[:3] - truth[n - 1, :3])
    print(f"loop: loop factor error {loop_err:.3f} m (accumulated offset {err_before[-1]:.3f} m)")
    assert loop_err < 0.3 * err_before[-1]
    # pose graph: odometry between consecutive keyframes, the loop between the first and the last
    w_odo = np.r_[np.full(3, 1 / 0.02), np.full(3, 1 / np.deg2rad(0.05))]
    w_loop = np.r_[np.full(3, 1 / 0.01), np.full(3, 1 / np.deg2rad(0.05))]
    edges = [(i, i + 1, _compose(_inverse(est[i]), est[i + 1]), w_odo) for i in range(n - 1)]
    edges.append((0, n - 1, _compose(_inverse(est[0]), t_loop), w_loop))
    opt = _pose_graph(est, edges)
    err_after = np.linalg.norm(opt[:, :3] - truth[:, :3], axis=1)
    print(f"loop: keyframe error mean {err_before.mean():.3f} -> {err_after.mean():.3f} m, max {err_before.max():.3f} -> {err_after.max():.3f} m")
    assert err_after.mean() < 0.6 * err_before.mean() and err_after.max() < 0.7 * err_before.max()
    # the map rebuilt at the corrected poses, against the map rebuilt at the true poses
    ids = np.arange(n, dtype=np.int32)
    ctx.map_from_keyframes(ctx, ids, opt, 1)
    assert np.array_equal(ctx.keyframe_poses(), opt)
    gt = _ctx(gpu_api)
    gt.map_set_origin(truth[0][:3])
    gt.map_from_keyframes(ctx, ids, truth, 1)
    gt_map = gt.map_download(0)
    far_live, far_rebuilt = _share_far(live_map, gt_map, 0.2), _share_far(ctx.map_download(0), gt_map, 0.2)
    print(f"loop: map points farther than planeRes from the ground-truth rebuild {far_live:.4f} -> {far_rebuilt:.4f}")
    assert far_rebuilt < 0.6 * far_live
    # the next live registration on the corrected map, back at the start
    prior = _compose(opt[-1], _compose(_inverse(truth[n - 1]), truth[0]))
    r = ctx.register(synth.make_scan(scene, "vlp16", truth[0], 6000, rmax=20.0), prior, 10, mf)
    nxt_err = np.linalg.norm(np.array(r.pose)[:3] - truth[0, :3])
    print(f"loop: next registration error {nxt_err:.3f} m")
    assert r.status == 0 and nxt_err < 0.1
    for x in (ctx, sub, gt):
        x.close()


@pytest.mark.gpu
def test_keyframe_shim_sequence(gpu_api, tmp_path):
    """tests/cpp/keyframe_test.cpp: keyframes from a live sequence, a submap of the first two, the last aligned against it, the map
    rebuilt with the loop result; the shim's T_w_lidar is the corrected last keyframe pose, and its keyframe poses are the
    registrations' poses."""
    import struct
    import subprocess
    from test_cpp_shim import _build, _sequence
    exe = _build(tmp_path, "keyframe_test")
    _, scans, priors = _sequence(5)
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiif", len(scans), 5, 0, 0.2))
        for s, p in zip(scans, priors):
            f.write(struct.pack("<i", len(s)))
            f.write(np.asarray(p, np.float64).tobytes())
            f.write(np.ascontiguousarray(s, np.float32).tobytes())
    out = subprocess.run([exe, str(path)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = [ln.split() for ln in out.stdout.strip().splitlines()]
    kf = [ln for ln in lines if ln[0] == "kf"]
    loop = [ln for ln in lines if ln[0] == "loop"][0]
    rebuilt = [ln for ln in lines if ln[0] == "rebuilt"][0]
    assert [int(ln[1]) for ln in kf] == list(range(len(scans) - 1))
    assert int(loop[1]) == 0
    assert int(rebuilt[1]) == len(kf) and int(rebuilt[2]) > 1000
    assert rebuilt[3:] == loop[2:]                                     # T_w_lidar: the corrected last keyframe
    for ln, p in zip(kf, priors[1:]):
        assert np.linalg.norm(np.array(ln[2:5], float) - np.asarray(p[:3])) < 0.3

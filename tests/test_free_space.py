"""so_map_clear_free_space* on the device: the removal set against the numpy restatement (tests/free_space_numpy.py), the order and
index of the carved store, the registered form in every undistortion mode, both stores and the block archive, a live loop with a
moving vehicle, and the argument errors."""
import numpy as np
import pytest

from superodom_b200 import synth
import free_space_numpy as F
import optimized_numpy as ON

pytestmark = pytest.mark.gpu


def _opts(api, sensor, **kw):
    o = F.opts_for(sensor, **kw)
    return api.free_space(**{n: getattr(o, n) for n, _ in api.FreeSpace._fields_}), o


def _box_points(box, leaf=0.2, seed=9):
    """Voxel-filtered surface samples of one box: what a parked object leaves in the map."""
    only = synth.Scene(room=np.asarray(box, np.float64) + np.array([-1, 1, -1, 1, -1, 1]), boxes=np.asarray(box, np.float64)[None])
    raw = synth.sample_surfaces(only, leaf, seed=seed)
    lo, hi = np.array([box[0], box[2], box[4]]) - 0.1, np.array([box[1], box[3], box[5]]) + 0.1
    raw = raw[((raw[:, :3] >= lo) & (raw[:, :3] <= hi)).all(1)]
    return synth.voxel_filter_blocks(np.c_[raw, np.ones(len(raw), np.float32)], leaf)


def _free_box(scene, pose, size=(4.5, 1.9, 1.6), dist=(5.0, 9.0), seed=0, avoid=None):
    """A box on the floor `dist` metres from the sensor, clear of the scene (and of `avoid`) and in its line of sight."""
    rng = np.random.default_rng(seed)
    for _ in range(2000):
        a, r = rng.uniform(-np.pi, np.pi), rng.uniform(*dist)
        c = pose[:2] + r * np.array([np.cos(a), np.sin(a)])
        box = np.array([c[0] - size[0] / 2, c[0] + size[0] / 2, c[1] - size[1] / 2, c[1] + size[1] / 2, -1.8, -1.8 + size[2]])
        if not scene.free(np.array([c[0], c[1], -1.0]), margin=max(size[:2]) / 2 + 0.5):
            continue
        if avoid is not None and np.hypot(*(c - 0.5 * np.array([avoid[0] + avoid[1], avoid[2] + avoid[3]]))) < 6.0:
            continue
        d = np.array([c[0], c[1], -1.0]) - pose[:3]
        if synth.raycast(scene, pose[:3], (d / np.linalg.norm(d))[None])[0] > np.linalg.norm(d):
            return box
    raise RuntimeError("no free box position")


def _scene_with(scene, box):
    return synth.Scene(room=scene.room, boxes=np.vstack([scene.boxes, np.asarray(box, np.float64)[None]]))


_CASES = {}


def _case(name, k=0):
    """static map + the points of a box that is no longer there; the scan sees through where it stood"""
    if (name, k) not in _CASES:
        scene, mp = synth.make_map_for(name)
        c = synth.make_case_on(scene, mp, name, k)
        box = _free_box(scene, c["pose_true"], seed=k)
        _CASES[(name, k)] = dict(scene=scene, static=mp, ghost=_box_points(box), case=c, box=box,
                                 map=np.vstack([mp, _box_points(box)]))
    return _CASES[(name, k)]


def _ctx(api, n_map, plane_res=0.2, **kw):
    return api.Context(max_map_points=max(1 << 20, 2 * n_map + 300000), max_scan_points=262144, plane_res=plane_res, **kw)


def _removed(before, after):
    """-> mask of the rows of `before` that are gone, and the check that `after` is `before` without them, bit for bit, in order"""
    keys_after = {r.tobytes() for r in after}
    gone = np.array([r.tobytes() not in keys_after for r in before])
    assert np.array_equal(before[~gone].view(np.uint32), after.view(np.uint32))
    return gone


@pytest.mark.parametrize("name", ["tiny", "cfg1", "cfg2"])
def test_removal_set_lies_between_the_restatement_bounds(gpu_api, name):
    d = _case(name)
    c = d["case"]
    sensor = c["cfg"]["sensor"]
    ctx = _ctx(gpu_api, len(d["map"]))
    ctx.map_set_points(d["map"])
    before = ctx.map_download()
    o, of = _opts(gpu_api, sensor)
    r = ctx.map_clear_free_space(c["scan_xyzi"], c["pose_true"], o)
    after = ctx.map_download()
    gone = _removed(before, after)
    lo, hi = F.bounds(before, c["scan_xyzi"], c["pose_true"], of)
    _, st = F.clear(before, c["scan_xyzi"], c["pose_true"], of)
    print(f"{name}: device removed {gone.sum()}, numpy lower {lo.sum()} upper {hi.sum()} (differ by {int(hi.sum() - lo.sum())}); "
          f"ghost points {len(d['ghost'])}; result {r}")
    assert gone.sum() > 0.2 * len(d["ghost"])
    assert not (lo & ~gone).any() and not (gone & ~hi).any()
    assert hi.sum() - lo.sum() <= 20
    assert r["n_removed"] == gone.sum() and r["n_after"] == (len(after), 0)
    assert r["n_image_points"] == st["n_image_points"] and r["n_pixels_hit"] == st["n_pixels_hit"]
    assert abs(r["n_candidates"] - st["n_candidates"]) <= hi.sum() - lo.sum() + 20


def test_carved_store_registers_as_the_oracle_with_the_kept_cloud(gpu_api):
    from oracle import oracle as O
    d = _case("cfg2")
    c = d["case"]
    ctx = _ctx(gpu_api, len(d["map"]))
    ctx.map_set_points(d["map"])
    r = ctx.map_clear_free_space(c["scan_xyzi"], c["pose_true"], _opts(gpu_api, "os1_128")[0])
    assert r["n_removed"] > 0
    kept = ctx.map_download()
    c2 = synth.make_case_on(d["scene"], d["static"], "cfg2", 3)
    g = ctx.register(c2["scan_xyzi"], c2["pose_prior"], 20)
    ro = O.OracleMap(kept).register(c2["scan_xyzi"], c2["pose_prior"], 0.2, 20, knn_mode=0)
    dp = np.abs(np.array(g.pose) - np.array(ro.pose)).max()
    print(f"carved cfg2 store: {r['n_removed']} removed; registration |gpu - oracle| = {dp:.2e}, {g.n_iterations} iterations")
    assert g.status == 0 and g.n_iterations == ro.n_iterations and dp < 1e-4
    # nothing removed: the store is left bit for bit, and a search gives what it gave
    ctx2 = _ctx(gpu_api, len(d["static"]))
    ctx2.map_set_points(d["static"])
    b0 = ctx2.map_download()
    k0 = ctx2.knn(c2["scan_xyzi"][:4096, :3] + 0.3, 5, 0.0)
    r0 = ctx2.map_clear_free_space(c["scan_xyzi"], c["pose_true"], _opts(gpu_api, "os1_128")[0])
    assert r0["n_removed"] == 0
    assert np.array_equal(b0.view(np.uint32), ctx2.map_download().view(np.uint32))
    k1 = ctx2.knn(c2["scan_xyzi"][:4096, :3] + 0.3, 5, 0.0)
    assert all(np.array_equal(a, b) for a, b in zip(k0, k1))


def _moving(name="cfg1", k=0):
    key = ("moving", name, k)
    if key not in _CASES:
        scene, mp = synth.make_map_for(name)
        pose = synth.random_sensor_pose(scene, 950 + k, 8.0)
        dd = synth.make_moving_scan(scene, synth.CONFIGS[name]["sensor"], pose, 5.0, 0.5, 60 + k)
        box = _free_box(scene, pose, seed=20 + k)
        dd.update(scene=scene, map=np.vstack([mp, _box_points(box)]), cfg=synth.CONFIGS[name])
        _CASES[key] = dd
    return _CASES[key]


@pytest.mark.parametrize("mode", ["none", "approximated", "optimized"])
def test_registered_form_equals_the_host_form(gpu_api, mode):
    d = _moving()
    o = _opts(gpu_api, "vlp16")[0]
    a, b = _ctx(gpu_api, len(d["map"])), _ctx(gpu_api, len(d["map"]))
    a.map_set_points(d["map"]); b.map_set_points(d["map"])
    scan, prior = d["scan_xyzi"], d["prior"]
    if mode == "none":
        pose = np.array(a.register(scan, prior, 5, 2000).pose)
        cloud = scan
    elif mode == "approximated":
        u = gpu_api.undistort(d["pose_prev"], 0.1)
        pose = np.array(a.register_undistort(scan, prior, u, 5, 2000).pose)
        cloud = b.undistort_points(scan, pose, u)
    else:
        r = a.register_optimized(scan, prior, gpu_api.motion(0.1), 5, 2000)
        pose = np.array(r.icp.pose)
        cloud = np.concatenate([ON.warp_points(scan, np.array(r.motion), 0.1), scan[:, 3:4]], 1)
    ra = a.map_clear_free_space_registered(pose, o)
    rb = b.map_clear_free_space(cloud, pose, o)
    print(f"{mode}: {ra}")
    assert ra == rb and ra["n_removed"] > 0
    assert np.array_equal(a.map_download().view(np.uint32), b.map_download().view(np.uint32))
    a.map_add_registered_scan(pose)                      # the record is still valid
    b.map_add_scan(cloud, pose)
    assert np.array_equal(a.map_download().view(np.uint32), b.map_download().view(np.uint32))


def test_both_stores_and_the_archive(gpu_api):
    d = _case("cfg1")
    c = d["case"]
    o = _opts(gpu_api, "vlp16")[0]
    edge = d["map"][::3]
    a, b = _ctx(gpu_api, len(d["map"])), _ctx(gpu_api, len(d["map"]))
    for x in (a, b):
        x.map_set_points(d["map"]); x.map_set_edge_points(edge)
    ra = a.map_clear_free_space(c["scan_xyzi"], c["pose_true"], o, stores=3)
    rb1 = b.map_clear_free_space(c["scan_xyzi"], c["pose_true"], o, stores=1)
    rb2 = b.map_clear_free_space(c["scan_xyzi"], c["pose_true"], o, stores=2)
    print(f"stores=3: {ra}; surf {rb1}; edge {rb2}")
    assert rb2["n_removed"] > 0 and ra["n_removed"] == rb1["n_removed"] + rb2["n_removed"]
    assert ra["n_after"] == rb2["n_after"]
    assert np.array_equal(a.map_download().view(np.uint32), b.map_download().view(np.uint32))
    # archive on, a copy of the map 2 km away lives in the archive: it is never carved and comes back unchanged
    far = d["map"].copy()
    far[:, 0] += 2000.0
    ctx = _ctx(gpu_api, len(d["map"]))
    ctx.map_archive(len(far) + 1024)
    ctx.map_set_points(np.vstack([d["map"], far]))
    all0 = ctx.map_download_all(0)
    win0 = ctx.map_download()
    r = ctx.map_clear_free_space(c["scan_xyzi"], c["pose_true"], o)
    assert r["n_removed"] > 0
    all1 = ctx.map_download_all(0)
    far0, far1 = all0[all0[:, 0] > 1000], all1[all1[:, 0] > 1000]
    assert np.array_equal(far0.view(np.uint32), far1.view(np.uint32))
    assert ctx.map_archive_info(0)[0] == len(far0)
    assert len(ctx.map_download()) == len(win0) - r["n_removed"]
    ctx.map_shift([2000.0, 0.0, 0.0])
    back = ctx.map_download()
    srt = lambda x: x[np.lexsort(x.view(np.uint32).T[::-1])]
    assert np.array_equal(srt(back).view(np.uint32), srt(far0).view(np.uint32))


def test_bad_arguments_leave_both_stores(gpu_api):
    d = _case("tiny")
    c = d["case"]
    ctx = _ctx(gpu_api, len(d["map"]))
    ctx.map_set_points(d["map"]); ctx.map_set_edge_points(d["map"][::4])
    before = ctx.map_download()
    bad = [dict(az_res_deg=0.0), dict(az_res_deg=float("nan")), dict(el_res_deg=-1.0), dict(el_res_deg=float("inf")),
           dict(el_min_deg=10.0, el_max_deg=10.0), dict(el_min_deg=10.0, el_max_deg=-10.0), dict(az_res_deg=0.001, el_res_deg=0.001),
           dict(dilate=-1), dict(dilate=5), dict(margin=-0.1), dict(margin_rel=-0.01), dict(min_range=5.0, max_range=5.0),
           dict(min_range=10.0, max_range=1.0)]
    for kw in bad:
        with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
            ctx.map_clear_free_space(c["scan_xyzi"], c["pose_true"], gpu_api.free_space(**kw))
    for stores in (0, 4, -1):
        with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
            ctx.map_clear_free_space(c["scan_xyzi"], c["pose_true"], None, stores=stores)
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
        ctx.map_clear_free_space_registered(c["pose_true"], gpu_api.free_space(dilate=7))
    assert np.array_equal(before.view(np.uint32), ctx.map_download().view(np.uint32))
    # a fresh context has no registered scan: nothing happens
    assert ctx.map_clear_free_space_registered(c["pose_true"])["n_removed"] == 0
    ctx.scan_prefilter(c["scan_xyzi"], 0.2, 0.2, auto_voxel_size=False, download=False)
    ctx.register(c["scan_xyzi"], c["pose_prior"], 5)
    ctx.scan_prefilter(c["scan_xyzi"], 0.2, 0.2, auto_voxel_size=False, download=False)       # overwrites the registered scan
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\)"):
        ctx.map_clear_free_space_registered(c["pose_true"])
    assert np.array_equal(before.view(np.uint32), ctx.map_download().view(np.uint32))


def test_live_loop_with_a_moving_vehicle(gpu_api):
    """register -> clear -> insert over 60 OS1-128 scans in a cfg1-sized scene: a vehicle parked at A, driving off, parked at B."""
    from scipy.spatial import cKDTree
    scene, static = synth.make_map_for("cfg1")
    pose0 = synth.random_sensor_pose(scene, 905, 5.0)
    A = _free_box(scene, pose0, seed=31)
    B = _free_box(scene, pose0, seed=32, avoid=A)
    n = 60

    def box_at(k):
        if k < 20:
            return A
        if k >= 40:
            return B
        t = (k - 19) / 21.0
        return A + t * (B - A)

    poses = []
    for k in range(n):                                        # the sensor creeps along x, 2 cm per scan, where the scene is free
        p = pose0.copy()
        p[0] += 0.02 * k
        poses.append(p)
    scans = [synth.make_scan(_scene_with(scene, box_at(k)), "os1_128", poses[k], 4000 + k) for k in range(n)]
    o = _opts(gpu_api, "os1_128")[0]
    out = {}
    for arm in ("clear", "plain"):
        ctx = _ctx(gpu_api, len(static) + 2000000)
        ctx.map_set_points(static)
        prev = poses[0]
        errs = []
        for k in range(n):
            r = ctx.register(scans[k], prev, 10, 2000)
            assert r.status == 0, (arm, k, r.status)
            pose = np.array(r.pose)
            errs.append(np.linalg.norm(pose[:3] - poses[k][:3]))
            if arm == "clear":
                ctx.map_clear_free_space_registered(pose, o)
            ctx.map_add_registered_scan(pose)
            prev = pose
        out[arm] = (ctx.map_download(), np.array(errs))
        ctx.close()
    tree = cKDTree(static[:, :3])
    boxes = [box_at(k) for k in range(n)]

    def near_box(p, b, m=0.3):
        return ((p[:, :3] >= np.array([b[0], b[2], b[4]]) - m) & (p[:, :3] <= np.array([b[1], b[3], b[5]]) + m)).all(1)

    res = {}
    for arm, (m, errs) in out.items():
        past = np.zeros(len(m), bool)
        for b in boxes:
            past |= near_box(m, b)
        far_static = tree.query(m[:, :3], k=1)[0] > 0.3
        ghost = past & far_static & ~near_box(m, boxes[-1])
        stat = ~past
        res[arm] = (int(ghost.sum()), int(stat.sum()))
        print(f"{arm}: {len(m)} map points, ghost {ghost.sum()}, static {stat.sum()}; position error per scan (m): "
              + " ".join(f"{e:.3f}" for e in errs))
    assert res["plain"][0] > 100
    assert res["clear"][0] <= 0.1 * res["plain"][0]
    assert res["plain"][1] - res["clear"][1] <= 0.001 * res["plain"][1]


def test_shim_localization_clears_before_inserting(tmp_path, gpu_api):
    """LidarSLAM::ClearFreeSpace: Localization carves the maps with the registered scan right before its inserts (the same maps as
    register -> so_map_clear_free_space_registered(stores 3) -> insert through the ABI); off, the maps are those of the plain loop."""
    import os
    import struct
    import subprocess
    from superodom_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = build.build()
    exe = str(tmp_path / "free_space_shim_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "free_space_shim_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    scene, _ = synth.make_map_for("tiny")
    pose0 = synth.random_sensor_pose(scene, 900, 4.0)
    box = _free_box(scene, pose0, seed=5)
    scans = [synth.make_scan(_scene_with(scene, box) if i < 2 else scene, "vlp16", pose0, 500 + i) for i in range(5)]
    priors = [pose0] + [synth.perturb_pose(pose0, 600 + i, 0.05, 0.5) for i in range(1, 5)]
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(scans)))
        for s, p in zip(scans, priors):
            f.write(struct.pack("<i", len(s)))
            f.write(np.asarray(p, np.float64).tobytes())
            f.write(np.ascontiguousarray(s, np.float32).tobytes())
    o = gpu_api.free_space(az_res_deg=0.4, el_res_deg=2.0, el_min_deg=-16.0, el_max_deg=16.0)
    for flag in ("off", "on"):
        out = subprocess.run([exe, str(path), flag, str(tmp_path / "map.bin")], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
        rows = [list(map(int, ln.split())) for ln in out.stdout.strip().splitlines()]
        shim_map = np.fromfile(tmp_path / "map.bin", np.float32).reshape(-1, 4)
        ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=1 << 17, plane_res=0.2, line_res=0.1)
        ctx.map_set_origin(priors[0][:3])
        ctx.map_add_scan(scans[0], priors[0])
        removed = []
        for i in range(1, len(scans)):
            pose = np.array(ctx.register(scans[i], priors[i], 5, 0).pose)
            if flag == "on":
                r = ctx.map_clear_free_space_registered(pose, o, stores=3)
                removed.append(r["n_removed"])
                assert rows[i][1] == r["n_removed"] and rows[i][2] == r["n_after"][0]
            ctx.map_add_registered_scan(pose)
            assert rows[i][3] == ctx.map_size()
        print(f"shim, clearing {flag}: removed per scan {[r[1] for r in rows]}, map {len(shim_map)} points")
        assert np.array_equal(shim_map.view(np.uint32), ctx.map_download().view(np.uint32))
        if flag == "on":
            assert sum(removed) > 0
        else:
            assert all(r[1] == 0 for r in rows)
        ctx.close()

"""so_map_clear_free_space_keyframes on the device: bit for bit the map that so_map_clear_free_space of each keyframe in turn leaves (both
stores, the index, the counts), across image tiles, on another context's prior map, and after a loop-closure rebuild that brought back
what the live clearing removed; the argument errors; and the shim's rebuildFromKeyframes(corrected, opts)."""
import numpy as np
import pytest

from superodom_b200 import synth
import free_space_numpy as F

pytestmark = pytest.mark.gpu

N_SCANS = 60


def _opts(api, **kw):
    o = F.opts_for("os1_128")
    return api.free_space(**{**{n: getattr(o, n) for n, _ in api.FreeSpace._fields_}, **kw})


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


def _ctx(api, n_map, plane_res=0.2, **kw):
    return api.Context(max_map_points=max(1 << 20, 2 * n_map + 300000), max_scan_points=262144, plane_res=plane_res, **kw)


def _near_box(p, b, m=0.3):
    return ((p[:, :3] >= np.array([b[0], b[2], b[4]]) - m) & (p[:, :3] <= np.array([b[1], b[3], b[5]]) + m)).all(1)


_SESSION = {}


def _session(api):
    """The live loop of test_live_loop_with_a_moving_vehicle (60 OS1-128 scans; a vehicle parked at A, driving off, parked at B), run
    with live clearing, every registered scan kept as a keyframe at its registered pose.  Returns the context that holds them."""
    if "ctx" in _SESSION:
        return _SESSION
    scene, static = synth.make_map_for("cfg1")
    pose0 = synth.random_sensor_pose(scene, 905, 5.0)
    A = _free_box(scene, pose0, seed=31)
    B = _free_box(scene, pose0, seed=32, avoid=A)

    def box_at(k):
        if k < 20:
            return A
        if k >= 40:
            return B
        return A + (k - 19) / 21.0 * (B - A)

    poses = []
    for k in range(N_SCANS):                                  # the sensor creeps along x, 2 cm per scan, where the scene is free
        p = pose0.copy()
        p[0] += 0.02 * k
        poses.append(p)
    scans = [synth.make_scan(_scene_with(scene, box_at(k)), "os1_128", poses[k], 4000 + k) for k in range(N_SCANS)]
    o = _opts(api)
    ctx = _ctx(api, len(static) + 2000000)
    ctx.map_set_points(static)
    ctx.keyframe_reserve(sum(len(s) for s in scans) + 1024, N_SCANS)
    prev = poses[0]
    for k in range(N_SCANS):
        r = ctx.register(scans[k], prev, 10, 2000)
        assert r.status == 0, (k, r.status)
        pose = np.array(r.pose)
        ctx.map_clear_free_space_registered(pose, o)
        assert ctx.keyframe_add_registered(pose) == k
        ctx.map_add_registered_scan(pose)
        prev = pose
    _SESSION.update(ctx=ctx, static=static, boxes=[box_at(k) for k in range(N_SCANS)], B=B, live=ctx.map_download(),
                    poses=ctx.keyframe_poses())
    return _SESSION


def _copy_session(api, s):
    """A second context holding the same keyframes, imported verbatim (a download / import round trip is bit-exact)."""
    src = s["ctx"]
    ctx = _ctx(api, len(s["static"]) + 2000000)
    n_frames, n_surf, n_edge = src.keyframe_info()
    ctx.keyframe_reserve(max(n_surf, n_edge) + 1024, n_frames)
    for i in range(n_frames):
        ctx.keyframe_import(src.keyframe_download(i, 0), s["poses"][i], src.keyframe_download(i, 1))
    return ctx


def _sequential(ctx, src, ids, poses, o, stores):
    """The definition: so_map_clear_free_space of each keyframe's downloaded surf cloud in turn -> summed results"""
    tot = dict(n_image_points=0, n_pixels_hit=0, n_removed=0)
    r = None
    for i, p in zip(ids, poses):
        r = ctx.map_clear_free_space(src.keyframe_download(int(i), 0), p, o, stores=stores)
        for k in tot:
            tot[k] += r[k]
    tot["n_after"] = r["n_after"]
    return tot


def _rebuild(ctx, ids, poses, edge_every=3):
    """so_map_from_keyframes of the context's own keyframes, then an edge store (every edge_every-th surf point) so that both stores
    hold points"""
    ctx.map_from_keyframes(ctx, ids, poses, stores=3)
    ctx.map_set_edge_points(ctx.map_download()[::edge_every].copy())


def _same_maps(a, b, probe):
    assert np.array_equal(a.map_download().view(np.uint32), b.map_download().view(np.uint32))
    assert a.map_size() == b.map_size()
    ka, kb = a.knn(probe, 5, 0.0), b.knn(probe, 5, 0.0)
    assert all(np.array_equal(x, y) for x, y in zip(ka, kb))


def _probe(s, n=8192, seed=3):
    rng = np.random.default_rng(seed)
    m = s["live"][rng.choice(len(s["live"]), n)]
    return (m[:, :3] + rng.normal(0, 0.3, (n, 3))).astype(np.float32)


def _check_equals_sequential(api, o, chunks=None):
    s = _session(api)
    a = s["ctx"]
    b = _copy_session(api, s)
    ids = np.arange(N_SCANS, dtype=np.int32)
    poses = s["poses"]
    _rebuild(a, ids, poses)
    _rebuild(b, ids, poses)
    assert np.array_equal(a.map_download().view(np.uint32), b.map_download().view(np.uint32))
    n_before = a.map_download()
    if chunks is None:
        ra = a.map_clear_free_space_keyframes(a, ids, poses, o, stores=3)
    else:                                                  # the same keyframes in calls of `chunks` ids
        ra = dict(n_image_points=0, n_pixels_hit=0, n_removed=0, n_tiles=0)
        for c0 in range(0, N_SCANS, chunks):
            r = a.map_clear_free_space_keyframes(a, ids[c0:c0 + chunks], poses[c0:c0 + chunks], o, stores=3)
            for k in ("n_image_points", "n_pixels_hit", "n_removed", "n_tiles"):
                ra[k] += r[k]
            ra["n_after"] = r["n_after"]
    rb = _sequential(b, b, ids, poses, o, 3)
    print(f"batched {ra}; sequential {rb}; map {len(n_before)} -> {len(a.map_download())}")
    assert ra["n_removed"] > 0
    for k in ("n_image_points", "n_pixels_hit", "n_removed", "n_after"):
        assert ra[k] == rb[k], (k, ra[k], rb[k])
    _same_maps(a, b, _probe(s))
    b.close()
    return ra, a.map_download()


def test_equals_the_sequential_calls_bit_for_bit(gpu_api):
    r, _ = _check_equals_sequential(gpu_api, _opts(gpu_api))
    assert r["n_tiles"] == 1 and r["n_keyframes"] == N_SCANS and r["n_candidates"] >= r["n_removed"] and r["time_ms"] > 0
    assert r["n_after"][1] > 0


def test_tiles_give_the_map_of_one_tile(gpu_api):
    """0.1 degree pixels: 3600 x 460 pixels, 6.6 MB an image, 40 images a tile, so the 60 keyframes take two tiles; the map equals the
    sequential calls' and that of calls of 30 keyframes, one tile each.  Pixels that fine are finer than the OS1-128's beams, so no
    5 x 5 neighbourhood is fully observed: dilate 0 tests the single pixel."""
    o = _opts(gpu_api, az_res_deg=0.1, el_res_deg=0.1, dilate=0)
    r, m2 = _check_equals_sequential(gpu_api, o)
    assert r["n_tiles"] >= 2
    r1, m1 = _check_equals_sequential(gpu_api, o, chunks=30)
    assert r1["n_tiles"] == 2 and r1["n_removed"] == r["n_removed"]
    assert np.array_equal(m1.view(np.uint32), m2.view(np.uint32))


def test_another_contexts_prior_map(gpu_api):
    """dst != src: a prior map (the static map and what the vehicle left at A) cleared with the session's keyframes, and a map with
    nothing to remove left bit for bit"""
    s = _session(gpu_api)
    src = s["ctx"]
    A = s["boxes"][0]
    seen = src.keyframe_download(0, 0, s["poses"][0])                   # the vehicle at A as the first keyframe saw it
    prior = np.vstack([s["static"], seen[_near_box(seen, A, 0.1)]]).astype(np.float32)
    ids = np.arange(N_SCANS, dtype=np.int32)[::-1].copy()              # any order, with a duplicate
    ids = np.concatenate([ids, ids[:3]])
    poses = s["poses"][ids]
    o = _opts(gpu_api)
    a, b = _ctx(gpu_api, len(prior)), _ctx(gpu_api, len(prior))
    for x in (a, b):
        x.map_set_points(prior)
        x.map_set_edge_points(prior[::4].copy())
    ra = a.map_clear_free_space_keyframes(src, ids, poses, o, stores=3)
    rb = _sequential(b, src, ids, poses, o, 3)
    print(f"prior map {len(prior)} points: batched {ra}; sequential {rb}")
    assert ra["n_removed"] > 0 and _near_box(prior, A).sum() > 0
    for k in ("n_image_points", "n_pixels_hit", "n_removed", "n_after"):
        assert ra[k] == rb[k], (k, ra[k], rb[k])
    _same_maps(a, b, _probe(s))
    # nothing to remove (a margin of a kilometre): every point tested, none removed, the store untouched
    c = _ctx(gpu_api, len(prior))
    c.map_set_points(prior)
    before = c.map_download()
    probe = _probe(s)
    k0 = c.knn(probe, 5, 0.0)
    r0 = c.map_clear_free_space_keyframes(src, ids, poses, _opts(gpu_api, margin=1000.0), stores=1)
    assert r0["n_removed"] == 0 and r0["n_candidates"] > 0
    assert np.array_equal(before.view(np.uint32), c.map_download().view(np.uint32))
    k1 = c.knn(probe, 5, 0.0)
    assert all(np.array_equal(x, y) for x, y in zip(k0, k1))
    for x in (a, b, c):
        x.close()


def test_the_rebuild_keeps_out_what_the_live_clearing_removed(gpu_api):
    """Live clearing keeps the vehicle's trail out of the live map; the rebuild from keyframes brings it back; the batched clearing
    takes it out again and loses almost nothing static."""
    from scipy.spatial import cKDTree
    s = _session(gpu_api)
    ctx = s["ctx"]
    ids = np.arange(N_SCANS, dtype=np.int32)
    tree = cKDTree(s["static"][:, :3])
    boxes, B = s["boxes"], s["B"]

    def count(m):
        past = np.zeros(len(m), bool)
        for b in boxes:
            past |= _near_box(m, b)
        far_static = tree.query(m[:, :3], k=1)[0] > 0.3
        return int((past & far_static & ~_near_box(m, B)).sum()), int((~past).sum()), int((_near_box(m, B) & far_static).sum())

    live = count(s["live"])
    ctx.map_from_keyframes(ctx, ids, s["poses"], stores=3)
    plain = count(ctx.map_download())
    r = ctx.map_clear_free_space_keyframes(ctx, ids, s["poses"], _opts(gpu_api), stores=3)
    cleared = count(ctx.map_download())
    print(f"ghost / static / vehicle at B: live {live}, rebuilt {plain}, rebuilt and cleared {cleared}; {r}")
    assert plain[0] > 100
    assert cleared[0] <= 0.1 * plain[0]
    assert plain[1] - cleared[1] <= 0.001 * plain[1]


def test_bad_arguments_leave_both_stores(gpu_api):
    import ctypes as C
    s = _session(gpu_api)
    src = s["ctx"]
    prior = s["static"]
    ctx = _ctx(gpu_api, len(prior))
    ctx.map_set_points(prior)
    ctx.map_set_edge_points(prior[::4].copy())
    before = ctx.map_download()
    ids = np.arange(4, dtype=np.int32)
    poses = s["poses"][:4].copy()
    err = r"\(-1\)"
    bad = [dict(az_res_deg=0.0), dict(el_res_deg=float("nan")), dict(el_min_deg=10.0, el_max_deg=10.0), dict(az_res_deg=0.001, el_res_deg=0.001),
           dict(dilate=5), dict(margin=-0.1), dict(margin_rel=float("inf")), dict(min_range=5.0, max_range=5.0)]
    for kw in bad:
        with pytest.raises(gpu_api.SuperOdomError, match=err):
            ctx.map_clear_free_space_keyframes(src, ids, poses, gpu_api.free_space(**kw))
    for stores in (0, 4, -1):
        with pytest.raises(gpu_api.SuperOdomError, match=err):
            ctx.map_clear_free_space_keyframes(src, ids, poses, None, stores=stores)
    for bad_ids in ([0, 1, -1], [0, N_SCANS]):
        with pytest.raises(gpu_api.SuperOdomError, match=err):
            ctx.map_clear_free_space_keyframes(src, np.array(bad_ids), s["poses"][:len(bad_ids)])
    for k, v in ((0, np.nan), (5, np.inf)):
        p = poses.copy()
        p[2, k] = v
        with pytest.raises(gpu_api.SuperOdomError, match=err):
            ctx.map_clear_free_space_keyframes(src, ids, p)
    p = poses.copy()
    p[1, 3:] = 0.0                                                        # a zero quaternion
    with pytest.raises(gpu_api.SuperOdomError, match=err):
        ctx.map_clear_free_space_keyframes(src, ids, p)
    with pytest.raises(gpu_api.SuperOdomError, match=err):              # no keyframe store in src
        ctx.map_clear_free_space_keyframes(ctx, ids, poses)
    o = gpu_api.free_space()
    L = ctx.L
    for args in ((None, 4, poses.ctypes.data_as(C.c_void_p)), (ids.ctypes.data_as(C.c_void_p), 4, None)):
        assert L.so_map_clear_free_space_keyframes(ctx.h, src.h, args[0], args[1], args[2], 1, C.byref(o), None) == -1
    assert L.so_map_clear_free_space_keyframes(ctx.h, src.h, ids.ctypes.data_as(C.c_void_p), 4, poses.ctypes.data_as(C.c_void_p), 1,
                                               None, None) == -1
    assert np.array_equal(before.view(np.uint32), ctx.map_download().view(np.uint32))
    r = ctx.map_clear_free_space_keyframes(src, np.zeros(0, np.int32), np.zeros((0, 7)), o, stores=3)   # no keyframes: nothing happens
    assert r["n_removed"] == 0 and r["n_keyframes"] == 0 and sum(r["n_after"]) == len(before)
    assert np.array_equal(before.view(np.uint32), ctx.map_download().view(np.uint32))
    ctx.close()


def test_shim_rebuild_clears_against_every_keyframe(tmp_path, gpu_api):
    """LidarSLAM::rebuildFromKeyframes(corrected, opts) after a live loop with ClearFreeSpace on: the map of the same ABI sequence, bit
    for bit (register -> clear registered -> keyframe -> insert; so_map_from_keyframes; so_map_clear_free_space_keyframes, stores 3)."""
    import os
    import struct
    import subprocess
    from superodom_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = build.build()
    exe = str(tmp_path / "keyframe_clear_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "keyframe_clear_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    scene, _ = synth.make_map_for("tiny")
    pose0 = synth.random_sensor_pose(scene, 900, 4.0)
    box = _free_box(scene, pose0, seed=5)
    scans = [synth.make_scan(_scene_with(scene, box) if i < 3 else scene, "vlp16", pose0, 500 + i) for i in range(7)]
    priors = [pose0] + [synth.perturb_pose(pose0, 600 + i, 0.05, 0.5) for i in range(1, 7)]
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(scans)))
        for sc, p in zip(scans, priors):
            f.write(struct.pack("<i", len(sc)))
            f.write(np.asarray(p, np.float64).tobytes())
            f.write(np.ascontiguousarray(sc, np.float32).tobytes())
    out = subprocess.run([exe, str(path), str(tmp_path / "map.bin")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    corrected = np.array([[float(v) for v in ln.split()[2:]] for ln in lines if ln.startswith("kf ")])
    clear = [int(v) for v in lines[-1].split()[1:]]
    shim_map = np.fromfile(tmp_path / "map.bin", np.float32).reshape(-1, 4)
    o = gpu_api.free_space(az_res_deg=0.4, el_res_deg=2.0, el_min_deg=-16.0, el_max_deg=16.0)
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=1 << 17, plane_res=0.2, line_res=0.1)
    ctx.keyframe_reserve(len(scans) << 17, len(scans))
    ctx.map_set_origin(priors[0][:3])
    ctx.map_add_scan(scans[0], priors[0])
    for i in range(1, len(scans)):
        pose = np.array(ctx.register(scans[i], priors[i], 5, 0).pose)
        ctx.map_clear_free_space_registered(pose, o, stores=3)
        ctx.keyframe_add_registered(pose)
        ctx.map_add_registered_scan(pose)
    ids = np.arange(len(corrected), dtype=np.int32)
    ctx.map_from_keyframes(ctx, ids, corrected, stores=3)
    r = ctx.map_clear_free_space_keyframes(ctx, ids, corrected, o, stores=3)
    print(f"shim rebuild + clear: {clear}; ABI {r}")
    assert clear == [r["n_keyframes"], r["n_removed"], r["n_after"][0], r["n_after"][1], r["n_tiles"]]
    assert len(corrected) == len(scans) - 1
    assert np.array_equal(shim_map.view(np.uint32), ctx.map_download().view(np.uint32))
    ctx.close()

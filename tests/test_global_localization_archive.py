"""Global localization over the whole archived prior map (so_global_opts.whole_map = 1): the search sees the window and the block
archive, and each kept candidate is registered in the window so_map_shift(prior) would give, with the window left at the winner.

Scene: three cfg2-sized rooms at x = -800, 0 and +800 m (1.70 km, about 3 M points), the archive on, the window in room A, so
that room C lies wholly in the archive.
CPU: the whole_map argument check and the struct layouts; the shim program builds.
GPU: so_map_bounds_all; scores, keys and bounds over a window face against the numpy restatements on the whole-map cloud; the
refinement against shift-then-so_register_batch; recovery in every room (and the failure without whole_map); determinism;
identity with the archive off or with every candidate in the current window; the insert afterwards; no winner; the shim."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import bnb_numpy as BN
import global_localization_numpy as GN
from conftest import get_case, quat_angle
from test_global_localization import _ctx, _global_bits, _icp_bits, _yaw_quat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO_ERR_ARG = -1
DEG = math.pi / 180.0
ROOM_X = (-800.0, 0.0, 800.0)
ROOM_A = [ROOM_X[0], 0.0, 0.0]
CAP = 1 << 22


# --------------------------------------------------------------------------------------------------------------- CPU
def test_whole_map_argument_and_layouts(tmp_path):
    from superodom_b200 import api
    for bad in (2, -1, 7):
        with pytest.raises(api.SuperOdomError) as ei:
            api.localize_global_size(api.global_opts(half_x=10.0, half_y=10.0, yaw_half=math.pi, whole_map=bad))
        assert ei.value.code == SO_ERR_ARG
    assert api.localize_global_size(api.global_opts(half_x=10.0, half_y=10.0, yaw_half=math.pi, whole_map=True))[1] == 1_180_980
    f = tmp_path / "sz.c"
    f.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "superodom_b200.h"\n'
                 'int main(void){printf("%zu %zu %zu %zu\\n", offsetof(so_global_opts, whole_map), offsetof(so_global_result, n_windows), '
                 'sizeof(so_global_opts), sizeof(so_global_result));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(f), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)]).split()))
    assert got == (api.GlobalOpts.whole_map.offset, api.GlobalResult.n_windows.offset, C.sizeof(api.GlobalOpts), C.sizeof(api.GlobalResult))


def _build_shim(tmp_path):
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "global_archive_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "global_archive_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


def test_shim_with_global_localize_in_whole_map_compiles(tmp_path):
    assert os.path.exists(_build_shim(tmp_path))


def _shift_origin(o, t):
    """LocalMap::shiftMap's rule: the origin so_map_shift(t) leaves when called at origin o."""
    out = []
    for a, dim in enumerate((21, 21, 11)):
        v = float(t[a]) + 25.0
        c = int(v / 50.0) - (1 if v < 0 else 0) + int(o[a])
        s = 0
        while c < 3:
            c, s = c + 1, s + 1
        while c >= dim - 3:
            c, s = c - 1, s - 1
        out.append(int(o[a]) + s)
    return tuple(out)


def test_shift_rule_restatement():
    assert _shift_origin((16, 10, 5), ROOM_A) == (19, 10, 5)          # room A at the window's low x face: three blocks in
    assert _shift_origin((19, 10, 5), [800.0, 0.0, 0.0]) == (1, 10, 5)           # room C: 18 blocks back
    assert _shift_origin((10, 10, 5), [10.0, -20.0, 0.3]) == (10, 10, 5)


# --------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def rooms():
    """The three rooms: scenes, the whole surf cloud and an edge cloud (every 10th surf point) so that both stores move."""
    from superodom_b200 import synth
    scenes, maps = [], []
    for k, x in enumerate(ROOM_X):                     # synth.make_map, with the block filter's grid placed on the room
        sc = synth.make_scene(52.0, seed=611 + k, center=(x, 0.0))
        raw = synth.sample_surfaces(sc, 0.2, seed=1234)
        xyzi = np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1)
        scenes.append(sc)
        maps.append(synth.voxel_filter_blocks(xyzi, 0.2, origin=(10 - int(round(x / 50.0)), 10, 5)))
    surf = np.ascontiguousarray(np.concatenate(maps), np.float32)
    return dict(scenes=scenes, surf=surf, edge=np.ascontiguousarray(surf[::10]))


def _scan(rooms, room, i):
    from superodom_b200 import synth
    pose = synth.random_sensor_pose(rooms["scenes"][room], 900 + 10 * room + i, 20.0)
    return synth.make_scan(rooms["scenes"][room], "os1_128", pose, 1000 + 10 * room + i), pose


def _ctx3(api, rooms, max_batch=16, edge=True, shift=True):
    """Archive on, origin in room A, the three rooms loaded, then (shift) so_map_shift in room A: room C is wholly archived."""
    ctx = api.Context(max_map_points=CAP, max_scan_points=262144, plane_res=0.2, line_res=0.1, max_batch=max_batch)
    ctx.map_archive(CAP)
    ctx.map_set_origin(ROOM_A)
    ctx.map_set_points(rooms["surf"])
    if edge:
        ctx.map_set_edge_points(rooms["edge"])
    if shift:
        ctx.map_shift(ROOM_A)
    return ctx


def _whole(api, ctx, z, yaw, whole=True, **kw):
    lo, hi, _ = ctx.map_bounds_all()
    center = np.r_[0.5 * (float(lo[0]) + float(hi[0])), 0.5 * (float(lo[1]) + float(hi[1])), z, _yaw_quat(yaw)]
    return center, api.whole_map_opts(lo, hi, center, yaw_half=math.pi, whole_map=whole, **kw)


def _set_origin_exact(ctx, o):
    ctx.map_set_origin([-50.0 * float(v) for v in o])
    assert tuple(ctx.map_origin()) == tuple(o)


def _cand_matches(c, r):
    """A candidate equals an so_icp_result: pose, status, SUCCESS count and final cost, bit for bit."""
    cost = r.iter_cost[r.n_iterations - 1] if r.n_iterations > 0 else 0.0
    return (np.array_equal(np.array(c.pose), np.array(r.pose)) and c.status == r.status and
            c.n_success == r.hist_reject_plane[0] and struct.pack("<d", c.cost) == struct.pack("<d", cost))


@pytest.fixture(scope="module")
def face_case(gpu_api):
    """cfg2 with the archive on and the window's -x face at x = -25 m cutting the room; a region across that face."""
    case = get_case("cfg2")
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=262144, plane_res=0.2, max_batch=1)
    ctx.map_archive(1 << 21)
    ctx.map_set_origin([0.0, 0.0, 0.0])
    ctx.map_set_points(case["map_xyzi"])
    assert ctx.map_archive_info(0)[0] > 0
    center = np.r_[-25.3, case["pose_true"][1], case["pose_true"][2], case["pose_true"][3:]]
    region = dict(half_x=3.0, half_y=2.0, yaw_half=20 * DEG, max_range=30.0)
    yield case, ctx, center, region
    ctx.close()


@pytest.mark.gpu
def test_map_bounds_all_equal_downloaded_whole_map(gpu_api, face_case):
    case, ctx, _, _ = face_case
    lo, hi, n = ctx.map_bounds_all()
    m = ctx.map_download_all(0)[:, :3]
    assert n == len(m) and lo.tobytes() == m.min(0).astype(np.float32).tobytes() and hi.tobytes() == m.max(0).astype(np.float32).tobytes()
    wlo, whi, wn = ctx.map_bounds()
    assert wn < n and wlo[0] > lo[0]
    off = _ctx(gpu_api, case, max_batch=1)
    a, b = off.map_bounds(), off.map_bounds_all()
    assert a[2] == b[2] and a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    off.close()


@pytest.mark.gpu
def test_scores_over_window_face_equal_numpy_on_whole_map(gpu_api, face_case):
    case, ctx, center, region = face_case
    whole_xyz = ctx.map_download_all(0)[:, :3]
    got, n_pts = ctx.localize_scores(case["scan_xyzi"], center, gpu_api.global_opts(whole_map=True, **region))
    want, n_want = GN.localize_scores_numpy(case["scan_xyzi"], center, whole_xyz, **region)
    assert n_pts == n_want > 0 and got.shape == want.shape
    bad = np.argwhere(got != want)
    assert len(bad) == 0, (len(bad), bad[:5])
    window_only, _ = ctx.localize_scores(case["scan_xyzi"], center, gpu_api.global_opts(**region))
    assert not np.array_equal(window_only, got)                                # the archived half of the room counts
    assert np.array_equal(window_only, GN.localize_scores_numpy(case["scan_xyzi"], center, ctx.map_download(0)[:, :3], **region)[0])


@pytest.mark.gpu
def test_keys_and_bounds_over_window_face(gpu_api, face_case):
    case, ctx, center, region = face_case
    g = gpu_api.global_opts(whole_map=True, **region)
    whole_xyz = ctx.map_download_all(0)[:, :3]
    scores, _ = GN.localize_scores_numpy(case["scan_xyzi"], center, whole_xyz, **region)
    P = GN.plan(**region)
    keys, st = ctx.localize_bnb_keys(case["scan_xyzi"], center, g)
    assert np.array_equal(keys, BN.prefix_keys(scores, min(P["n_hyp"], 64 * P["k"])))
    L = min(2, BN.lmax(P))
    got = ctx.localize_bnb_bounds(case["scan_xyzi"], center, L, g)
    want, _ = BN.bounds(case["scan_xyzi"], center, whole_xyz, L, **region)
    assert np.array_equal(got, want)


@pytest.mark.gpu
def test_refinement_equals_shift_then_register_batch(gpu_api, rooms):
    scan, pose_true = _scan(rooms, 2, 0)
    ctx = _ctx3(gpu_api, rooms)
    o0 = tuple(ctx.map_origin())
    assert ctx.map_archive_info(0)[0] > 0 and abs(ctx.map_bounds()[1][0]) < 500.0   # room C is not in the window
    before = [ctx.map_download_all(s).copy() for s in (0, 1)]
    center, g = _whole(gpu_api, ctx, pose_true[2], 0.4)
    pose, res, cands, st = ctx.localize_global_bnb(scan, center, 20, g)
    assert res.n_candidates == len(cands) > 1 and res.winner >= 0
    wins = [_shift_origin(o0, c.prior) for c in cands]
    assert res.n_windows == len(set(wins)) and tuple(ctx.map_origin()) == wins[res.winner]
    for s in (0, 1):
        after = ctx.map_download_all(s)
        assert after.shape == before[s].shape and np.array_equal(after, before[s])
    ref = _ctx3(gpu_api, rooms)
    for i, c in enumerate(cands):
        _set_origin_exact(ref, o0)
        ref.map_shift(np.array(c.prior[:3]))
        assert tuple(ref.map_origin()) == wins[i]
        r = ref.register_batch(scan, [len(scan)], np.array(c.prior)[None], 20)[0]
        assert _cand_matches(c, r), i
        if i == res.winner:
            assert _icp_bits(r) == _icp_bits(res.icp)
    print(f"room C scan: {res.n_candidates} candidates in {res.n_windows} windows {sorted(set(wins))}, winner {res.winner}, "
          f"err {np.linalg.norm(pose[:3] - pose_true[:3]):.4f} m, build {st.time_build_ms:.1f} ms, search {st.time_search_ms:.1f} ms, "
          f"refine {res.time_refine_ms:.1f} ms")
    ref.close()
    ctx.close()


@pytest.mark.gpu
def test_recovery_in_every_room(gpu_api, rooms):
    """8 scans (3 in room C), centre at the whole-map box centre with the true z and a seeded yaw: the best-ranked hypothesis of every
    scan is the true one, and its registration, made in its own window, lands within 5 cm / 0.5 deg.  The room-C scans with
    whole_map = 0 (the window only) have no candidate within that bound.

    The winner rule (most SUCCESS correspondences) is not asserted: the three rooms share one shelving lattice, and the same scan
    registered at its true pose gets about 12 % fewer SUCCESS correspondences 800 m from the world origin than at it (float
    precision of the plane rows), so a look-alike pose in the centre room can out-count the true one.  The winners are printed."""
    ctx = _ctx3(gpu_api, rooms)
    o0 = tuple(ctx.map_origin())
    plan = [(0, 0), (0, 1), (1, 0), (1, 1), (1, 2), (2, 0), (2, 1), (2, 2)]
    errors, room_c = [], []
    for room, i in plan:
        scan, truth = _scan(rooms, room, i)
        yaw = np.random.default_rng(9300 + 10 * room + i).uniform(-math.pi, math.pi)
        _set_origin_exact(ctx, o0)
        center, g = _whole(gpu_api, ctx, truth[2], yaw)
        pose, res, cands, st = ctx.localize_global_bnb(scan, center, 20, g)
        best = np.array(cands[0].pose)
        dt = float(np.linalg.norm(best[:3] - truth[:3]))
        da = float(quat_angle(best[3:], truth[3:])) / DEG
        print(f"room {'ABC'[room]} scan {i}: best-ranked status {cands[0].status}, err {dt:.4f} m {da:.4f} deg; winner {res.winner} "
              f"err {np.linalg.norm(pose[:3] - truth[:3]):.3f} m (SUCCESS {cands[res.winner].n_success} vs {cands[0].n_success}); "
              f"{res.n_hypotheses} hypotheses, search build {st.time_build_ms:.1f} ms + traversal {st.time_search_ms:.1f} ms, "
              f"refine {res.time_refine_ms:.1f} ms, n_windows {res.n_windows}, total {res.time_total_ms:.1f} ms")
        assert res.status == 0 and tuple(ctx.map_origin()) == _shift_origin(o0, cands[res.winner].prior)
        errors.append((room, i, cands[0].status, dt, da))
        if room == 2:
            room_c.append((scan, truth, center, g))
    for room, i, stt, dt, da in errors:
        assert stt == 0 and dt < 0.05 and da < 0.5, errors
    for scan, truth, center, g in room_c:
        _set_origin_exact(ctx, o0)
        g.whole_map = 0
        pose, res, cands, _ = ctx.localize_global_bnb(scan, center, 20, g)
        dt = float(np.linalg.norm(pose[:3] - truth[:3]))
        da = float(quat_angle(pose[3:], truth[3:])) / DEG
        print(f"room C, window only: status {res.status}, err {dt:.2f} m {da:.2f} deg")
        assert res.n_windows == 0 and not (res.status == 0 and dt < 0.05 and da < 0.5)
        assert not any(np.linalg.norm(np.array(c.pose[:3]) - truth[:3]) < 0.05 for c in cands)
    ctx.close()


def _stats_bits(st):
    from superodom_b200 import api
    c = api.BnbStats.from_buffer_copy(bytes(st))
    c.time_build_ms = c.time_search_ms = 0.0
    return bytes(c)


@pytest.mark.gpu
def test_deterministic_across_calls_and_batch_sizes(gpu_api, rooms):
    scan, truth = _scan(rooms, 2, 1)
    out = []
    for mb, calls in ((16, 2), (1, 1)):
        ctx = _ctx3(gpu_api, rooms, max_batch=mb)
        o0 = tuple(ctx.map_origin())
        for _ in range(calls):
            _set_origin_exact(ctx, o0)
            center, g = _whole(gpu_api, ctx, truth[2], -1.1)
            _, res, cands, st = ctx.localize_global_bnb(scan, center, 20, g)
            out.append((_global_bits(res, cands), _stats_bits(st), tuple(ctx.map_origin())))
        ctx.close()
    assert out[0][0][0] and out[0] == out[1] == out[2]


@pytest.mark.gpu
def test_identity_without_archive_and_within_one_window(gpu_api):
    case = get_case("cfg2", 1)
    from test_global_localization import _recovery_center
    center = _recovery_center(case, 1)
    region = dict(half_x=10.0, half_y=10.0, yaw_half=math.pi)
    off = _ctx(gpu_api, case)
    o_off = tuple(off.map_origin())
    for fn in (off.localize_global, lambda *a: off.localize_global_bnb(*a)[:3]):
        pose0, res0, c0 = fn(case["scan_xyzi"], center, 20, gpu_api.global_opts(**region))
        pose1, res1, c1 = fn(case["scan_xyzi"], center, 20, gpu_api.global_opts(whole_map=True, **region))
        assert res1.n_windows == 0 and _global_bits(res0, c0) == _global_bits(res1, c1) and np.array_equal(pose0, pose1)
        assert tuple(off.map_origin()) == o_off
    off.close()
    on = gpu_api.Context(max_map_points=1 << 21, max_scan_points=262144, plane_res=0.2, max_batch=16)
    on.map_archive(1 << 21)
    on.map_set_points(case["map_xyzi"])
    o0 = tuple(on.map_origin())
    pose0, res0, c0 = on.localize_global(case["scan_xyzi"], center, 20, gpu_api.global_opts(**region))
    pose1, res1, c1 = on.localize_global(case["scan_xyzi"], center, 20, gpu_api.global_opts(whole_map=True, **region))
    assert all(_shift_origin(o0, c.prior) == o0 for c in c1)
    assert res0.n_windows == 0 and res1.n_windows == 1 and tuple(on.map_origin()) == o0
    res1.n_windows = 0
    assert _global_bits(res0, c0) == _global_bits(res1, c1) and np.array_equal(pose0, pose1)
    on.close()


@pytest.mark.gpu
def test_insert_after_the_call_lands_in_the_winners_window(gpu_api, rooms):
    scan, truth = _scan(rooms, 2, 2)
    ctx = _ctx3(gpu_api, rooms)
    o0 = tuple(ctx.map_origin())
    center, g = _whole(gpu_api, ctx, truth[2], 2.3)
    pose, res, cands, _ = ctx.localize_global_bnb(scan, center, 20, g)
    assert res.status == 0
    ow = _shift_origin(o0, cands[res.winner].prior)
    assert ow != o0 and tuple(ctx.map_origin()) == ow
    ctx.map_add_registered_scan(pose)
    ref = _ctx3(gpu_api, rooms)
    ref.map_shift(np.array(cands[res.winner].prior[:3]))
    assert tuple(ref.map_origin()) == ow
    ref.map_add_scan(scan, pose)
    for s in (0, 1):
        assert np.array_equal(ctx.map_download_all(s), ref.map_download_all(s))
    ref.close()
    ctx.close()


@pytest.mark.gpu
def test_no_winner_leaves_the_window_and_the_sink(gpu_api, rooms):
    import torch
    scan, truth = _scan(rooms, 2, 0)
    ctx = _ctx3(gpu_api, rooms)
    o0 = tuple(ctx.map_origin())
    before = [ctx.map_download_all(s).copy() for s in (0, 1)]
    sink = torch.full((4, 8), -7.0, dtype=torch.float64, device="cuda")
    ctx.set_pose_sink(sink.data_ptr(), 4, 0)
    far = np.r_[0.0, 400.0, truth[2], _yaw_quat(0.3)]
    pose, res, cands, _ = ctx.localize_global_bnb(scan, far, 20, gpu_api.global_opts(half_x=2.0, half_y=2.0, yaw_half=math.pi, whole_map=True))
    torch.cuda.synchronize()
    assert res.status in (1, 2) and res.winner == -1 and np.array_equal(pose, far)
    assert tuple(ctx.map_origin()) == o0 and bool((sink == -7.0).all())
    for s in (0, 1):
        assert np.array_equal(ctx.map_download_all(s), before[s])
    ctx.set_pose_sink(None)
    ctx.close()


@pytest.mark.gpu
def test_shim_global_localize_in_whole_map_matches_abi(tmp_path, gpu_api, rooms):
    exe = _build_shim(tmp_path)
    scan, truth = _scan(rooms, 2, 1)
    m, s = rooms["surf"], np.ascontiguousarray(scan, np.float32)
    ctx = _ctx3(gpu_api, rooms, edge=False, shift=False)
    center, g = _whole(gpu_api, ctx, truth[2], 0.9)
    iters = 20
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiiifQ", len(m), len(s), iters, 0, 0.2, CAP))
        f.write(np.asarray(ROOM_A, np.float64).tobytes())
        f.write(np.asarray(center, np.float64).tobytes())
        f.write(bytes(gpu_api.global_opts(yaw_half=math.pi)))
        f.write(m.tobytes())
        f.write(s.tobytes())
    out = subprocess.run([exe, str(path)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    l1, l2, l3, l4 = out.stdout.strip().splitlines()
    rc, winner, *pose_s = l1.split()
    pose, res, cands, st = ctx.localize_global_bnb(s, center, iters, g)
    assert int(rc) == res.status == 0 and int(winner) == res.winner
    assert np.array_equal(np.array([float(v) for v in pose_s]), pose)
    assert np.array_equal(np.array([float(v) for v in l2.split()]), pose)
    assert [int(v) for v in l3.split()] == [st.lmax, st.leaves_scored, st.steps, res.n_windows]
    assert [int(v) for v in l4.split()] == list(ctx.map_origin())
    assert np.linalg.norm(np.array(cands[0].pose[:3]) - truth[:3]) < 0.05              # the best-ranked hypothesis is the true one
    ctx.close()

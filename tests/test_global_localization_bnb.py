"""Global localization by branch-and-bound (the search of every so_localize_global* call): the sorted key prefix of every
hypothesis' score, from an occupancy pyramid whose memory scales with the map; so_localize_global_bnb takes up to 2^32 hypotheses.

CPU: the numpy restatement of the bounds is a bound (every node's U >= its children's U and >= every exact score in it), the
stats struct layout, the C++ shim builds.
GPU: bounds equal the numpy restatement at every level; keys equal the prefix of the dense scores (so_localize_scores, or numpy
beyond so_localize_global's cap and for tall regions); so_localize_global equals so_localize_global_bnb bit for bit; the offset
table's capacity error comes before any device work; whole-map recovery; determinism; no side effects; soft statuses; map
bounds; shim."""
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
from test_global_localization import _ctx, _global_bits, _recovery_center, _with_rp, _yaw_quat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO_ERR_ARG, SO_ERR_CAPACITY = -1, -3
SO_STATUS_NOT_ENOUGH_FEATURES, SO_STATUS_NO_CORRESPONDENCES = 1, 2
DEG = math.pi / 180.0


# --------------------------------------------------------------------------------------------------------------- CPU
def _random_case(seed):
    """A small random map (boxes of points) and a scan of it from a random pose: sensor-frame scan, centre, map."""
    rng = np.random.default_rng(seed)
    n = 4000
    m = np.c_[rng.uniform(-6, 6, n), rng.uniform(-5, 5, n), rng.uniform(-1, 2, n)]
    m[: n // 3, 2] = -1.0                                                    # a floor: coarse levels saturate on it
    m[n // 3: n // 2, 0] = 4.0                                               # a wall
    yaw = rng.uniform(-math.pi, math.pi)
    t = np.r_[rng.uniform(-1, 1, 2), 0.3]
    c, s = math.cos(yaw), math.sin(yaw)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    scan = (m[rng.choice(n, 600, replace=False)] - t) @ R
    scan = np.c_[scan, np.zeros(len(scan))].astype(np.float32)
    center = np.r_[t + np.r_[rng.uniform(-0.5, 0.5, 2), 0.0], _yaw_quat(yaw + rng.uniform(-0.3, 0.3))]
    return scan, center, np.asarray(m, np.float32)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_numpy_bounds_bound_children_and_scores(seed):
    """U at level L+1 >= U of each of its (up to 4) children at level L, and U at every level >= every exact score in the node;
    level 0 is the exact score."""
    scan, center, m = _random_case(seed)
    region = dict(half_x=2.1, half_y=1.7, half_z=0.25 * (seed - 1), yaw_half=12 * DEG, yaw_step=4 * DEG, res=0.25, max_range=8.0,
                  score_points=300, dilate=seed % 2 + 1)
    P = GN.plan(**region)
    B = GN.bitmap(m, P, center)
    exact, n_pts = GN.localize_scores_numpy(scan, center, m, **region)
    assert n_pts > 100 and exact.max() > 0
    U = [BN.bounds(scan, center, m, L, B=B, **region)[0] for L in range(5)]
    assert np.array_equal(U[0], exact)
    ny, nx = exact.shape[2:]
    for L in range(1, 5):
        s = 1 << L
        up = np.repeat(np.repeat(U[L].astype(np.int64), s, axis=2), s, axis=3)[:, :, :ny, :nx]
        assert (up >= exact).all()
        child = np.repeat(np.repeat(U[L].astype(np.int64), 2, axis=2), 2, axis=3)[:, :, :U[L - 1].shape[2], :U[L - 1].shape[3]]
        assert (child >= U[L - 1]).all()
        assert (up > exact).any()                                             # a coarse window overestimates somewhere


def test_lmax_rule():
    assert BN.lmax(GN.plan(half_x=10.0, half_y=10.0, yaw_half=math.pi)) == 3        # 11 x 11 x 180 root nodes
    assert BN.lmax(GN.plan(half_x=1.0, half_y=1.0)) == 1
    assert BN.lmax(GN.plan(half_x=150.0, half_y=150.0, yaw_half=math.pi)) == 6      # 1201 shifts: 19 x 19 tiles x 180
    P = GN.plan(half_x=1.0, half_y=1.0, half_z=4000.0, yaw_half=math.pi, yaw_step=0.5 * DEG)
    assert BN.lmax(P) == 4                                                           # root tile covers every x/y shift


def test_bnb_stats_layout_matches_header(tmp_path):
    from superodom_b200 import api
    f = tmp_path / "sz.c"
    f.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "superodom_b200.h"\n'
                 'int main(void){printf("%zu %zu %zu %zu %zu %d\\n", sizeof(so_bnb_stats), offsetof(so_bnb_stats, scored), '
                 'offsetof(so_bnb_stats, leaves_scored), offsetof(so_bnb_stats, pyramid_bytes), offsetof(so_bnb_stats, time_search_ms), '
                 'SO_BNB_LEVELS);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(f), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)]).split()))
    S = api.BnbStats
    assert got == (C.sizeof(S), S.scored.offset, S.leaves_scored.offset, S.pyramid_bytes.offset, S.time_search_ms.offset, api.BNB_LEVELS)


def test_whole_map_opts_cover_the_box():
    from superodom_b200 import api
    g = api.whole_map_opts(np.float32([-50.5, -20.0, 0]), np.float32([52.25, 30.0, 8]), [1.0, 2.0, 0.5, 0, 0, 0, 1], yaw_half=math.pi, res=0.5)
    assert (g.half_x, g.half_y, g.yaw_half, g.res) == (51.5, 28.0, math.pi, 0.5)
    g = api.whole_map_opts(np.float32([0, 0, 0]), np.float32([1, 1, 1]), [5.0, 5.0, 0, 0, 0, 0, 1])
    assert (g.half_x, g.half_y) == (5.0, 5.0)


def _build_shim(tmp_path):
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "global_bnb_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "global_bnb_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


def test_shim_with_global_localize_in_map_compiles(tmp_path):
    assert os.path.exists(_build_shim(tmp_path))


# --------------------------------------------------------------------------------------------------------------- GPU
def _stats_bits(st):
    from superodom_b200 import api
    c = api.BnbStats.from_buffer_copy(bytes(st))
    c.time_build_ms = c.time_search_ms = 0.0
    return bytes(c)


def _check_stats(st, P, keys):
    assert st.lmax == BN.lmax(P) and st.root_nodes == BN.level_nodes(P, st.lmax)
    assert st.leaves_scored == st.scored[0] <= P["n_hyp"] and st.steps > 0
    assert st.kstar_score == 65535 - int(keys[-1] >> np.uint64(32))
    for L in range(st.lmax):
        assert st.scored[L] <= 4 * (st.scored[L + 1] - st.discarded[L + 1])


def _map_center(ctx, case):
    lo, hi, _ = ctx.map_bounds()
    return np.r_[0.5 * (float(lo[0]) + float(hi[0])), 0.5 * (float(lo[1]) + float(hi[1])), case["pose_true"][2]]


_BOUND_REGIONS = {
    "cfg1": ("cfg1", dict(half_x=1.0, half_y=1.0, half_z=0.25, yaw_half=math.pi, yaw_step=15 * DEG, max_range=15.0)),
    "cfg2_block_face_yaw_wrap": ("cfg2", dict(half_x=2.0, half_y=1.5, yaw_half=20 * DEG, dilate=2, score_points=2048, max_range=30.0)),
    "cfg2_overhanging_map_edge": ("cfg2", dict(half_x=6.0, half_y=6.0, yaw_half=30 * DEG, yaw_step=3 * DEG, max_range=25.0)),
    "cfg2_default": ("cfg2", dict(half_x=10.0, half_y=10.0, yaw_half=math.pi)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_BOUND_REGIONS))
def test_bounds_equal_numpy_at_every_level(gpu_api, name):
    cfg, region = _BOUND_REGIONS[name]
    case = get_case(cfg)
    ctx = _ctx(gpu_api, case, max_batch=1)
    if name == "cfg1":
        center = _with_rp(case["pose_true"], 3 * DEG, -2 * DEG)
        center[:3] += [0.37, -0.21, 0.05]
    elif name == "cfg2_block_face_yaw_wrap":
        center = _with_rp(np.r_[24.6, -3.1, case["pose_true"][2], _yaw_quat(175 * DEG)], -1.5 * DEG, 2.5 * DEG)
    elif name == "cfg2_overhanging_map_edge":            # the box reaches past the map's low x and y edges: windows straddle W's low side
        lo, _, _ = ctx.map_bounds()
        center = np.r_[float(lo[0]) + 2.3, float(lo[1]) + 1.6, case["pose_true"][2], _yaw_quat(0.4)]
    else:
        center = _recovery_center(case, 0)
    g = gpu_api.global_opts(**region)
    P = GN.plan(**region)
    map_xyz = ctx.map_download(0)[:, :3]
    B = GN.bitmap(map_xyz, P, center)
    if name == "cfg2_overhanging_map_edge":
        assert not B[:, :, :P["e"]].any() and not B[:, :P["e"], :].any()     # nothing of the map below the box's low corner
    lmax = BN.lmax(P)
    for L in range(lmax + 1):
        got = ctx.localize_bnb_bounds(case["scan_xyzi"], center, L, g)
        want, n_pts = BN.bounds(case["scan_xyzi"], center, map_xyz, L, B=B, **region)
        assert n_pts > 0 and got.shape == want.shape
        bad = np.argwhere(got != want)
        assert len(bad) == 0, (L, len(bad), bad[:5])
    with pytest.raises(gpu_api.SuperOdomError):
        ctx.localize_bnb_bounds(case["scan_xyzi"], center, lmax + 1, g)
    ctx.close()


def _keys_case(gpu_api, ctx, scan, center, g, **region):
    keys, st = ctx.localize_bnb_keys(scan, center, g)
    scores, _ = ctx.localize_scores(scan, center, g)
    P = GN.plan(**region)
    want = BN.prefix_keys(scores, min(P["n_hyp"], 64 * P["k"]))
    assert keys.dtype == np.uint64 and np.array_equal(keys, want), (len(keys), len(want), np.argwhere(keys != want)[:5])
    _check_stats(st, P, keys)
    return keys, st, scores


_KEY_REGIONS = {
    "default": dict(half_x=10.0, half_y=10.0, yaw_half=math.pi),
    "saturated": dict(yaw_half=math.pi, res=0.5, dilate=2, score_points=256),             # over the whole map
    "half_z": dict(half_x=3.0, half_y=2.0, half_z=0.5, yaw_half=30 * DEG),
    "k1": dict(half_x=10.0, half_y=10.0, yaw_half=math.pi, k=1),
    "k64": dict(half_x=10.0, half_y=10.0, yaw_half=math.pi, k=64),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_KEY_REGIONS))
def test_keys_equal_exhaustive_prefix(gpu_api, name):
    case = get_case("cfg2")
    ctx = _ctx(gpu_api, case, max_batch=1)
    region = dict(_KEY_REGIONS[name])
    center = _recovery_center(case, 0)
    if name == "saturated":
        lo, hi, _ = ctx.map_bounds()
        center = np.r_[_map_center(ctx, case), center[3:]]
        g = gpu_api.whole_map_opts(lo, hi, center, **region)
        region.update(half_x=g.half_x, half_y=g.half_y)
    keys, st, scores = _keys_case(gpu_api, ctx, case["scan_xyzi"], center, gpu_api.global_opts(**region), **region)
    top = scores.max()
    print(f"{name}: {scores.size} hypotheses, best {top} ({int((scores == top).sum())} at the top), lmax {st.lmax}, "
          f"leaves {st.leaves_scored} ({st.leaves_scored / scores.size:.3f}), steps {st.steps}")
    if name == "saturated":
        assert (scores == top).sum() > 1                                      # ties at the top: decided by index alone
    ctx.close()


@pytest.mark.gpu
def test_keys_whole_cfg2_map_at_6_deg(gpu_api):
    """The whole cfg2 map at 0.25 m and 6 deg (about 10^7 hypotheses, under so_localize_scores' 2^24 cap)."""
    case = get_case("cfg2")
    ctx = _ctx(gpu_api, case, max_batch=1)
    lo, hi, _ = ctx.map_bounds()
    center = np.r_[_map_center(ctx, case), _yaw_quat(0.7)]
    g = gpu_api.whole_map_opts(lo, hi, center, yaw_half=math.pi, yaw_step=6 * DEG)
    region = dict(half_x=g.half_x, half_y=g.half_y, yaw_half=math.pi, yaw_step=6 * DEG)
    keys, st, scores = _keys_case(gpu_api, ctx, case["scan_xyzi"], center, g, **region)
    assert 0.9e7 < scores.size < 2 ** 24
    print(f"whole map 6 deg: {scores.size} hypotheses, leaves scored {st.leaves_scored} ({st.leaves_scored / scores.size:.4f}), "
          f"steps {st.steps}, lmax {st.lmax}, scored per level {list(st.scored)[:st.lmax + 1]}")
    ctx.close()


@pytest.mark.gpu
def test_keys_no_map_and_empty_scan(gpu_api):
    """No map in the region: every score is 0, so the prefix is the first P indices.  An empty scan: the same."""
    case = get_case("cfg1")
    ctx = _ctx(gpu_api, case, max_batch=1)
    region = dict(half_x=2.0, half_y=2.0, yaw_half=math.pi, max_range=20.0)
    g = gpu_api.global_opts(**region)
    P = GN.plan(**region)
    want = (np.uint64(65535) << np.uint64(32)) | np.arange(min(P["n_hyp"], 64 * 16), dtype=np.uint64)
    far = np.r_[400.0, -300.0, 0.0, _yaw_quat(0.3)]
    keys, st = ctx.localize_bnb_keys(case["scan_xyzi"], far, g)
    assert np.array_equal(keys, want) and st.kstar_score == 0
    keys, st = ctx.localize_bnb_keys(np.zeros((0, 4), np.float32), case["pose_true"], g)
    assert np.array_equal(keys, want)
    ctx.close()


@pytest.mark.gpu
def test_keys_beyond_the_exhaustive_cap(gpu_api):
    """The whole cfg2 map at 0.5 m with 400 yaw steps: more than 2^24 hypotheses, which so_localize_global refuses.  The keys equal
    the numpy restatement's exhaustive prefix."""
    case = get_case("cfg2")
    ctx = _ctx(gpu_api, case, max_batch=1)
    lo, hi, _ = ctx.map_bounds()
    center = np.r_[_map_center(ctx, case), _yaw_quat(-2.1)]
    kw = dict(yaw_half=math.pi, yaw_step=2 * math.pi / 400, res=0.5, score_points=256)
    g = gpu_api.whole_map_opts(lo, hi, center, **kw)
    region = dict(half_x=g.half_x, half_y=g.half_y, **kw)
    with pytest.raises(gpu_api.SuperOdomError) as ei:
        gpu_api.localize_global_size(g)
    assert ei.value.code == SO_ERR_CAPACITY
    keys, st = ctx.localize_bnb_keys(case["scan_xyzi"], center, g)
    scores, n_pts = GN.localize_scores_numpy(case["scan_xyzi"], center, ctx.map_download(0)[:, :3], **region)
    assert scores.size > 2 ** 24 and n_pts > 100
    P = GN.plan(**region)
    assert np.array_equal(keys, BN.prefix_keys(scores, min(P["n_hyp"], 64 * P["k"])))
    _check_stats(st, P, keys)
    print(f"beyond the cap: {scores.size} hypotheses x {n_pts} points, leaves scored {st.leaves_scored} "
          f"({st.leaves_scored / scores.size:.4f}), steps {st.steps}")
    ctx.close()


@pytest.mark.gpu
def test_keys_z_heavy_region(gpu_api):
    """A tall region with small x/y at 4096 score points: NYAW * NZ * points * 16 B is above 1 GiB, so a table of score-point
    offsets per z shift would not fit; one per yaw does.  The dense scores equal the numpy restatement, the keys their prefix."""
    case = get_case("cfg2")
    ctx = _ctx(gpu_api, case, max_batch=1)
    region = dict(half_x=0.25, half_y=0.25, half_z=15.0, yaw_half=math.pi, score_points=4096)
    t = case["pose_true"]
    center = np.r_[t[0] + 0.1, t[1] - 0.05, t[2] + 0.3, t[3:]]
    P = GN.plan(**region)
    want, n_pts = GN.localize_scores_numpy(case["scan_xyzi"], center, ctx.map_download(0)[:, :3], **region)
    assert P["nz"] == 121 and P["nyaw"] * P["nz"] * n_pts * 16 > 1 << 30
    keys, st, scores = _keys_case(gpu_api, ctx, case["scan_xyzi"], center, gpu_api.global_opts(**region), **region)
    bad = np.argwhere(scores != want)
    assert len(bad) == 0, (len(bad), bad[:5])
    assert scores.max() > 0
    print(f"z-heavy: {scores.size} hypotheses x {n_pts} points, leaves scored {st.leaves_scored}, steps {st.steps}")
    ctx.close()


@pytest.mark.gpu
def test_offset_table_capacity_error_before_device_work(gpu_api):
    """NYAW * score points > 2^26 (20 000 yaw steps at 4096 points) is within so_localize_global_size's limits, but the offset table
    is above 1 GiB: so_localize_global, so_localize_global_bnb and so_localize_scores return SO_ERR_CAPACITY with no kernel launched
    and no byte copied."""
    case = get_case("cfg2")
    ctx = _ctx(gpu_api, case, max_batch=1)
    g = gpu_api.global_opts(yaw_half=math.pi, yaw_step=2 * math.pi / 20000, score_points=4096)
    dims, n_hyp, _ = gpu_api.localize_global_size(g)
    assert dims[3] == 20000 and n_hyp == 20000
    assert 20000 * len(GN.score_points(case["scan_xyzi"], 4096, 40.0)) > 1 << 26
    scan, center = case["scan_xyzi"], case["pose_true"]
    ctx.kernel_launches(reset=True)
    ctx.bytes_copied(reset=True)
    for call in (lambda: ctx.localize_global(scan, center, 5, g), lambda: ctx.localize_global_bnb(scan, center, 5, g),
                 lambda: ctx.localize_scores(scan, center, g)):
        with pytest.raises(gpu_api.SuperOdomError) as ei:
            call()
        assert f"({SO_ERR_CAPACITY})" in str(ei.value) and "offset table" in str(ei.value)
    assert ctx.kernel_launches() == 0 and ctx.bytes_copied() == (0, 0)
    ctx.close()


@pytest.mark.gpu
def test_result_equals_exhaustive_on_recovery_cases(gpu_api):
    """On the eight recovery cases of so_localize_global's test: the keys equal the prefix of the dense scores, and
    so_localize_global == so_localize_global_bnb bit for bit (timings zeroed), result and candidate list."""
    case0 = get_case("cfg2")
    ctx = _ctx(gpu_api, case0)
    region = dict(half_x=10.0, half_y=10.0, yaw_half=math.pi)
    g = gpu_api.global_opts(**region)
    for i in range(8):
        case = get_case("cfg2", i)
        center = _recovery_center(case, i)
        keys, _, _ = _keys_case(gpu_api, ctx, case["scan_xyzi"], center, g, **region)
        pose, res, cands = ctx.localize_global(case["scan_xyzi"], center, 20, g)
        pose_b, res_b, cands_b, st = ctx.localize_global_bnb(case["scan_xyzi"], center, 20, g)
        assert _global_bits(res, cands) == _global_bits(res_b, cands_b), i
        assert np.array_equal(pose, pose_b) and res.time_sort_ms == res_b.time_sort_ms == 0.0
        assert res.best_score == 65535 - int(keys[0] >> np.uint64(32))
        print(f"scan {i}: leaves {st.leaves_scored} of {res.n_hypotheses}, steps {st.steps}, search {st.time_search_ms:.2f} ms")
    ctx.close()


@pytest.mark.gpu
def test_whole_map_recovery_cfg2_os1_128(gpu_api):
    """8 OS1-128 scans, centre at the map centre with the true z and a seeded random yaw, region covering the whole map: every pose
    within 5 cm / 0.5 deg."""
    case0 = get_case("cfg2")
    ctx = _ctx(gpu_api, case0)
    lo, hi, _ = ctx.map_bounds()
    errors = []
    for i in range(8):
        case = get_case("cfg2", i)
        rng = np.random.default_rng(9100 + i)
        center = np.r_[_map_center(ctx, case), _yaw_quat(rng.uniform(-math.pi, math.pi))]
        g = gpu_api.whole_map_opts(lo, hi, center, yaw_half=math.pi)
        pose, res, cands, st = ctx.localize_global_bnb(case["scan_xyzi"], center, 20, g)
        dt = float(np.linalg.norm(pose[:3] - case["pose_true"][:3]))
        da = float(quat_angle(pose[3:], case["pose_true"][3:])) / DEG
        print(f"whole map scan {i}: status {res.status} winner {res.winner} of {res.n_candidates}, {res.n_hypotheses} hypotheses, "
              f"best {res.best_score} of {res.n_score_points}, err {dt:.4f} m {da:.4f} deg, leaves {st.leaves_scored} "
              f"({st.leaves_scored / res.n_hypotheses:.4f}), steps {st.steps}, search {st.time_search_ms:.1f} ms, "
              f"true offset {np.linalg.norm(center[:2] - case['pose_true'][:2]):.1f} m")
        errors.append((i, res.status, dt, da))
    ctx.close()
    for i, stt, dt, da in errors:
        assert stt == 0 and dt < 0.05 and da < 0.5, errors


@pytest.mark.gpu
def test_deterministic_across_calls_and_batch_sizes(gpu_api):
    case = get_case("cfg2", 1)
    center = _recovery_center(case, 1)
    g = gpu_api.global_opts(half_x=10.0, half_y=10.0, yaw_half=math.pi)
    ctx = _ctx(gpu_api, case, max_batch=16)
    _, res, cands, st = ctx.localize_global_bnb(case["scan_xyzi"], center, 20, g)
    _, res2, cands2, st2 = ctx.localize_global_bnb(case["scan_xyzi"], center, 20, g)
    assert res.status == 0 and _global_bits(res, cands) == _global_bits(res2, cands2)
    assert _stats_bits(st) == _stats_bits(st2)
    ctx.close()
    ctx1 = _ctx(gpu_api, case, max_batch=1)
    _, res1, cands1, st1 = ctx1.localize_global_bnb(case["scan_xyzi"], center, 20, g)
    assert _global_bits(res, cands) == _global_bits(res1, cands1) and _stats_bits(st) == _stats_bits(st1)
    ctx1.close()


@pytest.mark.gpu
def test_no_side_effects(gpu_api):
    """Map unchanged, pose sink rows and cursor unchanged, a following so_register equals a fresh context's, and the
    registered-scan insert at the returned pose equals so_map_add_scan of the same cloud."""
    import torch
    case = get_case("cfg2", 2)
    scan = case["scan_xyzi"]
    center = _recovery_center(case, 2)
    g = gpu_api.global_opts(half_x=10.0, half_y=10.0, yaw_half=math.pi)
    ctx = _ctx(gpu_api, case)
    before = ctx.map_download(0).copy()
    sink = torch.full((8, 8), -7.0, dtype=torch.float64, device="cuda")
    ctx.set_pose_sink(sink.data_ptr(), 8, 3)
    pose, res, _, _ = ctx.localize_global_bnb(scan, center, 20, g)
    torch.cuda.synchronize()
    assert res.status == 0
    assert np.array_equal(ctx.map_download(0), before)
    assert bool((sink == -7.0).all())
    prior = case["pose_prior"]
    r = ctx.register(scan, prior, 20)
    torch.cuda.synchronize()
    rows = sink.cpu().numpy()
    assert np.array_equal(rows[3, :7], np.array(r.pose_opt)) and (rows[4:] == -7.0).all() and (rows[:3] == -7.0).all()
    ctx.set_pose_sink(None)
    fresh = _ctx(gpu_api, case)
    rf = fresh.register(scan, prior, 20)
    assert np.array_equal(np.array(r.pose), np.array(rf.pose)) and r.n_iterations == rf.n_iterations
    fresh.close()
    ctx_a = _ctx(gpu_api, case)
    pose_a, _, _, _ = ctx_a.localize_global_bnb(scan, center, 20, g)
    assert np.array_equal(pose_a, pose)
    ctx_a.map_add_registered_scan(pose_a)
    ctx_b = _ctx(gpu_api, case)
    ctx_b.map_add_scan(scan, pose_a)
    assert np.array_equal(ctx_a.map_download(0), ctx_b.map_download(0))
    for c in (ctx, ctx_a, ctx_b):
        c.close()


@pytest.mark.gpu
def test_soft_statuses_and_argument_errors(gpu_api):
    case = get_case("cfg1")
    g = gpu_api.global_opts(half_x=2.0, half_y=2.0, yaw_half=math.pi, max_range=20.0)
    ctx = _ctx(gpu_api, case, max_batch=4)
    far = np.r_[400.0, -300.0, 0.0, _yaw_quat(0.3)]
    pose, res, cands, _ = ctx.localize_global_bnb(case["scan_xyzi"], far, 5, g)
    assert res.status == SO_STATUS_NO_CORRESPONDENCES and res.best_score == 0 and res.n_candidates == 0 and res.winner == -1
    assert np.array_equal(pose, far)
    ctx.close()
    empty = gpu_api.Context(max_map_points=1 << 16, max_scan_points=1 << 17, plane_res=0.2)
    lo, hi, n = empty.map_bounds()
    assert n == 0 and not lo.any() and not hi.any()
    pose, res, _, _ = empty.localize_global_bnb(case["scan_xyzi"], case["pose_prior"], 5, g)
    assert res.status == SO_STATUS_NO_CORRESPONDENCES and np.array_equal(pose, case["pose_prior"])
    pose, res, _, _ = empty.localize_global_bnb(np.zeros((0, 4), np.float32), case["pose_prior"], 5, g)
    assert res.status == SO_STATUS_NO_CORRESPONDENCES
    sparse = gpu_api.Context(max_map_points=1 << 16, max_scan_points=1 << 17, plane_res=0.2)
    sparse.map_set_points(case["map_xyzi"][::max(1, len(case["map_xyzi"]) // 40)][:40])
    pose, res, cands, _ = sparse.localize_global_bnb(case["scan_xyzi"], case["pose_true"], 5, g)
    assert res.best_score > 0 and res.n_candidates > 0
    assert res.status == SO_STATUS_NOT_ENOUGH_FEATURES and all(c.status == SO_STATUS_NOT_ENOUGH_FEATURES for c in cands)
    for bad_center, opts, code in (
            (np.r_[np.nan, 0, 0, 0, 0, 0, 1.0], g, SO_ERR_ARG),
            (case["pose_true"], gpu_api.global_opts(k=65), SO_ERR_ARG),
            (case["pose_true"], gpu_api.global_opts(half_x=4000.0, half_y=4000.0, yaw_half=math.pi), SO_ERR_CAPACITY)):
        with pytest.raises(gpu_api.SuperOdomError) as ei:
            sparse.localize_global_bnb(case["scan_xyzi"], bad_center, 5, opts)
        assert f"({code})" in str(ei.value)
        with pytest.raises(gpu_api.SuperOdomError):
            sparse.localize_bnb_keys(case["scan_xyzi"], bad_center, opts)
    empty.close()
    sparse.close()


@pytest.mark.gpu
def test_map_bounds_equal_downloaded_map(gpu_api):
    case = get_case("cfg2")
    ctx = _ctx(gpu_api, case, max_batch=1)
    lo, hi, n = ctx.map_bounds()
    m = ctx.map_download(0)[:, :3]
    assert n == len(m) and lo.dtype == np.float32
    assert lo.tobytes() == m.min(0).astype(np.float32).tobytes() and hi.tobytes() == m.max(0).astype(np.float32).tobytes()
    ctx.close()


@pytest.mark.gpu
def test_shim_global_localize_in_map_matches_abi(tmp_path, gpu_api):
    """LidarSLAM::globalLocalizeInMap returns the C ABI's pose bit for bit (whole-map region from so_map_bounds) and sets
    T_w_lidar and last_T_w_lidar; on that region so_localize_global gives the same result."""
    exe = _build_shim(tmp_path)
    case = get_case("cfg1", 1)
    center = _recovery_center(case, 1)
    opts = gpu_api.global_opts(yaw_half=math.pi, max_range=30.0)
    m = np.ascontiguousarray(case["map_xyzi"], np.float32)
    s = np.ascontiguousarray(case["scan_xyzi"], np.float32)
    iters, cap = 5, 2000
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiiif", len(m), len(s), iters, cap, 0.2))
        f.write(np.asarray(center, np.float64).tobytes())
        f.write(bytes(opts))
        f.write(m.tobytes())
        f.write(s.tobytes())
    out = subprocess.run([exe, str(path)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    l1, l2, l3 = out.stdout.strip().splitlines()
    rc, winner, *pose_s = l1.split()
    ctx = gpu_api.Context(max_map_points=1 << 22, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    ctx.map_add_surf(m)
    lo, hi, _ = ctx.map_bounds()
    g = gpu_api.whole_map_opts(lo, hi, center, yaw_half=math.pi, max_range=30.0)
    pose, res, cands, st = ctx.localize_global_bnb(s, center, iters, g, max_surface_features=cap)
    assert int(rc) == res.status == 0 and int(winner) == res.winner
    assert np.array_equal(np.array([float(v) for v in pose_s]), pose)
    assert np.array_equal(np.array([float(v) for v in l2.split()]), pose)
    assert [int(v) for v in l3.split()] == [st.lmax, st.leaves_scored, st.steps]
    assert np.linalg.norm(pose[:3] - case["pose_true"][:3]) < 0.05
    pose_x, res_x, cands_x = ctx.localize_global(s, center, iters, g, max_surface_features=cap)
    assert _global_bits(res, cands) == _global_bits(res_x, cands_x)
    ctx.close()

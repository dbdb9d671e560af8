"""Free-space clearing without a GPU: the numpy restatement (tests/free_space_numpy.py) on static scenes, where it must remove
nothing, the properties of the rule, and the ctypes layout of so_free_space / so_free_space_result against the header.

The static study sets the defaults of so_free_space_defaults (DESIGN.md §2 records its numbers): synth.make_map's maps sample every
face, hidden ones included, jittered by 2 cm and voxel-filtered, so any map point the rule removes at the true pose is a false removal."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from superodom_b200 import synth
import free_space_numpy as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_DT, ERR_DEG = 0.01, 0.05          # registration-sized pose error: 1 cm, 0.05 deg


def _pose_error(pose, seed):
    """pose (+) a 1 cm translation and a 0.05 deg rotation in random directions."""
    rng = np.random.default_rng(seed)
    u, v = rng.normal(size=3), rng.normal(size=3)
    q = synth.quat_mul(pose[3:], synth.quat_from_rotvec(np.deg2rad(ERR_DEG) * v / np.linalg.norm(v)))
    return np.concatenate([pose[:3] + ERR_DT * u / np.linalg.norm(u), q / np.linalg.norm(q)])


def _max_excess(map_xyz, scan, pose, o):
    """Largest (neighbourhood minimum - r_m) over the candidates: the smallest margin (margin_rel 0) that removes nothing."""
    img, hit, _, _ = F.range_image(scan, o)
    H, W = img.shape
    g = F._geom(o)
    q = F.to_sensor(map_xyz, pose)
    rm = np.sqrt((q * q).sum(1))
    az, el = F._angles(q)
    cu, ru = F._pixel_coords(az, el, g)
    col = np.minimum(np.floor(cu).astype(np.int64), W - 1)
    row = np.clip(np.floor(ru), -1e6, 1e6).astype(np.int64)
    known, mn, ok = F._neigh(img, hit, row, col, o.dilate)
    c = known & ok & (el >= g["el_min"]) & (el < g["el_max"]) & (rm >= o.min_range) & (rm <= o.max_range)
    return float((mn[c] - rm[c]).max())


STATIC = [("tiny", 0), ("tiny", 1), ("cfg1", 0), ("cfg1", 1), ("cfg2", 1), ("cfg2", 2)]
_MAPS = {}


def _map(name):
    if name not in _MAPS:
        _MAPS[name] = synth.make_map_for(name)
    return _MAPS[name]


@pytest.mark.parametrize("name,k", STATIC)
def test_static_scene_removes_nothing(name, k):
    """Exact pose, defaults (with the sensor's image geometry): nothing removed.  With a registration-sized pose error the count is
    printed and must stay at a handful; the smallest margin that still removes nothing at the exact pose is printed too."""
    scene, mp = _map(name)
    c = synth.make_case_on(scene, mp, name, k)
    sensor = synth.CONFIGS[name]["sensor"]
    o = F.opts_for(sensor)
    rem, st = F.clear(mp, c["scan_xyzi"], c["pose_true"], o)
    rem_err, st_err = F.clear(mp, c["scan_xyzi"], _pose_error(c["pose_true"], 50 + k), o)
    smallest = _max_excess(mp, c["scan_xyzi"], c["pose_true"], F.opts_for(sensor, margin=0.0, margin_rel=0.0))
    print(f"{name} scan {k}: {len(mp)} map points, {st['n_candidates']} candidates, removed {st['n_removed']} at the exact pose, "
          f"{st_err['n_removed']} with a {ERR_DT * 100:.0f} cm / {ERR_DEG} deg error; smallest margin removing nothing: {smallest:.3f} m")
    assert st["n_candidates"] > 0.2 * len(mp) or name != "cfg2"
    assert st["n_removed"] == 0
    assert st_err["n_removed"] <= 10
    assert smallest < o.margin


def _scene_with(scene, box):
    return synth.Scene(room=scene.room, boxes=np.vstack([scene.boxes, np.asarray(box, np.float64)[None]]))


def _box_map(scene, box, leaf=0.2, seed=9):
    """Voxel-filtered surface samples of the box alone (the map points a moving object leaves)."""
    only = synth.Scene(room=np.asarray(box, np.float64) + np.array([-1, 1, -1, 1, -1, 1]), boxes=np.asarray(box, np.float64)[None])
    raw = synth.sample_surfaces(only, leaf, seed=seed)
    lo = np.array([box[0], box[2], box[4]]) - 0.1
    hi = np.array([box[1], box[3], box[5]]) + 0.1
    raw = raw[((raw[:, :3] >= lo) & (raw[:, :3] <= hi)).all(1)]                 # the box's faces, not the room's
    return synth.voxel_filter_blocks(np.c_[raw, np.ones(len(raw), np.float32)], leaf)


@pytest.fixture(scope="module")
def tiny_setup():
    scene, mp = _map("tiny")
    pose = synth.random_sensor_pose(scene, 900, 4.0)
    # a 2 x 1.5 x 1.4 m box on the floor 6 m ahead of the sensor along x of the world, moved sideways until it is free of the scene
    for dy in np.arange(-3.0, 3.01, 0.5):
        cx, cy = pose[0] + 6.0, pose[1] + dy
        box = [cx - 1.0, cx + 1.0, cy - 0.75, cy + 0.75, -1.8, -0.4]
        if synth.Scene(room=scene.room, boxes=scene.boxes).free(np.array([cx, cy, -1.0]), margin=1.2):
            break
    return scene, mp, pose, np.array(box)


def test_box_seen_then_gone_is_removed(tiny_setup):
    """The box's faces inserted from a scan that saw it are removed once a scan from the same place sees through where it stood."""
    scene, mp, pose, box = tiny_setup
    o = F.opts_for("vlp16")
    with_box = synth.make_scan(_scene_with(scene, box), "vlp16", pose, 11)
    # what the insert of that scan added at the box: its returns that lie on the box
    R = synth.quat_to_R(pose[3:])
    w = with_box[:, :3].astype(np.float64) @ R.T + pose[:3]
    on_box = ((w >= np.array([box[0], box[2], box[4]]) - 0.05) & (w <= np.array([box[1], box[3], box[5]]) + 0.05)).all(1)
    ghost = np.c_[w[on_box], np.ones(on_box.sum())].astype(np.float32)
    assert len(ghost) > 100
    without = synth.make_scan(scene, "vlp16", pose, 12)
    rem, st = F.clear(np.vstack([mp, ghost]), without, pose, o)
    n_static = len(mp)
    # the rows where a (2 dilate + 1)^2 neighbourhood fits: the box's lowest points lie below the VLP-16's bottom beams
    q = F.to_sensor(ghost, pose)
    el = np.degrees(np.arctan2(q[:, 2], np.hypot(q[:, 0], q[:, 1])))
    row = np.floor((el - o.el_min_deg) / o.el_res_deg)
    fits = (row - o.dilate >= 0) & (row + o.dilate < F.dims(o)[1])
    frac = rem[n_static:][fits].mean()
    print(f"box returns in the map: {len(ghost)}, {fits.sum()} where a neighbourhood fits; removed {rem[n_static:].sum()} "
          f"({100 * frac:.1f} % of those), static removed {rem[:n_static].sum()}")
    assert fits.sum() > 50 and frac >= 0.9
    assert not rem[:n_static].any()


def test_occluded_points_are_never_removed(tiny_setup):
    """A box the scan does not see (it is in the map only) is carved where the scan saw past it, and never where something the scan
    saw stands in front of it: every removed point lies in front of the first surface along its own line of sight."""
    scene, mp, pose, box = tiny_setup
    o = F.opts_for("vlp16")
    ghost = _box_map(scene, box)
    scan = synth.make_scan(scene, "vlp16", pose, 13)
    allm = np.vstack([mp, ghost])
    rem, _ = F.clear(allm, scan, pose, o)
    d = allm[:, :3].astype(np.float64) - pose[:3]
    rm = np.linalg.norm(d, axis=1)
    surf = synth.raycast(scene, pose[:3], d / rm[:, None])              # range of the first static surface along each map point's ray
    occluded = surf < rm - 0.05
    print(f"ghost points {len(ghost)}, removed {rem[len(mp):].sum()}; occluded points {occluded.sum()}, removed among them "
          f"{(rem & occluded).sum()}")
    assert rem[len(mp):].sum() > 0.2 * len(ghost)        # its bottom face lies on the floor and its far faces are hidden
    assert not (rem & occluded).any()
    assert (surf[rem] > rm[rem]).all()


def test_unknown_pixels_never_carve(tiny_setup):
    """No return, no removal: with the scan's returns in a 30 deg azimuth sector deleted, nothing whose neighbourhood reaches the
    sector is removed, and an empty scan removes nothing at all."""
    scene, mp, pose, box = tiny_setup
    o = F.opts_for("vlp16")
    ghost = _box_map(scene, box)
    allm = np.vstack([mp, ghost])
    scan = synth.make_scan(scene, "vlp16", pose, 13)
    az_s = np.degrees(np.arctan2(scan[:, 1], scan[:, 0]))
    q = F.to_sensor(allm, pose)
    az_m = np.degrees(np.arctan2(q[:, 1], q[:, 0]))
    sector_m = np.abs(az_m - np.median(az_m[len(mp):])) <= 15.0 - 0.4 * (o.dilate + 1)    # inside the sector, beyond the neighbourhood
    lo, hi = np.median(az_m[len(mp):]) - 15.0, np.median(az_m[len(mp):]) + 15.0
    cut = scan[~((az_s >= lo) & (az_s <= hi))]
    rem, _ = F.clear(allm, cut, pose, o)
    rem_full, _ = F.clear(allm, scan, pose, o)
    assert rem_full[sector_m].sum() > 50                                # the sector does carve when it has returns
    assert not rem[sector_m].any()
    rem_empty, st = F.clear(allm, np.zeros((0, 4), np.float32), pose, o)
    assert not rem_empty.any() and st["n_pixels_hit"] == 0 and st["n_candidates"] == 0


def test_points_outside_the_span_and_the_range_are_untouched(tiny_setup):
    scene, mp, pose, box = tiny_setup
    ghost = _box_map(scene, box)
    allm = np.vstack([mp, ghost])
    scan = synth.make_scan(scene, "vlp16", pose, 13)
    q = F.to_sensor(allm, pose)
    rm = np.linalg.norm(q, axis=1)
    el = np.degrees(np.arctan2(q[:, 2], np.hypot(q[:, 0], q[:, 1])))
    base, _ = F.clear(allm, scan, pose, F.opts_for("vlp16"))
    assert base.sum() > 50
    near = F.opts_for("vlp16", min_range=float(np.median(rm[base])), max_range=float(np.max(rm[base])) - 0.5)
    rem, _ = F.clear(allm, scan, pose, near)
    assert rem.sum() > 0 and not rem[(rm < near.min_range) | (rm > near.max_range)].any()
    span = F.opts_for("vlp16", el_min_deg=-12.0, el_max_deg=-6.0)
    rem, _ = F.clear(allm, scan, pose, span)
    assert not rem[(el < -12.0) | (el >= -6.0)].any()


def test_azimuth_wraps_and_pixels_follow_the_floor_rule():
    """Pixel indices by hand: the azimuth -pi / +pi seam is column 0, the neighbourhood wraps across it, and an exact pixel edge
    belongs to the pixel above it."""
    o = F.Opts(az_res_deg=90.0, el_res_deg=30.0, el_min_deg=-45.0, el_max_deg=45.0, dilate=1, margin=0.1, margin_rel=0.0,
               min_range=0.0, max_range=100.0)
    assert F.dims(o) == (4, 3)
    pts = np.array([[-10.0, 0.0, 0.0], [-10.0, -1e-12, 0.0], [0.0, 10.0, 0.0], [10.0, 0.0, 0.0], [0.0, -10.0, 0.0]])
    img, hit, n, n_hit = F.range_image(np.c_[pts, np.ones(len(pts))].astype(np.float32), o)
    assert n == 5 and n_hit == 4 and np.array_equal(hit, np.isfinite(img))
    assert img[1, 0] == np.float32(10.0) and np.isfinite(img[1]).all() and not np.isfinite(img[0]).any()
    # every pixel of row 1 known but rows 0 and 2 unknown: a 3x3 neighbourhood never fits, dilate 0 does
    o0 = dataclasses_replace(o, dilate=0)
    rem, cand = F.removal_mask(np.array([[-5.0, 0.0, 0.0], [5.0, 0.0, 0.0]]), [0, 0, 0, 0, 0, 0, 1], img, hit, o0)
    assert cand.all() and rem.all()
    rem, cand = F.removal_mask(np.array([[-5.0, 0.0, 0.0]]), [0, 0, 0, 0, 0, 0, 1], img, hit, o)
    assert not cand.any() and not rem.any()


def dataclasses_replace(o, **kw):
    import dataclasses
    return dataclasses.replace(o, **kw)


def test_free_space_struct_layouts_match_header(tmp_path):
    from superodom_b200 import api
    f = tmp_path / "fs.c"
    fields = [n for n, _ in api.FreeSpace._fields_]
    rfields = ["n_image_points", "n_pixels_hit", "n_candidates", "n_removed", "n_after"]
    body = "".join(f'printf("%zu ", offsetof(so_free_space, {n}));' for n in fields)
    body += "".join(f'printf("%zu ", offsetof(so_free_space_result, {n}));' for n in rfields)
    f.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "superodom_b200.h"\nint main(void){'
                 'printf("%zu %zu ", sizeof(so_free_space), sizeof(so_free_space_result));' + body + 'return 0;}\n')
    exe = tmp_path / "fs"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(f), "-o", str(exe)])
    got = list(map(int, subprocess.check_output([str(exe)]).split()))
    want = [C.sizeof(api.FreeSpace), C.sizeof(api.FreeSpaceResult)]
    want += [getattr(api.FreeSpace, n).offset for n in fields] + [getattr(api.FreeSpaceResult, n).offset for n in rfields]
    assert got == want
    assert got[:2] == [36, 48]


def test_defaults_match_the_restatement():
    """so_free_space_defaults (host code, no GPU needed) and the restatement's Opts hold the same values."""
    from superodom_b200 import api, build
    build.build()
    o = api.free_space()
    ref = F.Opts()
    for n, _ in api.FreeSpace._fields_:
        assert getattr(o, n) == pytest.approx(getattr(ref, n), rel=1e-7), n
    assert math.isclose(o.margin, 0.3, rel_tol=1e-6) and o.dilate == 2

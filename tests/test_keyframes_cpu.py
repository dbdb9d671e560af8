"""Host side of the keyframe store and the map rebuilt from keyframes: the restatement in keyframe_map_numpy.py against the insert
restatement it must agree with, the new ABI entries declared and exported, and the shim's keyframe members compiling."""
import ctypes as C
import os
import subprocess

import numpy as np

import keyframe_map_numpy as KM
from map_archive_numpy import world_keys
from oracle import voxel_grid_numpy as vg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_ENTRIES = ["so_keyframe_reserve", "so_keyframe_add_registered", "so_keyframe_info", "so_keyframe_poses", "so_keyframe_download",
               "so_map_from_keyframes", "so_register_keyframes"]


def _cloud(rng, n, centre, spread):
    xyz = rng.normal(centre, spread, size=(n, 3))
    return np.concatenate([xyz, rng.uniform(1, 100, size=(n, 1))], 1).astype(np.float32)


def test_single_keyframe_into_empty_map_is_the_insert():
    rng = np.random.default_rng(3)
    c = _cloud(rng, 20000, (10.0, -20.0, 1.0), 30.0)
    c[5, 0] = np.nan
    for leaf in (0.2, 0.4, 0.1):
        win, arc = KM.map_from_keyframes([c], leaf)
        assert arc == {}
        assert np.array_equal(win, vg.map_insert(np.zeros((0, 4), np.float32), c, leaf)), leaf


def test_two_keyframes_are_one_filter_of_their_union():
    """Not a replay of inserts: the union is filtered once, so a voxel both keyframes reach averages every point once."""
    rng = np.random.default_rng(4)
    a, b = _cloud(rng, 5000, (0, 0, 0), 3.0), _cloud(rng, 5000, (0.5, 0, 0), 3.0)
    win, _ = KM.map_from_keyframes([a, b], 0.4)
    assert np.array_equal(win, vg.block_voxel_grid(np.concatenate([a, b]), 0.4))
    replay = vg.map_insert(vg.map_insert(np.zeros((0, 4), np.float32), a, 0.4), b, 0.4)
    assert len(win) == len(replay) and not np.array_equal(win, replay)


def test_empty_ids_give_an_empty_store():
    win, arc = KM.map_from_keyframes([], 0.2, archive=True)
    assert win.shape == (0, 4) and arc == {}
    assert KM.download_all(win, arc).shape == (0, 4)


def test_off_window_blocks_are_keyed_by_world_block():
    """With the archive on, a block outside the window goes to the archive under its world key (origin-free), filtered on its own;
    with it off, it is dropped."""
    rng = np.random.default_rng(5)
    near = _cloud(rng, 3000, (0, 0, 0), 5.0)
    far = _cloud(rng, 3000, (700.0, -40.0, 0.0), 4.0)            # 14 blocks east of the window's edge (origin (10, 10, 5))
    win, arc = KM.map_from_keyframes([near, far], 0.2, archive=True)
    assert np.array_equal(win, KM.map_from_keyframes([near], 0.2)[0])
    keys = world_keys(far[:, :3])
    assert sorted(arc) == sorted(set(int(k) for k in keys))
    for k, blk in arc.items():
        assert np.array_equal(blk, vg.voxel_grid(far[keys == k], 0.2))
    assert np.array_equal(KM.map_from_keyframes([near, far], 0.2, archive=False)[0], win)
    # the same blocks seen through another window: the archive keys do not change, the window's part moves
    win2, arc2 = KM.map_from_keyframes([near, far], 0.2, origin=(-4, 11, 5), archive=True)
    assert sorted(set(arc2) | set(int(k) for k in world_keys(win2[:, :3]))) == sorted(set(arc) | set(int(k) for k in world_keys(win[:, :3])))
    all1, all2 = KM.download_all(win, arc), KM.download_all(win2, arc2)
    assert np.array_equal(all1, all2)


def test_small_leaf_uses_the_absolute_index():
    """Below 0.04 m a 50 m block can overflow PCL's index; the restatement then orders by the absolute voxel, as the insert does."""
    rng = np.random.default_rng(6)
    c = _cloud(rng, 4000, (0, 0, 0), 8.0)
    c = c[(np.abs(c[:, :3]) < 24.0).all(1)]                      # one block
    assert vg.falls_back(c, 0.01)
    win, _ = KM.map_from_keyframes([c], 0.01)
    assert np.array_equal(win, vg.absolute_voxel_grid(c, 0.01))


def test_new_entries_declared_and_exported():
    from superodom_b200 import api, build
    from test_abi import _declared
    L = C.CDLL(build.build())
    decl = _declared()
    for name in NEW_ENTRIES:
        assert name in decl and name in api.EXPORTS and hasattr(L, name), name


def test_keyframe_shim_compiles_and_links(tmp_path):
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "keyframe_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "keyframe_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(exe)

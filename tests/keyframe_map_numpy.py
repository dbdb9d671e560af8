"""Restatement of so_map_from_keyframes (include/superodom_b200.h, "keyframes") on top of oracle/voxel_grid_numpy.py, apart from the
device code.  Input: the selected keyframes already in the world frame, in ids order (what so_keyframe_download(id, pose) returns).

    union      the keyframes in ids order, each in its point order; non-finite points dropped
    blocks     LocalMap's 50 m block of every point (world block w = g - origin); kept: the window's blocks, and every block in the
               archive's key range when the archive is on
    filter     each block's cloud (union order) through pcl::VoxelGrid at the store's leaf on its own; where PCL would fall back (its
               index overflows: leaves below 0.04 m) the absolute voxel index, as the map insert does
    window     the window's blocks, block by block (cube order = world key order), as the store's cloud
    archive    {world key: filtered block cloud} of the off-window blocks"""
import numpy as np

from map_archive_numpy import in_window, world_keys
from oracle import voxel_grid_numpy as vg

ARCHIVE_RANGE = 50.0 * (1 << 19)          # |x + 25| below this: the block lies in the archive's key range


def block_filter(cloud, leaf):
    """One block's filter: pcl::VoxelGrid, or the absolute-index order where PCL's index would overflow."""
    return vg.absolute_voxel_grid(cloud, leaf) if vg.falls_back(cloud, leaf) else vg.voxel_grid(cloud, leaf)


def map_from_keyframes(world_clouds, leaf, origin=vg.ORIGIN0, archive=False):
    """-> (window float32 [n, 4], {world key: float32 [m, 4]}) of the map of the union of world_clouds."""
    parts = [np.ascontiguousarray(c, np.float32).reshape(-1, 4) for c in world_clouds]
    u = np.concatenate(parts, 0) if parts else np.zeros((0, 4), np.float32)
    u = u[np.isfinite(u[:, :3]).all(1)]
    u = u[(np.abs(u[:, :3].astype(np.float64) + 25.0) < ARCHIVE_RANGE).all(1)]
    inside = in_window(u[:, :3], origin)
    if not archive:
        u, inside = u[inside], inside[inside]
    keys = world_keys(u[:, :3])
    order = np.argsort(keys, kind="stable")
    u, keys, inside = u[order], keys[order], inside[order]
    window, arc = [], {}
    cut = np.flatnonzero(np.diff(keys)) + 1
    for k, blk, ins in zip(keys[np.r_[0, cut]] if len(u) else [], np.split(u, cut), np.split(inside, cut)):
        f = block_filter(blk, leaf)
        if ins[0]:
            window.append(f)
        else:
            arc[int(k)] = f
    return (np.concatenate(window, 0) if window else np.zeros((0, 4), np.float32)), arc


def download_all(window, arc):
    """so_map_download_all of the result: window and archive blocks by world key, then by the order within the block."""
    blocks = dict(arc)
    if len(window):
        keys = world_keys(window[:, :3])
        cut = np.flatnonzero(np.diff(keys)) + 1
        for k, blk in zip(keys[np.r_[0, cut]], np.split(window, cut)):
            blocks[int(k)] = blk
    return np.concatenate([blocks[k] for k in sorted(blocks)], 0) if blocks else np.zeros((0, 4), np.float32)

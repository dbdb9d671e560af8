"""Restatement of a map store with the block archive on (include/superodom_b200.h, "block archive"): a LocalMap over an unbounded
block grid seen through the 21 x 21 x 11 window.  The window is the store's cloud in store order; the archive maps a world block key
to that block's cloud.  Built on oracle.map_insert_numpy (the insert), synth.block_of (the binning) and oracle.cube_order."""
import numpy as np

KEY_BITS = 20
KEY_OFF = 1 << (KEY_BITS - 1)


class CapacityError(Exception):
    pass


def world_blocks(xyz):
    """World block coordinate w = g - origin of every point (synth.block_of with origin 0)."""
    from superodom_b200 import synth
    return synth.block_of(np.ascontiguousarray(xyz, np.float32), (0, 0, 0)).astype(np.int64)


def world_keys(xyz):
    w = world_blocks(xyz) + KEY_OFF
    return (w[:, 2] << (2 * KEY_BITS)) | (w[:, 1] << KEY_BITS) | w[:, 0]


def in_window(xyz, origin):
    from superodom_b200 import synth
    return synth.block_linear(synth.block_of(np.ascontiguousarray(xyz, np.float32), origin)) >= 0


def _group(pts):
    """{key: block cloud in the order given}"""
    out = {}
    if len(pts) == 0:
        return out
    keys = world_keys(pts[:, :3])
    order = np.argsort(keys, kind="stable")
    keys, pts = keys[order], pts[order]
    cut = np.flatnonzero(np.diff(keys)) + 1
    for k, block in zip(keys[np.r_[0, cut]], np.split(pts, cut)):
        out[int(k)] = block
    return out


class ArchiveModel:
    def __init__(self, cap, max_map_points, origin=(10, 10, 5)):
        self.cap, self.max_map_points = cap, max_map_points
        self.origin = tuple(int(v) for v in origin)
        self.window = np.zeros((0, 4), np.float32)
        self.archive = {}

    def archived_points(self):
        return sum(len(b) for b in self.archive.values())

    def set_points(self, xyzi):
        """so_map_set_points: the window's part in order, the rest to the archive by block; non-finite points dropped."""
        p = np.ascontiguousarray(xyzi, np.float32)
        p = p[np.isfinite(p[:, :3]).all(1)]
        inside = in_window(p[:, :3], self.origin)
        if inside.sum() > self.max_map_points or (~inside).sum() > self.cap:
            raise CapacityError
        self.window, self.archive = p[inside], _group(p[~inside])

    def insert(self, new_xyzi, leaf):
        """so_map_add_*: the window's insert; points off the window are dropped."""
        from oracle.oracle import map_insert_numpy
        self.window = map_insert_numpy(self.window, new_xyzi, leaf, self.origin)

    def set_origin(self, origin):
        """The rebuild that applies an origin change: blocks leaving the window go to the archive, archived blocks the window now
        covers come back (in key order) behind the window's remaining points."""
        origin = tuple(int(v) for v in origin)
        keep = in_window(self.window[:, :3], origin)
        back = sorted(k for k, b in self.archive.items() if in_window(b[:1, :3], origin)[0])
        n_back = sum(len(self.archive[k]) for k in back)
        leaving = self.window[~keep]
        if self.archived_points() - n_back + len(leaving) > self.cap or keep.sum() + n_back > self.max_map_points:
            raise CapacityError
        restored = [self.archive.pop(k) for k in back]
        self.window = np.concatenate([self.window[keep]] + restored, 0) if restored else self.window[keep]
        self.archive.update(_group(leaving))
        self.origin = origin

    def download(self):
        """so_map_download(0) of a context whose other store is empty: the window in cube order."""
        from oracle.oracle import cube_order
        return self.window[cube_order(self.window, self.origin)]

    def download_all(self):
        """so_map_download_all: window and archive by world key, then by the order within the block."""
        blocks = dict(self.archive)
        blocks.update(_group(self.window))
        if not blocks:
            return np.zeros((0, 4), np.float32)
        return np.concatenate([blocks[k] for k in sorted(blocks)], 0)

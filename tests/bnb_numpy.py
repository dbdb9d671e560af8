"""numpy restatement of the branch-and-bound bounds of so_localize_global_bnb: the pyramid levels B_L and the node bounds U.

B_L(x, y, z) = OR over a, b in [0, 2^L) of B(x+a, y+b, z), with B the dilated occupancy bitmap of the whole search box
(global_localization_numpy.bitmap, read as 0 outside the box).  This is computed straight from the definition, a sliding-window
OR by prefix sums, not by the library's doubling.  A level-L node (yaw m, z shift k, x/y shift tile (a, b)) covers x shifts
[a 2^L, (a+1) 2^L) and y shifts [b 2^L, (b+1) 2^L); its bound is U = sum over score points of B_L at the point's voxel for
shift (a 2^L, b 2^L, k).  Shared by tests/test_global_localization_bnb.py and scripts/bench_reloc.py.
"""
from __future__ import annotations

import numpy as np

import global_localization_numpy as GN

ROOT_NODES = 1 << 16             # kBnbRoot: the root size the Lmax rule aims for


def _ceil_div(a, b):
    return -(-a // b)


def level_nodes(P, L):
    s = 1 << L
    return P["nyaw"] * P["nz"] * _ceil_div(P["nx"], s) * _ceil_div(P["ny"], s)


def lmax(P):
    """The smallest L >= 1 whose root level fits ROOT_NODES nodes, or at which one root tile covers every x/y shift."""
    L = 1
    while not ((_ceil_div(P["nx"], 1 << L) == 1 and _ceil_div(P["ny"], 1 << L) == 1) or level_nodes(P, L) <= ROOT_NODES):
        L += 1
    return L


def _window_or(A, s, axis):
    """OR of s consecutive elements along axis: out[i] = any(A[i : i + s]), len = A.shape[axis] - s + 1."""
    n = A.shape[axis] - s + 1
    c = np.cumsum(A, axis=axis, dtype=np.int32)
    c = np.concatenate([np.zeros_like(np.take(c, [0], axis=axis)), c], axis=axis)
    return (np.take(c, np.arange(s, s + n), axis=axis) - np.take(c, np.arange(n), axis=axis)) > 0


def level(B, L):
    """B_L of the box bitmap B [bz, by, bx] -> bool [bz, by + 2^L - 1, bx + 2^L - 1], element [z, y + 2^L - 1, x + 2^L - 1] = B_L(x, y, z)
    for x, y from -(2^L - 1) (windows starting below the box) to the box's end."""
    s = 1 << L
    Bp = np.pad(B, ((0, 0), (s - 1, s - 1), (s - 1, s - 1)))
    return _window_or(_window_or(Bp, s, 2), s, 1)


def bounds(scan_xyzi, center, map_xyz, L, half_x=0.0, half_y=0.0, half_z=0.0, yaw_half=0.0, B=None, **kw):
    """U of every level-L node -> (uint16 [nyaw, nz, ceil(ny / 2^L), ceil(nx / 2^L)], number of score points).  B: the box bitmap,
    if already computed."""
    P = GN.plan(half_x, half_y, half_z, yaw_half, **kw)
    pts = GN.score_points(scan_xyzi, P["score_points"], P["max_range"])
    _, _, qs = GN.yaw_quaternions(P, center)
    if B is None:
        B = GN.bitmap(map_xyz, P, center)
    s = 1 << L
    pad = 2
    BL = np.pad(level(B, L), pad)
    e, res = P["e"], P["res"]
    nz = P["nz"]
    nbx, nby = _ceil_div(P["nx"], s), _ceil_div(P["ny"], s)
    v = pts[:, :3].astype(np.float64)
    out = np.zeros((P["nyaw"], nz, nby, nbx), np.int64)
    for m, q in enumerate(qs):
        w = np.floor(GN._qrot(q, v) / res).astype(np.int64) + e + pad       # padded-box index of shift (0, 0, 0)
        assert (w >= 0).all() and (w[:, 2] + nz <= BL.shape[0]).all()
        acc = out[m]
        for p in range(len(w)):
            wx, wy, wz = w[p]
            y0, x0 = wy + s - 1, wx + s - 1                                     # B_L of box voxel y sits at row y + s - 1
            acc += BL[wz:wz + nz, y0:y0 + (nby - 1) * s + 1:s, x0:x0 + (nbx - 1) * s + 1:s]
    return out.astype(np.uint16), len(pts)


def prefix_keys(scores, n_keys):
    """The first n_keys of the ascending order of every hypothesis' key (65535 - score) << 32 | index, scores [nyaw, nz, ny, nx]."""
    s = scores.reshape(-1).astype(np.int64)
    order = np.lexsort((np.arange(len(s)), -s))[:n_keys]
    return ((65535 - s[order]).astype(np.uint64) << np.uint64(32)) | order.astype(np.uint64)

"""Numpy restatement of so_scan_extract_edges (LOAM edge selection, DESIGN.md §9), written apart from the device code.

Every step is float32 with each + - * / sqrt rounded on its own (numpy float32 arithmetic does not contract), sums left to
right as the definition writes them.  `extract_edges_loop` is the same definition as a plain per-point loop over Python floats
rounded through np.float32 after every operation; the CPU tests hold the two against each other.
"""
from __future__ import annotations

import numpy as np

F = np.float32
OCC_GAP2 = F(0.1)         # |q_{k+1} - q_k|^2 above this: an occlusion boundary candidate
OCC_RATIO = F(0.1)        # relative distance below which the farther side is occluded
PAR_RATIO = F(0.0002)     # parallel-beam test
NB_GAP2 = F(0.05)         # neighbour marks stop at a gap above this


def records_fields(records: np.ndarray, stride: int, time_offset: int, ring_offset: int):
    """(xyz float32 [n,3], time float32 [n], ring uint16 [n]) of raw records (a byte view of n records of `stride` bytes)."""
    b = np.ascontiguousarray(records).view(np.uint8).reshape(-1, stride)
    xyz = np.ascontiguousarray(b[:, 0:12]).view(np.float32).reshape(-1, 3)
    t = np.ascontiguousarray(b[:, time_offset:time_offset + 4]).view(np.float32).reshape(-1)
    ring = np.ascontiguousarray(b[:, ring_offset:ring_offset + 2]).view(np.uint16).reshape(-1)
    return xyz, t, ring


def _n2(d):
    """|v|^2 = (vx*vx + vy*vy) + vz*vz per row, float32."""
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _valid_order(xyz, t, ring, min_range):
    with np.errstate(over="ignore", invalid="ignore"):
        ok = np.isfinite(xyz).all(1) & np.isfinite(t) & (_n2(xyz) > F(min_range) * F(min_range))
    idx = np.flatnonzero(ok)
    tv = t[idx] + F(0.0)                      # -0 + 0 = +0: time compares as a value
    order = np.lexsort((idx, tv, ring[idx]))
    return idx[order]


def _ring_edges(q, thr, max_per_sector):
    """Accepted positions of one ring q [m,3] (float32), ascending."""
    m = len(q)
    if m - 6 - 5 < 6:
        return np.zeros(0, np.int64)
    excl = np.zeros(m, bool)
    with np.errstate(over="ignore", invalid="ignore"):
        # curvature, 5 <= k <= m-6
        k = np.arange(5, m - 5)
        s = q[k - 5].copy()
        for o in (-4, -3, -2, -1, 1, 2, 3, 4, 5):
            s = s + q[k + o]
        c = np.zeros(m, F)
        c[k] = _n2(s - F(10.0) * q[k])
        # occlusion, 5 <= k <= m-7
        for kk in range(5, m - 6):
            a, b = q[kk], q[kk + 1]
            d = b - a
            if _n2(d) > OCC_GAP2:
                ra, rb = np.sqrt(_n2(a)), np.sqrt(_n2(b))
                if ra > rb:
                    e = b - ((a * rb) / ra)
                    if np.sqrt(_n2(e)) / rb < OCC_RATIO:
                        excl[max(kk - 5, 0):kk + 1] = True
                else:
                    e = ((b * ra) / rb) - a
                    if np.sqrt(_n2(e)) / ra < OCC_RATIO:
                        excl[kk + 1:min(kk + 7, m)] = True
        # parallel beam, 5 <= k <= m-6
        n2 = _n2(q)
        dprev = _n2(q[k] - q[k - 1])
        dnext = _n2(q[k + 1] - q[k])
        lim = PAR_RATIO * n2[k]
        excl[k[(dprev > lim) & (dnext > lim)]] = True
        gap = np.zeros(m, F)                  # gap[p] = |q_p - q_{p-1}|^2
        gap[1:] = _n2(q[1:] - q[:-1])
    a, z = 5, m - 6
    acc = []
    for j in range(6):
        sp = a + (z - a) * j // 6
        ep = a + (z - a) * (j + 1) // 6 - 1
        pos = np.arange(sp, ep + 1)
        cand = pos[c[pos] > F(thr)]           # NaN is never a candidate
        cand = cand[np.lexsort((cand, -c[cand].astype(np.float64)))]
        n_acc = 0
        for kk in cand:
            if n_acc >= max_per_sector:
                break
            if excl[kk]:
                continue
            acc.append(kk)
            n_acc += 1
            excl[kk] = True
            for l in range(1, 6):
                if gap[kk + l] > NB_GAP2:
                    break
                excl[kk + l] = True
            for l in range(1, 6):
                if gap[kk - l + 1] > NB_GAP2:
                    break
                excl[kk - l] = True
    return np.sort(np.array(acc, np.int64))


def extract_edges(xyz, t, ring, min_range=0.0, edge_threshold=0.1, max_per_sector=20):
    """-> float32 [k,4] {x, y, z, time}: the accepted points ordered by (ring, position)."""
    xyz = np.ascontiguousarray(xyz, F)
    t = np.ascontiguousarray(t, F)
    ring = np.ascontiguousarray(ring, np.uint16)
    sel = _valid_order(xyz, t, ring, min_range)
    out = []
    r = ring[sel]
    bounds = np.flatnonzero(np.r_[True, r[1:] != r[:-1], True]) if len(sel) else np.zeros(1, np.int64)
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        ids = sel[lo:hi]
        keep = _ring_edges(xyz[ids], edge_threshold, max_per_sector)
        out.append(ids[keep])
    ids = np.concatenate(out) if out else np.zeros(0, np.int64)
    return np.concatenate([xyz[ids], t[ids, None]], 1).astype(F)


# ------------------------------------------------------------------------------------------------ per-point loop version
def _f(v):
    return float(F(v))


def _sub3(a, b):
    return (_f(a[0] - b[0]), _f(a[1] - b[1]), _f(a[2] - b[2]))


def _nrm2(v):
    return _f(_f(_f(v[0] * v[0]) + _f(v[1] * v[1])) + _f(v[2] * v[2]))


def extract_edges_loop(xyz, t, ring, min_range=0.0, edge_threshold=0.1, max_per_sector=20):
    """The definition as a straightforward loop over points (slow; small scans only)."""
    pts = []
    mr2 = _f(_f(min_range) * _f(min_range))
    for i in range(len(xyz)):
        p = tuple(float(v) for v in np.asarray(xyz[i], F))
        ti = float(F(t[i]))
        if not all(np.isfinite(p)) or not np.isfinite(ti):
            continue
        with np.errstate(over="ignore"):
            if not _nrm2(p) > mr2:
                continue
        pts.append((int(ring[i]), ti + 0.0, i, p, ti))
    pts.sort(key=lambda e: (e[0], e[1], e[2]))
    res = []
    i = 0
    while i < len(pts):
        j = i
        while j < len(pts) and pts[j][0] == pts[i][0]:
            j += 1
        q = [e[3] for e in pts[i:j]]
        m = len(q)
        if m >= 17:
            c = [0.0] * m
            for k in range(5, m - 5):
                s = q[k - 5]
                for o in (-4, -3, -2, -1, 1, 2, 3, 4, 5):
                    s = (_f(s[0] + q[k + o][0]), _f(s[1] + q[k + o][1]), _f(s[2] + q[k + o][2]))
                ten = (_f(10.0 * q[k][0]), _f(10.0 * q[k][1]), _f(10.0 * q[k][2]))
                c[k] = _nrm2(_sub3(s, ten))
            ex = [False] * m
            for k in range(5, m - 6):
                if _nrm2(_sub3(q[k + 1], q[k])) > _f(0.1):
                    ra, rb = _f(np.sqrt(F(_nrm2(q[k])))), _f(np.sqrt(F(_nrm2(q[k + 1]))))
                    if ra > rb:
                        e = tuple(_f(q[k + 1][a] - _f(_f(q[k][a] * rb) / ra)) for a in range(3))
                        if _f(_f(np.sqrt(F(_nrm2(e)))) / rb) < _f(0.1):
                            for u in range(max(k - 5, 0), k + 1):
                                ex[u] = True
                    else:
                        e = tuple(_f(_f(_f(q[k + 1][a] * ra) / rb) - q[k][a]) for a in range(3))
                        if _f(_f(np.sqrt(F(_nrm2(e)))) / ra) < _f(0.1):
                            for u in range(k + 1, min(k + 7, m)):
                                ex[u] = True
            for k in range(5, m - 5):
                lim = _f(_f(0.0002) * _nrm2(q[k]))
                if _nrm2(_sub3(q[k], q[k - 1])) > lim and _nrm2(_sub3(q[k + 1], q[k])) > lim:
                    ex[k] = True
            a, z = 5, m - 6
            acc = []
            for sec in range(6):
                sp = a + (z - a) * sec // 6
                ep = a + (z - a) * (sec + 1) // 6 - 1
                order = sorted(range(sp, ep + 1), key=lambda k: (-c[k], k))
                n_acc = 0
                for k in order:
                    if not c[k] > _f(edge_threshold) or n_acc >= max_per_sector:
                        break
                    if ex[k]:
                        continue
                    acc.append(k)
                    n_acc += 1
                    ex[k] = True
                    for l in range(1, 6):
                        if _nrm2(_sub3(q[k + l], q[k + l - 1])) > _f(0.05):
                            break
                        ex[k + l] = True
                    for l in range(1, 6):
                        if _nrm2(_sub3(q[k - l], q[k - l + 1])) > _f(0.05):
                            break
                        ex[k - l] = True
            for k in sorted(acc):
                e = pts[i + k]
                res.append([e[3][0], e[3][1], e[3][2], e[4]])
        i = j
    return np.array(res, F).reshape(-1, 4)

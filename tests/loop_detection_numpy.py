"""Numpy restatement of loop detection (so_loop_candidates, so_keyframe_descriptors; DESIGN.md, "Loop detection"), written apart from
the device code.

Descriptor (Scan Context) of a sensor-frame cloud at pose q:
  - levelling: R = R(q) (quaternion normalised), psi = atan2(R10, R00), L = Rz(-psi) R, taken as cos psi = R00 / h, sin psi = R10 / h
    with h = sqrt(R00^2 + R10^2) (psi = 0 when h = 0); v = L p with every row summed ((a + b) + c); non-finite points skipped;
  - rho = hypot(vx, vy), skipped when rho >= max_range; ring floor(rho / max_range * rings), at most rings - 1;
  - az = atan2(vy, vx) folded to [-pi, pi); sector floor((az + pi) / (2 pi / sectors)), at most sectors - 1;
  - cell: max over its points of max(0, float32(vz + height_offset)); 0 when empty.  Column norms: sqrt of the squares summed in ring
    order.

`describe_bounds` gives two images the device's must lie between, for the rounding differences of atan2 and hypot: a point within eps
bin of a ring or sector edge (the azimuth seam included, whose two sides are sectors sectors - 1 and 0) or of max_range is left out of
the lower image and put into every cell it may fall in in the upper one.

The distance and the search loop in the device's fixed order (dot over rings, cosines over ascending query columns), so they are
compared bit for bit.  `search` takes one pair at a time; `search_many` gives the same rows with the arithmetic vectorised over
[candidates, shifts] (rings and columns still summed one at a time, in order), fast enough for thousands of keyframes.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np


@dataclasses.dataclass
class Opts:
    """Mirror of so_loop_opts; the defaults are so_loop_opts_defaults'."""
    rings: int = 20
    sectors: int = 60
    max_range: float = 80.0
    height_offset: float = 2.0
    exclude_recent: int = 30

    def kw(self):
        return dataclasses.asdict(self)


def levelling(pose7) -> np.ndarray:
    """L = Rz(-psi) R(q), row-major [3, 3], in the host's expression order."""
    qx, qy, qz, qw = (float(v) for v in pose7[3:7])
    nq = math.sqrt(qx * qx + qy * qy + qz * qz + qw * qw)
    x, y, z, w = qx / nq, qy / nq, qz / nq, qw / nq
    R = [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
         2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
         2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]
    h = math.sqrt(R[0] * R[0] + R[3] * R[3])
    cs, sn = (R[0] / h, R[3] / h) if h > 0 else (1.0, 0.0)
    L = [0.0] * 9
    for k in range(3):
        L[k] = cs * R[k] + sn * R[3 + k]
        L[3 + k] = cs * R[3 + k] - sn * R[k]
        L[6 + k] = R[6 + k]
    return np.array(L, np.float64).reshape(3, 3)


def _bins(xyz, pose7, o: Opts):
    p32 = np.asarray(xyz, np.float32)[:, :3]
    p32 = p32[np.isfinite(p32).all(1)]
    p = p32.astype(np.float64)
    L = levelling(pose7)
    v = [(L[r, 0] * p[:, 0] + L[r, 1] * p[:, 1]) + L[r, 2] * p[:, 2] for r in range(3)]
    rho = np.hypot(v[0], v[1])
    ru = (rho / float(o.max_range)) * float(o.rings)
    az = np.arctan2(v[1], v[0])
    az = np.where(az >= math.pi, az - 2 * math.pi, az)
    cu = (az + math.pi) / ((2.0 * math.pi) / float(o.sectors))
    val = np.maximum(np.float32(0), (v[2] + float(o.height_offset)).astype(np.float32))
    return rho, ru, cu, val


def describe_bounds(xyz, pose7, o: Opts, eps: float = 1e-9):
    """-> (lower, upper) float32 images [rings, sectors]; eps = 0 gives the one image of numpy's own roundings twice."""
    Nr, Ns = int(o.rings), int(o.sectors)
    rho, ru, cu, val = _bins(xyz, pose7, o)
    inside = rho < float(o.max_range)
    near_far = np.abs(ru - Nr) < eps if eps > 0 else np.zeros(len(ru), bool)
    ring = np.minimum(np.floor(ru), Nr - 1).astype(np.int64)
    sector = np.minimum(np.floor(cu), Ns - 1).astype(np.int64)
    fr, fc = ru - np.floor(ru), cu - np.floor(cu)
    if eps > 0:
        amb_r = (fr < eps) | (fr > 1 - eps)
        seam = (cu < eps) | (cu > Ns - eps)
        amb_c = (fc < eps) | (fc > 1 - eps) | seam
    else:
        amb_r = amb_c = seam = np.zeros(len(ru), bool)
    alt_r = np.clip(np.where(fr < 0.5, ring - 1, ring + 1), 0, Nr - 1)
    alt_c = np.where(seam, np.where(sector == 0, Ns - 1, 0), np.where(fc < 0.5, sector - 1, sector + 1) % Ns)
    lo = np.zeros(Nr * Ns, np.float32)
    hi = np.zeros(Nr * Ns, np.float32)
    sure = inside & ~near_far & ~amb_r & ~amb_c
    np.maximum.at(lo, ring[sure] * Ns + sector[sure], val[sure])
    maybe = inside | near_far
    for rr in (ring, alt_r):
        for cc in (sector, alt_c):
            m = maybe & ((rr == ring) | amb_r) & ((cc == sector) | amb_c)
            r2 = np.minimum(rr[m], Nr - 1)
            np.maximum.at(hi, r2 * Ns + cc[m], val[m])
    return lo.reshape(Nr, Ns), hi.reshape(Nr, Ns)


def describe(xyz, pose7, o: Opts) -> np.ndarray:
    return describe_bounds(xyz, pose7, o, eps=0.0)[0]


def norms(img) -> np.ndarray:
    """Column norms [sectors]: squares summed in ring order in FP64."""
    a = np.asarray(img, np.float32).astype(np.float64)
    acc = np.zeros(a.shape[1])
    for r in range(a.shape[0]):
        acc = acc + a[r] * a[r]
    return np.sqrt(acc)


def distances(a, b, na=None, nb=None):
    """d(a, b, s) and n_pairs for every shift s -> (d [sectors] float64, n [sectors] int), in the device's order."""
    A, B = np.asarray(a, np.float32).astype(np.float64), np.asarray(b, np.float32).astype(np.float64)
    na = norms(a) if na is None else na
    nb = norms(b) if nb is None else nb
    Nr, Ns = A.shape
    cols = (np.arange(Ns)[None, :] + np.arange(Ns)[:, None]) % Ns          # [s, j] -> candidate column
    dot = np.zeros((Ns, Ns))
    for r in range(Nr):
        dot = dot + A[r][None, :] * B[r][cols]
    nbc = nb[cols]
    valid = (na[None, :] != 0) & (nbc != 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        cos = np.where(valid, dot / np.where(valid, na[None, :] * nbc, 1.0), 0.0)
    acc = np.zeros(Ns)
    for j in range(Ns):
        acc = acc + cos[:, j]
    n = valid.sum(1)
    with np.errstate(invalid="ignore", divide="ignore"):
        d = np.where(n > 0, 1.0 - acc / np.maximum(n, 1).astype(np.float64), 1.0)
    return d, n


def pair(a, b, na=None, nb=None):
    """-> (distance, shift, n_pairs): the minimum over shifts, ties to the lowest shift."""
    d, n = distances(a, b, na, nb)
    s = int(np.argmin(d))
    return float(d[s]), s, int(n[s])


def yaw_of(shift: int, sectors: int) -> float:
    y = float(shift) * ((2.0 * math.pi) / float(sectors))
    return y - 2.0 * math.pi if y > math.pi else y


def search(descs, queries, k: int, exclude_recent: int):
    """descs [frames, rings, sectors] (the device's images) -> [(id, distance, shift, n_pairs, yaw)] * k per query."""
    nrm = [norms(d) for d in descs]
    Ns = descs.shape[2]
    out = []
    for q in queries:
        m = max(int(q) - int(exclude_recent), 0)
        rows = []
        for b in range(m):
            d, s, n = pair(descs[q], descs[b], nrm[q], nrm[b])
            rows.append((d, b, s, n))
        rows.sort(key=lambda t: (t[0], t[1]))
        best = [(b, d, s, n, yaw_of(s, Ns)) for d, b, s, n in rows[:k]]
        best += [(-1, 1.0, 0, 0, 0.0)] * (k - len(best))
        out.append(best)
    return out


def _norms_all(A):
    """norms() of every image of A [frames, rings, sectors] float64, squares summed in ring order."""
    acc = np.zeros((A.shape[0], A.shape[2]))
    for r in range(A.shape[1]):
        acc = acc + A[:, r] * A[:, r]
    return np.sqrt(acc)


def _row(A, nrm, q, m, k, Ns, chunk_elems=1 << 22):
    """search()'s row of query q against candidates 0 .. m-1, vectorised over [candidates, shifts] in the same order of operations."""
    if m == 0:
        return [(-1, 1.0, 0, 0, 0.0)] * k
    from numpy.lib.stride_tricks import sliding_window_view
    Nr = A.shape[1]
    na = nrm[q]
    dq, sq, nq = np.empty(m), np.empty(m, np.int64), np.empty(m, np.int64)
    step = max(1, chunk_elems // (Ns * Ns))
    for c0 in range(0, m, step):
        # the candidate's columns twice over: [.., s, j] of a window view is column (j + s) mod sectors, without a copy
        B2 = np.concatenate([A[c0:min(c0 + step, m)]] * 2, 2)[..., :2 * Ns - 1]
        nb2 = np.concatenate([nrm[c0:min(c0 + step, m)]] * 2, 1)[:, :2 * Ns - 1]
        c = len(B2)
        W = sliding_window_view(B2, Ns, axis=2)                             # [candidate, ring, s, j]
        dot = np.zeros((c, Ns, Ns))                                         # [candidate, s, j]
        prod = np.empty_like(dot)
        for r in range(Nr):
            np.multiply(A[q, r][None, None, :], W[:, r], out=prod)
            np.add(dot, prod, out=dot)
        nbc = sliding_window_view(nb2, Ns, axis=1)
        valid = (na[None, None, :] != 0) & (nbc != 0)
        with np.errstate(invalid="ignore", divide="ignore"):
            cos = np.where(valid, dot / np.where(valid, na[None, None, :] * nbc, 1.0), 0.0)
        acc = np.zeros((c, Ns))
        for j in range(Ns):
            acc = acc + cos[:, :, j]
        n = valid.sum(2)
        with np.errstate(invalid="ignore", divide="ignore"):
            d = np.where(n > 0, 1.0 - acc / np.maximum(n, 1).astype(np.float64), 1.0)
        s = np.argmin(d, 1)                                                 # the lowest shift of a tie
        at = np.arange(c)
        dq[c0:c0 + c], sq[c0:c0 + c], nq[c0:c0 + c] = d[at, s], s, n[at, s]
    ids = np.arange(m)
    order = np.lexsort((ids, dq))[:k]
    best = [(int(b), float(dq[b]), int(sq[b]), int(nq[b]), yaw_of(int(sq[b]), Ns)) for b in order]
    return best + [(-1, 1.0, 0, 0, 0.0)] * (k - len(best))


def search_many(descs, queries, k: int, exclude_recent: int):
    """search() for many candidates and queries: the same rows, bit for bit, with each distinct query's row computed once."""
    A = np.asarray(descs, np.float32).astype(np.float64)
    nrm = _norms_all(A)
    Ns = A.shape[2]
    rows = {}
    out = []
    for q in queries:
        q = int(q)
        if q not in rows:
            rows[q] = _row(A, nrm, q, max(q - int(exclude_recent), 0), k, Ns)
        out.append(list(rows[q]))
    return out

"""Stored outputs of the reference's own k-NN (flann/octree.h, compiled verbatim into oracle/_ref) for the parity tests.

The reference octree is not an exact search, but it agrees with the exact search on most queries.  So every reference
array is stored as the rows where it differs from the oracle's exact search (knn_mode=0) on the same queries (integer
rows as the difference to the exact row), plus a SHA-256 of the whole reference array.  A test recomputes the exact search, applies the stored rows and checks the digest,
which pins the reconstruction to the reference bit for bit.  ICP neighbour traces are stored per iteration together with
the pose the iteration searched from; in a differing trace row each id is stored as its rank among the exact 16 nearest
map points of that query (the octree misses close neighbours, it does not invent far ones), and as a raw id otherwise.

Regenerate (needs the oracle/_ref build, i.e. the reference tree at build time):
    python tests/ref_octree_golden.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PATH = os.path.join(HERE, "golden", "ref_octree.npz")
REGISTER_CASES = [("cfg1", 2000), ("cfg1", 0), ("cfg2", 0), ("cfg3", 0)]
# cases whose whole neighbour trace is stored; cfg3's (240 000 points, ~60 000 octree ids unlike the exact search's)
# would be some 200 KB, so for cfg3 only the registration result and the first iteration's mismatch rows are kept
TRACE_CASES = REGISTER_CASES[:3]
RESULT_FIELDS = ("iter_n_surf", "iter_lm_steps", "iter_lm_successful", "iter_lm_termination", "iter_cost")

_data = None


def digest(a) -> str:
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str(a.dtype).encode() + str(a.shape).encode() + a.tobytes()).hexdigest()


def load():
    global _data
    if _data is None:
        with np.load(PATH) as z:
            _data = {k: z[k] for k in z.files}
    return _data


def patched(key, exact):
    """The reference array `key`: `exact` with the stored differing rows applied, checked against the stored digest."""
    g = load()
    out = np.array(exact, copy=True)
    rows = g[key + ".rows"]
    out[rows] = out[rows] + g[key + ".vals"] if out.dtype.kind == "i" else g[key + ".vals"]
    assert digest(out) == str(g[key + ".sha256"]), f"{key}: exact search + stored rows != the reference's output"
    return out


def trace_from_corr(corr):
    """Neighbour ids as the oracle's nn_trace records them: -1 for points without a search result."""
    return np.where(corr["status"][:, None] < 0, -1, corr["nn"])


def knn(om, key, q, k=5):
    """Reference octree k-NN (ids, d2) on queries q, rebuilt from the exact search."""
    i0, d0, _ = om.knn(q, k, 0)
    return patched(key + ".idx", i0), patched(key + ".d2", d0)


def register_result(om, name, case, cap):
    """The octree-in-the-loop registration of a case: (result fields, correspondence status at the prior pose, points
    whose octree neighbour set at the prior pose differs from the exact search's, the exact search's correspondences there)."""
    g = load()
    key = f"{name}_cap{cap}"
    cfg = case["cfg"]
    oc0 = om.correspond(case["scan_xyzi"], case["pose_prior"], cfg["plane_res"], cap, 0, n_threads=8)[0]
    status = patched(key + ".status0", oc0["status"])
    res = {f: g[f"{key}.{f}"] for f in RESULT_FIELDS + ("hist_obs", "hist_reject_plane", "pose", "cov")}
    res["status"], res["n_iterations"] = int(g[key + ".status"]), int(g[key + ".n_iterations"])
    return res, status, g[key + ".nn0_mismatch"], oc0


def register_trace(om, name, case, cap):
    """The octree's neighbour ids of every ICP iteration [iterations, points, 5], rebuilt from the exact search at the pose
    each iteration searched from."""
    g = load()
    key = f"{name}_cap{cap}"
    cfg = case["cfg"]
    n = int(g[key + ".n_iterations"])
    poses = g[key + ".poses"]
    trace = np.stack([trace_from_corr(om.correspond(case["scan_xyzi"], poses[i], cfg["plane_res"], cap, 0, n_threads=8)[0])
                      for i in range(n)])
    flat = trace.reshape(-1, 5)
    rows = g[key + ".trace.rows"]
    flat[rows] = decode_ids(g[key + ".trace.codes"], g[key + ".trace.raw"], _candidates(om, case["scan_xyzi"], poses, rows))
    assert digest(flat) == str(g[key + ".trace.sha256"]), f"{key}: exact search + stored rows != the reference's trace"
    return trace


def _candidates(om, scan, poses, rows):
    """Exact 16 nearest map ids of the queries behind flat trace rows (row = iteration * n_points + point)."""
    from oracle import oracle as O
    it, pt = np.divmod(rows.astype(np.int64), len(scan))
    cand = np.full((len(rows), 16), -2, np.int64)
    for i in np.unique(it):
        m = it == i
        q = O.transform_scan_numpy(scan[pt[m]], poses[i])[:, :3]
        cand[m] = om.knn(q, 16, 0)[0]
    return cand


def encode_ids(ref, cand):
    """ids -> uint8 codes: rank in the candidate row, 254 for -1, 255 for an id stored raw (in order)."""
    codes = np.full(ref.shape, 255, np.uint8)
    raw = []
    for r in range(len(ref)):
        for j, v in enumerate(ref[r]):
            hit = np.flatnonzero(cand[r] == v)
            if v == -1:
                codes[r, j] = 254
            elif len(hit):
                codes[r, j] = hit[0]
            else:
                raw.append(v)
    return codes, np.array(raw, np.int32)


def decode_ids(codes, raw, cand):
    out = np.take_along_axis(cand, np.minimum(codes, 15).astype(np.int64), 1)
    out[codes == 254] = -1
    out[codes == 255] = raw
    return out


# ---------------------------------------------------------------------------------------------------------------------
def _put(out, key, ref, exact):
    ref, exact = np.asarray(ref), np.asarray(exact)
    assert ref.shape == exact.shape and ref.dtype == exact.dtype, key
    diff = (ref != exact).reshape(len(ref), -1).any(1)
    out[key + ".rows"] = np.flatnonzero(diff).astype(np.int32)
    # integer ids: the difference to the exact row (mostly zeros: the octree usually misses one neighbour of five)
    out[key + ".vals"] = (ref[diff] - exact[diff]).astype(np.int32) if ref.dtype.kind == "i" else ref[diff]
    out[key + ".sha256"] = np.array(digest(ref))


def generate():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    from conftest import get_case
    from oracle import oracle as O
    from test_oracle import _x_dominant_map
    O.build()
    assert O.has_ref_octree(), "needs the oracle/_ref build (the reference's octree compiled verbatim)"
    out = {}
    # tests/test_oracle.py::test_reference_octree_pins_the_knn_restatement
    xyzi = _x_dominant_map()
    m = O.OracleMap(xyzi)
    rng = np.random.default_rng(2)
    q = xyzi[::13, :3] + rng.normal(0, 0.1, size=xyzi[::13, :3].shape).astype(np.float32)
    i0, d0, _ = m.knn(q, 5, 0)
    i2, d2, _ = m.knn(q, 5, 2)
    _put(out, "xdom.idx", i2, i0)
    _put(out, "xdom.d2", d2, d0)
    c = get_case("cfg1")
    m = O.OracleMap(c["map_xyzi"])
    q = c["map_xyzi"][::37, :3] + rng.normal(0, 0.1, size=c["map_xyzi"][::37, :3].shape).astype(np.float32)
    i0, d0, _ = m.knn(q, 5, 0)
    i2, d2, _ = m.knn(q, 5, 2)
    _put(out, "cfg1_warehouse.idx", i2, i0)
    _put(out, "cfg1_warehouse.d2", d2, d0)
    # tests/test_gpu_parity.py: the hall case, where the octree is exact
    c = get_case("hall")
    cfg = c["cfg"]
    rng = np.random.default_rng(0)
    base = c["map_xyzi"][::7, :3]
    q = base + rng.normal(0, 0.12, size=base.shape).astype(np.float32)
    m = O.OracleMap(c["map_xyzi"])
    i0, d0, _ = m.knn(q, 5, 0)
    i2, d2, _ = m.knn(q, 5, 2)
    _put(out, "hall.idx", i2, i0)
    _put(out, "hall.d2", d2, d0)
    rr = m.register(c["scan_xyzi"], c["pose_prior"], cfg["plane_res"], cfg["max_iterations"], 0, knn_mode=2)
    out["hall.pose"], out["hall.n_iterations"] = np.array(rr.pose), np.array(rr.n_iterations)
    # tests/test_reference_octree_parity.py
    for name, cap in REGISTER_CASES:
        c = get_case(name)
        cfg, scan, prior, pr = c["cfg"], c["scan_xyzi"], c["pose_prior"], c["cfg"]["plane_res"]
        key = f"{name}_cap{cap}"
        om = O.OracleMap(c["map_xyzi"], ref_octree=True)
        trace = np.zeros((cfg["max_iterations"], len(scan), 5), np.int64)
        ro = om.register(scan, prior, pr, cfg["max_iterations"], cap, knn_mode=2, n_threads=8, nn_trace=trace)
        n = ro.n_iterations
        # pose iteration i searched from = the pose a registration stopped after i iterations returns
        poses = [np.asarray(prior, np.float64)] + [np.array(om.register(scan, prior, pr, i, cap, knn_mode=2, n_threads=8).pose_opt)
                                                   for i in range(1, n)]
        for i in range(n):
            t2 = trace_from_corr(om.correspond(scan, poses[i], pr, cap, 2, n_threads=8)[0])
            assert np.array_equal(t2, trace[i]), (key, i, "per-iteration pose does not reproduce the trace")
        if (name, cap) in TRACE_CASES:
            exact = np.stack([trace_from_corr(om.correspond(scan, poses[i], pr, cap, 0, n_threads=8)[0]) for i in range(n)])
            ref, exact = trace[:n].reshape(-1, 5), exact.reshape(-1, 5)
            rows = np.flatnonzero((ref != exact).any(1)).astype(np.int32)
            codes, raw = encode_ids(ref[rows], _candidates(om, scan, poses, rows))
            assert np.array_equal(decode_ids(codes, raw, _candidates(om, scan, poses, rows)), ref[rows])
            out[key + ".trace.rows"], out[key + ".trace.codes"], out[key + ".trace.raw"] = rows, codes, raw
            out[key + ".trace.sha256"] = np.array(digest(ref))
            out[key + ".poses"] = np.stack(poses)
        oc2 = om.correspond(scan, prior, pr, cap, 2, n_threads=8)[0]
        oc0 = om.correspond(scan, prior, pr, cap, 0, n_threads=8)[0]
        _put(out, key + ".status0", oc2["status"], oc0["status"])
        out[key + ".nn0_mismatch"] = np.flatnonzero((np.sort(oc2["nn"], 1) != np.sort(oc0["nn"], 1)).any(1)).astype(np.int32)
        out[key + ".n_iterations"], out[key + ".status"] = np.array(n), np.array(ro.status)
        for f in RESULT_FIELDS:
            out[f"{key}.{f}"] = np.array(getattr(ro, f)[:n])
        for f in ("hist_obs", "hist_reject_plane", "pose", "cov"):
            out[f"{key}.{f}"] = np.array(getattr(ro, f))
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    generate()

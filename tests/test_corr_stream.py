"""The solve's correspondence record (superodom_b200/csrc/so_corr_tiles.h, DESIGN.md section 4): the tile rule that places each scan's
points, and the results of the kernels that write and read the record, which must not move by a bit when its layout changes.

The GPU tests compare SHA-256 digests of each case's outputs with tests/golden/corr_stream_digests.json, which holds the digests the
library gave when the record still stored {n, d} (56 B per point).  `python tests/test_corr_stream.py --write-golden PATH` writes that
file from whatever library SO_LIB_PATH (or the in-tree build) names."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden", "corr_stream_digests.json")

TILE_TEST = r"""
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "so_corr_tiles.h"
// argv: capacity in points, then the scans' sizes; the scans are laid out back to back after a lead of `lead` points of an
// earlier scan (so the first one starts at an odd offset).  Checks that no two scans share a slot and that every slot is in bounds
// of a buffer sized for the whole batch, and that every scan starts on a tile boundary.
int main(int argc, char** argv) {
    const size_t lead = size_t(std::atoll(argv[1]));
    std::vector<uint32_t> n;
    for (int i = 2; i < argc; ++i) n.push_back(uint32_t(std::atoll(argv[i])));
    size_t total = lead;
    for (uint32_t v : n) total += v;
    const size_t cap = so::corr_tile_cap(total, n.size() + 1) * so::kCorrTile;
    std::vector<unsigned char> used(cap, 0);
    size_t off = 0;
    for (size_t s = 0; s <= n.size(); ++s) {
        const uint32_t m = s == 0 ? uint32_t(lead) : n[s - 1];
        const size_t first = so::corr_first(uint32_t(s), uint32_t(off));
        if (first % so::kCorrTile) { std::printf("scan %zu unaligned\n", s); return 1; }
        for (uint32_t i = 0; i < m; ++i) {
            if (first + i >= cap) { std::printf("scan %zu out of bounds\n", s); return 2; }
            if (used[first + i]++) { std::printf("scan %zu overlaps\n", s); return 3; }
        }
        off += m;
    }
    std::printf("ok %zu\n", cap);
    return 0;
}
"""


@pytest.mark.parametrize("sizes", [[1], [255], [256], [257], [131072], [1, 255, 256, 257, 131072], [257] * 64, [1] * 300,
                                   [131072] * 3 + [1]])
@pytest.mark.parametrize("lead", [0, 1, 255, 257, 12345])
def test_tile_rule_no_overlap_in_bounds(tmp_path, sizes, lead):
    src = tmp_path / "corr_tiles_test.cpp"
    src.write_text(TILE_TEST)
    exe = tmp_path / "corr_tiles_test"
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-O1", "-I", os.path.join(ROOT, "superodom_b200", "csrc"), str(src),
                           "-o", str(exe)])
    out = subprocess.check_output([str(exe), str(lead)] + [str(v) for v in sizes], text=True)
    assert out.startswith("ok"), out


# ---- GPU cases --------------------------------------------------------------------------------------------------------------------

def _digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _icp_bytes(r):
    """A result struct's bytes without its wall and device times (the only fields that vary between identical runs)."""
    icp = getattr(r, "icp", r)
    icp.time_ms = 0.0
    icp.time_total_ms = 0.0
    return np.frombuffer(bytes(r), np.uint8)


_cfg2 = {}


def _cfg2_cases(n):
    from superodom_b200 import synth
    if "scene" not in _cfg2:
        _cfg2["scene"], _cfg2["map"] = synth.make_map_for("cfg2")
    while len(_cfg2.setdefault("cases", [])) < n:
        _cfg2["cases"].append(synth.make_case_on(_cfg2["scene"], _cfg2["map"], "cfg2", len(_cfg2["cases"])))
    return _cfg2["map"], _cfg2["cases"][:n]


def _ctx(map_xyzi, max_batch=8):
    from superodom_b200 import api
    ctx = api.Context(max_map_points=len(map_xyzi) + 1024, max_scan_points=262144, max_batch=max_batch, plane_res=0.2)
    ctx.map_set_points(map_xyzi)
    return ctx


def _timed(scan, seed):
    """The scan with a per-point time column (x, y, z, intensity, t): t in [0, 0.1) s, a seeded permutation of the scan order."""
    t = np.random.default_rng(seed).permutation(len(scan)).astype(np.float32) * np.float32(0.1 / len(scan))
    return np.ascontiguousarray(np.concatenate([scan[:, :4], t[:, None]], 1))


def case_correspond():
    """so_correspond on a cfg2 scan, iteration 0 and iteration 1 (seeded): every reported plane, offset, weight and label."""
    m, cs = _cfg2_cases(1)
    ctx = _ctx(m)
    c = cs[0]
    out = []
    for seed in (None, c["pose_true"]):
        corr, ho, hr = ctx.correspond(c["scan_xyzi"], c["pose_prior"], 0, seed_pose=seed)
        out.append(_digest(corr["n"], corr["d"], corr["w"], corr["status"], corr["obs"], corr["nn"], corr["nn_d2"], ho, hr))
    H, g, cost = ctx.evaluate(c["pose_true"])
    out.append(_digest(H, g, np.array([cost])))
    ctx.close()
    return out


def case_register_modes():
    """One cfg2 scan registered in mode NONE, APPROXIMATED, OPTIMIZED and degeneracy-aware."""
    from superodom_b200 import api
    m, cs = _cfg2_cases(2)
    ctx = _ctx(m)
    out = []
    for c in cs:
        s5 = _timed(c["scan_xyzi"], 5)
        out.append(_digest(_icp_bytes(ctx.register(c["scan_xyzi"], c["pose_prior"], 20))))
        out.append(_digest(_icp_bytes(ctx.register_undistort(s5, c["pose_prior"], api.undistort(c["pose_prior"], 0.1), 20, time_col=4))))
        out.append(_digest(_icp_bytes(ctx.register_optimized(s5, c["pose_prior"], api.motion(0.1), 20, time_col=4))))
        out.append(_digest(_icp_bytes(ctx.register_degeneracy(c["scan_xyzi"], c["pose_prior"], api.degeneracy(0.1, 0.1), 20))))
    ctx.close()
    return out


def _batch(m, cs, sizes):
    """Scans cut to `sizes` points (odd sizes: every scan after the first starts at an odd offset and ends in a ragged tile)."""
    scans = [np.ascontiguousarray(c["scan_xyzi"][:k]) for c, k in zip(cs, sizes)]
    return np.concatenate(scans, 0), np.array(sizes, np.uint32), np.stack([c["pose_prior"] for c in cs]), scans


BATCH_SIZES = [130001, 4097, 131072, 65537, 257, 100003]


def case_register_batch():
    """A 6-scan batch with odd sizes, in modes NONE, APPROXIMATED, OPTIMIZED and degeneracy-aware."""
    from superodom_b200 import api
    m, cs = _cfg2_cases(len(BATCH_SIZES))
    flat, n, poses, _ = _batch(m, cs, BATCH_SIZES)
    ctx = _ctx(m)
    f5 = _timed(flat, 6)
    out = [_digest(*[_icp_bytes(r) for r in ctx.register_batch(flat, n, poses, 20)]),
           _digest(*[_icp_bytes(r) for r in ctx.register_batch_undistort(f5, n, poses, [api.undistort(p, 0.1) for p in poses], 20, time_col=4)]),
           _digest(*[_icp_bytes(r) for r in ctx.register_batch_optimized(f5, n, poses, [api.motion(0.1)] * len(n), 20, time_col=4)]),
           _digest(*[_icp_bytes(r) for r in ctx.register_batch_degeneracy(flat, n, poses, [api.degeneracy(0.1, 0.1)] * len(n), 20)])]
    ctx.close()
    return out


def _rows(seed, counts, specials):
    """so_solve rows of len(counts) problems: planes through a box seen from a perturbed pose; `specials` sets row weights to 0,
    NaN and -0.0 at fixed positions of every problem."""
    from superodom_b200 import api
    rng = np.random.default_rng(seed)
    rows = np.zeros(int(sum(counts)), api.SOLVE_ROW_DTYPE)
    probs = np.zeros(len(counts), api.SOLVE_PROBLEM_DTYPE)
    off = 0
    for b, k in enumerate(counts):
        nrm = rng.normal(size=(k, 3))
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        p = rng.uniform(-20, 20, size=(k, 3)).astype(np.float32)
        rows["p"][off:off + k] = p
        rows["n"][off:off + k] = nrm
        rows["d"][off:off + k] = -(nrm * p.astype(np.float64)).sum(1) + rng.normal(scale=0.02, size=k)
        rows["w"][off:off + k] = rng.uniform(0.2, 1.0, size=k)
        if specials:
            for j, v in zip((0, k // 2, k - 1), (0.0, np.nan, -0.0)):
                rows["w"][off + j] = v
        probs["n_rows"][b] = k
        probs["lm_max_iterations"][b] = 12
        q = rng.normal(scale=0.02, size=3)
        probs["pose"][b] = [rng.normal(scale=0.1), rng.normal(scale=0.1), rng.normal(scale=0.1), *q, np.sqrt(1 - (q * q).sum())]
        probs["x0"][b] = probs["pose"][b]
        off += k
    return rows, probs


SOLVE_COUNTS = [1, 255, 256, 257, 3001, 65537, 4097, 131072]


def case_solve():
    """so_solve and so_solve_optimized on given rows: odd row counts (odd offsets, ragged tiles), weights 0, NaN and -0.0."""
    from superodom_b200 import api
    m, _ = _cfg2_cases(1)
    ctx = _ctx(m, max_batch=len(SOLVE_COUNTS))
    out = []
    for specials in (False, True):
        rows, probs = _rows(11, SOLVE_COUNTS, specials)
        out.append(_digest(ctx.solve(rows, probs)))
        out.append(_digest(ctx.solve(rows, probs, [api.degeneracy(0.1, 0.1)] * len(probs))))
        op = np.zeros(len(probs), api.SOLVE_OPTIMIZED_PROBLEM_DTYPE)
        op["n_rows"] = probs["n_rows"]
        op["lm_max_iterations"] = probs["lm_max_iterations"]
        op["pose"] = probs["pose"]
        op["motion"] = [0, 0, 0, 0, 0, 0, 1]
        op["motion_prior"] = [0, 0, 0, 0, 0, 0, 1]
        op["dt"] = 0.1
        times = np.random.default_rng(12).uniform(0, 0.1, size=len(rows)).astype(np.float32)
        out.append(_digest(ctx.solve_optimized(rows, times, op)))
    ctx.close()
    return out


CASES = {"correspond": case_correspond, "register_modes": case_register_modes, "register_batch": case_register_batch, "solve": case_solve}


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_bits_as_before(name):
    assert CASES[name]() == _golden()[name]


@pytest.mark.gpu
def test_scan_alone_and_in_batch():
    """A scan's registration does not depend on the batch it travels in or where in it (its record tiles start elsewhere)."""
    m, cs = _cfg2_cases(len(BATCH_SIZES))
    flat, n, poses, scans = _batch(m, cs, BATCH_SIZES)
    ctx = _ctx(m)

    def key(r):
        return np.array(list(r.pose_opt) + list(r.iter_cost)[:r.n_iterations] + list(r.cov) + [r.n_iterations, r.status])

    batch = [key(r) for r in ctx.register_batch(flat, n, poses, 20)]
    for k in (0, 1, 4, 5):
        alone = key(ctx.register_batch(scans[k], n[k:k + 1], poses[k:k + 1], 20)[0])
        assert np.array_equal(alone, batch[k]), k
    ctx.close()


if __name__ == "__main__" and "--write-golden" in sys.argv:
    path = sys.argv[sys.argv.index("--write-golden") + 1]
    res = {name: fn() for name, fn in CASES.items()}
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))

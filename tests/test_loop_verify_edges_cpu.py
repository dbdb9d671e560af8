"""CPU self-checks of the loop-verification restatement (loop_verify_numpy.py) that test_loop_verify_edges.py compares the device
with: the two-stage sum against a literal transcription of k_verify_overlap's tree and k_verify_sum for every grid size from 1 to 3000
and against math.fsum; "a conflict of any image" against the kernel's in-order loop that stops at the first removal; and the submap ids
against so_verify_rule.h's verify_range / verify_eligible, compiled."""
import math
import os
import subprocess

import numpy as np

import loop_verify_numpy as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _literal_cta(vals):
    """k_verify_overlap's reduction, thread by thread: s_sum[t] = d2 (0 past n), then for h = 32 .. 1 threads t < h add s_sum[t + h]."""
    n = len(vals)
    out = []
    for b in range((n + 63) // 64):
        s = [float(vals[b * 64 + t]) if b * 64 + t < n else 0.0 for t in range(64)]
        h = 32
        while h > 0:
            for t in range(h):
                s[t] += s[t + h]
            h >>= 1
        out.append(s[0])
    return out


def _literal_sum(partials):
    """k_verify_sum, thread by thread."""
    n = len(partials)
    per = (n + 256 - 1) // 256
    s_run = []
    for t in range(256):
        a = t * per
        e = min(n, a + per)
        v = 0.0
        k = a
        while k < e:
            v += float(partials[k])
            k += 1
        s_run.append(v)
    t = 0.0
    for k in range(256):
        t += s_run[k]
    return t


def _values(rng, n):
    """Positive values over 30 binary orders of magnitude, so that a different order of addition gives a different sum."""
    return rng.uniform(0.5, 1.0, n) * np.exp2(rng.integers(-20, 10, n).astype(np.float64))


def test_sum_restatement_equals_the_kernels_for_every_grid():
    rng = np.random.default_rng(5)
    orders_matter = 0
    for grid in range(1, 3001):
        p = _values(rng, grid)
        got = V.verify_sum(p)
        assert got == _literal_sum(p), grid
        exact = math.fsum(p)
        assert abs(got - exact) <= (grid - 1) * 2.0 ** -53 * float(p.sum()) * 1.0000001, grid
        per_floor = grid // 256                                      # the sum of a kernel that rounds the run length down
        floor_sum = sum(sum(p[t * per_floor:min(grid, t * per_floor + per_floor)]) for t in range(256))
        if grid % 256:
            assert floor_sum != got, grid
        orders_matter += float(np.cumsum(p)[-1]) != got
    assert orders_matter > 1000                                    # the fixed order is observable: plain in-order sums differ


def test_cta_tree_restatement_equals_the_kernel():
    rng = np.random.default_rng(6)
    for n in list(range(1, 200)) + [64 * 256, 64 * 256 + 1, 64 * 2100 + 17]:
        v = _values(rng, n)
        v[rng.random(n) < 0.3] = 0.0                               # non-inliers add 0
        got = V.cta_partials(v)
        want = _literal_cta(v) if n < 20000 else None
        if want is not None:
            assert got.tolist() == want, n
        assert len(got) == (n + 63) // 64
        # a tree over 32 lanes only, or plain in-order sums, give other bits for some CTA
        if n >= 64:
            s = np.zeros(((n + 63) // 64, 64))
            s.reshape(-1)[:n] = v
            assert not np.array_equal(got, s[:, :32].sum(1)), n
    full = V.cta_partials(np.ones(64 * 3 + 5))
    assert full.tolist() == [64.0, 64.0, 64.0, 5.0]


def test_any_image_equals_the_in_order_loop():
    """k_verify_conflict: images in order, *cand set by every image that observes the point, stopping at the first removal."""
    rng = np.random.default_rng(7)
    for trial in range(300):
        n_img, n = int(rng.integers(1, 18)), 200
        cand = rng.random((n_img, n)) < rng.uniform(0, 1)
        rem = cand & (rng.random((n_img, n)) < rng.uniform(0, 0.5))
        lc = np.zeros(n, bool)
        lr = np.zeros(n, bool)
        for i in range(n):
            c = r = False
            for j in range(n_img):
                if r:
                    break
                r = bool(rem[j, i])
                c = c or bool(cand[j, i])
            lc[i], lr[i] = c, r
        assert np.array_equal(lc, cand.any(0)) and np.array_equal(lr, rem.any(0)), trial


def test_submap_ids_equal_the_rule_header(tmp_path):
    src = tmp_path / "ids.cpp"
    src.write_text(
        '#include <cstdio>\n#include "so_verify_rule.h"\n'
        "int main() {\n"
        "  for (int q = 0; q < 14; ++q) for (int c = 0; c < 14; ++c) for (int w = 0; w <= 8; ++w)\n"
        "  for (int b = -1; b < 14; ++b) for (int e = b; e <= 14; ++e) for (int x = 0; x < 4; ++x) {\n"
        "    if ((b < 0) != (e < 0) || (b < 0 && e != -1)) continue;\n"
        "    const so::VerifyRange r = so::verify_range(q, b < 0 ? 0 : b, e, x * 3);\n"
        "    std::printf(\"%d %d %d %d %d %d:\", q, c, w, b, e, x * 3);\n"
        "    for (long k = long(c) - w; k <= long(c) + w; ++k) if (k >= 0 && so::verify_eligible(r, q, int(k))) std::printf(\" %ld\", k);\n"
        "    std::printf(\"\\n\");\n"
        "  }\n"
        "  return 0;\n"
        "}\n")
    exe = tmp_path / "ids"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "superodom_b200", "csrc"), str(src),
                           "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(out) > 50000
    nonempty = 0
    for line in out:
        head, ids = line.split(":")
        q, c, w, b, e, x = (int(v) for v in head.split())
        want = [int(v) for v in ids.split()]
        got = V.submap_ids(q, c, w, max(b, 0), e, x)
        assert got == want, line
        assert all(V.verify_eligible(V.verify_range(q, max(b, 0), e, x), q, k) for k in got)
        nonempty += bool(got)
    assert nonempty > 10000

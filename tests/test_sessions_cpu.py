"""Sessions without a device: the session file of include/superodom_b200/KeyframeIO.hpp (bit-exact round trips, hostile files rejected
under AddressSanitizer), the host-only rules of so_pose_graph_check_constant, the layouts and exports of the new entry points, and the
constant-set restatement of sessions_numpy.py against central differences and against PoseGraph(fixed=k)."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import pose_graph_numpy as PG
import sessions_numpy as SN
import test_ceres_restatement as CR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_ENTRIES = ["so_keyframe_import", "so_loop_candidates_range", "so_pose_graph_check_constant", "so_pose_graph_solve_constant"]


# ------------------------------------------------------------------------------------------------------------- the session file
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("kfio") / "keyframe_io_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-Wall", "-Werror", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "keyframe_io_test.cpp"), "-o", out])
    return out


def _file(frames, edges=b"", n_edges=None, magic=b"SOKF", version=1, n_frames=None):
    """A session file from the layout KeyframeIO.hpp documents: frames = [(pose7, surf [n, 4], edge [m, 4])], edges = packed records."""
    head = magic + struct.pack("<IQQ", version, len(frames) if n_frames is None else n_frames,
                               len(edges) // 360 if n_edges is None else n_edges)
    table = b"".join(struct.pack("<7dQQ", *p, len(s), len(e)) for p, s, e in frames)
    clouds = b"".join(np.ascontiguousarray(s, "<f4").tobytes() + np.ascontiguousarray(e, "<f4").tobytes() for _, s, e in frames)
    return head + table + clouds + edges


def _edges(m, seed=0):
    rng = np.random.default_rng(seed)
    return b"".join(struct.pack("<ii7d36dd", int(rng.integers(0, 50)), int(rng.integers(0, 50)), *rng.normal(size=7), *rng.normal(size=36),
                                float(rng.uniform(0, 2))) for _ in range(m))


def _frames(n, seed=0, max_points=40):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        s = rng.normal(0, 10, (int(rng.integers(0, max_points)), 4)).astype(np.float32)
        e = rng.normal(0, 10, (int(rng.integers(0, max_points)) if k % 3 else 0, 4)).astype(np.float32)      # empty edge clouds
        if len(s):
            s[0, 0] = np.nan                                              # clouds are kept verbatim, non-finite points included
        out.append((np.r_[rng.normal(0, 100, 3), rng.normal(size=4)], s, e))
    return out


def _copy(exe, tmp_path, data):
    src, dst = tmp_path / "in.sokf", tmp_path / "out.sokf"
    src.write_bytes(data)
    r = subprocess.run([exe, "copy", str(src), str(dst)], capture_output=True, text=True)
    return r, (dst.read_bytes() if r.returncode == 0 else None)


@pytest.mark.parametrize("n, m", [(0, 0), (1, 0), (5, 3), (1000, 0), (1000, 999)])
def test_session_file_round_trip(exe, tmp_path, n, m):
    frames = _frames(n, seed=n + m)
    data = _file(frames, _edges(m, seed=m))
    r, back = _copy(exe, tmp_path, data)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["ok", str(n), str(m), str(sum(len(s) + len(e) for _, s, e in frames))]
    assert back == data


def _hostile(frames, edges):
    good = _file(frames, edges)
    big = 1 << 63
    nan_pose = [(np.r_[np.nan, frames[0][0][1:]], frames[0][1], frames[0][2])] + frames[1:]
    inf_pose = [(np.r_[frames[0][0][:6], np.inf], frames[0][1], frames[0][2])] + frames[1:]
    zero_q = [(np.r_[frames[0][0][:3], 0.0, 0.0, 0.0, 0.0], frames[0][1], frames[0][2])] + frames[1:]
    table_at = 24
    wrap = bytearray(good)                                                # two point counts whose sum wraps 2^64
    struct.pack_into("<QQ", wrap, table_at + 56, (1 << 64) - 1, 2)
    huge_points = bytearray(good)
    struct.pack_into("<Q", huge_points, table_at + 56, 1 << 60)
    return {
        "empty": b"", "short_header": good[:23], "magic": b"SOKX" + good[4:], "version": good[:4] + struct.pack("<I", 2) + good[8:],
        "frames_over_file": _file(frames, edges, n_frames=len(frames) + 1), "frames_huge": _file(frames, edges, n_frames=big),
        "frames_wrap": _file(frames, edges, n_frames=(1 << 64) // 72 + 1), "edges_huge": _file(frames, edges, n_edges=big),
        "edges_over_file": _file(frames, edges, n_edges=len(edges) // 360 + 1), "points_wrap": bytes(wrap),
        "points_huge": bytes(huge_points), "truncated_table": good[:24 + 71], "truncated_cloud": good[:-len(edges) - 1],
        "truncated_edge": good[:-1], "padded": good + b"\0", "nan_pose": _file(nan_pose, edges), "inf_pose": _file(inf_pose, edges),
        "zero_quaternion": _file(zero_q, edges),
    }


@pytest.mark.parametrize("case", ["empty", "short_header", "magic", "version", "frames_over_file", "frames_huge", "frames_wrap",
                                  "edges_huge", "edges_over_file", "points_wrap", "points_huge", "truncated_table", "truncated_cloud",
                                  "truncated_edge", "padded", "nan_pose", "inf_pose", "zero_quaternion"])
def test_session_file_rejects_hostile_input(exe, tmp_path, case):
    """Each file is rejected with a message and without a sanitizer report (the helper is built with AddressSanitizer and UBSan)."""
    frames = _frames(4, seed=9, max_points=10)
    frames[0] = (frames[0][0], np.ones((3, 4), np.float32), np.ones((2, 4), np.float32))
    r, _ = _copy(exe, tmp_path, _hostile(frames, _edges(2))[case])
    assert r.returncode == 1, (case, r.returncode, r.stderr)
    assert "readKeyframeSession" in r.stderr and "Sanitizer" not in r.stderr and "runtime error" not in r.stderr, r.stderr


def test_missing_session_file(exe, tmp_path):
    r = subprocess.run([exe, "copy", str(tmp_path / "none.sokf"), str(tmp_path / "out.sokf")], capture_output=True, text=True)
    assert r.returncode == 1 and "cannot open" in r.stderr


# ------------------------------------------------------------------------------------------------------------- entry points
def test_new_entries_declared_and_exported():
    from superodom_b200 import api, build
    from test_abi import _declared
    L = C.CDLL(build.build())
    decl = _declared()
    for name in NEW_ENTRIES:
        assert name in decl and name in api.EXPORTS and hasattr(L, name), name


def test_session_shim_compiles_and_links(tmp_path):
    from superodom_b200 import build
    lib = build.build()
    out = str(tmp_path / "session_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "session_test.cpp"), "-o", out, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)


def test_loop_candidate_layout_is_unchanged(tmp_path):
    """The range search returns the existing so_loop_candidate records: the dtype still matches the header."""
    from superodom_b200 import api
    f = tmp_path / "s.c"
    f.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "superodom_b200.h"\nint main(void){printf("%zu %zu %zu\\n", '
                 'sizeof(so_loop_candidate), offsetof(so_loop_candidate, yaw), sizeof(so_pose_edge));return 0;}\n')
    x = tmp_path / "s"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(f), "-o", str(x)])
    size, yaw, edge = (int(v) for v in subprocess.check_output([str(x)]).split())
    assert size == api.LOOP_CANDIDATE_DTYPE.itemsize and yaw == api.LOOP_CANDIDATE_DTYPE.fields["yaw"][1]
    assert edge == api.POSE_EDGE_DTYPE.itemsize == 360                      # the session file's edge record


def _code(fn):
    from superodom_b200 import api
    with pytest.raises(api.SuperOdomError) as e:
        fn()
    return e.value.code, str(e.value)


def _good(n=4):
    return PG.to_array([PG.edge(k, k + 1, [0.1, 0, 0, 0, 0, 0, 1.0], np.ones(6)) for k in range(n - 1)])


@pytest.mark.parametrize("case, needle", [
    ("none", "no constant node"), ("all", "no free node"), ("disc", "not connected to any constant node"),
    ("disc_other", "not connected to any constant node"), ("n1", "two nodes"), ("iters", "max_iterations"), ("self", "i == j"),
])
def test_constant_check_rejects(case, needle):
    from superodom_b200 import api
    api.load_library()
    n, e, mask, iters = 4, _good(), np.array([1, 0, 0, 0], np.uint8), 50
    if case == "none":
        mask[:] = 0
    elif case == "all":
        mask[:] = 1
    elif case == "disc":                                                  # {0, 1} held, {2, 3} free and apart
        e = e[[0, 2]]
    elif case == "disc_other":                                            # {0, 1} free and apart, {2, 3} held
        e, mask = e[[0, 2]], np.array([0, 0, 1, 0], np.uint8)
    elif case == "n1":
        n, e, mask = 1, e[:0], np.array([1], np.uint8)
    elif case == "iters":
        iters = -1
    elif case == "self":
        e[1]["j"] = e[1]["i"]
    code, msg = _code(lambda: api.pose_graph_check_constant(n, e, mask, iters))
    assert code == -1 and needle in msg, msg


def test_constant_check_accepts():
    """A constant node in every component, any number of them, every node constant when nothing is solved, a mask value other than 1."""
    from superodom_b200 import api
    e = _good(6)[[0, 1, 3, 4]]                                             # {0, 1, 2} and {3, 4, 5}
    api.pose_graph_check_constant(6, e, np.array([0, 7, 0, 0, 0, 1], np.uint8))
    api.pose_graph_check_constant(6, _good(6), np.ones(6, np.uint8), max_iterations=0)
    api.pose_graph_check_constant(6, _good(6), np.array([1, 1, 1, 0, 1, 1], np.uint8))


def test_constant_solve_rejects_before_device_work():
    """The solve's argument errors come before the context is touched: a NULL context still reports the mask's rule first only
    after its own NULL check, and a wrong mask length is refused by the binding."""
    from superodom_b200 import api
    L = api.load_library()
    x = np.tile(np.r_[0, 0, 0, 0, 0, 0, 1.0], (4, 1))
    e = _good()
    m = np.zeros(4, np.uint8)
    assert L.so_pose_graph_solve_constant(None, api._p(x), 4, api._p(e), 3, api._p(m), None, api._p(x), None, None) == -1
    assert "NULL ctx" in L.so_last_error().decode()
    with pytest.raises(ValueError):
        api.pose_graph_check_constant(4, e, np.zeros(3, np.uint8))


# ------------------------------------------------------------------------------------------------------------- the restatement
def test_constant_set_restatement_gradient():
    """The objective and gradient over the free nodes only, against central differences in the tangent of Plus."""
    rng = np.random.default_rng(5)
    init, edges, _ = PG.drifted(rng, 9, loops=3, cauchy=1.0, drift=(0.1, 0.03))
    mask = np.array([1, 0, 0, 1, 0, 0, 0, 1, 0], np.uint8)
    prob = SN.ConstantPoseGraph(init, PG.to_array(edges), mask)
    x = prob.x0()
    assert len(x) == 7 * 6
    cost, res, J = prob.linearise(x)
    g = J.T @ res
    h = 1e-6
    num = np.zeros_like(g)
    for k in range(len(g)):
        d = np.zeros_like(g)
        d[k] = h
        num[k] = (prob.cost(CR._plus_blocks(x, d)) - prob.cost(CR._plus_blocks(x, -d))) / (2 * h)
    assert abs(cost - prob.cost(x)) <= 1e-12 * cost
    assert np.abs(num - g).max() <= 1e-5 * max(1.0, np.abs(g).max()), np.abs(num - g).max()
    # constant nodes stay where they are given
    X = prob.nodes(x + 0.01)
    assert np.array_equal(X[mask == 1], prob.init[mask == 1])


@pytest.mark.parametrize("fixed", [0, 4, 8])
def test_one_node_set_is_the_fixed_problem(fixed):
    rng = np.random.default_rng(6 + fixed)
    init, edges, _ = PG.drifted(rng, 9, loops=2, drift=(0.05, 0.01))
    E = PG.to_array(edges)
    mask = np.zeros(9, np.uint8)
    mask[fixed] = 1
    a, b = PG.PoseGraph(init, E, fixed), SN.ConstantPoseGraph(init, E, mask)
    assert np.array_equal(a.free, b.free) and np.array_equal(a.col, b.col) and np.array_equal(a.x0(), b.x0())
    ra, rb = CR.solve_full(a, a.x0(), 20), CR.solve_full(b, b.x0(), 20)
    assert np.array_equal(ra["x"], rb["x"]) and ra["termination"] == rb["termination"]

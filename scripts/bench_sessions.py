"""Multi-session costs on prefiltered OS1-128 cfg2 keyframes: importing an earlier session's keyframes (so_keyframe_import), reading
and writing its session file (KeyframeIO.hpp, through tests/cpp/keyframe_io_test.cpp), the loop search of the live session's keyframes
over the earlier session's ids (so_loop_candidates_range) beside the prefix search over as many candidates (so_loop_candidates), the
joined pose graph with the earlier half constant (so_pose_graph_solve_constant) beside the same graph with one fixed node, and the
merged rebuild of both sessions' keyframes (so_map_from_keyframes, both stores).  Wall time is around calls that end in a device
synchronise (median of --reps); device time is what CUDA events report (loop search, pose graph) or the kernels and copies
torch.profiler records in a run of its own.  Prints one JSON line with the card and its power limit, read in the same run.

    python scripts/bench_sessions.py [--frames 1000] [--reps 5]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pose_graph_numpy as PG  # noqa: E402
from superodom_b200 import api, synth  # noqa: E402


def device_ms(fn):
    """Summed device time (ms) of the kernels and copies one call of fn records under torch.profiler."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(float(getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0) or 0.0)
               for e in prof.events() if getattr(e, "device_type", None) == DeviceType.CUDA) / 1e3


def wall_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000, help="keyframes per session")
    ap.add_argument("--scans", type=int, default=8, help="distinct OS1-128 scans the keyframes are drawn from")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    n = a.frames
    out = {"card": card(), "frames_per_session": n}
    scene, map_xyzi = synth.make_map_for("cfg2")
    src = api.Context(max_map_points=1 << 22, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    src.map_set_points(map_xyzi)
    src.keyframe_reserve(a.scans << 18, a.scans)
    truth = []
    for i in range(a.scans):
        c = synth.make_case_on(scene, map_xyzi, "cfg2", i)
        src.scan_prefilter(c["scan_xyzi"], 0.1, 0.2, auto_voxel_size=False, download=False)
        r = src.register_prefiltered(c["pose_true"], 20, 0)
        src.keyframe_add_registered(np.array(r.pose))
        truth.append(np.array(r.pose))
    clouds = [src.keyframe_download(i, 0) for i in range(a.scans)]
    src.close()
    rng = np.random.default_rng(0)
    poses = np.array([np.r_[truth[i % a.scans][:3] + rng.normal(0, 0.05, 3), truth[i % a.scans][3:]] for i in range(2 * n)])
    out["points_per_keyframe"] = float(np.mean([len(c) for c in clouds]))
    ctx = api.Context(max_map_points=1 << 22, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    cap = 2 * n * max(len(c) for c in clouds) + 1

    def import_session():
        ctx.keyframe_reserve(0, 0)
        ctx.keyframe_reserve(cap, 2 * n)
        for i in range(n):
            ctx.keyframe_import(clouds[i % a.scans], poses[i])
    out["import_wall_ms"] = wall_ms(import_session, a.reps)
    out["import_device_ms"] = device_ms(import_session)
    # the session file of n keyframes, read and written back by the compiled reader / writer
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "keyframe_io_test")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                               os.path.join(ROOT, "tests", "cpp", "keyframe_io_test.cpp"), "-o", exe])
        path = os.path.join(d, "a.sokf")
        with open(path, "wb") as f:
            f.write(b"SOKF" + struct.pack("<IQQ", 1, n, 0))
            for i in range(n):
                f.write(struct.pack("<7dQQ", *poses[i], len(clouds[i % a.scans]), 0))
            for i in range(n):
                f.write(np.ascontiguousarray(clouds[i % a.scans], "<f4").tobytes())
        out["file_bytes"] = os.path.getsize(path)
        out["file_read_write_wall_ms"] = wall_ms(lambda: subprocess.check_call([exe, "copy", path, os.path.join(d, "b.sokf")],
                                                                                stdout=subprocess.DEVNULL), a.reps)
    # the live session's keyframes after the earlier one's
    for i in range(n, 2 * n):
        ctx.keyframe_import(clouds[i % a.scans], poses[i])
    opts = dict(max_range=80.0, exclude_recent=0)
    ctx.loop_candidates(np.arange(2 * n), 5, **opts)                                  # every descriptor computed once
    _, st = ctx.loop_candidates([2 * n - 1], 5, stats=True, ids=(0, n), **opts)
    out["range_one_query_ms"] = st["time_search_ms"]
    _, st = ctx.loop_candidates([n], 5, stats=True, **opts)                         # the prefix of query n: the same n candidates
    out["prefix_one_query_ms"] = st["time_search_ms"]
    qs = np.arange(n, 2 * n, dtype=np.int32)
    out["range_all_queries_ms"] = float(np.median([ctx.loop_candidates(qs, 5, stats=True, ids=(0, n), **opts)[1]["time_search_ms"]
                                                   for _ in range(a.reps)]))
    same = np.full(n, n, np.int32)
    out["prefix_all_queries_ms"] = float(np.median([ctx.loop_candidates(same, 5, stats=True, **opts)[1]["time_search_ms"]
                                                    for _ in range(a.reps)]))
    # the joined graph: 2n nodes, n of them constant, against one fixed node
    init, edges, _ = PG.drifted(np.random.default_rng(1), 2 * n, loops=2 * n // 10, false_loops=2 * n // 100, cauchy=1.0,
                                drift=(0.05, 0.01))
    E = PG.to_array(edges)
    mask = (np.arange(2 * n) < n).astype(np.uint8)
    for name, kw in (("constant", dict(constant=mask)), ("fixed", dict(fixed=0))):
        ctx.pose_graph_solve(init, E, **kw)
        rs = []
        w = wall_ms(lambda: rs.append(ctx.pose_graph_solve(init, E, **kw)[1]), a.reps)
        out[f"graph_{name}_wall_ms"] = w
        out[f"graph_{name}_device_ms"] = float(np.median([r["time_ms"] for r in rs]))
        out[f"graph_{name}_iterations"] = rs[-1]["iterations"]
        out[f"graph_{name}_pcg_iterations"] = int(rs[-1]["pcg_iterations"])
    # the merged rebuild of both sessions, both stores
    ids = np.arange(2 * n, dtype=np.int32)
    ctx.map_set_origin(poses[-1][:3])

    def rebuild():
        ctx.map_from_keyframes(ctx, ids, poses, 3)
    rebuild()
    out["merged_rebuild_wall_ms"] = wall_ms(rebuild, a.reps)
    out["merged_rebuild_device_ms"] = device_ms(rebuild)
    out["merged_map_points"] = ctx.map_size()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Free-space clearing of a map rebuilt from keyframes (so_map_clear_free_space_keyframes): the rebuild (so_map_from_keyframes, surf store,
archive on) and the batched clearing against every keyframe, for N prefiltered OS1-128 keyframes made as scripts/bench_keyframes.py
makes them, and for the smallest N the same clearing done the old way, one so_map_clear_free_space per keyframe (download the keyframe,
upload it, image it, carve, compact).  Wall time is around calls that end in a device synchronise; the batched call's device time is its
own CUDA-event time, the sequential loop's the kernels and copies torch.profiler records in a run of its own.  Prints one JSON line with
the card and its power limit.

    python scripts/bench_keyframe_clear.py [--frames 100,1000] [--reps 5]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from superodom_b200 import api, synth  # noqa: E402
from bench_keyframes import card, device_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="100,1000")
    ap.add_argument("--scans", type=int, default=8, help="distinct OS1-128 scans the keyframes are drawn from")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    frames = [int(v) for v in a.frames.split(",")]
    n_max = max(frames)
    scene, map_xyzi = synth.make_map_for("cfg2")
    ctx = api.Context(max_map_points=1 << 22, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    ctx.map_set_points(map_xyzi)
    cases = [synth.make_case_on(scene, map_xyzi, "cfg2", i) for i in range(a.scans)]
    per = [ctx.scan_prefilter(c["scan_xyzi"], 0.1, 0.2, auto_voxel_size=False, download=False)[0] for c in cases]
    ctx.keyframe_reserve(n_max * max(per) + 1, n_max)
    while ctx.keyframe_info()[0] < n_max:                      # the scans in turn, each registered and kept
        c = cases[ctx.keyframe_info()[0] % a.scans]
        ctx.scan_prefilter(c["scan_xyzi"], 0.1, 0.2, auto_voxel_size=False, download=False)
        r = ctx.register_prefiltered(c["pose_true"], 20, 0)
        ctx.keyframe_add_registered(np.array(r.pose))
    n_kf, n_pts, _ = ctx.keyframe_info()
    # a trajectory of 0.5 m steps with a slow turn (bench_keyframes.py), so the map spreads over many blocks
    rng = np.random.default_rng(1)
    th = np.cumsum(rng.normal(0.0, 0.02, n_kf))
    xy = np.cumsum(0.5 * np.stack([np.cos(th), np.sin(th)], 1), 0)
    poses = np.array([np.r_[xy[i], 0.0, synth.quat_from_rotvec(np.array([0, 0, th[i]]))] for i in range(n_kf)])
    o = api.free_space()                                      # the OS1-128 defaults
    dst = api.Context(max_map_points=1 << 25, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    dst.map_archive(1 << 25)
    rows = []
    for n in frames:
        ids = np.arange(n, dtype=np.int32)
        rebuild_ms, clear_ms, clear_dev = [], [], []
        res = None
        for rep in range(a.reps + 1):                          # the first round warms up
            t0 = time.perf_counter()
            dst.map_from_keyframes(ctx, ids, poses[:n], 1)
            t1 = time.perf_counter()
            res = dst.map_clear_free_space_keyframes(ctx, ids, poses[:n], o, 1)
            t2 = time.perf_counter()
            if rep:
                rebuild_ms.append((t1 - t0) * 1e3)
                clear_ms.append((t2 - t1) * 1e3)
                clear_dev.append(res["time_ms"])
        row = dict(frames=n, keyframe_points=int(sum(ctx.keyframe_download(i).shape[0] for i in range(n))),
                   map_points_before=int(res["n_after"][0] + res["n_removed"]), removed=int(res["n_removed"]),
                   candidates=int(res["n_candidates"]), tiles=int(res["n_tiles"]),
                   rebuild_wall_ms=float(np.median(rebuild_ms)), clear_wall_ms=float(np.median(clear_ms)),
                   clear_device_ms=float(np.median(clear_dev)))
        if n == min(frames):                                   # the old way: one call per keyframe, through the host
            batched = dst.map_download()

            def sequential():
                for i in range(n):
                    dst.map_clear_free_space(ctx.keyframe_download(i), poses[i], o, 1)

            seq_ms = []
            for rep in range(a.reps + 1):
                dst.map_from_keyframes(ctx, ids, poses[:n], 1)
                t0 = time.perf_counter()
                sequential()
                if rep:
                    seq_ms.append((time.perf_counter() - t0) * 1e3)
            assert np.array_equal(batched.view(np.uint32), dst.map_download().view(np.uint32)), "the two forms differ"
            dst.map_from_keyframes(ctx, ids, poses[:n], 1)
            row.update(sequential_wall_ms=float(np.median(seq_ms)), sequential_device_ms=device_ms(sequential))
        rows.append(row)
    print(json.dumps(dict(card=card(), keyframe_points=int(n_pts / max(n_kf, 1)), clear=rows)))
    for c in (ctx, dst):
        c.close()


if __name__ == "__main__":
    main()

"""Loop-detection costs (so_loop_candidates, so_keyframe_descriptors) on prefiltered OS1-128 keyframes at the default options: describing
one keyframe, one query against 1 000 and 10 000 keyframes, all pairs of 1 000, and a live step (prefilter, register, insert) with
addKeyframe plus one query against one without.  Device time is the call's CUDA-event stage times (so_loop_stats); wall time is around
calls that end in a device synchronise.  Prints one JSON line with the card and its power limit.

    python scripts/bench_loop_detect.py [--frames 1000,10000] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from superodom_b200 import api, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def timed(fn, reps):
    """-> (median wall ms, median of the stats key) over reps calls of fn, which returns so_loop_stats as a dict."""
    wall, dev = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        st = fn()
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(st)
    return float(np.median(wall)), {k: float(np.median([d[k] for d in dev])) for k in dev[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="1000,10000")
    ap.add_argument("--scans", type=int, default=8, help="distinct OS1-128 scans the keyframes are drawn from")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    frames = [int(v) for v in a.frames.split(",")]
    n_max = max(frames)
    scene, map_xyzi = synth.make_map_for("cfg2")
    scans, truth = [], []
    for i in range(a.scans):
        c = synth.make_case_on(scene, map_xyzi, "cfg2", i)
        scans.append(c["scan_xyzi"])
        truth.append(c["pose_true"])
    ctx = api.Context(max_map_points=1 << 22, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    ctx.map_set_points(map_xyzi)
    per = [ctx.scan_prefilter(s, 0.1, 0.2, auto_voxel_size=False, download=False)[0] for s in scans]
    ctx.keyframe_reserve((n_max + 64) * max(per), n_max + 64)
    opts = api.loop_opts()
    k = 0

    def step(keep):
        nonlocal k
        i = k % a.scans
        ctx.scan_prefilter(scans[i], 0.1, 0.2, auto_voxel_size=False, download=False)
        r = ctx.register_prefiltered(truth[i], 20, 0)
        if keep:
            q = ctx.keyframe_add_registered(np.array(r.pose))
            ctx.loop_candidates([q], 10, opts)
        ctx.map_add_registered_scan(np.array(r.pose))
        k += 1
        return r

    # keyframes: every scan once, then copies up to n_max (a copy costs the search what a distinct keyframe costs)
    for i in range(a.scans):
        step(True)
    for _ in range(3):
        step(False)
    t_plain, t_keep = [], []
    for _ in range(3 * a.reps):
        t0 = time.perf_counter(); step(False); t_plain.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter(); step(True); t_keep.append((time.perf_counter() - t0) * 1e3)
    live = dict(without_keyframe_ms=float(np.median(t_plain)), with_keyframe_and_query_ms=float(np.median(t_keep)),
                keyframes=int(ctx.keyframe_info()[0]))
    poses = ctx.keyframe_poses()
    while ctx.keyframe_info()[0] <= n_max:                            # ids 0 .. n_max: query n against ids 0 .. n - 1
        ctx.keyframe_add_registered(poses[-1])
    n_kf, n_pts, _ = ctx.keyframe_info()
    ctx.loop_candidates([n_kf - 1], 10, opts)                         # describes every keyframe once
    # describing one keyframe: a one-keyframe store whose options alternate, so every call describes it again
    one = api.Context(max_map_points=1 << 20, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    one.keyframe_reserve(max(per) + 1, 1)
    one.scan_prefilter(scans[0], 0.1, 0.2, auto_voxel_size=False, download=False)
    one.register_prefiltered(truth[0], 1, 0)
    one.keyframe_add_registered(truth[0])
    flip = [0]

    def describe():
        flip[0] ^= 1
        return one.loop_candidates([0], 1, api.loop_opts(height_offset=2.0 + 0.5 * flip[0]), stats=True)[1]

    describe()
    d_wall, d_dev = timed(describe, 5 * a.reps)
    out = dict(card=card(), keyframe_points=int(n_pts / max(n_kf, 1)), options=dict(rings=opts.rings, sectors=opts.sectors,
               max_range=opts.max_range), describe_one=dict(wall_ms=d_wall, device_ms=d_dev["time_describe_ms"]), query={}, live_step=live)
    excl0 = api.loop_opts(exclude_recent=0)
    for n in frames:
        def q1():
            return ctx.loop_candidates([n], 10, excl0, stats=True)[1]  # keyframe n against ids 0 .. n-1
        q1()
        w, d = timed(q1, a.reps)
        out["query"][str(n)] = dict(wall_ms=w, device_ms=d["time_search_ms"], products=n * opts.rings * opts.sectors ** 2)
    n_all = min(frames)
    ids = np.arange(n_all, dtype=np.int32)

    def all_pairs():
        return ctx.loop_candidates(ids, 10, excl0, stats=True)[1]
    all_pairs()
    w, d = timed(all_pairs, max(1, a.reps // 2))
    out["all_pairs"] = dict(keyframes=n_all, wall_ms=w, device_ms=d["time_search_ms"],
                            products=n_all * (n_all - 1) // 2 * opts.rings * opts.sectors ** 2)
    print(json.dumps(out))
    one.close()
    ctx.close()


if __name__ == "__main__":
    main()

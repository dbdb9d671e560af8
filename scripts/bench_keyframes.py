"""Keyframe costs (so_keyframe_*, so_map_from_keyframes, so_register_keyframes): the rebuild of the map from N prefiltered OS1-128
keyframes at new poses (surf store, archive on), the loop-verification submap plus one keyframe registered against it,
and what so_keyframe_add_registered adds to a live-loop step (so_register_prefiltered + so_map_add_registered_scan).  Wall time is
around calls that end in a device synchronise (the rebuild reads its sizes back; the registration reads its results); device time
is the kernels and copies torch.profiler records in a run of its own.  Prints one JSON line with the card and its power limit.

    python scripts/bench_keyframes.py [--frames 100,500,1000] [--reps 5]
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


def device_ms(fn):
    """Summed device time (ms) of the kernels, copies and sets one call of fn records under torch.profiler."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.events():
        if getattr(e, "device_type", None) == DeviceType.CUDA:
            tot += float(getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0) or 0.0)
    return tot / 1e3


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
    ap.add_argument("--frames", default="100,500,1000")
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
    per = []
    for s in scans:
        per.append(ctx.scan_prefilter(s, 0.1, 0.2, auto_voxel_size=False, download=False)[0])
    ctx.keyframe_reserve(n_max * max(per) + 1, n_max)
    # live step (prefilter, register, insert) with and without keeping the keyframe, interleaved so both see the same map
    k = 0

    def step(keep):
        nonlocal k
        i = k % a.scans
        ctx.scan_prefilter(scans[i], 0.1, 0.2, auto_voxel_size=False, download=False)
        r = ctx.register_prefiltered(truth[i], 20, 0)
        if keep:
            ctx.keyframe_add_registered(np.array(r.pose))
        ctx.map_add_registered_scan(np.array(r.pose))
        k += 1
        return r

    for _ in range(3):
        step(False)
    t_plain, t_keep = [], []
    for _ in range(3 * a.reps):
        t_plain.append(wall_ms(lambda: step(False), 1))
        t_keep.append(wall_ms(lambda: step(True), 1))
    live_plain, live_keep = float(np.median(t_plain)), float(np.median(t_keep))
    r = step(False)
    while ctx.keyframe_info()[0] < n_max - 1:
        ctx.keyframe_add_registered(np.array(r.pose))
    add_dev = device_ms(lambda: ctx.keyframe_add_registered(np.array(r.pose)))
    n_kf, n_pts, _ = ctx.keyframe_info()
    # rebuild at new poses: a trajectory of 0.5 m steps with a slow turn, so the union spreads over many blocks
    rng = np.random.default_rng(1)
    th = np.cumsum(rng.normal(0.0, 0.02, n_kf))
    xy = np.cumsum(0.5 * np.stack([np.cos(th), np.sin(th)], 1), 0)
    poses = np.array([np.r_[xy[i], 0.0, synth.quat_from_rotvec(np.array([0, 0, th[i]]))] for i in range(n_kf)])
    dst = api.Context(max_map_points=1 << 25, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    dst.map_archive(1 << 25)
    rebuild = []
    for n in frames:
        ids = np.arange(n, dtype=np.int32)
        f = lambda: dst.map_from_keyframes(ctx, ids, poses[:n], 1)    # noqa: E731
        f()
        pts = sum(ctx.keyframe_download(i).shape[0] for i in range(n))
        rebuild.append(dict(frames=n, union_points=int(pts), wall_ms=wall_ms(f, a.reps), device_ms=device_ms(f), map_points=dst.map_size(),
                            archive_points=dst.map_archive_info(0)[0]))
    # loop verification: a submap of 10 keyframes, one keyframe registered against it
    sub = api.Context(max_map_points=1 << 21, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    sub_ids = np.arange(10, dtype=np.int32)
    kf_poses = ctx.keyframe_poses()
    sub_poses = kf_poses[:10]
    prior = synth.perturb_pose(kf_poses[3], 7, 0.1, 1.0)
    build = lambda: sub.map_from_keyframes(ctx, sub_ids, sub_poses, 1)  # noqa: E731
    align = lambda: sub.register_keyframes(ctx, [3], [prior], 20, 0)   # noqa: E731
    build()
    align()
    loop = dict(submap_keyframes=10, build_wall_ms=wall_ms(build, a.reps), build_device_ms=device_ms(build),
                align_wall_ms=wall_ms(align, a.reps), align_device_ms=device_ms(align))
    print(json.dumps(dict(card=card(), keyframe_points=int(n_pts / max(n_kf, 1)), rebuild=rebuild, loop=loop,
                          live_step_wall_ms=dict(without_keyframe=live_plain, with_keyframe=live_keep, add_device_ms=add_dev))))
    for c in (ctx, dst, sub):
        c.close()


if __name__ == "__main__":
    main()

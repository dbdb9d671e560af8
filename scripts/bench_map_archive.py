"""Block archive cost (so_map_archive): wall and device time (torch.profiler, summed kernels and copies) per map shift with the archive (eviction + restore + index) against the same shift
without it (drop + index), on the cfg2 map and on a street map of several million points; live-loop time per scan (register +
insert, no shift) with and without the archive; the archive's memory.  Every shift call synchronises (the rebuild reads its sizes
back), so wall time per call is what the caller waits.  Prints one JSON line.

    python scripts/bench_map_archive.py [--reps 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from superodom_b200 import api, synth  # noqa: E402


def street(n_points, seed=5):
    """Patches of points along a 3 km street, 40 m wide, 10 m high"""
    rng = np.random.default_rng(seed)
    per = 2000
    c = np.stack([rng.uniform(-1500, 1500, n_points // per), rng.uniform(-20, 20, n_points // per), rng.uniform(-2, 8, n_points // per)], 1)
    p = (c[:, None, :] + rng.uniform(0, 1, size=(len(c), per, 3)) * np.array([6.0, 6.0, 0.5])).reshape(-1, 3)
    return np.concatenate([p, np.ones((len(p), 1))], 1).astype(np.float32)


def device_ms(events):
    """Summed device time (ms) of the kernels, copies and sets a torch.profiler trace recorded (every stream of the device)."""
    from torch.autograd import DeviceType
    tot = 0.0
    for e in events:
        if getattr(e, "device_type", None) == DeviceType.CUDA:
            tot += float(getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0) or 0.0)
    return tot / 1e3


def shift_times(cloud, archive, a_x, b_x, reps, plane_res=0.2):
    """Median milliseconds of the rebuild that applies an origin change from window A (so_map_set_origin(a_x)) to window B
    (b_x) and back, timed around so_map_set_origin + the read that rebuilds (so_map_counts_5x5).  Without the archive the cloud
    is reloaded at A (untimed) before every timed change to B, so each timed rebuild drops the blocks the archive run evicts."""
    ctx = api.Context(max_map_points=max(len(cloud), 1 << 20), max_scan_points=65536, plane_res=plane_res)
    if archive:
        ctx.map_archive(len(cloud))
    ctx.map_set_origin([a_x, 0.0, 0.0])
    ctx.map_set_points(cloud)
    ts = []
    for _ in range(reps):
        for x in (b_x, a_x):
            if not archive:
                if x == a_x:
                    continue
                ctx.map_set_origin([a_x, 0.0, 0.0])
                ctx.map_set_points(cloud)
            t0 = time.perf_counter()
            ctx.map_set_origin([x, 0.0, 0.0])
            ctx.map_counts_5x5([10, 10, 5])
            ts.append(time.perf_counter() - t0)
    # device time: the same changes once more under torch.profiler (CUPTI sees the context's own streams)
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    dev = []
    for x in ((b_x, a_x) if archive else (b_x,)) * 3:
        if not archive:
            ctx.map_set_origin([a_x, 0.0, 0.0])
            ctx.map_set_points(cloud)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctx.map_set_origin([x, 0.0, 0.0])
            ctx.map_counts_5x5([10, 10, 5])
        dev.append(device_ms(prof.events()))
    ctx.map_set_origin([b_x, 0.0, 0.0])
    ctx.map_counts_5x5([10, 10, 5])                                   # applies the change
    n = ctx.map_size()
    info = ctx.map_archive_info(0)
    ctx.close()
    return float(np.median(ts)) * 1e3, n, info, float(np.median(dev))


def live_loop(archive, reps):
    c0 = synth.make_case("cfg1")
    ctx = api.Context(max_map_points=1 << 21, max_scan_points=1 << 17, plane_res=0.2)
    if archive:
        ctx.map_archive(1 << 21)
    ctx.map_set_points(c0["map_xyzi"])
    scan, prior = c0["scan_xyzi"], c0["pose_prior"]
    for _ in range(3):
        ctx.register(scan, prior, 5, 2000)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = ctx.register(scan, prior, 5, 2000)
        ctx.map_add_registered_scan(np.array(r.pose))
        ts.append(time.perf_counter() - t0)
    ctx.close()
    return float(np.median(ts)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    cfg2 = synth.make_case("cfg2")["map_xyzi"]
    big = street(4_000_000)
    out = {"gpu": os.environ.get("SO_GPU_NAME", "H100")}
    # cfg2 (x in [-52, 52] m): window B leaves out the blocks below x = -25 m; street: B moves the window 400 m (8 block columns)
    for name, cloud, ax, bx in [("cfg2", cfg2, -100.0, 0.0), ("street", big, -1500.0, -1100.0)]:
        t_on, n_on, info, d_on = shift_times(cloud, True, ax, bx, a.reps)
        t_off, n_off, _, d_off = shift_times(cloud, False, ax, bx, a.reps)
        out[name] = {"points": len(cloud), "origin_x": [ax, bx], "ms_per_change_archive": round(t_on, 3),
                     "ms_per_change_no_archive": round(t_off, 3), "device_ms_per_change_archive": round(d_on, 3),
                     "device_ms_per_change_no_archive": round(d_off, 3),
                     "window_points_at_B": n_on, "window_points_at_B_no_archive": n_off, "archive_points": info[0], "archive_blocks": info[1],
                     "archive_bytes_per_store": info[2] * 16}
    out["live_ms_per_scan_archive"] = round(live_loop(True, 4 * a.reps), 4)
    out["live_ms_per_scan_no_archive"] = round(live_loop(False, 4 * a.reps), 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

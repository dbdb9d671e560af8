"""Map-store call times of two builds of the library, measured in one run with alternating worker processes.

    python scripts/bench_map.py --old path/to/libA.so [--new path/to/libB.so] [--rounds 3] [--reps 10]

Each round starts one worker per library (alternating which goes first); a worker loads its library through SO_LIB_PATH, warms
every call up once and times it --reps times (host wall clock around calls that end in a stream synchronise):
  set_cfg2       so_map_set_points of the 1 M-point cfg2 map (upload + index build)
  add_cfg5       so_map_add_surf of the 5.4 M-point cfg5 raw cloud into an empty store (voxel filter + index)
  shift_rebuild  the rebuild a so_map_shift forces on the cfg2 map (origin moved by one block)
  prefilter      so_scan_prefilter of one OS1-128 scan at leaf 0.2, result left on the device
and runs the live loop of tests/tools/live_loop.py once (its ms_insert_median and ms_prefilter_median).  Prints one JSON line:
the card and its power limit, and per library and workload the median and the spread (min, max) over all rounds' samples."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        return "unknown"


def _time(fn, reps, setup=None):
    out = []
    for r in range(reps + 1):                                   # the first call warms up
        if setup:
            setup()
        t0 = time.perf_counter()
        fn()
        if r:
            out.append((time.perf_counter() - t0) * 1e3)
    return out


def worker(reps: int, live_scans: int) -> dict:
    from superodom_b200 import api, synth
    sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
    import live_loop
    scene2, map2 = synth.make_map_for("cfg2")
    raw = synth.sample_surfaces(synth.make_scene(58.0, seed=77), 0.1, seed=1234)
    raw4 = np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1)
    scan = synth.make_scan(scene2, "os1_128", synth.random_sensor_pose(scene2, 901, 10.0), 8000)
    empty = np.zeros((0, 4), np.float32)
    out = {}
    ctx = api.Context(max_map_points=len(raw4) + 1024, max_scan_points=len(scan), plane_res=0.2)
    out["set_cfg2"] = _time(lambda: ctx.map_set_points(map2), reps)

    def reset_shift():
        ctx.map_set_origin([-500.0, -500.0, -250.0])                  # origin (10, 10, 5), the initial one
        ctx.map_set_points(map2)
    out["shift_rebuild"] = _time(lambda: ctx.map_shift([-410.0, 0.0, 0.0]), reps, reset_shift)
    out["prefilter"] = _time(lambda: ctx.scan_prefilter(scan, 0.1, 0.2, auto_voxel_size=False, download=False), reps)
    ctx.close()
    ctx = api.Context(max_map_points=len(raw4) + 1024, max_scan_points=1024, plane_res=0.1)
    out["add_cfg5"] = _time(lambda: ctx.map_add_surf(raw4), reps, lambda: ctx.map_set_points(empty))
    ctx.close()
    live = live_loop.run(api, synth, n_scans=live_scans)
    out["live_insert"] = [live["ms_insert_median"]]
    out["live_prefilter"] = [live["ms_prefilter_median"]]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old", required=True, help="the library to compare against")
    ap.add_argument("--new", default=os.path.join(ROOT, "superodom_b200", "libsuperodom_b200.so"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--live-scans", type=int, default=60)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        print(json.dumps(worker(a.reps, a.live_scans)))
        return
    libs = {"old": a.old, "new": a.new}
    samples = {k: {} for k in libs}
    for r in range(a.rounds):
        for tag in (("old", "new") if r % 2 == 0 else ("new", "old")):
            env = dict(os.environ, SO_LIB_PATH=libs[tag])
            res = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--old", a.old, "--reps", str(a.reps),
                                  "--live-scans", str(a.live_scans)], env=env, check=True, capture_output=True, text=True)
            for k, v in json.loads(res.stdout.strip().splitlines()[-1]).items():
                samples[tag].setdefault(k, []).extend(v)
    out = {"card": _card(), "rounds": a.rounds, "reps": a.reps, "unit": "ms"}
    for tag, s in samples.items():
        out[tag] = {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)} for k, v in s.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

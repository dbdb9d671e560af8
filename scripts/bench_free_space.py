"""Cost of free-space clearing on cfg2 (OS1-128 scan of 131 072 rays, about 1 M-point map), on the GPU.

  python scripts/bench_free_space.py [--reps N] [--scans N] [--out DIR]

  - per call of so_map_clear_free_space_registered(stores 1) beside so_map_add_registered_scan on the same map: device time (CUDA
    events, profile class 3, profiling on in a pass of its own) and wall time (the calls end in a device synchronise);
  - the live loop register -> [clear] -> insert per scan, with and without clearing.
Each timed call starts from the same map: the cfg2 map plus the points of a vehicle-sized box the scan sees through.  Prints the card
and its power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from superodom_b200 import api, synth  # noqa: E402
import free_space_numpy as F  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                    # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    scene, mp = synth.make_map_for("cfg2")
    c = synth.make_case_on(scene, mp, "cfg2", 1)
    pose = c["pose_true"]
    # a 4.5 x 1.9 x 1.6 m box 7 m from the sensor, in the map only
    for ang in np.linspace(-np.pi, np.pi, 73):
        ctr = pose[:2] + 7.0 * np.array([np.cos(ang), np.sin(ang)])
        if scene.free(np.array([ctr[0], ctr[1], -1.0]), margin=2.8):
            break
    box = np.array([ctr[0] - 2.25, ctr[0] + 2.25, ctr[1] - 0.95, ctr[1] + 0.95, -1.8, -0.2])
    only = synth.Scene(room=box + np.array([-1, 1, -1, 1, -1, 1]), boxes=box[None])
    raw = synth.sample_surfaces(only, 0.2, seed=9)
    raw = raw[((raw[:, :3] >= box[[0, 2, 4]] - 0.1) & (raw[:, :3] <= box[[1, 3, 5]] + 0.1)).all(1)]
    the_map = np.vstack([mp, synth.voxel_filter_blocks(np.c_[raw, np.ones(len(raw), np.float32)], 0.2)])
    o = F.opts_for("os1_128")
    opts = api.free_space(**{n: getattr(o, n) for n, _ in api.FreeSpace._fields_})
    ctx = api.Context(max_map_points=1 << 22, max_scan_points=262144, plane_res=0.2)
    res = dict(card=card(), map_points=len(the_map), scan_points=len(c["scan_xyzi"]))

    def one(kind, profile):
        ctx.map_set_points(the_map)
        ctx.register(c["scan_xyzi"], c["pose_prior"], 20)
        ctx.profile_enable(profile)
        ctx.profile_get(3, reset=True)
        t0 = time.perf_counter()
        out = ctx.map_clear_free_space_registered(pose, opts) if kind == "clear" else ctx.map_add_registered_scan(pose)
        wall = (time.perf_counter() - t0) * 1e3
        dev = ctx.profile_get(3, reset=True)[0]
        ctx.profile_enable(False)
        return wall, dev, out

    for kind in ("clear", "insert"):                          # warm-up
        one(kind, False); one(kind, True)
    walls = {"clear": [], "insert": []}
    devs = {"clear": [], "insert": []}
    removed = None
    for _ in range(a.reps):
        for kind in ("clear", "insert"):                      # alternate the two
            w, _, out = one(kind, False)
            walls[kind].append(w)
            if kind == "clear":
                removed = out["n_removed"]
            devs[kind].append(one(kind, True)[1])
    for kind in walls:
        res[f"{kind}_wall_ms_median"] = float(np.median(walls[kind]))
        res[f"{kind}_device_ms_median"] = float(np.median(devs[kind]))
    res["removed_per_clear"] = int(removed)
    # live loop: register -> [clear] -> insert over scans from nearby poses
    poses = [synth.random_sensor_pose(scene, 3000 + k, 20.0) for k in range(a.scans)]
    scans = [synth.make_scan(scene, "os1_128", p, 3100 + k) for k, p in enumerate(poses)]
    priors = [synth.perturb_pose(p, 3200 + k, 0.05, 0.5) for k, p in enumerate(poses)]
    for arm in ("plain", "clear", "plain", "clear"):
        ctx.map_set_points(the_map)
        ts = []
        for s, p in zip(scans, priors):
            t0 = time.perf_counter()
            r = ctx.register(s, p, 20)
            if arm == "clear":
                ctx.map_clear_free_space_registered(np.array(r.pose), opts)
            ctx.map_add_registered_scan(np.array(r.pose))
            ts.append((time.perf_counter() - t0) * 1e3)
        res[f"loop_{arm}_ms_per_scan_median"] = float(np.median(ts[2:]))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_free_space.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Degeneracy-aware registration: accuracy sweep of the thresholds and cost against so_register (DESIGN.md section 8).

  python scripts/bench_degeneracy.py [--scans 6] [--repeat 20]

Part 1, accuracy: thresholds 0.02 / 0.05 / 0.1 / 0.2 / 0.3 (both blocks) with constrain = 1, against so_register, on the corridor
without poles (priors 0.15 m off along it) and on cfg1 / cfg2: along- and across-corridor (x / y) position error and the flagged
counts of the last ICP iteration.  Part 2, cost: a capped VLP-16 cfg1 scan (device and wall time, median of --repeat) and 64- and
256-scan cfg2 batches (scans/s).  Prints one JSON line per row; the card and its power limit are printed first and belong beside
every number."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from superodom_b200 import api, synth  # noqa: E402

THRESHOLDS = (0.02, 0.05, 0.1, 0.2, 0.3)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})"


def corridor(n_scans):
    sc = synth.make_corridor_scene(poles=False)
    raw = synth.sample_surfaces(sc, 0.2)
    surf = synth.voxel_filter_blocks(np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1), 0.2)
    rng = np.random.default_rng(9100)
    cases = []
    for s in range(n_scans):
        yaw = rng.uniform(-0.2, 0.2)
        T = np.array([rng.uniform(-20, 20), rng.uniform(-0.8, 0.8), rng.uniform(-0.3, 0.3), 0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)])
        rec = synth.make_ring_scan(sc, "os1_128", T, 9200 + s)
        prior = synth.perturb_pose(T, 9300 + s)
        prior[0] += 0.15
        cases.append(dict(scan=np.ascontiguousarray(np.concatenate([rec[:, :3], rec[:, 5:6]], 1)), T=T, prior=prior))
    return surf, cases


def scenes(n_scans):
    surf, cases = corridor(n_scans)
    yield "corridor", surf, cases, 20, 0
    for name in ("cfg1", "cfg2"):
        scene, m = synth.make_map_for(name)
        cs = [synth.make_case_on(scene, m, name, i) for i in range(n_scans)]
        cfg = synth.CONFIGS[name]
        yield name, m, [dict(scan=c["scan_xyzi"], T=c["pose_true"], prior=c["pose_prior"]) for c in cs], cfg["max_iterations"], cfg["max_surface_features"]


def accuracy(n_scans):
    for name, m, cases, iters, cap in scenes(n_scans):
        ctx = api.Context(max_map_points=max(1 << 20, 2 * len(m)), max_scan_points=262144, plane_res=0.2)
        ctx.map_set_points(m)
        for thr in (None,) + THRESHOLDS:
            ex, ey, fp, fo = [], [], [], []
            for c in cases:
                if thr is None:
                    r = ctx.register(c["scan"], c["prior"], iters, cap)
                    flags = (0, 0)
                else:
                    d = ctx.register_degeneracy(c["scan"], c["prior"], api.degeneracy(thr, thr), iters, cap)
                    r, flags = d.icp, (bin(d.flags_pos).count("1"), bin(d.flags_ori).count("1"))
                ex.append(abs(r.pose[0] - c["T"][0])); ey.append(abs(r.pose[1] - c["T"][1]))
                fp.append(flags[0]); fo.append(flags[1])
            print(json.dumps(dict(part="accuracy", scene=name, threshold=thr, err_x_max=max(ex), err_x_median=float(np.median(ex)),
                                  err_y_max=max(ey), flagged_pos=fp, flagged_ori=fo)), flush=True)
        ctx.close()


def cost(repeat):
    scene, m = synth.make_map_for("cfg1")
    c = synth.make_case_on(scene, m, "cfg1", 0)
    ctx = api.Context(max_map_points=max(1 << 20, 2 * len(m)), max_scan_points=262144, plane_res=0.2)
    ctx.map_set_points(m)
    d = api.degeneracy(0.1, 0.1)
    for arm in ("so_register", "so_register_degeneracy"):
        dev, wall = [], []
        for _ in range(repeat + 3):
            t0 = time.perf_counter()
            r = ctx.register(c["scan_xyzi"], c["pose_prior"], 5, 2000, skip_map_checks=True) if arm == "so_register" else \
                ctx.register_degeneracy(c["scan_xyzi"], c["pose_prior"], d, 5, 2000, skip_map_checks=True).icp
            wall.append((time.perf_counter() - t0) * 1e3); dev.append(r.time_ms)
        print(json.dumps(dict(part="cost", case="cfg1 capped single", arm=arm, device_ms=float(np.median(dev[3:])),
                              wall_ms=float(np.median(wall[3:])))), flush=True)
    ctx.close()
    scene, m = synth.make_map_for("cfg2")
    cs = [synth.make_case_on(scene, m, "cfg2", i) for i in range(16)]
    for n in (64, 256):
        ctx = api.Context(max_map_points=max(1 << 20, 2 * len(m)), max_scan_points=262144, max_batch=n, plane_res=0.2)
        ctx.map_set_points(m)
        pick = [cs[i % len(cs)] for i in range(n)]
        scans = np.ascontiguousarray(np.concatenate([p["scan_xyzi"] for p in pick]))
        npts = [len(p["scan_xyzi"]) for p in pick]
        poses = np.array([p["pose_prior"] for p in pick])
        for arm in ("so_register_batch", "so_register_batch_degeneracy"):
            ts = []
            for _ in range(4):
                t0 = time.perf_counter()
                if arm == "so_register_batch":
                    ctx.register_batch(scans, npts, poses, 20, 0, skip_map_checks=True)
                else:
                    ctx.register_batch_degeneracy(scans, npts, poses, [d] * n, 20, 0, skip_map_checks=True)
                ts.append(time.perf_counter() - t0)
            print(json.dumps(dict(part="cost", case=f"cfg2 batch {n}", arm=arm, scans_per_s=n / float(np.median(ts[1:])))), flush=True)
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=6)
    ap.add_argument("--repeat", type=int, default=20)
    a = ap.parse_args()
    print(json.dumps(dict(card=card())), flush=True)
    accuracy(a.scans)
    cost(a.repeat)


if __name__ == "__main__":
    main()

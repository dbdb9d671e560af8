"""Edge extraction (so_scan_extract_edges): call times, the live loop with and without edges, and the corridor accuracy.

    python scripts/bench_edges.py [--calls 200] [--scans 40] [--out result.json]

  extract      per-scan extractor time on a VLP-16 ring scan (cfg1 scene, 28 800 records) and an OS1-128 one (cfg2 scene, 131 072):
               device time (profile class 3: CUDA events around the kernels, the count read-back and the voxel filter, profiling on)
               and wall time (host clock around the whole call, profiling off), median and spread over --calls calls each
  live_loop    per-scan time of the cfg1 live loop: [extract edges], so_register with the host surf cloud [and the edge cloud],
               so_map_add_registered_scan, [so_map_add_scan_edge]; both arms on the same scans, alternating, median over --scans
  corridor     tests/test_edge_features.corridor_runs: along-corridor error and pos_inv_cond of 8 OS1-128 scans, planes only / with edges
Prints one JSON line with the card name and power limit read in the same run."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        return "unknown"


def _stats(v):
    v = np.asarray(v, np.float64)
    return dict(median=round(float(np.median(v)), 4), min=round(float(v.min()), 4), max=round(float(v.max()), 4), n=int(len(v)))


def bench_extract(api, synth, calls):
    out = {}
    for name, (half, sensor) in {"vlp16": (17.5, "vlp16"), "os1_128": (52.0, "os1_128")}.items():
        scene, _ = synth.make_map(half, 0.2)
        rec = synth.make_ring_scan(scene, sensor, synth.random_sensor_pose(scene, 900, 10.0), 1000)
        ctx = api.Context(max_map_points=1 << 16, max_scan_points=262144)
        for leaf in (0.0, 0.1):
            for _ in range(10):
                ctx.scan_extract_edges(rec, voxel_leaf=leaf)
            wall = []
            for _ in range(calls):
                t0 = time.perf_counter()
                e = ctx.scan_extract_edges(rec, voxel_leaf=leaf)
                wall.append((time.perf_counter() - t0) * 1e3)
            ctx.profile_enable(True)
            ctx.profile_get(3, reset=True)
            dev = []
            for _ in range(calls):
                ctx.scan_extract_edges(rec, voxel_leaf=leaf)
                dev.append(ctx.profile_get(3, reset=True)[0])
            ctx.profile_enable(False)
            out[f"{name}_leaf{leaf}"] = dict(records=len(rec), edges=len(e), device_ms=_stats(dev), wall_ms=_stats(wall))
        ctx.close()
    return out


def bench_live_loop(api, synth, n_scans):
    from conftest import get_case
    case = get_case("cfg1", 0)
    scene, surf_map = case["scene"], case["map_xyzi"]
    poses = [synth.random_sensor_pose(scene, 4000 + i, 10.0) for i in range(n_scans)]
    recs = [synth.make_ring_scan(scene, "vlp16", T, 4100 + i) for i, T in enumerate(poses)]
    scans = [np.ascontiguousarray(np.concatenate([r[:, :3], r[:, 5:6]], 1)) for r in recs]
    priors = [synth.perturb_pose(T, 4200 + i) for i, T in enumerate(poses)]
    ctxs = {}
    for arm in ("planes", "edges"):
        c = api.Context(max_map_points=1 << 21, max_scan_points=262144, plane_res=0.2, line_res=0.1)
        c.map_set_points(surf_map)
        c.map_set_resolution(0.1, 0.2)
        ctxs[arm] = c
    times = {"planes": [], "edges": []}
    errs = {"planes": [], "edges": []}
    for i in range(n_scans):
        for arm in (("planes", "edges") if i % 2 == 0 else ("edges", "planes")):
            c = ctxs[arm]
            t0 = time.perf_counter()
            if arm == "edges":
                e = c.scan_extract_edges(recs[i])
                r = c.register(scans[i], priors[i], 5, 2000, edge_xyzi=e)
                c.map_add_registered_scan(np.array(r.pose))
                c.map_add_scan_edge(e, np.array(r.pose))
            else:
                r = c.register(scans[i], priors[i], 5, 2000)
                c.map_add_registered_scan(np.array(r.pose))
            dt = (time.perf_counter() - t0) * 1e3
            if i >= 4:                                    # the first scans warm up the graphs and grow the edge store
                times[arm].append(dt)
            errs[arm].append(float(np.linalg.norm(np.array(r.pose)[:3] - poses[i][:3])))
    for c in ctxs.values():
        c.close()
    return {arm: dict(ms=_stats(times[arm]), pos_err_m=_stats(errs[arm])) for arm in times}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--scans", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from superodom_b200 import api, synth
    assert api.device_available(), "no sm_90 device"
    res = dict(card=_card(), extract=bench_extract(api, synth, a.calls), live_loop=bench_live_loop(api, synth, a.scans))
    import test_edge_features as T
    res["corridor"] = T.corridor_runs(api)
    res["card_after"] = _card()
    line = json.dumps(res, default=float)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

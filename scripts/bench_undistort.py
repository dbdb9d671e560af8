"""Cost and value of within-scan motion compensation (so_register_undistort*, so_register_optimized*) on the GPU.

Prints one JSON line: the card and its power limit; capped VLP-16 single-scan latency of so_register, so_register_undistort
(APPROXIMATED) and so_register_optimized (OPTIMIZED), alternating calls, medians of the host wall time and of the device time
between the schedule's events; 64- and 256-scan cfg2 batch time for the three; per-launch times of profile classes 7 and 8 and
of the search and fit (a separate profiling run); the pose error against ground truth at several speeds for NONE and
APPROXIMATED; and, for OPTIMIZED, the pose error in four velocity scenarios over a sweep of motion_info."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from superodom_b200 import api, synth  # noqa: E402


def _card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        return "unknown"


def _err(pose, truth):
    d = abs(float(np.dot(pose[3:], truth[3:])))
    return float(np.linalg.norm(np.asarray(pose[:3]) - truth[:3])), float(2 * np.arccos(min(1.0, d)))


def _qmul(a, b):
    return np.array([a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1], a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2],
                     a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0], a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]])


def _compose(a, b):
    return np.concatenate([a[:3] + synth.quat_to_R(a[3:]) @ b[:3], _qmul(a[3:], b[3:])])


def _inverse(a):
    qc = np.array([-a[3], -a[4], -a[5], a[6]])
    return np.concatenate([-(synth.quat_to_R(qc) @ a[:3]), qc])


def _delta(prev, cur):
    """D0 = prev^-1 * cur, what a caller that has the previous registration passes"""
    return _compose(_inverse(np.asarray(prev, np.float64)), np.asarray(cur, np.float64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--batch-reps", type=int, default=10)
    ap.add_argument("--info", type=float, default=api.DEFAULT_MOTION_INFO, help="motion_info of the timed OPTIMIZED calls")
    ap.add_argument("--info-sweep", type=float, nargs="*", default=[0.0, 1e-3, 1e-2, 0.1, 1.0, 10.0])
    a = ap.parse_args()
    out = {"card": _card()}

    # ---- single capped VLP-16 scan (the live loop)
    scene, map_xyzi = synth.make_map_for("cfg1")
    pose = synth.random_sensor_pose(scene, 950, 8.0)
    d = synth.make_moving_scan(scene, "vlp16", pose, 1.5, 0.3, 60)
    ctx = api.Context(max_map_points=1 << 21, max_scan_points=262144, plane_res=0.2)
    ctx.map_set_points(map_xyzi)
    u = api.undistort(d["pose_prev"], 0.1)
    mo = api.motion(0.1, _delta(d["pose_prev"], d["prior"]), [a.info] * 6)
    wall = {"none": [], "approx": [], "opt": []}
    dev = {"none": [], "approx": [], "opt": []}
    for i in range(a.reps + 20):
        for m in ("none", "approx", "opt"):
            r = (ctx.register(d["scan_xyzi"], d["prior"], 5, 2000) if m == "none" else
                 ctx.register_undistort(d["scan_xyzi"], d["prior"], u, 5, 2000) if m == "approx" else
                 ctx.register_optimized(d["scan_xyzi"], d["prior"], mo, 5, 2000).icp)
            if i >= 20:
                wall[m].append(r.time_total_ms)
                dev[m].append(r.time_ms)
    out["single_capped_vlp16_ms"] = {m: {"wall_median": float(np.median(wall[m])), "device_median": float(np.median(dev[m]))} for m in wall}

    # ---- cfg2 batches
    scene2, map2 = synth.make_map_for("cfg2")
    base = []
    for k in range(16):
        p = synth.random_sensor_pose(scene2, 970 + k, 20.0)
        base.append(synth.make_moving_scan(scene2, "os1_128", p, 1.5, 0.3, 80 + k))
    for nb in (64, 256):
        ds = [base[k % len(base)] for k in range(nb)]
        flat = np.ascontiguousarray(np.concatenate([x["scan_xyzi"] for x in ds]))
        npts = [len(x["scan_xyzi"]) for x in ds]
        priors = np.stack([x["prior"] for x in ds])
        us = [api.undistort(x["pose_prev"], 0.1) for x in ds]
        ms_ = [api.motion(0.1, _delta(x["pose_prev"], x["prior"]), [a.info] * 6) for x in ds]
        bctx = api.Context(max_map_points=1 << 22, max_scan_points=max(npts), max_batch=nb, plane_res=0.2)
        bctx.map_set_points(map2)
        t = {"none": [], "approx": [], "opt": []}
        for i in range(a.batch_reps + 2):
            for m in ("none", "approx", "opt"):
                res = (bctx.register_batch(flat, npts, priors, 20, 0, skip_map_checks=True) if m == "none"
                       else bctx.register_batch_undistort(flat, npts, priors, us, 20, 0, skip_map_checks=True) if m == "approx"
                       else [x.icp for x in bctx.register_batch_optimized(flat, npts, priors, ms_, 20, 0, skip_map_checks=True)])
                if i >= 2:
                    t[m].append(res[0].time_total_ms)
        out[f"cfg2_batch{nb}_ms"] = {m: float(np.median(v)) for m, v in t.items()}
        if nb == 64:
            # class 7 is the warp; its keys keep the kernel names of the first runs (k_undistort, k_motion_warp), so runs compare
            bctx.profile_enable(True)
            bctx.profile_get(7, reset=True)
            bctx.register_batch_undistort(flat, npts, priors, us, 20, 0, skip_map_checks=True)
            ms, n = bctx.profile_get(7)
            kn, knn_n = bctx.profile_get(0)
            kf, kf_n = bctx.profile_get(5)
            out["cfg2_batch64_per_launch_ms"] = {"k_undistort": ms / max(n, 1), "k_knn_scan": kn / max(knn_n, 1), "k_fit": kf / max(kf_n, 1)}
            for c in (0, 5, 7, 8):
                bctx.profile_get(c, reset=True)
            bctx.register_batch_optimized(flat, npts, priors, ms_, 20, 0, skip_map_checks=True)
            per = {k: bctx.profile_get(c) for k, c in (("k_knn_scan", 0), ("k_fit", 5), ("k_motion_warp", 7), ("k_motion_eval+step", 8))}
            out["cfg2_batch64_optimized_per_launch_ms"] = {k: v[0] / max(v[1], 1) for k, v in per.items()}
            bctx.profile_enable(False)
        bctx.close()

    # ---- accuracy against speed
    acc = []
    for name, sensor, it, mf, sc, mp in (("cfg1", "vlp16", 5, 2000, scene, map_xyzi), ("cfg2", "os1_128", 20, 0, scene2, map2)):
        actx = api.Context(max_map_points=1 << 22, max_scan_points=262144, plane_res=0.2)
        actx.map_set_points(mp)
        for speed, yaw in ((0.0, 0.0), (1.5, 0.3), (5.0, 0.5), (10.0, 0.5)):
            en, ea = [], []
            for k in range(4):
                p = synth.random_sensor_pose(sc, 990 + k, 8.0 if name == "cfg1" else 20.0)
                x = synth.make_moving_scan(sc, sensor, p, speed, yaw, 300 + k)
                rn = actx.register(x["scan_xyzi"], x["prior"], it, mf)
                ra = actx.register_undistort(x["scan_xyzi"], x["prior"], api.undistort(x["pose_prev"], 0.1), it, mf)
                en.append(_err(np.array(rn.pose), x["pose_true"]))
                ea.append(_err(np.array(ra.pose), x["pose_true"]))
            acc.append({"case": name, "speed": speed, "yaw_rate": yaw,
                        "none_m": float(np.mean([e[0] for e in en])), "approx_m": float(np.mean([e[0] for e in ea])),
                        "none_rad": float(np.mean([e[1] for e in en])), "approx_rad": float(np.mean([e[1] for e in ea]))})
        actx.close()
    out["accuracy_mean_of_4"] = acc

    # ---- OPTIMIZED in four velocity scenarios (the previous registration's velocity right, starting from rest, braking, still),
    # over a sweep of motion_info; mean of 4 scans per row
    opt = []
    for name, sensor, it, mf, sc, mp in (("cfg1", "vlp16", 5, 2000, scene, map_xyzi), ("cfg2", "os1_128", 20, 0, scene2, map2)):
        actx = api.Context(max_map_points=1 << 22, max_scan_points=262144, plane_res=0.2)
        actx.map_set_points(mp)
        for scenario, speed in (("constant", 5.0), ("start", 1.5), ("start", 5.0), ("start", 10.0), ("brake", 5.0), ("still", 0.0)):
            xs = []
            for k in range(4):
                p = synth.random_sensor_pose(sc, 990 + k, 8.0 if name == "cfg1" else 20.0)
                sweep = 0.0 if scenario in ("brake", "still") else speed
                x = synth.make_moving_scan(sc, sensor, p, sweep, 0.3 if sweep else 0.0, 300 + k)
                if scenario == "constant":
                    D0, prev = _delta(x["pose_prev"], x["pose_true"]), x["pose_prev"]
                elif scenario == "brake":
                    D0 = np.array([0.5, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])         # 5 m/s straight ahead over 0.1 s
                    prev = _compose(x["pose_true"], _inverse(D0))
                else:
                    D0, prev = np.array([0.0, 0, 0, 0, 0, 0, 1]), x["pose_true"]
                xs.append((x, D0, prev))
            row = {"case": name, "scenario": scenario, "speed": speed,
                   "approx_m": float(np.mean([_err(np.array(actx.register_undistort(x["scan_xyzi"], x["prior"], api.undistort(prev, 0.1), it, mf).pose),
                                                   x["pose_true"])[0] for x, D0, prev in xs]))}
            for info in a.info_sweep:
                e = [_err(np.array(actx.register_optimized(x["scan_xyzi"], x["prior"], api.motion(0.1, D0, [info] * 6), it, mf).icp.pose), x["pose_true"])[0]
                     for x, D0, prev in xs]
                row[f"opt_m_info_{info:g}"] = float(np.mean(e))
            opt.append(row)
        actx.close()
    out["optimized_scenarios_mean_of_4"] = opt
    print(json.dumps(out))


if __name__ == "__main__":
    main()

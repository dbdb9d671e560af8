#!/usr/bin/env python3
"""bench_reloc.py -- global localization (so_localize_global) on synthetic maps, one JSON line per workload:

  default  the cfg2 map (1 M points), one OS1-128 scan, half 10 m in x and y at 0.25 m, the full circle at 2 deg
           = 81 x 81 x 180 = 1 180 980 hypotheses x 1024 score points;
  small    the cfg1 map, one VLP-16 scan, half 1 m in x and y, 0.25 m in z, the full circle at 15 deg, max_range 15 m
           = 9 x 9 x 3 x 24 = 5 832 hypotheses (where the search's per-step read-backs weigh most);
  z        the default scan and centre with half 5 m in x and y and 2 m in z = 41 x 41 x 17 x 180 = 5 143 860 hypotheses.

Per workload: median whole-call wall time over --calls calls after --warmup calls, the per-stage device times (CUDA events in the
call; profile class 6 from one extra profiled call), the search statistics of so_localize_global_bnb on the same call, the
recovery error against the truth, and the card name and power limit read in the same run.  --cpu adds one single-thread run of
the numpy restatement of the default search's scoring (tests/global_localization_numpy.py) for a speed-up figure.  Writes nothing.
The library is the in-tree build, or the one SO_LIB_PATH names.

--whole-map adds so_localize_global_bnb searches over whole maps: the cfg2 map (0.25 m, 2 deg, centre at the map centre with the
true z and a seeded yaw) and a 300 m x 300 m synthetic map (synth.make_map(150.0, 0.2)), each with its per-level statistics, the
share of hypotheses whose leaves were scored and the recovery error.  One more JSON line per map.
--archive adds whole-map searches (so_global_opts.whole_map = 1) over three cfg2-sized rooms at x = -800, 0 and +800 m (1.70 km,
about 3 M points) held in the window and the block archive, window in room A: a scan in room C (the refinement moves the window)
and a scan in room A (no move).  Per case, medians over --calls calls of the build device time (bounds, segment raster, dilation,
levels, offsets), the traversal, the refinement wall time and n_windows, and the whole call; one JSON line per case.
"""
import argparse
import json
import math
import os
import sys
import time

for v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
    os.environ.setdefault(v, "1")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def card():
    name, limit = None, None
    try:
        import torch
        name = torch.cuda.get_device_name(0)
    except Exception:
        pass
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(0)
        limit = nv.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
        if name is None:
            name = nv.nvmlDeviceGetName(h)
            name = name.decode() if isinstance(name, bytes) else name
    except Exception:
        pass
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--scan", type=int, default=0, help="scan index of every workload")
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--whole-map", action="store_true", help="also run so_localize_global_bnb over the whole cfg2 and 300 m maps")
    ap.add_argument("--archive", action="store_true", help="also run whole-map searches over a 1.7 km three-room map in the block archive")
    a = ap.parse_args()
    from superodom_b200 import api, synth
    import global_localization_numpy as GN
    name, limit = card()
    scene, map_xyzi = synth.make_map_for("cfg2")
    case = synth.make_case_on(scene, map_xyzi, "cfg2", a.scan)
    truth = case["pose_true"]
    rng = np.random.default_rng(7100 + a.scan)
    d = rng.uniform(-8.0, 8.0, 2)
    dyaw = rng.uniform(-math.pi, math.pi)
    q = synth.quat_mul(np.array([0.0, 0.0, math.sin(dyaw / 2), math.cos(dyaw / 2)]), truth[3:])
    center = np.r_[truth[0] + d[0], truth[1] + d[1], truth[2], q / np.linalg.norm(q)]
    off = f"centre {np.linalg.norm(d):.2f} m / {math.degrees(dyaw):.1f} deg off"
    scene1, map1 = synth.make_map_for("cfg1")
    case1 = synth.make_case_on(scene1, map1, "cfg1", a.scan)
    t1 = case1["pose_true"]
    center1 = np.r_[t1[:3] + np.array([0.37, -0.21, 0.05]), t1[3:]]
    work = (("default", map_xyzi, case, center, off, dict(half_x=10.0, half_y=10.0, yaw_half=math.pi)),
            ("small", map1, case1, center1, "centre 0.43 m off", dict(half_x=1.0, half_y=1.0, half_z=0.25, yaw_half=math.pi,
                                                                     yaw_step=15 * math.pi / 180, max_range=15.0)),
            ("z", map_xyzi, case, center, off, dict(half_x=5.0, half_y=5.0, half_z=2.0, yaw_half=math.pi)))
    for label, m, cs, c, where, region in work:
        out = localize_workload(m, cs, c, region, a.calls, a.warmup)
        out["workload"] = f"{label}: {out['workload']}, {where}"
        if a.cpu and label == "default":
            ctx = api.Context(max_map_points=len(m) + (1 << 18), max_scan_points=262144, plane_res=0.2)
            ctx.map_set_points(m)
            t0 = time.perf_counter()
            GN.localize_scores_numpy(cs["scan_xyzi"], c, ctx.map_download(0)[:, :3], **region)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            ctx.close()
            out["cpu_numpy_scoring_ms"] = cpu_ms
            out["speedup_search_vs_cpu"] = cpu_ms / sum(out["stage_ms_median"][k] for k in ("raster", "dilate", "score"))
        print(json.dumps(dict(out, card=name, power_limit_w=limit)))
    if a.whole_map:
        ctx = api.Context(max_map_points=len(map_xyzi) + (1 << 18), max_scan_points=262144, plane_res=0.2, max_batch=16)
        ctx.map_set_points(map_xyzi)
        print(json.dumps(dict(whole_map(ctx, "cfg2 map", case, a.calls, a.warmup), card=name, power_limit_w=limit)))
        ctx.close()
        t0 = time.perf_counter()
        scene3, map3 = synth.make_map(150.0, 0.2)
        gen_s = time.perf_counter() - t0
        case3 = synth.make_case_on(scene3, map3, "cfg2", a.scan)
        ctx = api.Context(max_map_points=len(map3) + (1 << 18), max_scan_points=262144, plane_res=0.2, max_batch=16)
        ctx.map_set_points(map3)
        r = whole_map(ctx, f"300 m x 300 m synthetic map ({len(map3)} pts, generated in {gen_s:.1f} s)", case3, max(3, a.calls // 4), 1)
        print(json.dumps(dict(r, card=name, power_limit_w=limit)))
        ctx.close()
    if a.archive:
        for r in archive_cases(a.calls, a.warmup):
            print(json.dumps(dict(r, card=name, power_limit_w=limit)))


def localize_workload(map_xyzi, case, center, region, calls, warmup):
    """so_localize_global on one region: whole-call wall times, stage times, class-6 profile, and one so_localize_global_bnb call
    for the search statistics."""
    from superodom_b200 import api
    g = api.global_opts(**region)
    dims, n_hyp, _ = api.localize_global_size(g)
    ctx = api.Context(max_map_points=len(map_xyzi) + (1 << 18), max_scan_points=262144, plane_res=case["cfg"]["plane_res"], max_batch=16)
    ctx.map_set_points(map_xyzi)
    scan, truth = case["scan_xyzi"], case["pose_true"]
    for _ in range(warmup):
        ctx.localize_global(scan, center, 20, g)
    wall, st = [], {k: [] for k in ("raster", "dilate", "score", "refine")}
    for _ in range(calls):
        t0 = time.perf_counter()
        pose, res, cands = ctx.localize_global(scan, center, 20, g)      # returns after a device synchronise
        wall.append((time.perf_counter() - t0) * 1e3)
        for k in st:
            st[k].append(getattr(res, f"time_{k}_ms"))
    ctx.profile_get(6, reset=True)
    ctx.profile_enable(True)
    ctx.localize_global(scan, center, 20, g)
    ctx.profile_enable(False)
    prof_ms, prof_n = ctx.profile_get(6, reset=True)
    _, _, _, bst = ctx.localize_global_bnb(scan, center, 20, g)
    ctx.close()
    ns = sorted((c.n_success for c in cands if c.status == 0), reverse=True)
    return {"workload": f"{len(map_xyzi)}-point map, scan of {len(scan)} pts, search {dims} = {n_hyp} hypotheses x "
                        f"{res.n_score_points} score points",
            "calls": calls, "warmup": warmup,
            "wall_ms_median": float(np.median(wall)), "wall_ms_min": float(np.min(wall)), "wall_ms_max": float(np.max(wall)),
            "stage_ms_median": {k: float(np.median(v)) for k, v in st.items()},
            "profile_class6_ms": prof_ms, "profile_class6_launches": prof_n,
            "leaf_fraction": bst.leaves_scored / n_hyp, "stats": _stats(bst),
            "status": res.status, "n_candidates": res.n_candidates, "best_score": res.best_score,
            "winner_success": ns[0] if ns else 0, "runner_up_success": ns[1] if len(ns) > 1 else 0,
            "err_m": float(np.linalg.norm(pose[:3] - truth[:3])),
            "err_deg": math.degrees(2.0 * math.acos(min(1.0, abs(float(np.dot(pose[3:], truth[3:]))))))}


def _stats(st):
    L = st.lmax
    return {"lmax": L, "root_nodes": st.root_nodes, "scored": list(st.scored)[:L + 1], "discarded": list(st.discarded)[:L + 1],
            "leaves_scored": st.leaves_scored, "steps": st.steps, "kstar_score": st.kstar_score, "pyramid_bytes": st.pyramid_bytes,
            "build_ms": st.time_build_ms, "search_ms": st.time_search_ms}


def whole_map(ctx, label, case, calls, warmup):
    """so_localize_global_bnb over the whole map from its centre (true z, seeded yaw), 0.25 m and 2 deg."""
    from superodom_b200 import api
    truth = case["pose_true"]
    lo, hi, n_map = ctx.map_bounds()
    yaw = np.random.default_rng(9100).uniform(-math.pi, math.pi)
    center = np.r_[0.5 * (float(lo[0]) + float(hi[0])), 0.5 * (float(lo[1]) + float(hi[1])), truth[2],
                   0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2)]
    g = api.whole_map_opts(lo, hi, center, yaw_half=math.pi)
    for _ in range(warmup):
        ctx.localize_global_bnb(case["scan_xyzi"], center, 20, g)
    wall, search = [], []
    for _ in range(calls):
        t0 = time.perf_counter()
        pose, res, cands, st = ctx.localize_global_bnb(case["scan_xyzi"], center, 20, g)
        wall.append((time.perf_counter() - t0) * 1e3)
        search.append(st.time_build_ms + st.time_search_ms)
    return {"workload": f"{label}: whole-map search {g.half_x:.2f} x {g.half_y:.2f} m half-extents = {res.n_hypotheses} hypotheses x "
                        f"{res.n_score_points} score points", "calls": calls,
            "wall_ms_median": float(np.median(wall)), "wall_ms_range": [float(np.min(wall)), float(np.max(wall))],
            "bnb_ms_median": float(np.median(search)), "bnb_ms_range": [float(np.min(search)), float(np.max(search))],
            "leaf_fraction": st.leaves_scored / res.n_hypotheses, "stats": _stats(st),
            "status": res.status, "best_score": res.best_score, "n_candidates": res.n_candidates,
            "true_offset_m": float(np.linalg.norm(center[:2] - truth[:2])),
            "err_m": float(np.linalg.norm(pose[:3] - truth[:3])),
            "err_deg": math.degrees(2.0 * math.acos(min(1.0, abs(float(np.dot(pose[3:], truth[3:]))))))}


def three_rooms():
    """Three cfg2-sized rooms at x = -800, 0, +800 m (synth.make_map with the block filter's grid on each room): scenes and the
    whole cloud."""
    from superodom_b200 import synth
    scenes, maps = [], []
    for k, x in enumerate((-800.0, 0.0, 800.0)):
        sc = synth.make_scene(52.0, seed=611 + k, center=(x, 0.0))
        raw = synth.sample_surfaces(sc, 0.2, seed=1234)
        xyzi = np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1)
        scenes.append(sc)
        maps.append(synth.voxel_filter_blocks(xyzi, 0.2, origin=(10 - int(round(x / 50.0)), 10, 5)))
    return scenes, np.ascontiguousarray(np.concatenate(maps), np.float32)


def archive_cases(calls, warmup):
    """Whole-map search over the three rooms, window in room A (so_map_set_origin, the load, so_map_shift there).  Before every call
    the window is put back in room A and rebuilt (untimed), so each call starts from the same state."""
    from superodom_b200 import api, synth
    scenes, cloud = three_rooms()
    cap = 1 << 22
    ctx = api.Context(max_map_points=cap, max_scan_points=262144, plane_res=0.2, max_batch=16)
    ctx.map_archive(cap)
    ctx.map_set_origin([-800.0, 0.0, 0.0])
    ctx.map_set_points(cloud)
    ctx.map_shift([-800.0, 0.0, 0.0])
    o0 = [int(v) for v in ctx.map_origin()]
    lo, hi, n_map = ctx.map_bounds_all()
    out = []
    for room, label in ((2, "room C: the window moves"), (0, "room A: no move")):
        truth = synth.random_sensor_pose(scenes[room], 900 + 10 * room, 20.0)
        scan = synth.make_scan(scenes[room], "os1_128", truth, 1000 + 10 * room)
        yaw = np.random.default_rng(9300 + room).uniform(-math.pi, math.pi)
        center = np.r_[0.5 * (float(lo[0]) + float(hi[0])), 0.5 * (float(lo[1]) + float(hi[1])), truth[2], 0.0, 0.0,
                       math.sin(yaw / 2), math.cos(yaw / 2)]
        g = api.whole_map_opts(lo, hi, center, yaw_half=math.pi, whole_map=True)
        rec = {k: [] for k in ("build", "search", "refine", "wall")}
        for it in range(warmup + calls):
            ctx.map_set_origin([-50.0 * v for v in o0])
            ctx.map_counts_5x5([10, 10, 5])                               # applies the origin change outside the timed call
            t0 = time.perf_counter()
            pose, res, cands, st = ctx.localize_global_bnb(scan, center, 20, g)
            wall = (time.perf_counter() - t0) * 1e3
            if it >= warmup:
                for k, v in (("build", st.time_build_ms), ("search", st.time_search_ms), ("refine", res.time_refine_ms), ("wall", wall)):
                    rec[k].append(v)
        out.append({"workload": f"three-room map ({n_map} pts, {hi[0] - lo[0]:.0f} m x {hi[1] - lo[1]:.0f} m), whole-map search "
                                f"{res.n_hypotheses} hypotheses x {res.n_score_points} score points, scan in {label}",
                    "calls": calls, "build_device_ms_median": float(np.median(rec["build"])),
                    "traversal_device_ms_median": float(np.median(rec["search"])),
                    "refine_wall_ms_median": float(np.median(rec["refine"])), "wall_ms_median": float(np.median(rec["wall"])),
                    "wall_ms_range": [float(np.min(rec["wall"])), float(np.max(rec["wall"]))],
                    "n_windows": res.n_windows, "n_candidates": res.n_candidates, "status": res.status,
                    "err_m": float(np.linalg.norm(pose[:3] - truth[:3])),
                    "err_deg": math.degrees(2.0 * math.acos(min(1.0, abs(float(np.dot(pose[3:], truth[3:])))))),
                    "best_ranked_err_m": float(np.linalg.norm(np.array(cands[0].pose[:3]) - truth[:3]))})
    ctx.close()
    return out


if __name__ == "__main__":
    main()

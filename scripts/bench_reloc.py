#!/usr/bin/env python3
"""bench_reloc.py -- global localization (so_localize_global) on the cfg2 map (1 M points) with one OS1-128 scan and the default
search: half 10 m in x and y at 0.25 m, the full circle at 2 deg = 81 x 81 x 180 = 1 180 980 hypotheses x 1024 score points.

Prints one JSON line: median whole-call wall time over --calls calls after --warmup calls, the per-stage device times (CUDA events
in the call; profile class 6 from one extra profiled call), hypotheses/s and bitmap lookups/s of the scoring kernel, the bitmap
size, the recovery error against the truth, and the card name and power limit read in the same run.  --cpu adds one single-thread
run of the numpy restatement of the search (tests/global_localization_numpy.py) for a speed-up figure.  Writes nothing.

--bnb adds so_localize_global_bnb on the same search, timed in alternation with the exhaustive call (whole call and search stage).
--whole-map adds branch-and-bound searches over whole maps: the cfg2 map (0.25 m, 2 deg, centre at the map centre with the true z
and a seeded yaw) and a 300 m x 300 m synthetic map (synth.make_map(150.0, 0.2)), each with its per-level statistics, the share of
hypotheses whose leaves were scored and the recovery error.  Either flag prints one more JSON line per workload.
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
    ap.add_argument("--scan", type=int, default=0, help="cfg2 scan index")
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--bnb", action="store_true", help="also time so_localize_global_bnb against the exhaustive call")
    ap.add_argument("--whole-map", action="store_true", help="also run branch-and-bound searches over the whole cfg2 and 300 m maps")
    ap.add_argument("--archive", action="store_true", help="also run whole-map searches over a 1.7 km three-room map in the block archive")
    a = ap.parse_args()
    from superodom_b200 import api, synth
    import global_localization_numpy as GN
    scene, map_xyzi = synth.make_map_for("cfg2")
    case = synth.make_case_on(scene, map_xyzi, "cfg2", a.scan)
    truth = case["pose_true"]
    rng = np.random.default_rng(7100 + a.scan)
    d = rng.uniform(-8.0, 8.0, 2)
    dyaw = rng.uniform(-math.pi, math.pi)
    q = synth.quat_mul(np.array([0.0, 0.0, math.sin(dyaw / 2), math.cos(dyaw / 2)]), truth[3:])
    center = np.r_[truth[0] + d[0], truth[1] + d[1], truth[2], q / np.linalg.norm(q)]
    region = dict(half_x=10.0, half_y=10.0, yaw_half=math.pi)
    g = api.global_opts(**region)
    dims, n_hyp, bitmap_bytes = api.localize_global_size(g)
    ctx = api.Context(max_map_points=len(map_xyzi) + (1 << 18), max_scan_points=262144, plane_res=0.2, max_batch=16)
    ctx.map_set_points(map_xyzi)
    scan = case["scan_xyzi"]
    for _ in range(a.warmup):
        ctx.localize_global(scan, center, 20, g)
    wall, st = [], {k: [] for k in ("raster", "dilate", "score", "sort", "refine")}
    for _ in range(a.calls):
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
    med = {k: float(np.median(v)) for k, v in st.items()}
    ns = sorted((c.n_success for c in cands if c.status == 0), reverse=True)
    name, limit = card()
    out = {
        "workload": f"cfg2 map ({len(map_xyzi)} pts), OS1-128 scan {a.scan} ({len(scan)} pts), centre {np.linalg.norm(d):.2f} m / "
                    f"{math.degrees(dyaw):.1f} deg off, default search {dims} = {n_hyp} hypotheses x {res.n_score_points} score points",
        "card": name, "power_limit_w": limit,
        "calls": a.calls, "warmup": a.warmup,
        "wall_ms_median": float(np.median(wall)), "wall_ms_min": float(np.min(wall)), "wall_ms_max": float(np.max(wall)),
        "stage_ms_median": med,
        "profile_class6_ms": prof_ms, "profile_class6_launches": prof_n,
        "hypotheses_per_s": n_hyp / (med["score"] * 1e-3),
        "lookups_per_s": n_hyp * res.n_score_points / (med["score"] * 1e-3),
        "bitmap_bytes": bitmap_bytes,
        "status": res.status, "n_candidates": res.n_candidates, "best_score": res.best_score,
        "winner_success": ns[0] if ns else 0, "runner_up_success": ns[1] if len(ns) > 1 else 0,
        "err_m": float(np.linalg.norm(pose[:3] - truth[:3])),
        "err_deg": math.degrees(2.0 * math.acos(min(1.0, abs(float(np.dot(pose[3:], truth[3:])))))),
    }
    if a.cpu:
        t0 = time.perf_counter()
        GN.localize_scores_numpy(scan, center, ctx.map_download(0)[:, :3], **region)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        out["cpu_numpy_search_ms"] = cpu_ms
        out["speedup_search_vs_cpu"] = cpu_ms / (med["raster"] + med["dilate"] + med["score"] + med["sort"])
    if a.bnb:
        bnb_out = bnb_vs_exhaustive(ctx, scan, center, truth, g, a.calls, a.warmup)
    ctx.close()
    print(json.dumps(out))
    if a.bnb:
        print(json.dumps(dict(bnb_out, card=name, power_limit_w=limit)))
    if a.whole_map:
        ctx = api.Context(max_map_points=len(map_xyzi) + (1 << 18), max_scan_points=262144, plane_res=0.2, max_batch=16)
        ctx.map_set_points(map_xyzi)
        print(json.dumps(dict(whole_map(ctx, "cfg2 map", case, a.calls, a.warmup, out["hypotheses_per_s"]), card=name, power_limit_w=limit)))
        ctx.close()
        t0 = time.perf_counter()
        scene3, map3 = synth.make_map(150.0, 0.2)
        gen_s = time.perf_counter() - t0
        case3 = synth.make_case_on(scene3, map3, "cfg2", a.scan)
        ctx = api.Context(max_map_points=len(map3) + (1 << 18), max_scan_points=262144, plane_res=0.2, max_batch=16)
        ctx.map_set_points(map3)
        r = whole_map(ctx, f"300 m x 300 m synthetic map ({len(map3)} pts, generated in {gen_s:.1f} s)", case3, max(3, a.calls // 4), 1, out["hypotheses_per_s"])
        print(json.dumps(dict(r, card=name, power_limit_w=limit)))
        ctx.close()
    if a.archive:
        for r in archive_cases(a.calls, a.warmup):
            print(json.dumps(dict(r, card=name, power_limit_w=limit)))


def _stats(st):
    L = st.lmax
    return {"lmax": L, "root_nodes": st.root_nodes, "scored": list(st.scored)[:L + 1], "discarded": list(st.discarded)[:L + 1],
            "leaves_scored": st.leaves_scored, "steps": st.steps, "kstar_score": st.kstar_score, "pyramid_bytes": st.pyramid_bytes,
            "build_ms": st.time_build_ms, "search_ms": st.time_search_ms}


def bnb_vs_exhaustive(ctx, scan, center, truth, g, calls, warmup):
    """The default search both ways, alternating call by call; the two results must be bit-identical apart from timings."""
    for _ in range(warmup):
        ctx.localize_global(scan, center, 20, g)
        ctx.localize_global_bnb(scan, center, 20, g)
    wall = {"exhaustive": [], "bnb": []}
    search = {"exhaustive": [], "bnb": []}
    same = True
    for _ in range(calls):
        t0 = time.perf_counter()
        pose, res, _ = ctx.localize_global(scan, center, 20, g)
        wall["exhaustive"].append((time.perf_counter() - t0) * 1e3)
        search["exhaustive"].append(res.time_raster_ms + res.time_dilate_ms + res.time_score_ms + res.time_sort_ms)
        t0 = time.perf_counter()
        pose_b, res_b, _, st = ctx.localize_global_bnb(scan, center, 20, g)
        wall["bnb"].append((time.perf_counter() - t0) * 1e3)
        search["bnb"].append(res_b.time_raster_ms + res_b.time_dilate_ms + res_b.time_score_ms)
        same &= bool(np.array_equal(pose, pose_b)) and res.winner == res_b.winner and res.best_score == res_b.best_score
    return {"workload": "default cfg2 search, exhaustive vs branch-and-bound, alternating", "calls": calls,
            "wall_ms_median": {k: float(np.median(v)) for k, v in wall.items()},
            "wall_ms_range": {k: [float(np.min(v)), float(np.max(v))] for k, v in wall.items()},
            "search_ms_median": {k: float(np.median(v)) for k, v in search.items()},
            "search_ms_range": {k: [float(np.min(v)), float(np.max(v))] for k, v in search.items()},
            "same_result": same, "n_hypotheses": res.n_hypotheses, "leaf_fraction": st.leaves_scored / res.n_hypotheses,
            "stats": _stats(st)}


def whole_map(ctx, label, case, calls, warmup, exhaustive_rate):
    """Branch-and-bound over the whole map from its centre (true z, seeded yaw), 0.25 m and 2 deg.  exhaustive_rate: hypotheses/s of
    the exhaustive scoring kernel in this run, for the time an exhaustive search of the same region would take if it were allowed."""
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
            "exhaustive_rate_equivalent_ms": res.n_hypotheses / exhaustive_rate * 1e3,
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

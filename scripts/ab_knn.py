"""A/B harness for k-NN kernel variants (run under gpurun; pick the library with SO_LIB_PATH, label the line with TAG).

    SO_LIB_PATH=superodom_b200/lib_variant.so TAG=variant python scripts/ab_knn.py [B] [--parity] [--cfg5]

Prints one line: per-launch times of the k-NN / fit / evaluate kernel classes on a B-scan cfg2 batch (profiling mode: CUDA events
around every launch that has work), the unprofiled step time, optionally the cfg5 microbench times and a quick parity check
against the oracle (neighbour ids / d2 bit-equal, registration pose equal) -- a variant that is fast but wrong is not a result.
"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from superodom_b200 import api, synth  # noqa: E402

args = [a for a in sys.argv[1:] if not a.startswith("--")]
B = int(args[0]) if args else 16
out = {"tag": os.environ.get("TAG", ""), "lib": os.path.basename(api.LIB_PATH), "B": B}
map_xyzi, scans, priors, truths = bench.make_inputs(0, B)
n_points = np.array([len(s) for s in scans], np.uint32)
flat = np.ascontiguousarray(np.concatenate(scans, 0))
ctx = api.Context(max_map_points=len(map_xyzi) + 1024, max_scan_points=int(n_points.max()), max_batch=B, plane_res=0.2)
ctx.map_set_points(map_xyzi)
for _ in range(3):
    res = ctx.register_batch(flat, n_points, priors, 20, 0, skip_map_checks=True)
t = time.perf_counter()
for _ in range(5):
    res = ctx.register_batch(flat, n_points, priors, 20, 0, skip_map_checks=True)
out["step_ms"] = (time.perf_counter() - t) / 5 * 1e3
out["scans_per_s_e2e"] = B / out["step_ms"] * 1e3
ctx.profile_enable(True)
for k in range(6):
    ctx.profile_get(k, reset=True)
res = ctx.register_batch(flat, n_points, priors, 20, 0, skip_map_checks=True)
ctx.profile_enable(False)
names = {0: "knn", 5: "fit", 4: "first_eval", 1: "evaluate", 3: "scan_order"}
for k, nm in names.items():
    ms, n = ctx.profile_get(k)
    out[nm + "_ms_per_launch"] = ms / max(n, 1)
    out[nm + "_launches"] = int(n)
out["err_vs_truth"] = float(np.abs(np.array([list(r.pose) for r in res])[:, :3] - truths[:, :3]).max())
out["icp_iters_mean"] = float(np.mean([r.n_iterations for r in res]))
ctx.close()

if "--parity" in sys.argv:
    from oracle import oracle as O
    par = {}
    for name in ("tiny", "cfg1"):
        c = synth.make_case(name)
        cx = api.Context(max_map_points=max(1 << 20, len(c["map_xyzi"]) + 1024), max_scan_points=262144, plane_res=0.2)
        cx.map_set_points(c["map_xyzi"])
        om = O.OracleMap(c["map_xyzi"], ref_octree=False)
        rng = np.random.default_rng(0)
        base = c["map_xyzi"][::5, :3]
        q = base + rng.normal(0, 0.12, size=base.shape).astype(np.float32)
        gi, gd = cx.knn(q, 5, 0.0)
        oi, od, of = om.knn(q, 5, 0)
        g = gi.astype(np.int64)
        g[gi == 0xFFFFFFFF] = -1
        par[name + "_knn_exact"] = bool(np.array_equal(g[of], oi[of]) and np.array_equal(gd[of], od[of]))
        bound = np.float32(3 * np.float32(0.2))
        gi, gd = cx.knn(q, 5, float(bound))
        g = gi.astype(np.int64)
        g[gi == 0xFFFFFFFF] = -1
        keep = (od <= bound) & of[:, None]
        par[name + "_knn_bounded"] = bool(np.array_equal(g[keep], oi[keep]) and (gi[~keep] == 0xFFFFFFFF).all())
        gc, gho, ghr = cx.correspond(c["scan_xyzi"], c["pose_prior"], 0)
        oc, oho, ohr = om.correspond(c["scan_xyzi"], c["pose_prior"], 0.2, 0, 0, n_threads=8)
        ok = oc["status"] == 0
        par[name + "_corr"] = bool(np.array_equal(gc["status"].astype(np.int64), np.where(oc["status"] < 0, 255, oc["status"])) and
                                   np.array_equal(gc["nn"][ok].astype(np.int64), oc["nn"][ok]) and np.array_equal(gho, oho))
        r = cx.register(c["scan_xyzi"], c["pose_prior"], 5, 0)
        ro = om.register(c["scan_xyzi"], c["pose_prior"], 0.2, 5, 0, knn_mode=0, n_threads=8)
        par[name + "_pose"] = bool(np.abs(np.array(r.pose) - np.array(ro.pose)).max() < 1e-9 and r.n_iterations == ro.n_iterations and
                                   list(r.hist_reject_plane) == list(ro.hist_reject_plane))
        cx.close()
    out["parity"] = par
    out["parity_all"] = all(par.values())

if "--cfg5" in sys.argv:
    import torch
    cache = "/tmp/superodom_b200_bench_inputs/cfg5_map.npy"
    kctx = None
    if os.path.exists(cache):
        map5 = np.load(cache)
    else:
        scene = synth.make_scene(58.0, seed=77)
        raw = synth.sample_surfaces(scene, 0.1, seed=1234)
        kctx = api.Context(max_map_points=len(raw) + 1024, max_scan_points=1024, plane_res=0.1)
        kctx.map_add_surf(np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1))
        map5 = kctx.map_download(0)
        kctx.close()
        os.makedirs(os.path.dirname(cache), exist_ok=True)
        np.save(cache, map5)
    kctx = api.Context(max_map_points=len(map5) + 1024, max_scan_points=1024, plane_res=0.1)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    kctx.set_stream(stream.cuda_stream)
    kctx.map_set_points(map5)
    NQ = 10_000_000
    q4 = bench.cfg5_queries(map5, 0, NQ)
    dq = torch.from_numpy(q4).cuda()
    didx = torch.empty((NQ, 5), dtype=torch.int32, device="cuda")
    dd2 = torch.empty((NQ, 5), dtype=torch.float32, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for name, bound in (("cfg5_bounded_ms", float(np.float32(3 * np.float32(0.1)))), ("cfg5_exact_ms", 0.0)):
        ts = []
        for it in range(6):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            kctx.knn_device(dq.data_ptr(), NQ, 5, bound, didx.data_ptr(), dd2.data_ptr())
            e1.record()
            torch.cuda.synchronize()
            if it >= 2:
                ts.append(e0.elapsed_time(e1))
        out[name] = float(np.median(ts))
    out["cfg5_checksum"] = int(didx.to(torch.int64).sum().item())          # equal across variants = same neighbours
    kctx.close()
print(json.dumps(out), flush=True)

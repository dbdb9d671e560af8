"""BASELINE cfg5: k-NN microbench -- 10 M queries, k=5, vs a 5 M-point map; HBM GB/s against the measured peak.

Queries = map points + N(0,(0.1 m)^2) (seed 3000), in map order (block / voxel order, i.e. spatially coherent, as a
scan is).  Reports the radius-bounded (sqrt(3*0.1)) and the exact unbounded variant, each with device-resident
queries/results (CUDA events around so_knn_device, L2 flushed between iterations), plus -- with --cpu -- the CPU
comparators on a bounded sample: the reference's own octree (oracle/_ref, verbatim) and scipy cKDTree (the exact
kd-tree stand-in for pcl::KdTreeFLANN, SURVEY 8d).

    python tests/tools/bench_knn.py [--cpu]                 # 1 GPU
    torchrun --nproc-per-node N tests/tools/bench_knn.py    # queries split over N GPUs, map replicated
"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

import bench  # noqa: E402
from superodom_b200 import api, synth  # noqa: E402

NQ = 10_000_000
rank = int(os.environ.get("RANK", "0"))
world = int(os.environ.get("WORLD_SIZE", "1"))
local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
t0 = time.time()
scene, map_xyzi = synth.make_map(58.0, 0.1)              # leaf 0.1, ~5 M points over 9 blocks
M = len(map_xyzi)
rng = np.random.default_rng(3000)
reps = (NQ + M - 1) // M
q = np.concatenate([map_xyzi[:, :3] + rng.normal(0, 0.1, size=(M, 3)).astype(np.float32) for _ in range(reps)], 0)[:NQ]
if world > 1:
    per = (NQ + world - 1) // world                      # queries split evenly (contiguous), map replicated (SURVEY 8e)
    q = q[rank * per:(rank + 1) * per]
nq = len(q)
q4 = np.concatenate([q, np.zeros((nq, 1), np.float32)], 1)
print(f"[rank {rank}] map {M} pts, {nq} queries, gen {time.time() - t0:.1f}s", file=sys.stderr)
ctx = api.Context(device=local, max_map_points=M + 1024, max_scan_points=1024, plane_res=0.1)
stream = torch.cuda.Stream()                           # a real (non-legacy) stream shared by torch events and the library
torch.cuda.set_stream(stream)
ctx.set_stream(stream.cuda_stream)
ctx.map_set_points(map_xyzi)
dq = torch.from_numpy(q4).cuda()
didx = torch.empty((nq, 5), dtype=torch.int32, device="cuda")
dd2 = torch.empty((nq, 5), dtype=torch.float32, device="cuda")
peak = bench._peaks()[0]
try:
    peak = float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass
out = {"config": "cfg5", "map_points": M, "queries": NQ, "k": 5, "n_gpus": world, "peak_gbs_per_gpu": peak}
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for name, bound in (("bounded", float(np.float32(3 * np.float32(0.1)))), ("exact", 0.0)):
    times = []
    for it in range(8):
        flush.zero_()                                    # L2 flush between timed iterations
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        ctx.knn_device(dq.data_ptr(), nq, 5, bound, didx.data_ptr(), dd2.data_ptr())
        e1.record()
        torch.cuda.synchronize()
        if it >= 3:
            times.append(e0.elapsed_time(e1))
    ms = float(np.median(times))
    if world > 1:
        t = torch.tensor([ms], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    # algorithmic bytes (SURVEY 8d): 16 B query + k*8 B result per query + the map streamed once per GPU
    alg = NQ * (16 + 5 * 8) + world * 16 * M
    out[name] = {"ms": ms, "Mqueries_per_s": NQ / ms / 1e3, "algorithmic_GB": alg / 1e9, "achieved_GBps": alg / ms / 1e6,
                 "frac_of_peak": alg / ms / 1e6 / (peak * world), "found5_frac_rank0": float((didx[:, 4] != -1).float().mean().item())}
if rank == 0 and "--cpu" in sys.argv:
    from oracle import oracle as O
    ns = 200_000
    om = O.OracleMap(map_xyzi)
    mode = 2 if O.has_ref_octree() else 0
    t = time.time()
    oi, od, of = om.knn(q[:ns], 5, mode)
    dt = time.time() - t
    out["cpu_reference_octree_1thread"] = {"Mqueries_per_s": ns / dt / 1e6, "sample": ns, "verbatim_reference_header": bool(O.has_ref_octree())}
    gi = didx[:ns].cpu().numpy().astype(np.int64)       # last GPU pass was the exact variant
    oi0, od0, _ = om.knn(q[:ns], 5, 0)
    out["gpu_exact_equals_oracle_exact"] = bool(np.array_equal(gi, oi0))
    out["octree_vs_exact_mismatch_queries"] = int((np.sort(oi, 1) != np.sort(oi0, 1)).any(1).sum())
    from scipy.spatial import cKDTree
    t = time.time()
    tree = cKDTree(map_xyzi[:, :3])
    tb = time.time() - t
    t = time.time()
    tree.query(q[:2_000_000], k=5, workers=-1)
    dt = time.time() - t
    out["cpu_scipy_ckdtree_allcores"] = {"Mqueries_per_s": 2.0 / dt, "build_s": tb, "cores": os.cpu_count()}
if rank == 0:
    print(json.dumps(out))
if world > 1:
    dist.destroy_process_group()

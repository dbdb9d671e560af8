"""Achieved bandwidth of the solve's evaluation passes at the bench shape (DESIGN.md sections 4 and 6).

  python scripts/bench_corr_stream.py [--batch 256] [--rounds 3] [--bytes-per-point 44]

One device-resident registration call of --batch cfg2 scans (the scans bench.py's timed step starts with), profiled launch by
launch (profile_enable): profile class 4 is the first evaluation of each solve (k_evaluate<PH_CORR> + k_lm_step), class 1 one LM
evaluation (k_evaluate<PH_EVAL> + k_lm_step).  The points a class evaluated are counted from the scans' own results: every ICP
iteration of a scan opens one solve (class 4 reads all its points once) and each LM step of that solve is one class 1 pass.  An
invalid LM step (rare) is counted although it evaluates nothing, so the class 1 rate is an upper bound.  The rate is the stream's
bytes (--bytes-per-point per evaluated point) over the class time, which includes the short k_lm_step: a lower bound on the
evaluation kernel's own rate.  SO_LIB_PATH selects the library (A/B runs).  Prints one JSON line per round; the card and its
power limit are printed first and belong beside every number."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from superodom_b200 import api  # noqa: E402

HBM_GBPS = 3350.0                 # H100 SXM data sheet (HBM3), 700 W card


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bytes-per-point", type=int, default=44, help="correspondence-stream bytes one evaluation reads per point")
    args = ap.parse_args()
    import torch
    import bench                                                    # the bench's seeded inputs and its input cache
    print(json.dumps({"card": card(), "library": api.LIB_PATH}), flush=True)
    map_xyzi, scans, priors, _ = bench.make_inputs(0, args.batch)
    n_points = np.array([len(s) for s in scans], np.uint32)
    ctx = api.Context(max_map_points=len(map_xyzi) + 1024, max_scan_points=int(n_points.max()), max_batch=args.batch, plane_res=0.2)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    ctx.map_set_points(map_xyzi)
    d_scans = torch.from_numpy(np.ascontiguousarray(np.concatenate(scans, 0))).cuda()

    def call():
        return ctx.register_batch_device(d_scans.data_ptr(), n_points, priors, 20, 0, skip_map_checks=True)

    for _ in range(2):
        call()
    torch.cuda.synchronize()
    for rnd in range(args.rounds):
        ctx.profile_enable(True)
        for k in (1, 4):
            ctx.profile_get(k, reset=True)
        res = call()
        ctx.profile_enable(False)
        row = {"round": rnd}
        pts4 = sum(int(n) * int(r.n_iterations) for r, n in zip(res, n_points))
        pts1 = sum(int(n) * sum(int(r.iter_lm_steps[i]) for i in range(r.n_iterations)) for r, n in zip(res, n_points))
        for cls, pts in ((4, pts4), (1, pts1)):
            ms, n = ctx.profile_get(cls)
            gbps = pts * args.bytes_per_point / (ms * 1e-3) / 1e9 if ms > 0 else 0.0
            row[f"class{cls}"] = {"launches": int(n), "ms_per_launch": ms / max(n, 1), "points_per_launch": pts / max(n, 1),
                                  "GBps": gbps, "share_of_hbm_peak": gbps / HBM_GBPS}
        row["bytes_per_point"] = args.bytes_per_point
        print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

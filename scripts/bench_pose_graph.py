"""Time so_pose_graph_solve on seeded drifted trajectories, beside the CPU time of the exact-step restatement on the same host.

  python scripts/bench_pose_graph.py [--reps R] [--out FILE] [--no-cpu]

Graphs: a random walk of n keyframes (n = 1 000 and 10 000) with odometry edges between consecutive keyframes, the start chained
from the odometry with drift, and L loop edges (L = 10, 100, 1 000) between random non-adjacent keyframes measured from the truth; one
in ten loop edges is false (a wrong Z between unrelated keyframes) and every loop edge is Cauchy-weighted (c = 1).  Per graph: device
time (CUDA events, so_pose_graph_result.time_ms) and wall time of one solve (median of R), trust-region and PCG iterations, and the
CPU time of tests/pose_graph_numpy.solve_sparse (the restatement's rules with a sparse direct solve; not GTSAM, which is not
available).  The card's name and power limit are read in the same run."""
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

import pose_graph_numpy as PG  # noqa: E402
from superodom_b200 import api  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             check=True).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        return "unknown", "unknown"


def graph(n, loops, seed):
    rng = np.random.default_rng(seed)
    n_false = loops // 10
    init, edges, truth = PG.drifted(rng, n, loops=loops - n_false, false_loops=n_false, cauchy=1.0, drift=(0.03, 0.004))
    return init, PG.to_array(edges)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    name, power = card()
    print(json.dumps(dict(card=name, power_limit=power)), flush=True)
    ctx = api.Context(max_map_points=1 << 16, max_scan_points=1 << 12)
    rows = []
    for n in (1000, 10000):
        for loops in (10, 100, 1000):
            init, E = graph(n, loops, seed=n + loops)
            ctx.pose_graph_solve(init, E)                                  # warm-up: allocation and module load
            dev, wall = [], []
            for _ in range(a.reps):
                t = time.perf_counter()
                X, r = ctx.pose_graph_solve(init, E)
                wall.append((time.perf_counter() - t) * 1e3)
                dev.append(r["time_ms"])
            row = dict(n=n, edges=len(E), loops=loops, device_ms=float(np.median(dev)), wall_ms=float(np.median(wall)),
                       iterations=r["iterations"], pcg_iterations=int(r["pcg_iterations"]), termination=r["termination"],
                       initial_cost=r["initial_cost"], final_cost=r["final_cost"])
            if not a.no_cpu:
                prob = PG.PoseGraph(init, E)
                t = time.perf_counter()
                ref = PG.solve_sparse(prob, prob.x0(), 50)
                row["restatement_cpu_ms"] = (time.perf_counter() - t) * 1e3
                row["restatement_iterations"] = ref["iterations"]
                row["max_pose_diff_vs_restatement"] = float(np.abs(X - prob.nodes(ref["x"])).max())
            rows.append(row)
            print(json.dumps(row), flush=True)
    ctx.close()
    res = dict(card=name, power_limit=power, rows=rows)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

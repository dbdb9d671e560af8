"""Device time per registration and pose error of the edge / compensation arms on moving OS1-128 corridor scans taken through
extraction: (a) edges without compensation (so_register), (b) planes with APPROXIMATED (so_register_undistort), (c) edges with
APPROXIMATED (so_register_undistort_edges), (d) edges with OPTIMIZED (so_register_optimized_edges).  Reads the card name and power limit in the same run.  Prints one JSON line.

    python scripts/bench_edges_undistort.py [--scans 6] [--repeat 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=6)
    ap.add_argument("--repeat", type=int, default=20)
    a = ap.parse_args()
    from superodom_b200 import api
    # the corridor setup and the four arms are the accuracy test's (tests/test_undistortion_edges.py), as scripts/bench_edges.py reuses
    # tests/test_edge_features.corridor_runs; the device times are the median over --repeat registrations of the run's last scan
    from test_undistortion_edges import corridor_arms
    rows, timing = corridor_arms(api, n_scans=a.scans, timing_repeat=a.repeat)
    summ = {k: dict(err_max=max(r["err_" + k] for r in rows), err_median=float(np.median([r["err_" + k] for r in rows])))
            for k in ("a", "b", "c", "d")}
    print(json.dumps(dict(card=card(), time=timing, accuracy=summ, rows=rows)))


if __name__ == "__main__":
    main()

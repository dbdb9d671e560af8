"""Time so_scan_prefilter of two builds of the library in one process, alternating call by call.

    python scripts/bench_prefilter.py A.so B.so [--calls 200]

Scans: the cfg1 VLP-16 scan (28 800 points) and the cfg2 OS1-128 scan (131 072 points) at leaf 0.2, the filtered cloud left on the
device (download=False, as the live loop calls it).  Per call: host wall time around the call, which ends in a stream
synchronise.  Prints one JSON line: per scan and library the median and quartiles in ms, whether the two builds' filtered clouds
are bit-equal, and the GPU's name and power limit."""
import importlib.util
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def load_api(lib, tag):
    os.environ["SO_LIB_PATH"] = os.path.abspath(lib)
    spec = importlib.util.spec_from_file_location(f"so_api_{tag}", os.path.join(ROOT, "superodom_b200", "api.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.load_library()
    return mod


def main():
    libs = [a for a in sys.argv[1:] if a.endswith(".so")]
    calls = int(sys.argv[sys.argv.index("--calls") + 1]) if "--calls" in sys.argv else 200
    from superodom_b200 import synth
    apis = [load_api(lib, k) for k, lib in enumerate(libs)]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": gpu, "libs": [os.path.basename(x) for x in libs], "calls": calls, "scans": {}}
    for name in ("cfg1", "cfg2"):
        scan = synth.make_case(name)["scan_xyzi"]
        ctxs = [a.Context(max_map_points=1 << 20, max_scan_points=len(scan), plane_res=0.2) for a in apis]
        filtered = [c.scan_prefilter(scan, 0.1, 0.2, False)[0] for c in ctxs]
        for _ in range(20):                                             # warm-up of every build
            for c in ctxs:
                c.scan_prefilter(scan, 0.1, 0.2, False, download=False)
        t = [[] for _ in ctxs]
        for _ in range(calls):
            for k, c in enumerate(ctxs):
                t0 = time.perf_counter()
                c.scan_prefilter(scan, 0.1, 0.2, False, download=False)
                t[k].append((time.perf_counter() - t0) * 1e3)
        out["scans"][name] = {"points": len(scan), "out_points": len(filtered[0]),
                              "bit_equal": all(np.array_equal(f.view(np.uint32), filtered[0].view(np.uint32)) for f in filtered),
                              "ms": {out["libs"][k]: [float(np.percentile(x, q)) for q in (25, 50, 75)] for k, x in enumerate(t)}}
        for c in ctxs:
            c.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Build the sm_90a shared library IN-TREE: superodom_b200/libsuperodom_b200.so (C ABI, no torch types)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.environ.get("SO_LIB_OUT") or os.path.join(HERE, "libsuperodom_b200.so")
SOURCES = ["so_icp.cu", "so_map.cu", "so_scan.cu", "so_reloc.cu", "so_global.cu", "so_undistort.cu", "so_motion.cu", "so_features.cu", "so_free.cu", "so_keyframes.cu", "so_loop.cu", "so_api.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))] + [os.path.join(HERE, "..", "include", "superodom_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", os.environ.get("SO_OBJ_SUFFIX", "") + ".o"))
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, *os.environ.get("SO_NVCC_EXTRA", "").split(), "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {src}")
    # the arch flag also goes to the link step: without it nvcc adds an (empty) device-link stub for its default architecture
    subprocess.check_call([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs, "-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

"""Destroying a context returns its device memory: every buffer a context allocates, at creation or on first use of a feature, is
freed by so_destroy.

GPU: three cycles of create -> use every lazily allocating feature once -> destroy in one process; this process's device memory
after the third cycle equals that after the first (within 4 MiB).  The memory is read per process with nvidia-smi's query of the
compute apps, not from the device's free memory, which other processes on the same GPU move; the test skips when nvidia-smi does
not list this process."""
import os
import subprocess

import numpy as np
import pytest

from conftest import get_case

TOLERANCE_MIB = 4


def _own_used_mib():
    """This process's device memory in MiB as nvidia-smi reports it, or None when it is not listed."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,used_memory", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=120).stdout
    except (OSError, subprocess.SubprocessError):
        return None
    for line in out.splitlines():
        fields = [f.strip() for f in line.split(",")]
        if len(fields) == 2 and fields[0] == str(os.getpid()) and fields[1].isdigit():
            return int(fields[1])
    return None


def _cycle(api, case, rec, edge_map):
    """One context through every feature that allocates on first use, then destroyed."""
    ctx = api.Context(max_map_points=len(case["map_xyzi"]) + (1 << 18), max_scan_points=262144, plane_res=case["cfg"]["plane_res"])
    try:
        prior = case["pose_prior"]
        scan = case["scan_xyzi"]
        n = len(scan)
        ctx.map_set_points(case["map_xyzi"])
        ctx.map_set_edge_points(edge_map)
        ctx.knn_graph()                                         # the neighbour graph, then a search that queues on it
        ctx.register(scan, prior, 3)
        ctx.keyframe_reserve(4 * n, 8)
        strided = np.c_[scan[:, :4], np.zeros(n, np.float32)]  # 20-byte records, capped: pinned staging and the deferred upload
        ctx.register(strided, prior, 5, 2000)
        ids = [ctx.keyframe_add_registered(prior)]
        edges = ctx.scan_extract_edges(rec)                     # edge extraction; w = the point's time
        timed = np.c_[scan[:, :3], np.linspace(0.0, 0.1, n, dtype=np.float32)]
        ctx.register_undistort_edges(timed, edges, prior, api.undistort(prior, 0.1), 5, time_col=3)
        ids.append(ctx.keyframe_add_registered(prior))
        ctx.register_optimized_edges(timed, edges, prior, api.motion(0.1), 5, time_col=3)
        ids.append(ctx.keyframe_add_registered(prior))
        ctx.register_degeneracy(scan, prior, api.degeneracy(0.1, 0.1), 5)
        ctx.map_clear_free_space(scan, prior)
        ctx.map_archive(len(case["map_xyzi"]) + (1 << 16))
        ctx.map_shift(np.r_[1000.0, 0.0, 0.0])                  # the map's blocks leave the window for the archive ...
        ctx.map_shift(prior[:3])                                 # ... and come back
        ctx.map_from_keyframes(ctx, ids, np.tile(prior, (len(ids), 1)))
        ctx.loop_candidates([ids[-1]], 2, exclude_recent=0)
        ctx.localize_global(scan, prior, 5, api.global_opts(half_x=2.0, half_y=2.0, yaw_half=0.2))
        ctx.knn(case["map_xyzi"][:4096, :3], 5)
        ctx.knn_graph_stats(True)
        ctx.knn_graph_stats(False)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_destroy_returns_device_memory(gpu_api):
    from superodom_b200 import synth
    case = get_case("cfg1")
    rec = synth.make_ring_scan(case["scene"], "vlp16", case["pose_true"], 11)
    edge_map = synth.make_edge_map(case["scene"], 0.2)
    used = []
    for _ in range(3):
        _cycle(gpu_api, case, rec, edge_map)
        used.append(_own_used_mib())
    if used[0] is None or used[2] is None:
        pytest.skip("nvidia-smi does not list this process's device memory")
    print(f"device memory after each cycle: {used} MiB")
    assert abs(used[2] - used[0]) <= TOLERANCE_MIB, used

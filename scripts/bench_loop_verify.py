"""Loop verification costs (so_loop_verify): one call over k candidates (k = 1, 5, 16; half_window 2) on
  - the VLP-16 hall keyframes of the drifted loop (tests/test_loop_detection.py: 60 keyframes around the cfg2 hall), query 59, and
  - prefiltered OS1-128 keyframes of the cfg2 hall as scripts/bench_keyframes.py makes them (registered against the prior map), the last
    keyframe as the query.
Candidates are keyframes spread over the eligible ids.  Wall time is the median around calls (each candidate ends in a device
synchronise); device time is the kernels, copies and sets torch.profiler records in a run of its own, and events is the sum of the
results' time_ms (CUDA events from the first to the last command of each candidate on the scratch stream).  Prints one JSON line with
the card and its power limit.

    python scripts/bench_loop_verify.py [--reps 5]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from superodom_b200 import api, synth  # noqa: E402
from bench_keyframes import card, device_ms, wall_ms  # noqa: E402

VLP16 = dict(el_res_deg=2.0, el_min_deg=-16.0, el_max_deg=16.0)


def _cands(query, ids):
    c = np.zeros(len(ids), api.LOOP_CANDIDATE_DTYPE)
    c["query"], c["id"] = query, ids
    return c


def _measure(ctx, scratch, query, eligible, opts, reps):
    out = {}
    for k in (1, 5, 16):
        ids = np.linspace(0, eligible - 1, k).round().astype(np.int32)
        c = _cands(query, ids)
        ctx.loop_verify(scratch, c, opts)                              # warm-up: buffers, CUDA graphs of the registration
        res = ctx.loop_verify(scratch, c, opts)
        out[k] = dict(wall_ms=wall_ms(lambda: ctx.loop_verify(scratch, c, opts), reps),
                      device_ms=device_ms(lambda: ctx.loop_verify(scratch, c, opts)),
                      events_ms=float(sum(r.time_ms for r in res)),
                      query_points=int(res[0].n_query_points), submap_points=int(np.mean([r.n_submap_points for r in res])))
    return out


def vlp16_hall(reps):
    from test_loop_detection import _closure
    _, _, _, q, _, ctx, _ = _closure(api, False)                       # the tests' gpu_api fixture is the api module
    scratch = api.Context(max_map_points=1 << 21, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    r = _measure(ctx, scratch, q, q - 30, api.loop_verify_opts(image=VLP16, exclude_recent=30), reps)
    scratch.close()
    ctx.close()
    return r


def os1_hall(reps, n_kf=40, n_scans=8):
    scene, map_xyzi = synth.make_map_for("cfg2")
    ctx = api.Context(max_map_points=1 << 22, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    ctx.map_set_points(map_xyzi)
    ctx.keyframe_reserve(n_kf << 17, n_kf)
    for i in range(n_kf):
        c = synth.make_case_on(scene, map_xyzi, "cfg2", i % n_scans)
        ctx.scan_prefilter(c["scan_xyzi"], 0.1, 0.2, auto_voxel_size=False, download=False)
        r = ctx.register_prefiltered(c["pose_true"], 20, 0)
        ctx.keyframe_add_registered(np.array(r.pose))
    scratch = api.Context(max_map_points=1 << 22, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    q = n_kf - 1
    r = _measure(ctx, scratch, q, q, api.loop_verify_opts(id_begin=0, id_end=q), reps)
    scratch.close()
    ctx.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(dict(card=card(), vlp16_hall=vlp16_hall(a.reps), os1_128_prefiltered=os1_hall(a.reps))))


if __name__ == "__main__":
    main()

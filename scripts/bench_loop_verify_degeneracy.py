"""Degeneracy-aware loop verification (so_loop_verify_degeneracy) against plain verification (so_loop_verify):
  - time per candidate, the two calls alternating (thresholds 0.2 / 0.1), on the VLP-16 hall loop (tests/test_loop_detection.py,
    query 59, its top 5 candidates) and on the out-and-back corridor revisit (tests/loop_corridor.py), bare and with poles (there
    also without the 2 m offset);
  - sqrt(i_min / i_max) of the translation and the rotation block at the end of the alignment, for the true revisits of the hall
    (forward and reverse loop), the corridor with poles and the bare corridor: the recommended thresholds come from these ratios;
  - on each corridor revisit, per threshold: what is flagged, how far the alignment moved along the corridor, whether plain verification
    accepts, the edges' errors along the corridor, and the keyframe errors of the pose graph solved without a loop edge, with the
    plain edge and with the projected edge (so_loop_edge_information).
Prints one JSON line with the card and its power limit.

    python scripts/bench_loop_verify_degeneracy.py [--reps 10] [--thresholds 0.1,0.2,0.3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from superodom_b200 import api  # noqa: E402
from bench_keyframes import card  # noqa: E402
import loop_corridor as LC  # noqa: E402


def _scratch():
    return api.Context(max_map_points=1 << 21, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)


def _alternate(ctx, scratch, cands, opts, d, reps):
    """Median wall time per candidate (ms) of plain and degeneracy-aware verification, the two alternating call by call"""
    ctx.loop_verify(scratch, cands, opts)                              # warm-up of both
    ctx.loop_verify_degeneracy(scratch, cands, d, opts)
    n = sum(int(c["id"]) >= 0 for c in cands)
    tp, td = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        ctx.loop_verify(scratch, cands, opts)
        tp.append((time.perf_counter() - t0) * 1e3 / n)
        t0 = time.perf_counter()
        ctx.loop_verify_degeneracy(scratch, cands, d, opts)
        td.append((time.perf_counter() - t0) * 1e3 / n)
    return dict(candidates=n, plain_ms=float(np.median(tp)), degeneracy_ms=float(np.median(td)),
                plain_min_ms=float(np.min(tp)), degeneracy_min_ms=float(np.min(td)))


def hall(reps, d):
    from test_loop_detection import LOOP_OPTS, _closure
    out = {}
    for reverse in (False, True):
        _, _, _, q, _, ctx, true_near = _closure(api, reverse)
        scratch = _scratch()
        o = api.loop_verify_opts(image=LC.VLP16)
        cands = ctx.loop_candidates([q], 5, **LOOP_OPTS)[0]
        if not reverse:
            out["time"] = _alternate(ctx, scratch, cands, o, d, reps)
        one = cands[:1]                                                # the best match: the true revisit (tests/test_loop_verify.py)
        res, deg = ctx.loop_verify_degeneracy(scratch, one, api.degeneracy(0.0, 0.0, False), o)
        pr, orr = LC.ratios(deg[0])
        out["reverse" if reverse else "forward"] = dict(id=int(res[0].id), accepted=int(res[0].accepted), pos_ratio=pr, ori_ratio=orr)
        scratch.close()
        ctx.close()
    return out


def corridor(reps, poles, thresholds, d, cand=LC.CAND):
    ctx = LC.context(api, poles)
    scratch = _scratch()
    o = api.loop_verify_opts(image=LC.VLP16)
    c = LC.candidate(api, LC.QUERY, cand)
    plain = ctx.loop_verify(scratch, c, o)[0]
    res, deg = ctx.loop_verify_degeneracy(scratch, c, api.degeneracy(0.0, 0.0, False), o)
    pr, orr = LC.ratios(deg[0])
    out = dict(pos_ratio=pr, ori_ratio=orr, pos_info=list(deg[0].pos_info), ori_info=list(deg[0].ori_info),
               pos_axis0=list(deg[0].pos_axes[0:3]), plain_accepted=int(plain.accepted), plain_status=int(plain.reg.status),
               plain_overlap=plain.overlap, plain_conflict=(plain.conflict_query, plain.conflict_map),
               plain_along_error=LC.along_error(plain.rel7, cand), time=_alternate(ctx, scratch, c, o, d, reps))
    prior = ctx.loop_prior(c[0])
    out["plain_move_x"] = float(plain.reg.pose_opt[0] - prior[0])
    _, e0, _ = LC.solve(api, ctx)
    _, ep, wp = LC.solve(api, ctx, (cand, LC.QUERY, plain.rel7, LC.loop_sqrt_info()))
    S = LC.loop_sqrt_info()

    def summary(e):
        return {k: dict(mean=float(v.mean()), max=float(v.max()), query=float(v[LC.QUERY])) for k, v in e.items()}
    out["graph_no_loop"] = summary(e0)
    out["graph_plain"] = dict(summary(ep), rho1=wp)
    out["per_threshold"] = {}
    for thr in thresholds:
        r, g = ctx.loop_verify_degeneracy(scratch, c, api.degeneracy(thr, thr), o)
        r, g = r[0], g[0]
        ax = np.array(g.pos_axes).reshape(3, 3)
        flagged = [k for k in range(3) if g.flags_pos >> k & 1]
        row = dict(flags_pos=int(g.flags_pos), flags_ori=int(g.flags_ori), accepted=int(r.accepted), status=int(r.reg.status),
                   overlap=r.overlap, conflict=(r.conflict_query, r.conflict_map),
                   axis_x=[float(abs(ax[k][0])) for k in flagged], move_x=float(r.reg.pose_opt[0] - prior[0]),
                   along_error=LC.along_error(r.rel7, cand), same_as_plain=r.reg.n_iterations == plain.reg.n_iterations and
                   bytes(r.reg.pose) == bytes(plain.reg.pose) and bytes(r.rel7) == bytes(plain.rel7))
        Sp = api.loop_edge_information(np.array(r.reg.pose), g, S)
        _, ej, wj = LC.solve(api, ctx, (cand, LC.QUERY, r.rel7, Sp))
        row["graph_projected"] = dict(summary(ej), rho1=wj)
        row["x_vs_no_loop_max"] = float(np.abs(ej["x"] - e0["x"]).max())
        out["per_threshold"][str(thr)] = row
    scratch.close()
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--thresholds", default="0.1,0.2,0.3")
    a = ap.parse_args()
    thr = [float(v) for v in a.thresholds.split(",")]
    d = api.degeneracy(0.2, 0.1)                                       # the recommended thresholds (DESIGN.md section 4)
    print(json.dumps(dict(card=card(), hall=hall(a.reps, d), corridor_poles=corridor(a.reps, True, thr, d),
                          corridor_poles_no_offset=corridor(a.reps, True, thr, d, 0), corridor_bare=corridor(a.reps, False, thr, d))))


if __name__ == "__main__":
    main()

"""Degeneracy-aware loop verification (so_register_keyframes_degeneracy, so_loop_verify_degeneracy, so_loop_edge_information):
the keyframe form equals so_register_degeneracy on the downloaded keyframe; with nothing flagged or nothing constrained verification
is so_loop_verify's bit for bit; in the bare corridor the alignment is held along the corridor, and the loop edge built with
so_loop_edge_information leaves that direction to odometry while it still corrects the rest.  Thresholds 0.2 (translation) and 0.1
(rotation) are the recommended ones (DESIGN.md section 4, "Loop verification", from scripts/bench_loop_verify_degeneracy.py)."""
import numpy as np
import pytest

import loop_corridor as LC
from test_keyframes import _ctx, _err, _keyframes
from test_loop_detection import LOOP_OPTS, _closure

SO_ERR_ARG = -1
THR = (0.2, 0.1)


def _icp_bits(api, r):
    c = api.IcpResult.from_buffer_copy(bytes(r))
    c.time_ms = 0.0
    c.time_total_ms = 0.0
    return bytes(c)


def _deg_bits(api, r):
    """the degeneracy report of a so_degeneracy_result (everything after icp)"""
    return bytes(r)[api.DegeneracyResult.iter_n_flag_pos.offset:]


def _verify_bits(api, res):
    out = []
    for r in res:
        c = api.LoopVerifyResult.from_buffer_copy(r)
        c.time_ms = 0.0
        c.reg.time_ms = 0.0
        c.reg.time_total_ms = 0.0
        out.append(bytes(c))
    return out


def _same_solve(a, b):
    """pose, covariance, iteration counts and the solve record of two so_icp_results, bit for bit"""
    return all(bytes(getattr(a, f)) == bytes(getattr(b, f)) for f in ("pose", "pose_opt", "cov", "iter_lm_steps", "iter_lm_successful",
                                                                      "iter_lm_termination", "iter_cost", "iter_n_surf")) and \
        (a.status, a.n_iterations) == (b.status, b.n_iterations)


def _flagged(deg, n_iterations):
    return sum(deg.iter_n_flag_pos[:n_iterations]) + sum(deg.iter_n_flag_ori[:n_iterations])


def _scratch(api):
    return _ctx(api, max_map_points=1 << 21)


# ------------------------------------------------------------------------------------------------------ 1. keyframe input
@pytest.mark.gpu
@pytest.mark.parametrize("mf", [0, 2000])
def test_keyframes_equal_register_degeneracy(gpu_api, mf):
    """cfg1 keyframes at thresholds 0.9, so that reduced solves run: one keyframe per call is so_register_degeneracy on the
    downloaded keyframe bit for bit; several in one call agree with the single calls; constrain = 0 is so_register_keyframes."""
    from superodom_b200 import synth
    api = gpu_api
    src, case, _ = _keyframes(api, "cfg1", 4, 2000)
    poses = src.keyframe_poses()
    sub = _ctx(api, max_batch=4)
    sub.map_from_keyframes(src, [0, 1], poses[:2], 1)
    d = api.degeneracy(0.9, 0.9)
    priors = {i: synth.perturb_pose(poses[i], 40 + i, 0.1, 1.0) for i in (2, 3)}
    for i, prior in priors.items():
        a = sub.register_keyframes_degeneracy(src, [i], [prior], d, 5, mf)[0]
        b = sub.register_degeneracy(src.keyframe_download(i, 0), prior, d, 5, mf)
        assert a.icp.status == 0 and _flagged(a, a.icp.n_iterations) > 0, i
        assert _same_solve(a.icp, b.icp), i
        assert _deg_bits(api, a) == _deg_bits(api, b), i
        off = sub.register_keyframes_degeneracy(src, [i], [prior], api.degeneracy(0.9, 0.9, False), 5, mf)[0]
        plain = sub.register_keyframes(src, [i], [prior], 5, mf)[0]
        assert _icp_bits(api, off.icp) == _icp_bits(api, plain), i
        assert _flagged(off, off.icp.n_iterations) > 0                 # reported, not used
    for ids in ([3, 2], [2, 3]):                                       # a gather and in place
        rs = sub.register_keyframes_degeneracy(src, ids, [priors[i] for i in ids], [d, api.degeneracy(0.5, 0.9)], 5, mf)
        for i, dd, r in zip(ids, (d, api.degeneracy(0.5, 0.9)), rs):
            one = sub.register_keyframes_degeneracy(src, [i], [priors[i]], dd, 5, mf)[0]
            assert np.allclose(np.array(r.icp.pose), np.array(one.icp.pose), atol=1e-9), (ids, i)
            assert r.flags_pos == one.flags_pos and r.flags_ori == one.flags_ori
    sub.close()
    src.close()


@pytest.mark.gpu
def test_keyframes_equal_register_degeneracy_in_the_bare_corridor(gpu_api):
    api = gpu_api
    ctx = LC.context(api, False)
    poses = ctx.keyframe_poses()
    sub = _scratch(api)
    ids = [0, 1, 2, 3, 4]
    sub.map_set_origin(poses[LC.CAND][:3])
    sub.map_from_keyframes(ctx, ids, poses[ids], 1)
    prior = ctx.loop_prior(LC.candidate(api)[0])
    d = api.degeneracy(*THR)
    a = sub.register_keyframes_degeneracy(ctx, [LC.QUERY], [prior], d, 20, 0)[0]
    b = sub.register_degeneracy(ctx.keyframe_download(LC.QUERY, 0), prior, d, 20, 0)
    assert a.flags_pos & 1 and abs(a.pos_axes[0]) > 0.99
    assert _same_solve(a.icp, b.icp) and _deg_bits(api, a) == _deg_bits(api, b)
    sub.close()
    ctx.close()


@pytest.mark.gpu
def test_keyframe_argument_errors(gpu_api):
    api = gpu_api
    src, case, _ = _keyframes(api, "cfg1", 2, 2000)
    poses = src.keyframe_poses()
    sub = _ctx(api)
    sub.map_from_keyframes(src, [0], poses[:1], 1)
    sub.kernel_launches(reset=True)
    for d in (api.degeneracy(float("nan"), 0.1), api.degeneracy(-0.1, 0.1), api.degeneracy(0.1, 1.0), api.Degeneracy(0.1, 0.1, 2, 0)):
        assert _err(api, lambda: sub.register_keyframes_degeneracy(src, [1], [poses[1]], d, 5)) == SO_ERR_ARG
    assert _err(api, lambda: sub.register_keyframes_degeneracy(src, [9], [poses[1]], api.degeneracy(0.1, 0.1), 5)) == SO_ERR_ARG
    assert sub.kernel_launches() == 0
    L = api.load_library()
    assert L.so_register_keyframes_degeneracy(sub.h, src.h, None, 0, None, None, None, None) == SO_ERR_ARG
    sub.close()
    src.close()


# ------------------------------------------------------------------------------------------------------ 2. nothing flagged
@pytest.mark.gpu
def test_nothing_flagged_is_loop_verify(gpu_api):
    """The hall loop's top 5 candidates (the true revisit and four false ones) and a skipped slot: with nothing constrained, or
    nothing flagged, every field equals so_loop_verify's; at the recommended thresholds so do the candidates where nothing was
    flagged."""
    api = gpu_api
    scene, truth, est, q, off, ctx, true_near = _closure(api, False)
    cands = np.concatenate([ctx.loop_candidates([q], 5, **LOOP_OPTS)[0], np.zeros(1, api.LOOP_CANDIDATE_DTYPE)])
    cands[-1]["query"], cands[-1]["id"] = q, -1
    scratch = _scratch(api)
    o = api.loop_verify_opts(image=LC.VLP16)
    plain = _verify_bits(api, ctx.loop_verify(scratch, cands, o))
    for d in (api.degeneracy(0.9, 0.9, False), api.degeneracy(0.0, 0.0, True)):
        res, deg = ctx.loop_verify_degeneracy(scratch, cands, d, o)
        assert _verify_bits(api, res) == plain, (d.pos_threshold, d.constrain)
        assert bytes(deg[-1]) == bytes(api.DegeneracyResult())              # the skipped slot: zeroed
        for r, g in zip(res[:-1], deg[:-1]):
            assert _icp_bits(api, g.icp) == _icp_bits(api, r.reg)
            if r.reg.n_iterations > 0:
                assert g.pos_info[2] > 0 and (d.constrain == 1 or _flagged(g, r.reg.n_iterations) > 0)
    res, deg = ctx.loop_verify_degeneracy(scratch, cands, api.degeneracy(*THR), o)
    got = _verify_bits(api, res)
    for k, (r, g) in enumerate(zip(res[:-1], deg[:-1])):
        n = _flagged(g, r.reg.n_iterations)
        pr, orr = LC.ratios(g)
        print(f"hall candidate {r.id}: accepted {r.accepted}, flagged {n}, ratios {pr:.3f} / {orr:.3f}")
        if n == 0:
            assert got[k] == plain[k], r.id
    print(f"true revisit {true_near}: best candidate {res[0].id}, accepted {res[0].accepted}")
    scratch.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------------ 3. the corridor
@pytest.mark.gpu
def test_bare_corridor_edge_leaves_the_axis_to_odometry(gpu_api):
    """Measured (H100 80GB HBM3, 700 W): the alignment's translation ratio is 0.143 (x flagged at 0.2, the axis 0.7 degrees off x)
    and it moves 0.001 mm along that axis; plain verification accepts the candidate (overlap 0.999, no conflict) with rel7 2.000 m off along
    the corridor.  Graph errors (mean over the keyframes, m / rad): no loop x 0.245, y 0.367, yaw 0.049; plain edge x 0.536, y 0.216,
    yaw 0.047 (rho' 0.35); projected edge x 0.247, y 0.172, yaw 0.046 (rho' 0.52), x within 4.3 mm of the no-loop solve."""
    api = gpu_api
    ctx = LC.context(api, False)
    scratch = _scratch(api)
    o = api.loop_verify_opts(image=LC.VLP16)
    c = LC.candidate(api)
    prior = ctx.loop_prior(c[0])
    plain = ctx.loop_verify(scratch, c, o)[0]
    res, deg = ctx.loop_verify_degeneracy(scratch, c, api.degeneracy(*THR), o)
    r, g = res[0], deg[0]
    axis = np.array(g.pos_axes[0:3])
    move = float(np.dot(np.array(r.reg.pose[:3]) - prior[:3], axis))
    print(f"bare corridor: ratios {LC.ratios(g)}, flags {g.flags_pos}/{g.flags_ori}, axis {axis}, moved {move * 1e3:.3f} mm; plain "
          f"accepted {plain.accepted} overlap {plain.overlap:.4f} conflicts {plain.conflict_query:.4f}/{plain.conflict_map:.4f}, along "
          f"error {LC.along_error(plain.rel7):.4f} m; degeneracy-aware accepted {r.accepted}, along error {LC.along_error(r.rel7):.4f} m")
    assert g.flags_pos & 1 and abs(axis[0]) > 0.99 and abs(move) < 1e-3
    assert plain.accepted and abs(LC.along_error(plain.rel7) - 2.0) < 0.01       # what the measurement showed
    assert r.accepted                                                            # the accept rule is unchanged
    S = LC.loop_sqrt_info()
    Sp = api.loop_edge_information(np.array(r.reg.pose), g, S)
    _, e0, _ = LC.solve(api, ctx)
    _, ep, wp = LC.solve(api, ctx, (LC.CAND, LC.QUERY, plain.rel7, S))
    _, ej, wj = LC.solve(api, ctx, (LC.CAND, LC.QUERY, r.rel7, Sp))
    for tag, e, w in (("no loop", e0, None), ("plain", ep, wp), ("projected", ej, wj)):
        print(f"  {tag}: " + ", ".join(f"{k} mean {v.mean():.4f} max {v.max():.4f}" for k, v in e.items()) + f", rho' {w}")
    assert np.abs(ej["x"] - e0["x"]).max() < 0.01                                # x left to odometry
    assert ej["x"].mean() < ep["x"].mean() and ej["x"][LC.QUERY] < ep["x"][LC.QUERY]
    for k in ("y", "yaw"):
        assert ej[k].mean() <= e0[k].mean() and ej[k][LC.QUERY] <= e0[k][LC.QUERY], k
    # repeated calls give the same bytes
    again, deg2 = ctx.loop_verify_degeneracy(scratch, c, api.degeneracy(*THR), o)
    assert _verify_bits(api, res) == _verify_bits(api, again) and _deg_bits(api, g) == _deg_bits(api, deg2[0])
    assert _icp_bits(api, g.icp) == _icp_bits(api, deg2[0].icp)
    scratch.close()
    ctx.close()


@pytest.mark.gpu
def test_corridor_with_poles(gpu_api):
    """The corridor with poles, measured (H100 80GB HBM3, 700 W).  At thresholds 0.1 nothing is flagged, at the query's own place
    (candidate 0) or 2 m from it, and the results are plain verification's bit for bit.  The recommended 0.2 flags two translation
    directions even at the query's own place: the weakest is the vertical (ratio 0.175; a VLP-16 in a 6 m corridor sees the floor
    only beyond 6.7 m), and the poles, 0.1 m thick, do not lift the corridor's axis above 0.2 either.  Flagging a direction the
    alignment did measure costs the loop edge that information, not a wrong edge; the decision is unchanged (accepted).  At 2 m
    the query's poles fall half way between the submap's (they are 4 m apart) and x is flagged as in the bare corridor (ratio 0.141);
    plain verification rejects that candidate, by its query conflict (0.056)."""
    api = gpu_api
    ctx = LC.context(api, True)
    scratch = _scratch(api)
    o = api.loop_verify_opts(image=LC.VLP16)
    for cand in (0, LC.CAND):
        c = LC.candidate(api, LC.QUERY, cand)
        plain = ctx.loop_verify(scratch, c, o)
        res, deg = ctx.loop_verify_degeneracy(scratch, c, api.degeneracy(0.1, 0.1), o)
        assert _flagged(deg[0], res[0].reg.n_iterations) == 0, cand
        assert _verify_bits(api, res) == _verify_bits(api, plain), cand
        res, deg = ctx.loop_verify_degeneracy(scratch, c, api.degeneracy(*THR), o)
        g = deg[0]
        print(f"poles, candidate {cand}: ratios {LC.ratios(g)}, flags {g.flags_pos}/{g.flags_ori}, axes {list(g.pos_axes)}, plain "
              f"accepted {plain[0].accepted} conflicts {plain[0].conflict_query:.4f}/{plain[0].conflict_map:.4f}, accepted "
              f"{res[0].accepted}, along error {LC.along_error(res[0].rel7, cand):.4f} m")
        assert res[0].accepted == plain[0].accepted == (1 if cand == 0 else 0), cand
        if cand == 0:
            assert g.flags_pos == 3 and g.flags_ori == 0 and abs(g.pos_axes[2]) > 0.99
        else:
            assert g.flags_pos & 1 and abs(g.pos_axes[0]) > 0.99
    scratch.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------------ 4. errors
@pytest.mark.gpu
def test_verify_argument_errors(gpu_api):
    api = gpu_api
    ctx = LC.context(api, False)
    scratch = _scratch(api)
    c = LC.candidate(api)
    for x in (ctx, scratch):
        x.kernel_launches(reset=True)
    for d in (api.degeneracy(float("nan"), 0.1), api.degeneracy(0.1, 1.0), api.Degeneracy(0.1, 0.1, 2, 0)):
        assert _err(api, lambda: ctx.loop_verify_degeneracy(scratch, c, d, image=LC.VLP16)) == SO_ERR_ARG
    assert _err(api, lambda: ctx.loop_verify_degeneracy(ctx, c, api.degeneracy(0.2, 0.1), image=LC.VLP16)) == SO_ERR_ARG
    assert _err(api, lambda: ctx.loop_verify_degeneracy(scratch, c, api.degeneracy(0.2, 0.1), half_window=9)) == SO_ERR_ARG
    o = api.loop_verify_opts()
    L = api.load_library()
    assert L.so_loop_verify_degeneracy(ctx.h, scratch.h, api._p(c), 1, api.C.byref(o), None, None, None) == SO_ERR_ARG
    for x in (ctx, scratch):
        assert x.kernel_launches() == 0
    assert ctx.loop_verify_degeneracy(scratch, c[:0], api.degeneracy(0.2, 0.1)) == ([], [])
    scratch.close()
    ctx.close()

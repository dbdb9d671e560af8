"""The restatements and scenes of test_free_space_keyframes_edges.py, without a GPU: the union restatement against a literal loop of
free_space_numpy.clear per entry, the tile plan against so_free_rule.h, and each builder producing what its case claims."""
import math
import re

import numpy as np

import free_space_keyframe_sets as K
import free_space_numpy as F


def _literal(stores, clouds, poses, o):
    """Each entry in turn with free_space_numpy.clear on every point it has not removed yet: removal masks per store; candidates
    collected as a set of (store, point) so that a point counts once"""
    removed = [np.zeros(len(s), bool) for s in stores]
    cands = set()
    for cloud, pose in zip(clouds, poses):
        img, hit, _, _ = F.range_image(cloud, o)
        for k, s in enumerate(stores):
            live = np.nonzero(~removed[k])[0]
            rem, _ = F.clear(s[live], cloud, pose, o)
            _, cand = F.removal_mask(s[live], pose, img, hit, o)
            cands |= {(k, int(i)) for i in live[cand]}
            removed[k][live[rem]] = True
    return removed, cands


def test_union_restatement_equals_the_per_entry_loop():
    c = K.spread_case(seed=19, n_keyframes=60)
    stores = [c["surf"], c["edge"]]
    order = np.random.default_rng(2).permutation(60)[:45]
    clouds, poses = [c["clouds"][i] for i in order], c["poses"][order]
    rs = K.restate(stores, clouds, poses, c["opts"])
    removed, cands = _literal(stores, clouds, poses, c["opts"])
    assert rs["n_ambiguous_map"] == 0 and rs["n_ambiguous_scan"] == 0
    for k in range(2):
        assert np.array_equal(rs["removed"][k], removed[k])
    assert rs["n_removed"] > 10 and rs["n_candidates"] == len(cands) > rs["n_removed"]
    # a candidate that an earlier entry removed is not counted again by a later entry: the per-call sum is larger
    per_call = sum(F.clear(np.vstack(stores), cl, p, c["opts"])[1]["n_candidates"] for cl, p in zip(clouds, poses))
    assert per_call > rs["n_candidates"]


def test_tile_plan_matches_the_header():
    with open(f"{K.ROOT}/superodom_b200/csrc/so_free_rule.h") as f:
        assert re.search(r"kFreeTileBytes = size_t\(256\) << 20;", f.read())
    assert K.tile_bytes() == 256 << 20
    assert K.tile_plan(13, K.BIG) == (4, 4) and K.tile_plan(4, K.BIG) == (4, 1) and K.tile_plan(5, K.BIG) == (4, 2)
    assert F.dims(K.BIG) == (4096, 4096) and F.dims(K.COARSE) == (180, 20)
    per, n = K.tile_plan(320, K.COARSE)
    assert per == (256 << 20) // (4 * 3600) and n == 1
    assert K.tile_plan(1, F.opts_for("os1_128"))[0] == 648                 # DESIGN.md: 648 images of the OS1-128 defaults


def test_block_restatement():
    """free_coord's int() then c--: a point on a negative face lands in the block below it (x = -75), one on the face at 0 above it (x = -25)"""
    f = np.array([[-75.0, 0, 0], [-25.0, 0, 0], [25.0, 0, 0], [75.0, 0, 0], [-525.0, 0, 0], [524.99, 0, 0], [525.0, 0, 0]])
    b = K.grid_block(f)
    assert list(b[:4] % 21) == [8, 10, 11, 12] and b[4] == -1 and b[5] % 21 == 20 and b[6] == -1
    gx = [K.grid_coord(np.array([v + 25.0]), 10)[0] for v in f[:, 0]]
    assert gx == [8, 10, 11, 12, -1, 20, 21]
    lo, hi = K.block_box(b[:4])
    assert (lo[:, 0] <= f[:4, 0]).all() and (f[:4, 0] <= hi[:, 0]).all()


def test_spread_case_exercises_the_cull():
    c = K.spread_case()
    blocks = np.unique(np.r_[K.grid_block(c["surf"]), K.grid_block(c["edge"])])
    blocks = blocks[blocks >= 0]
    lists = K.cull_lists(blocks, c["poses"], c["opts"].max_range)
    cnt = lists.sum(1)
    assert len(c["poses"]) >= 300 and ((cnt > 0) & (cnt < len(c["poses"]))).sum() > 1000 and (cnt == 0).sum() > 100
    t = c["poses"][:, :3]
    outside = (np.abs(t[:, 0]) >= 525) | (np.abs(t[:, 1]) >= 525) | (np.abs(t[:, 2]) >= 275)
    reach_any = lists.any(0)
    assert (outside & reach_any).sum() >= 10 and (outside & ~reach_any).sum() >= 5
    roll_pitch = np.array([abs(2 * math.asin(max(-1.0, min(1.0, q)))) for q in np.hypot(c["poses"][:, 3], c["poses"][:, 4])])
    assert (roll_pitch > 0.2).sum() > 20


def test_face_cases():
    """Points exactly on faces (both signs, int() and c-- on the negative ones), r_m at float(max_range) and one float32 step
    either side (and one FP64 step where the keyframe's coordinate holds it), exact; one keyframe's pixel holds its own point only"""
    for axis in (0, 1):
        c = K.face_case(axis)
        o = c["opts"]
        m = c["surf"]
        f = m[:, axis].astype(np.float64)
        assert np.array_equal((f - 25.0) % 50.0, np.zeros(len(f))) and (f < 0).sum() >= 20 and (f > 0).sum() >= 20
        r = np.array([K.device_range(m[i:i + 1], p)[0] for i, p in enumerate(c["poses"])])
        lim = float(np.float32(o.max_range))
        step = float(np.nextafter(np.float32(lim), np.float32(100))) - lim
        assert set(np.round((r - lim) / step, 6)) >= {-1.0, 0.0, 1.0}
        assert (r == lim).sum() >= 12 and (np.abs(r - lim) < 1e-13).sum() > (r == lim).sum()
        for i, p in enumerate(c["poses"]):                     # r_m is the FP64 difference: exact in every form
            assert float(np.linalg.norm(F.to_sensor(m[i:i + 1], p))) == r[i]
        rs = K.restate([m, None], c["clouds"], c["poses"], o, exact_gate=True)
        assert rs["n_ambiguous_map"] == 0 and rs["n_ambiguous_scan"] == 0
        assert np.array_equal(rs["removed"][0], c["want"]) and np.array_equal(c["want"], r <= lim)
        for e, (cl, p) in enumerate(zip(c["clouds"], c["poses"])):
            img, hit, _, _ = F.range_image(cl, o)
            _, cand = F.removal_mask(m, p, img, hit, o)
            assert set(np.nonzero(cand)[0]) <= {e}


def test_face_near_case():
    """Every keyframe is more than max_range from its point by the FP64 difference (the box distance), yet the rotation puts some
    points at r_m <= max_range; no keyframe's patch reaches another keyframe's point"""
    c = K.face_near_case(np.random.default_rng(5))
    o = c["opts"]
    m = c["surf"]
    lim = float(np.float32(o.max_range))
    d = np.array([abs(float(m[i, 0]) - p[0]) for i, p in enumerate(c["poses"])])
    r = np.array([K.device_range(m[i:i + 1], p)[0] for i, p in enumerate(c["poses"])])
    assert (d > lim).all() and 10 <= (r <= lim).sum() < len(r)
    lo, hi = K.block_box(K.grid_block(m), pad=False)
    assert ((lo[:, 0] == m[:, 0]) | (hi[:, 0] == m[:, 0])).all()    # on a face of its own block
    for e, (cl, p) in enumerate(zip(c["clouds"], c["poses"])):
        img, hit, _, _ = F.range_image(cl, o)
        q = F.to_sensor(m, p)
        near = np.sqrt((q * q).sum(1)) < lim - 1e-6
        _, cand = F.removal_mask(m, p, img, hit, o)
        assert not (cand & near).any()


def test_seam_case():
    """Each designed point kind is a candidate / removed by exactly the entries its layout names; no ambiguous point"""
    c = K.seam_case()
    o = c["opts"]
    clouds = [c["keyframes"][nm][0] for nm in c["ids"]]
    assert [len(cl) == 0 for cl in clouds] == [nm.startswith("E") for nm in c["names"]]
    assert all(len(cl) == 0 for cl in clouds[8:12])                       # tile 2 holds only empty keyframes
    assert c["ids"][3] == c["ids"][4] and not np.array_equal(c["poses"][3], c["poses"][4])
    for cl in clouds:
        if len(cl):
            assert np.isfinite(cl[0, :3]).all() and (~np.isfinite(cl[:, :3]).all(1)).sum() == 9
            assert (np.abs(cl[:, :3]).sum(1) == 0).sum() == 2
    stores = [c["surf"], c["edge"]]
    per_entry = []
    for cl, p in zip(clouds, c["poses"]):
        img, hit, _, _ = F.range_image(cl, o)
        per_entry.append([F.removal_mask(s, p, img, hit, o) for s in stores])
        assert F.edge_points(cl, o).sum() == 0
        for s in stores:
            assert F.edge_points(s, o, p).sum() == 0
    for k in range(2):
        for kd, inter in enumerate(K.SEAM_KINDS.values()):
            m = c["kinds"][k] == kd
            assert m.sum() >= 6
            for e in range(len(clouds)):
                rem, cand = per_entry[e][k]
                how = dict(inter).get(e)
                assert cand[m].all() == (how is not None) and cand[m].any() == (how is not None), (kd, e)
                assert rem[m].all() == (how == "behind") and rem[m].any() == (how == "behind"), (kd, e)

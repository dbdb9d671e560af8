"""so_scan_extract_edges: LOAM edge features of ring-ordered raw scans on the device (DESIGN.md §9).

The device output must equal the numpy restatement (tests/edge_features_numpy.py) bit for bit; the restatement itself is held
against a plain per-point loop on the CPU.  Then the buffers the extractor must leave alone, its argument errors, registration
parity against the oracle with real edge clouds, and the corridor the edge rows exist for."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import edge_features_numpy as EN
from conftest import get_case, quat_angle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRIDE, TOFF, ROFF = 32, 20, 24


def _fields(rec):
    return EN.records_fields(rec, STRIDE, TOFF, ROFF)


def _ref(rec, **kw):
    return EN.extract_edges(*_fields(rec), **kw)


def _set_rings(rec, ring):
    rec = rec.copy()
    rec.view(np.uint16)[:, 12] = np.asarray(ring, np.uint16)
    return rec


def _small_scan():
    """4 VLP-16 rings of the first 300 columns of a cfg1 scan, with a 17- and a 16-point ring, a zero return and a repeated point."""
    from superodom_b200 import synth
    case = get_case("cfg1", 0)
    rec = synth.make_ring_scan(case["scene"], "vlp16", case["pose_true"], 11)
    ring = rec.view(np.uint16)[:, 12]
    col = np.rint(rec[:, 5] / np.float32(0.1) * 1800).astype(np.int64)
    keep = (ring < 4) & (col < 300) | (ring == 4) & (col < 17) | (ring == 5) & (col < 16)
    rec = rec[keep].copy()
    rec[7, :3] = 0.0
    rec[40, :3] = rec[39, :3]
    return rec


# --------------------------------------------------------------------------------------------------------------- CPU
def test_restatement_matches_per_point_loop():
    rec = _small_scan()
    xyz, t, ring = _fields(rec)
    for kw in ({}, dict(edge_threshold=0.02, max_per_sector=3), dict(min_range=5.0)):
        a = EN.extract_edges(xyz, t, ring, **kw)
        b = EN.extract_edges_loop(xyz, t, ring, **kw)
        assert len(a) > 0 and a.shape == b.shape, kw
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), kw


def test_ring_scan_orders_hold_the_same_points():
    from superodom_b200 import synth
    sc = synth.make_corridor_scene()
    pose = np.array([0.3, 0.2, 0.1, 0.0, 0.0, 0.0, 1.0])
    a = synth.make_ring_scan(sc, "vlp16", pose, 5, "column")
    b = synth.make_ring_scan(sc, "vlp16", pose, 5, "ring")
    ka = np.lexsort((a[:, 5], a.view(np.uint16)[:, 12]))
    kb = np.lexsort((b[:, 5], b.view(np.uint16)[:, 12]))
    assert np.array_equal(a[ka, :3], b[kb, :3]) and np.array_equal(a[ka, 5], b[kb, 5])
    assert len(np.unique(a.view(np.uint16)[:, 12])) == 16
    # (ring, time) is unique per point
    assert len(np.unique(a.view(np.uint16)[:, 12].astype(np.int64) * 10**9 + np.rint(a[:, 5] * 1e7).astype(np.int64))) == len(a)
    # the corridor keeps the "no face plane within 1 m of the origin" rule
    faces = np.r_[sc.room, sc.boxes.ravel()]
    assert np.abs(faces).min() >= 1.0


def test_struct_layout_matches_header(tmp_path):
    from superodom_b200 import api
    f = tmp_path / "sz.c"
    f.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "superodom_b200.h"\n'
                 'int main(void){printf("%zu %zu\\n", sizeof(so_edge_opts), offsetof(so_edge_opts, max_per_sector));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(f), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)]).split()))
    assert got == (C.sizeof(api.EdgeOpts), api.EdgeOpts.max_per_sector.offset)


def _build_edge_test(tmp_path):
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "edge_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "edge_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


def test_edge_shim_compiles(tmp_path):
    assert os.path.exists(_build_edge_test(tmp_path))


# --------------------------------------------------------------------------------------------------------------- GPU
def _ctx(api, max_scan_points=262144, max_map_points=1 << 20, **kw):
    return api.Context(max_map_points=max_map_points, max_scan_points=max_scan_points, **kw)


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _ring_case(name, idx, order):
    from superodom_b200 import synth
    case = get_case(name, idx)
    rec = synth.make_ring_scan(case["scene"], case["cfg"]["sensor"], case["pose_true"], 300 + idx, "ring" if order == "ring" else "column")
    if order == "shuffled":
        rec = rec[np.random.default_rng(idx).permutation(len(rec))]
    return rec


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg1", "cfg2"])
def test_bit_exact_in_every_record_order(gpu_api, name):
    ctx = _ctx(gpu_api)
    for idx in range(2):
        outs = []
        for order in ("column", "ring", "shuffled"):
            rec = _ring_case(name, idx, order)
            got = ctx.scan_extract_edges(rec)
            ref = _ref(rec)
            assert len(ref) > 100 and _bits_equal(got, ref), (name, idx, order, len(got), len(ref))
            outs.append(got)
        assert _bits_equal(outs[0], outs[1]) and _bits_equal(outs[0], outs[2])
    ctx.close()


@pytest.mark.gpu
def test_bit_exact_corridor_and_options(gpu_api):
    from superodom_b200 import synth
    sc = synth.make_corridor_scene()
    ctx = _ctx(gpu_api)
    for i, sensor in enumerate(["vlp16", "os1_128"]):
        pose = np.array([1.0 + 3 * i, 0.4, 0.2, 0.0, 0.0, np.sin(0.15), np.cos(0.15)])
        rec = synth.make_ring_scan(sc, sensor, pose, 40 + i)
        for kw in ({}, dict(min_range=4.0), dict(edge_threshold=0.5), dict(max_per_sector=5), dict(edge_threshold=0.03, max_per_sector=40)):
            got = ctx.scan_extract_edges(rec, **kw)
            ref = _ref(rec, **kw)
            assert len(ref) > 50 and _bits_equal(got, ref), (sensor, kw, len(got), len(ref))
    ctx.close()


@pytest.mark.gpu
def test_bit_exact_defects_and_ring_sizes(gpu_api):
    from superodom_b200 import synth
    ctx = _ctx(gpu_api, max_scan_points=1 << 17)
    # raw sweep with NaN / inf / zero / repeated points and real rings (its ring column holds small integers as floats)
    d = synth.make_raw_sweep(60_000, seed=4300)
    rec = _set_rings(d["points"], np.arange(60_000) % 64)
    rec[::997, 5] = -0.0                                      # -0 times sort as +0
    ref = _ref(rec)
    assert len(ref) > 0 and _bits_equal(ctx.scan_extract_edges(rec), ref)
    # the same defects in a real ring scan: repeats, zero returns, NaN / inf coordinates and times
    case = get_case("cfg1", 1)
    full = synth.make_ring_scan(case["scene"], "vlp16", case["pose_true"], 77)
    rec = full.copy()
    rng = np.random.default_rng(4301)
    k = rng.choice(np.arange(16, len(rec)), size=600, replace=False)
    rec[k[:300], :3] = rec[k[:300] - 16, :3]                  # the same point again, one column later
    rec[k[300:450], :3] = 0.0
    rec[k[450:500], 0] = np.nan
    rec[k[500:550], 2] = np.inf
    rec[k[550:], 5] = np.nan
    ref = _ref(rec)
    assert len(ref) > 100 and _bits_equal(ctx.scan_extract_edges(rec), ref)
    # rings of 0 (absent), 16 and 17 points next to a full ring, then one 65 536-point ring
    r = full.view(np.uint16)[:, 12]
    parts = [full[r == 3], full[r == 5][:16], full[r == 7][:17], full[r == 9][:40]]
    rec = np.concatenate(parts)
    got, ref = ctx.scan_extract_edges(rec), _ref(rec)
    assert _bits_equal(got, ref) and len(ref) > 0
    assert len(ctx.scan_extract_edges(parts[1])) == len(_ref(parts[1])) == 0                  # a 16-point ring yields nothing
    a = np.arange(65536) * (2 * np.pi / 65536)                 # one beam at -3 deg, 65 536 columns
    el = np.deg2rad(-3.0)
    d = np.stack([np.cos(el) * np.cos(a), np.cos(el) * np.sin(a), np.full_like(a, np.sin(el))], 1)
    rr = synth.raycast(case["scene"], case["pose_true"][:3], d @ synth.quat_to_R(case["pose_true"][3:]).T)
    rr = rr + np.random.default_rng(5).normal(0.0, 0.01, len(rr))
    one = np.zeros((65536, 8), np.float32)
    one[:, :3] = d * rr[:, None]
    one[:, 5] = np.arange(65536, dtype=np.float32) * np.float32(1e-6)
    one = _set_rings(one, np.full(65536, 2))
    got, ref = ctx.scan_extract_edges(one), _ref(one)
    assert len(ref) > 50 and _bits_equal(got, ref)
    # empty and all-invalid inputs
    assert len(ctx.scan_extract_edges(np.zeros((0, 8), np.float32))) == 0
    bad = full[:500].copy()
    bad[:, 0] = np.nan
    assert len(ctx.scan_extract_edges(bad)) == 0
    ctx.close()


@pytest.mark.gpu
def test_voxel_leaf_equals_prefilter_reference(gpu_api, oracle_mod):
    ctx = _ctx(gpu_api)
    for name in ("cfg1", "cfg2"):
        rec = _ring_case(name, 0, "column")
        plain = ctx.scan_extract_edges(rec)
        got = ctx.scan_extract_edges(rec, voxel_leaf=0.1)
        ref = oracle_mod.adjust_voxel_size_numpy(plain, 0.1, 0.1, auto_voxel_size=False)[0]
        assert 0 < len(got) <= len(plain) and _bits_equal(got, ref), name
        # ... and bit-equal to so_scan_prefilter's filter of the same cloud
        pf, _, _, _ = ctx.scan_prefilter(plain, 0.1, 0.1, auto_voxel_size=False)
        assert _bits_equal(got, pf)
    ctx.close()


@pytest.mark.gpu
def test_extraction_leaves_the_scan_buffers_alone(gpu_api):
    case = get_case("cfg1", 0)
    rec = _ring_case("cfg1", 0, "column")
    pose = case["pose_prior"]

    def run(extract):
        ctx = _ctx(gpu_api, plane_res=0.2)
        ctx.map_set_points(case["map_xyzi"])
        ctx.scan_prefilter(case["scan_xyzi"], 0.1, 0.2, auto_voxel_size=False, download=False)
        if extract:
            assert len(ctx.scan_extract_edges(rec, voxel_leaf=0.1)) > 0
        r = ctx.register_prefiltered(pose, 5)
        ctx.map_add_registered_scan(np.array(r.pose))
        m = ctx.map_download(0)
        ctx.close()
        return r, m

    r0, m0 = run(False)
    r1, m1 = run(True)
    assert bytes(r0)[: gpu_api.IcpResult.time_ms.offset] == bytes(r1)[: gpu_api.IcpResult.time_ms.offset]
    assert _bits_equal(m0, m1) and len(m1) > len(case["map_xyzi"])


@pytest.mark.gpu
def test_argument_errors(gpu_api):
    L = gpu_api.load_library()
    ctx = _ctx(gpu_api, max_scan_points=4096)
    rec = np.zeros((16, 8), np.float32)
    out = np.zeros((16, 4), np.float32)
    n = C.c_size_t()

    def call(pts=rec, cnt=16, stride=32, toff=20, roff=24, opts=None, o=out, cap=16, nout=C.byref(n)):
        return L.so_scan_extract_edges(ctx.h, None if pts is None else pts.ctypes.data_as(C.c_void_p), cnt, stride, toff, roff,
                                       None if opts is None else C.byref(opts), None if o is None else o.ctypes.data_as(C.c_void_p), cap, nout)

    E = gpu_api.EdgeOpts
    assert call() == 0
    assert call(pts=None) == -1 and call(pts=None, cnt=0) == 0
    assert call(o=None) == -1 and call(nout=None) == -1
    assert call(stride=11) == -1 and call(toff=29) == -1 and call(roff=31) == -1          # the stride does not hold the fields
    assert call(toff=8) == -1 and call(roff=10) == -1                                      # overlapping x, y, z
    assert call(toff=20, roff=22) == -1                                                     # overlapping each other
    for bad in (E(-1.0, 0, 0, 0), E(0, -0.1, 0, 0), E(0, 0, -0.1, 0), E(0, 0, 0, -1), E(float("nan"), 0, 0, 0), E(0, float("inf"), 0, 0),
                E(0, 0, float("nan"), 0)):
        assert call(opts=bad) == -1
    big = np.zeros((4097, 8), np.float32)
    assert call(pts=big, cnt=4097) == -3
    ctx.close()


@pytest.mark.gpu
def test_edge_shim_matches_abi(tmp_path, gpu_api):
    exe = _build_edge_test(tmp_path)
    rec = _ring_case("cfg1", 0, "column")
    ctx = _ctx(gpu_api)
    for leaf in (0.0, 0.1):
        path, outp = tmp_path / "raw.bin", tmp_path / "out.bin"
        with open(path, "wb") as f:
            f.write(struct.pack("<if", len(rec), leaf))
            f.write(rec.tobytes())
        res = subprocess.run([exe, str(path), str(outp)], capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        raw = open(outp, "rb").read()
        k = struct.unpack("<i", raw[:4])[0]
        got = np.frombuffer(raw[4:], np.float32).reshape(k, 4)
        assert _bits_equal(got, ctx.scan_extract_edges(rec, voxel_leaf=leaf)) and k > 0
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# registration with extracted edge clouds
# ---------------------------------------------------------------------------------------------------------------
def _edge_map_by_extraction(ctx, oracle_mod, scene, sensor, poses, seed0):
    ref = np.zeros((0, 4), np.float32)
    from superodom_b200 import synth
    for i, T in enumerate(poses):
        e = ctx.scan_extract_edges(synth.make_ring_scan(scene, sensor, T, seed0 + i))
        ctx.map_add_scan_edge(e, T)
        ref = oracle_mod.map_insert_numpy(ref, oracle_mod.transform_scan_numpy(e, T), 0.1)
    return ref


@pytest.mark.gpu
@pytest.mark.parametrize("name,cap", [("cfg1", 2000), ("cfg1", 0), ("cfg2", 0)])
def test_registration_parity_with_extracted_edges(gpu_api, oracle_mod, name, cap):
    from superodom_b200 import synth
    case = get_case(name, 0)
    cfg = case["cfg"]
    ctx = _ctx(gpu_api, max_map_points=max(1 << 20, len(case["map_xyzi"]) * 2), plane_res=0.2, line_res=0.1)
    ctx.map_set_points(case["map_xyzi"])
    ctx.map_set_resolution(0.1, 0.2)
    poses = [synth.random_sensor_pose(case["scene"], 6100 + i, 12.0) for i in range(10)]
    em = _edge_map_by_extraction(ctx, oracle_mod, case["scene"], cfg["sensor"], poses, 6200)
    es = ctx.scan_extract_edges(synth.make_ring_scan(case["scene"], cfg["sensor"], case["pose_true"], 6300))
    assert len(em) > 1000 and len(es) > 200
    om = oracle_mod.OracleMap(case["map_xyzi"])
    om.set_edge_points(em)
    r = ctx.register(case["scan_xyzi"], case["pose_prior"], cfg["max_iterations"], cap, edge_xyzi=es)
    ro = om.register(case["scan_xyzi"], case["pose_prior"], 0.2, cfg["max_iterations"], cap, knn_mode=0, edge_xyzi=es, line_res=0.1)
    assert np.abs(np.array(r.pose)[:3] - np.array(ro.pose)[:3]).max() <= 1e-4
    assert quat_angle(np.array(r.pose)[3:], np.array(ro.pose)[3:]) <= 1e-4
    n = ro.n_iterations
    assert r.n_iterations == n and r.status == ro.status == 0
    assert list(r.iter_lm_steps[:n]) == list(ro.iter_lm_steps[:n]) and list(r.iter_lm_successful[:n]) == list(ro.iter_lm_successful[:n])
    assert list(r.iter_n_edge[:n]) == list(ro.iter_n_edge[:n]) and list(r.hist_reject_line) == list(ro.hist_reject_line)
    assert r.iter_n_edge[0] > 100
    cg, co = np.array(r.cov).reshape(6, 6), np.array(ro.cov).reshape(6, 6)
    assert np.abs(cg - co).max() <= 1e-6 * np.abs(co).max()
    ctx.close()


def corridor_runs(api, oracle_mod=None, n_scans=8, log=None):
    """8 seeded OS1-128 scans in the corridor, priors 0.15 m off along it plus the usual perturbation, registered with planes only
    and with extracted edges against a corridor map (surf: sampled faces; edges: extracted from mapping scans at true poses).
    -> list of dicts (along-corridor error and pos_inv_cond per arm)."""
    from superodom_b200 import synth
    sc = synth.make_corridor_scene()
    raw = synth.sample_surfaces(sc, 0.2)
    surf = synth.voxel_filter_blocks(np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1), 0.2)
    ctx = api.Context(max_map_points=max(1 << 20, 2 * len(surf)), max_scan_points=262144, plane_res=0.2, line_res=0.1)
    ctx.map_set_points(surf)
    ctx.map_set_resolution(0.1, 0.2)
    for i, x in enumerate(np.arange(-40.0, 40.1, 8.0)):
        T = np.array([x + 0.7, 0.3 * ((i % 3) - 1), 0.1, 0.0, 0.0, 0.0, 1.0])
        ctx.map_add_scan_edge(ctx.scan_extract_edges(synth.make_ring_scan(sc, "os1_128", T, 8000 + i)), T)
    rng = np.random.default_rng(8100)
    rows = []
    for s in range(n_scans):
        yaw = rng.uniform(-0.2, 0.2)
        T = np.array([rng.uniform(-20, 20), rng.uniform(-0.8, 0.8), rng.uniform(-0.3, 0.3), 0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)])
        rec = synth.make_ring_scan(sc, "os1_128", T, 8200 + s)
        scan = np.ascontiguousarray(np.concatenate([rec[:, :3], rec[:, 5:6]], 1))
        edges = ctx.scan_extract_edges(rec)
        prior = synth.perturb_pose(T, 8300 + s)
        prior[0] += 0.15
        rp = ctx.register(scan, prior, 20, 0)
        re = ctx.register(scan, prior, 20, 0, edge_xyzi=edges)
        rows.append(dict(err_planes=abs(rp.pose[0] - T[0]), err_edges=abs(re.pose[0] - T[0]), cond_planes=rp.pos_inv_cond,
                         cond_edges=re.pos_inv_cond, n_edges=len(edges), n_edge_rows=re.iter_n_edge[max(re.n_iterations - 1, 0)],
                         status=(rp.status, re.status)))
    ctx.close()
    return rows


@pytest.mark.gpu
def test_corridor_edges_tighten_the_along_corridor_direction(gpu_api):
    """The pole faces are not rejected as collinear: planes alone already take the 0.15 m along-corridor offset down to about 3 cm
    (measured 1.3-3.2 cm, DESIGN.md §9).  The edge rows lower the error further on every scan (0.7-2.8 cm) and raise pos_inv_cond."""
    rows = corridor_runs(gpu_api)
    for r in rows:
        print(r)
    for r in rows:
        assert r["status"] == (0, 0) and r["n_edge_rows"] > 300, r
        assert r["err_edges"] < r["err_planes"] and r["err_edges"] < 0.035, r
        assert r["cond_edges"] > r["cond_planes"], r
    assert np.median([r["err_edges"] for r in rows]) < 0.025

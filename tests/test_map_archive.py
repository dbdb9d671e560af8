"""The block archive (so_map_archive): a map store that keeps the blocks its 21 x 21 x 11 window drops and restores them when the
window comes back, against the restatement in map_archive_numpy.py; registrations against restored blocks; the capacity rule; the
shim's localization-mode order with a prior map saved and read back as a PCD file."""
import os
import subprocess

import numpy as np
import pytest

from conftest import get_case
from map_archive_numpy import ArchiveModel, CapacityError

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANE, LINE = 0.2, 0.1
IDENTITY = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])


def _gi(idx):
    g = idx.astype(np.int64)
    g[idx == 0xFFFFFFFF] = -1
    return g


def _patches(rng, n_patches, per, lo, hi, size=(12.0, 12.0, 1.0)):
    """Dense patches (so that k-NN finds neighbours) scattered over [lo, hi]"""
    c = rng.uniform(lo, hi, size=(n_patches, 3))
    p = (c[:, None, :] + rng.uniform(0, 1, size=(n_patches, per, 3)) * np.asarray(size)).reshape(-1, 3)
    return np.concatenate([p, rng.uniform(0, 255, size=(len(p), 1))], 1).astype(np.float32)


# a cloud about 3 km long in x, 900 m in y and 700 m in z: every shift below moves blocks out of the window and back in
def _scene(seed):
    rng = np.random.default_rng(seed)
    return rng, _patches(rng, 260, 1500, [-1500.0, -450.0, -350.0], [1500.0, 450.0, 350.0])


STEPS = [("insert", None), ("shift", [600.0, 0.0, 0.0]), ("shift", [1300.0, 0.0, 0.0]), ("insert", None),
         ("shift", [-1400.0, 0.0, 0.0]), ("shift", [-200.0, 500.0, 0.0]), ("shift", [0.0, -450.0, 0.0]),
         ("shift", [0.0, 0.0, 320.0]), ("shift", [0.0, 0.0, -330.0]), ("insert", None), ("origin", [1450.0, -300.0, 0.0]),
         ("origin", [-900.0, 420.0, 100.0]), ("origin", [0.0, 0.0, 0.0])]


def _run(gpu_api, oracle_mod, edge, seed=31, check=True):
    rng, cloud = _scene(seed)
    cap = 1 << 22
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=65536, plane_res=PLANE, line_res=LINE)
    ctx.map_archive(cap)
    ctx.map_set_origin([0.0, 0.0, 0.0])
    model = ArchiveModel(cap, 1 << 21, ctx.map_origin())
    (ctx.map_set_edge_points if edge else ctx.map_set_points)(cloud)
    model.set_points(cloud)
    store = 1 if edge else 0
    leaf = LINE if edge else PLANE
    trace = []

    def compare(step):
        got, got_all = ctx.map_download(0), ctx.map_download_all(store)
        trace.append((got, got_all))
        if not check:
            return
        exp = model.download()
        assert got.shape == exp.shape and np.array_equal(got, exp), step
        exp_all = model.download_all()
        assert got_all.shape == exp_all.shape and np.array_equal(got_all, exp_all), step
        assert ctx.map_archive_info(store)[:2] == (model.archived_points(), len(model.archive)), step
        assert ctx.map_archive_info(1 - store)[:2] == (0, 0)
        if edge and len(model.window):                                  # the edge store's 10-NN line search over the window
            q = model.window[::97] + np.concatenate([rng.normal(0, 0.05, size=(len(model.window[::97]), 3)), np.zeros((len(model.window[::97]), 1))], 1).astype(np.float32)
            om = oracle_mod.OracleMap()
            om.set_origin(model.origin)
            om.set_edge_points(model.window)
            gc, ghr = ctx.correspond_edge(q, IDENTITY)
            oc, ohr = om.correspond_edge(q, IDENTITY, LINE)
            searched = oc["nn"][:, 0] >= 0
            assert searched.any() and np.array_equal(ghr, ohr), step
            assert np.array_equal(gc["status"].astype(np.int32), oc["status"]), step
            assert np.array_equal(gc["nn"][searched].astype(np.int64), oc["nn"][searched]), step
        if not edge and len(model.window):
            q = model.window[::97, :3] + rng.normal(0, 0.1, size=model.window[::97, :3].shape).astype(np.float32)
            om = oracle_mod.OracleMap()
            om.set_origin(model.origin)
            om.set_points(model.window)
            gi, gd = ctx.knn(q, 5, 0.0)
            oi, od, of = om.knn(q, 5, 0)
            assert of.any()
            assert np.array_equal(_gi(gi)[of], oi[of]) and np.array_equal(gd[of], od[of]), step
            assert (gi[~of] == 0xFFFFFFFF).all(), step

    compare("load")
    assert model.archived_points() > 0 and len(model.window) > 0
    for i, (what, t) in enumerate(STEPS):
        if what == "insert":                                            # new points around the window's centre and some off it
            o = np.asarray(ctx.map_origin(), np.float64)
            centre = -o * 50.0 + np.array([500.0, 500.0, 250.0])
            new = _patches(rng, 30, 800, centre - [700.0, 700.0, 300.0], centre + [700.0, 700.0, 300.0])
            (ctx.map_add_edge if edge else ctx.map_add_surf)(new)
            model.insert(new, leaf)
        elif what == "shift":
            ctx.map_shift(t)
            model.set_origin(ctx.map_origin())
        else:
            ctx.map_set_origin(t)
            model.set_origin(ctx.map_origin())
        compare(f"{i}: {what} {t}")
    ctx.close()
    return trace


@pytest.mark.parametrize("store", ["surf", "edge"])
def test_archive_matches_the_restatement(gpu_api, oracle_mod, store):
    """Loads, inserts, shifts along x, y and z both ways and set_origin jumps over a 3 km cloud: after every step the window (in cube
    order), the whole map (window + archive by world block), the archive's counts and the search over the window (surf: 5-NN; edge:
    the 10-NN line search) equal the unbounded-store model."""
    _run(gpu_api, oracle_mod, store == "edge")


def test_archive_runs_are_deterministic(gpu_api, oracle_mod):
    """Two runs of the same sequence give bit-equal downloads after every step."""
    a = _run(gpu_api, oracle_mod, False, seed=32, check=False)
    b = _run(gpu_api, oracle_mod, False, seed=32, check=False)
    assert len(a) == len(b)
    for (w0, all0), (w1, all1) in zip(a, b):
        assert np.array_equal(w0, w1) and np.array_equal(all0, all1)


RESULT_FIELDS = ["pose", "pose_opt", "status", "n_iterations", "iter_n_surf", "iter_n_edge", "iter_dtrans", "iter_drot", "iter_lm_steps",
                 "iter_lm_successful", "iter_lm_termination", "iter_cost", "hist_obs", "hist_reject_plane", "hist_reject_line", "cov",
                 "pos_err", "pos_dir", "pos_inv_cond", "ori_err_deg", "ori_dir", "ori_inv_cond", "map_surf_5x5", "map_edge_5x5"]


def _fields(r):
    return [np.asarray(getattr(r, f)).tobytes() if hasattr(getattr(r, f), "__len__") else np.float64(getattr(r, f)).tobytes()
            for f in RESULT_FIELDS]


def _live_sequence(ctx):
    """A live loop far from the start: four tiny-case scans re-posed around x = 1500 m (clear of every block near the start),
    registered one by one (the map shifts to each prior) and inserted, then the window shifted further along y."""
    for i in range(4):
        c = get_case("tiny", i)
        pose = np.array(c["pose_true"], np.float64)
        pose[0] += 1500.0
        if i == 0:
            ctx.map_shift(pose[:3])
            ctx.map_add_scan(c["scan_xyzi"], pose)
            continue
        prior = np.array(c["pose_prior"], np.float64)
        prior[0] += 1500.0
        r = ctx.register(c["scan_xyzi"], prior, 5, 0)
        ctx.map_add_registered_scan(np.array(r.pose))
    ctx.map_shift([1500.0, 700.0, 0.0])


@pytest.mark.parametrize("archive", [True, False])
def test_revisit_gives_the_same_registrations(gpu_api, archive):
    """Probe scans registered as a frozen-map batch before and after an excursion of the window more than 1 km away: with the
    archive the probe blocks come back unchanged and every so_icp_result field but the timings and positions equals the first run's,
    bit for bit; without it the probes find no map."""
    case = get_case("cfg1")
    probes = [get_case("cfg1", i) for i in range(4)]
    scans = np.concatenate([p["scan_xyzi"] for p in probes], 0)
    n_points = [len(p["scan_xyzi"]) for p in probes]
    poses = np.stack([p["pose_prior"] for p in probes])
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=1 << 17, max_batch=4, plane_res=PLANE, line_res=LINE)
    if archive:
        ctx.map_archive(1 << 21)
    ctx.map_set_points(case["map_xyzi"])
    before = ctx.register_batch(scans, n_points, poses, 5, 0, skip_map_checks=True)
    assert all(r.iter_n_surf[0] > 0 for r in before)
    _live_sequence(ctx)
    assert (ctx.map_archive_info(0)[0] >= len(case["map_xyzi"])) if archive else ctx.map_archive_info(0)[0] == 0
    assert ctx.map_size() < len(case["map_xyzi"])                     # the start's blocks have left the window
    ctx.map_shift([0.0, 0.0, 0.0])
    after = ctx.register_batch(scans, n_points, poses, 5, 0, skip_map_checks=True)
    for r0, r1 in zip(before, after):
        if archive:
            assert _fields(r0) == _fields(r1)
        else:
            assert r1.status != 0 or r1.iter_n_surf[0] == 0
    ctx.close()


def test_archive_capacity(gpu_api):
    """An eviction the archive has no room for fails with SO_ERR_CAPACITY and so does every later map read; growing the archive
    recovers the store with nothing lost.  A load whose parts exceed the window or the archive fails before any change."""
    rng, cloud = _scene(33)
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=65536, plane_res=PLANE, line_res=LINE)
    ctx.map_set_origin([0.0, 0.0, 0.0])
    model = ArchiveModel(1 << 22, 1 << 21, ctx.map_origin())
    model.set_points(cloud)
    n_off = model.archived_points()
    ctx.map_archive(n_off)
    ctx.map_set_points(cloud)                                          # the archive holds exactly the off-window part
    assert ctx.map_archive_info(0) == (n_off, len(model.archive), n_off)
    small = ArchiveModel(n_off - 1, 1 << 21, ctx.map_origin())
    with pytest.raises(CapacityError):
        small.set_points(cloud)
    ctx.map_archive(0)
    ctx.map_archive(n_off - 1)
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-3\)"):
        ctx.map_set_points(cloud)
    ctx.map_archive(n_off)
    ctx.map_set_points(cloud)
    before = ctx.map_download(0)
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-3\)"):       # a load the archive cannot hold changes nothing
        ctx.map_set_points(np.concatenate([cloud, _patches(rng, 2, 100, [3000.0, 0, 0], [3100.0, 10, 10])]))
    assert np.array_equal(ctx.map_download(0), before) and ctx.map_archive_info(0)[0] == n_off
    ctx.map_set_origin([5000.0, 0.0, 0.0])                             # the whole window leaves; nothing comes back
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-3\)"):       # the read that applies it: an eviction beyond the archive
        ctx.map_download(0)
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-3\)"):
        ctx.map_shift([5000.0, 0.0, 0.0])
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-3\)"):
        ctx.knn(cloud[:10, :3], 5, 0.0)
    ctx.map_archive(1 << 22)                                           # grown: the pending eviction goes through, nothing lost
    model.set_origin(ctx.map_origin())
    assert np.array_equal(ctx.map_download(0), model.download())
    assert np.array_equal(ctx.map_download_all(0), model.download_all())
    ctx.close()


def test_insert_after_a_restore_is_checked_against_the_grown_window(gpu_api):
    """An insert that fits the window before a pending origin change but not after it (the change restores archived blocks) fails
    with SO_ERR_CAPACITY: the change is applied, nothing is inserted and nothing is written past the store."""
    rng, cloud = _scene(35)
    ctx0 = gpu_api.Context(max_map_points=1 << 21, max_scan_points=4096, plane_res=PLANE, line_res=LINE)
    o_a, o_b = ctx0.map_set_origin([0.0, 0.0, 0.0]), ctx0.map_set_origin([-500.0, 0.0, 0.0])
    ctx0.close()
    a, b = ArchiveModel(1 << 22, 1 << 21, o_a), ArchiveModel(1 << 22, 1 << 21, o_b)
    a.set_points(cloud)
    b.set_points(cloud)
    (t_small, small), (t_big, big) = sorted([([0.0, 0.0, 0.0], a), ([-500.0, 0.0, 0.0], b)], key=lambda x: len(x[1].window))
    assert len(big.window) > len(small.window) + 1000
    m = len(big.window) + 500
    n = m - len(small.window)                                             # fits beside the window before the change, not after
    ctx = gpu_api.Context(max_map_points=m, max_scan_points=n, plane_res=PLANE, line_res=LINE)
    ctx.map_archive(1 << 22)
    ctx.map_set_origin(t_small)
    ctx.map_set_points(cloud)
    assert ctx.map_size() == len(small.window)
    ctx.map_set_origin(t_big)
    new = _patches(rng, 1, n, [10.0, 10.0, 0.0], [10.0, 10.0, 0.0])
    with pytest.raises(gpu_api.SuperOdomError, match=r"\(-3\)"):
        ctx.map_add_surf(new)
    small.set_origin(ctx.map_origin())
    assert ctx.map_size() == len(small.window) == len(big.window)
    assert np.array_equal(ctx.map_download(0), small.download())
    assert np.array_equal(ctx.map_download_all(0), small.download_all())
    ctx.close()


# A 1.8 km corridor sampled at 0.4 m (720 k points), loaded in localization mode's order from a start 650 m from its -x end; scans
# along it in both directions, registered one after another (the window follows each prior)
STREET_START = -250.0
STREET_XS = [-250.0, -400.0, -550.0, -700.0, -850.0, -100.0, 100.0, 300.0, 500.0, 700.0, 880.0]
STREET_FAIL_WITHOUT = [-400.0, -550.0, -700.0, -850.0, 880.0]      # past the start block's -x face, and beyond the window (x > 775 m)
STREET_BOUND_M = 0.05                                                  # measured on an H100: 0.007-0.026 m


def _street():
    from superodom_b200 import synth
    sc = synth.make_scene(900.0, seed=77, half_extent_y=10.0)
    raw = synth.sample_surfaces(sc, 0.4)
    prior = np.concatenate([raw, np.ones((len(raw), 1), np.float32)], 1).astype(np.float32)
    scans = []
    for k, x in enumerate(STREET_XS):
        rng = np.random.default_rng(700 + k)
        yaw = float(rng.uniform(-0.3, 0.3))
        pose = np.concatenate([[x, float(rng.uniform(-1.5, 1.5)), 0.0], synth.quat_from_rotvec(np.array([0.0, 0.0, yaw]))])
        assert sc.free(pose[:3])
        scans.append((synth.make_scan(sc, "vlp16", pose, 800 + k), pose, synth.perturb_pose(pose, 900 + k)))
    return prior, scans


def _street_ctx(gpu_api, prior, archive):
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=1 << 16, plane_res=0.4, line_res=0.2)
    if archive:
        ctx.map_archive(1 << 20)
    ctx.map_set_origin([STREET_START, 0.0, 0.0])                          # setOrigin(start), then the prior-map load
    ctx.map_set_points(prior)
    return ctx


def test_localization_on_a_prior_map_longer_than_the_window(gpu_api):
    """With the archive every scan along the corridor converges within STREET_BOUND_M of the truth (the largest error measured on
    an H100 is in DESIGN.md section 4); without it the load keeps only the window, and the scans past the start block's -x face and
    beyond the window fail (NOT_ENOUGH_FEATURES, no correspondences, or off by more than a metre)."""
    prior, scans = _street()
    ctx = _street_ctx(gpu_api, prior, True)
    assert ctx.map_size() < len(prior) and ctx.map_size() + ctx.map_archive_info(0)[0] == len(prior)
    errs = []
    for scan, truth, guess in scans:
        r = ctx.register(scan, guess, 20, 0)
        errs.append(float(np.linalg.norm(np.array(r.pose)[:3] - truth[:3])))
        assert r.status == 0, (truth[0], r.status)
    print("street: position error per scan (m):", " ".join(f"{x:+.0f}:{e:.4f}" for x, e in zip(STREET_XS, errs)))
    assert max(errs) < STREET_BOUND_M, errs
    ctx.close()
    for scan, truth, guess in scans:
        if truth[0] not in STREET_FAIL_WITHOUT:
            continue
        ctx = _street_ctx(gpu_api, prior, False)
        r = ctx.register(scan, guess, 20, 0)
        err = float(np.linalg.norm(np.array(r.pose)[:3] - truth[:3]))
        assert r.status != 0 or err > 1.0, (truth[0], r.status, err)
        ctx.close()


def _sequence_results(gpu_api, archive_cap, off_after=False):
    """Loads, inserts, shifts inside the window and registrations of the tiny case: nothing ever leaves the window."""
    c0 = get_case("tiny", 0)
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=1 << 17, plane_res=PLANE, line_res=LINE)
    if archive_cap is not None:
        ctx.map_archive(archive_cap)
        if off_after:
            ctx.map_archive(0)
    ctx.map_set_origin(c0["pose_true"][:3])
    ctx.map_add_scan(c0["scan_xyzi"], c0["pose_true"])
    ctx.map_set_points(np.concatenate([ctx.map_download(0), c0["map_xyzi"][::2]]))
    out = [ctx.map_download(0)]
    q = c0["map_xyzi"][::7, :3] + np.float32(0.05)
    for i in range(1, 4):
        c = get_case("tiny", i)
        r = ctx.register(c["scan_xyzi"], c["pose_prior"], 5, 0)
        ctx.map_add_registered_scan(np.array(r.pose))
        out += [np.frombuffer(b"".join(_fields(r)), np.uint8), ctx.map_download(0), *ctx.knn(q, 5, 0.0)]
    ctx.map_shift([5.0, -3.0, 0.0])
    out += [ctx.map_download(0), ctx.map_origin()]
    if archive_cap is not None:
        assert ctx.map_archive_info(0)[:2] == (0, 0)
    ctx.close()
    return out


def test_archive_off_or_idle_changes_nothing(gpu_api):
    """With the archive on but no block ever leaving the window, or turned on and off again, a sequence of loads, inserts, shifts
    and registrations gives what a context without it gives: downloads, k-NN and so_icp_results (timings aside), bit for bit."""
    ref = _sequence_results(gpu_api, None)
    for cap, off in [(1 << 20, False), (1 << 20, True)]:
        got = _sequence_results(gpu_api, cap, off)
        assert len(got) == len(ref)
        for a, b in zip(ref, got):
            assert np.array_equal(a, b)


def test_shim_prior_map_beyond_the_window(gpu_api, tmp_path):
    """LidarSlam.hpp in localization mode's order -- setArchive, setOrigin(start), readPointCloud + loadPriorMap -- keeps the whole
    prior map; after a far shift and the return the whole map is unchanged, and writePointCloud(getWholeMap()) saves it bit for bit."""
    from superodom_b200 import build
    lib = build.build()
    exe = str(tmp_path / "archive_shim_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "archive_shim_test.cpp"), "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)])
    _, cloud = _scene(34)
    prior = tmp_path / "prior.pcd"
    hdr = (f"VERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\nCOUNT 1 1 1 1\nWIDTH {len(cloud)}\nHEIGHT 1\n"
           f"POINTS {len(cloud)}\nDATA binary\n")
    prior.write_bytes(hdr.encode() + cloud.tobytes())
    out = subprocess.run([exe, str(prior), str(tmp_path / "out.pcd"), "1600"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows = [list(map(int, ln.split())) for ln in out.stdout.split("\n") if ln.strip()]
    model = ArchiveModel(1 << 22, 1 << 20, (0, 0, 0))
    model.set_points(cloud)
    assert rows[0] == [len(model.window), model.archived_points(), len(cloud)]
    assert rows[1][2] == rows[2][2] == len(cloud) and rows[1][:2] != rows[0][:2]
    assert rows[1][0] + rows[1][1] == rows[2][0] + rows[2][1] == len(cloud)
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=4096, plane_res=0.4)
    ctx.map_archive(1 << 22)
    ctx.map_set_origin([0.0, 0.0, 0.0])
    ctx.map_set_points(cloud)
    whole = ctx.map_download_all(0)
    assert np.array_equal(whole, model.download_all())
    raw = (tmp_path / "out.pcd").read_bytes()
    body = raw[raw.index(b"DATA binary\n") + len(b"DATA binary\n"):]
    assert np.array_equal(np.frombuffer(body, np.float32).reshape(-1, 4), whole)
    ctx.close()

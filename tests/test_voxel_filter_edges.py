"""The device's pcl::VoxelGrid filters against the restatement in oracle/voxel_grid_numpy.py, bit for bit, where kernels go wrong: points on
and one ulp off voxel faces, products x * (1/leaf) that round onto an integer, dense voxels whose float sums depend on their order,
voxel indices at the edges of narrow key layouts, PCL's int32 overflow test on both sides of its threshold, non-finite input, the
leaf rule's thresholds, block faces of the map inserts, and a window far from the world origin.

Filters: so_scan_prefilter (fixed leaf and automatic), so_scan_extract_edges with voxel_leaf, and the surf and edge map inserts."""
import numpy as np
import pytest

from oracle import voxel_grid_numpy as vg
from conftest import get_case

pytestmark = pytest.mark.gpu

INF = np.float32(np.inf)


def _same(got, ref):
    got = np.ascontiguousarray(got, np.float32).reshape(-1, 4)
    ref = np.ascontiguousarray(ref, np.float32).reshape(-1, 4)
    return got.shape == ref.shape and np.array_equal(got.view(np.uint32), ref.view(np.uint32))


def _ctx(api, **kw):
    kw.setdefault("plane_res", 0.2)
    return api.Context(max_map_points=1 << 20, max_scan_points=1 << 17, **kw)


def _prefilter(ctx, cloud, leaf):
    out, lr, pr, _ = ctx.scan_prefilter(cloud, 0.1, leaf, False)
    assert pr == np.float32(leaf)
    m, _, _, _ = ctx.scan_prefilter(cloud, 0.1, leaf, False, download=False)     # the count left for so_register_prefiltered
    assert m == len(out)
    return out


def _xyzi(xyz, rng):
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    return np.concatenate([xyz, rng.uniform(0, 255, size=(len(xyz), 1)).astype(np.float32)], 1)


def _face_values(leaf, ks):
    """k * leaf in float32 and one ulp either side, for every k; with the floats a few ulps below k * leaf whose float product
    with 1/leaf rounds up onto k.  Returns (values, number of the round-up values)."""
    inv = vg.inverse_leaf(leaf)
    vals, up = [np.float32(0.0), np.float32(-0.0)], 0
    for k in ks:
        c = np.float32(k * leaf)
        vals += [np.nextafter(c, -INF), c, np.nextafter(c, INF)]
        x = c
        for _ in range(4):
            x = np.nextafter(x, -INF)
            if np.float32(x * inv) == np.float32(k) and np.float64(x) * np.float64(inv) < k:
                vals.append(x)
                up += 1
    return np.array(vals, np.float32), up


# --------------------------------------------------------------------------------------------------- scan pre-filter
@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.25, 0.3, 0.4, 0.8])
def test_voxel_faces(gpu_api, leaf):
    """Coordinates on voxel faces, one ulp off them, +-0 and negatives, in every axis; points repeated with other intensities."""
    rng = np.random.default_rng(int(leaf * 100))
    vals, up = _face_values(leaf, range(-40, 41))
    if leaf != 0.25:                                     # 1/0.25 = 4: every product is exact, nothing rounds
        assert up > 0
    c = _xyzi(rng.choice(vals, size=(6000, 3)), rng)
    c = np.concatenate([c, _xyzi(c[::3, :3], rng)], 0)
    ctx = _ctx(gpu_api)
    ref = vg.voxel_grid(c, leaf)
    assert not vg.falls_back(c, leaf) and len(ref) < len(c)
    assert _same(_prefilter(ctx, c, leaf), ref)
    ctx.close()


def test_dense_voxel(gpu_api):
    """10 000 points in one voxel with intensities 1e6 next to 1e-3 (the float sum depends on its order), next to single-point
    voxels."""
    rng = np.random.default_rng(3)
    dense = _xyzi(rng.uniform(0.2001, 0.3999, size=(10000, 3)), rng)
    dense[:, 3] = np.where(np.arange(10000) % 2 == 0, np.float32(1e6), np.float32(1e-3)) * rng.uniform(0.5, 1.5, 10000).astype(np.float32)
    fwd = np.float32(0)
    for v in dense[:, 3]:
        fwd = np.float32(fwd + v)
    bwd = np.float32(0)
    for v in dense[::-1, 3]:
        bwd = np.float32(bwd + v)
    assert fwd != bwd                                    # accumulation order shows in the result
    single = _xyzi((np.arange(300)[:, None] * np.float32(0.2) + np.float32(2.1)) * np.array([1, -1, 1], np.float32), rng)
    c = np.concatenate([single[:150], dense, single[150:]], 0)
    ctx = _ctx(gpu_api)
    ref = vg.voxel_grid(c, 0.2)
    assert len(ref) == 301
    assert _same(_prefilter(ctx, c, 0.2), ref)
    ctx.close()


def _flat(leaf, idx, rng, axes=1):
    """Two points in each voxel (i, 0, 0) -- or (i, j, 0) with axes=2 -- i, j in idx: centre and a point nearer its lower face."""
    inv = vg.inverse_leaf(leaf)
    idx = np.asarray(idx, np.int64)
    grid = np.stack(np.meshgrid(idx, idx, indexing="ij"), -1).reshape(-1, 2) if axes == 2 else np.stack([idx, np.zeros_like(idx)], 1)
    pts = []
    for f in (0.5, 0.2):
        xyz = np.zeros((len(grid), 3), np.float32)
        xyz[:, 0] = ((grid[:, 0] + f) * leaf).astype(np.float32)
        xyz[:, 1] = ((grid[:, 1] + f) * leaf).astype(np.float32) if axes == 2 else np.float32(0.3 * leaf)
        xyz[:, 2] = np.float32(0.3 * leaf)
        assert np.array_equal(np.floor(xyz[:, :2] * inv).astype(np.int64), grid)
        pts.append(_xyzi(xyz, rng))
    return np.concatenate(pts, 0), len(grid)


NARROW = [-4097, -4096, -1, 0, 4095, 4096]
WIDE = [-65537, -65536, -4097, -4096, 0, 4095, 4096, 65535, 65536]


@pytest.mark.parametrize("leaf", [0.2, 0.25])
@pytest.mark.parametrize("idx,axes", [(NARROW, 1), (WIDE, 1), (NARROW, 2), ([-8193, -8192, 0, 8191, 8192], 2)])
def test_key_ranges(gpu_api, leaf, idx, axes):
    """Voxel indices at +-4096 and +-65536 on flat clouds that PCL filters (dy = dz = 1), and at +-4096 and +-8192 on flat clouds
    with dz = 1: every voxel stays its own."""
    rng = np.random.default_rng(len(idx) * axes)
    c, n_vox = _flat(leaf, idx, rng, axes)
    ref = vg.voxel_grid(c, leaf)
    assert not vg.falls_back(c, leaf) and len(ref) == n_vox
    ctx = _ctx(gpu_api)
    assert _same(_prefilter(ctx, c, leaf), ref)
    ctx.close()


def test_far_pair(gpu_api):
    """(0.1, 0.1, 0.1) and (26 214.5, 0.1, 0.1) at leaf 0.2 are 131 072 voxels apart: two points out, each unchanged."""
    c = np.array([[0.1, 0.1, 0.1, 1.0], [26214.5, 0.1, 0.1, 2.0]], np.float32)
    ctx = _ctx(gpu_api)
    out = _prefilter(ctx, c, 0.2)
    assert _same(out, c) and _same(out, vg.voxel_grid(c, 0.2))
    ctx.close()


def _threshold_cloud(z_top, rng):
    """At leaf 0.25 (every product exact): x, y in [0, 255.75] and z in [0, z_top], NaN rows in between."""
    c = _xyzi(np.concatenate([rng.uniform(0, 255.75, size=(2000, 2)), rng.uniform(0, z_top, size=(2000, 1))], 1), rng)
    c[0, :3] = 0.0
    c[1, :3] = (255.75, 255.75, z_top)
    c = np.concatenate([c, _xyzi(c[::4, :3], rng)], 0)                  # voxels of two points
    c[7::211, 1] = np.nan
    return c


def test_overflow_threshold(gpu_api):
    """dx dy dz = 1024 * 1024 * 2048 = 2^31 returns the input verbatim, NaN rows included; 1024 * 1024 * 2047 is filtered."""
    rng = np.random.default_rng(5)
    ctx = _ctx(gpu_api)
    over = _threshold_cloud(511.75, rng)
    assert vg.extent(over, 0.25) == (1024, 1024, 2048) and vg.falls_back(over, 0.25)
    out = _prefilter(ctx, over, 0.25)
    assert _same(out, over) and np.isnan(out[7, 1])
    under = _threshold_cloud(511.5, rng)
    assert vg.extent(under, 0.25) == (1024, 1024, 2047) and not vg.falls_back(under, 0.25)
    ref = vg.voxel_grid(under, 0.25)
    assert len(ref) < len(under) - 400 and np.isfinite(ref).all()
    assert _same(_prefilter(ctx, under, 0.25), ref)
    # +-4096 voxels on all three axes: 8194^3 cells, PCL falls back
    c, _ = _flat(0.25, NARROW, rng, 2)
    c[::5, 2] = np.float32(4096.3 * 0.25)
    c[1::5, 2] = np.float32(-4096.7 * 0.25)
    assert vg.falls_back(c, 0.25)
    assert _same(_prefilter(ctx, c, 0.25), c)
    ctx.close()


def test_scaled_scan_falls_back(gpu_api):
    """The cfg1 scan with every 997th point scaled by 400 spans about 7e13 voxels at leaf 0.2: returned as it came."""
    s = get_case("cfg1")["scan_xyzi"].copy()
    s[::1000, 0] = np.nan
    s[5::997, :3] *= np.float32(400.0)
    assert vg.falls_back(s, 0.2)
    ctx = _ctx(gpu_api)
    assert _same(_prefilter(ctx, s, 0.2), s)
    ctx.close()


def test_non_finite_input(gpu_api):
    """NaN and +-inf in each coordinate are skipped; a cloud of non-finite points alone and the empty cloud give nothing."""
    rng = np.random.default_rng(6)
    c = _xyzi(rng.uniform(-5, 5, size=(3000, 3)), rng)
    k = 0
    for a in range(3):
        for v in (np.nan, np.inf, -np.inf):
            c[k::97, a] = v
            k += 1
    ref = vg.voxel_grid(c, 0.2)
    assert len(ref) > 0 and np.isfinite(ref).all()
    ctx = _ctx(gpu_api)
    assert _same(_prefilter(ctx, c, 0.2), ref)
    bad = c[~np.isfinite(c[:, :3]).all(1)]
    assert len(bad) > 9
    assert len(_prefilter(ctx, bad, 0.2)) == 0
    assert len(_prefilter(ctx, np.zeros((0, 4), np.float32), 0.2)) == 0
    ctx.close()


def _stat_cloud(x, y, z):
    return np.array([[x, y, z, 1.0], [-x, -y, -z, 2.0]], np.float32)


def test_auto_statistic(gpu_api):
    """The leaf rule with auto on: a NaN point (statistic NaN, leaves unchanged), statistics of exactly 25 and 65 (unchanged) and
    one ulp of mean|x| past each (changed)."""
    five = np.float32(5.0)
    lo, hi = np.nextafter(five, np.float32(0)), np.nextafter(five, INF)
    nan = _stat_cloud(5, 5, 1)
    nan[0, 1] = np.nan
    cases = [(nan, None, (0.2, 0.4)), (_stat_cloud(5, 5, 1), 25.0, (0.2, 0.4)), (_stat_cloud(5, 13, 1), 65.0, (0.2, 0.4)),
             (_stat_cloud(lo, 5, 1), None, (0.1, 0.2)), (_stat_cloud(hi, 13, 1), None, (0.4, 0.8))]
    ctx = _ctx(gpu_api)
    for c, stat, leaves in cases:
        avg_ref = vg.adjust_statistic(c)
        if stat is not None:
            assert avg_ref == stat
        assert vg.adjust_leaves(avg_ref, 0.2, 0.4) == tuple(float(np.float32(v)) for v in leaves)
        out, lr, pr, avg = ctx.scan_prefilter(c, 0.2, 0.4, True)
        assert (np.isnan(avg) and np.isnan(avg_ref)) or avg == avg_ref, (avg, avg_ref)
        assert (lr, pr) == (np.float32(leaves[0]), np.float32(leaves[1]))
        assert _same(out, vg.voxel_grid(c, leaves[1]))
    ctx.close()


# ------------------------------------------------------------------------------------------------------ edge extraction
@pytest.mark.parametrize("leaf", [0.01, 0.02, 0.03, 0.05, 0.1, 0.25, 0.3, 0.8])
def test_edge_voxel_leaf(gpu_api, leaf):
    """so_scan_extract_edges with voxel_leaf: the restatement of the plain edge cloud; at leaf 0.01 the cloud's 4 450 x 4 620 x 840
    voxels pass 2^31 and at 0.02 its 2 221 x 2 309 x 419 do: the cloud comes back unfiltered."""
    from superodom_b200 import synth
    case = get_case("cfg1", 0)
    rec = synth.make_ring_scan(case["scene"], "vlp16", case["pose_true"], 11)
    ctx = _ctx(gpu_api)
    plain = ctx.scan_extract_edges(rec)
    got = ctx.scan_extract_edges(rec, voxel_leaf=leaf)
    assert vg.falls_back(plain, leaf) == (leaf <= 0.02)
    assert _same(got, vg.voxel_grid(plain, leaf))
    ctx.close()


# ---------------------------------------------------------------------------------------------------------- map inserts
def _ulps(values):
    c = np.asarray(values, np.float32)
    return np.concatenate([np.nextafter(c, -INF), c, np.nextafter(c, INF)])


def _block_face_cloud(leaf, rng, centre_x=0.0):
    """Points with one coordinate on a block face (centre + 25 + 50 k m, k = -3..2), on a voxel face next to it, or one ulp off
    either; the other two coordinates on or next to voxel faces around the centre."""
    faces = [25.0 + 50.0 * k + j * leaf for k in range(-3, 3) for j in (-2, -1, 0, 1, 2)]
    near = [k * leaf for k in range(-8, 9)]
    parts = []
    for a in range(3):
        off = centre_x if a == 0 else 0.0
        xyz = np.stack([rng.choice(_ulps(np.add(near, centre_x if b == 0 else 0.0)), size=1500) for b in range(3)], 1)
        xyz[:, a] = rng.choice(_ulps(np.add(faces, off)), size=1500)
        parts.append(xyz)
    return _xyzi(np.concatenate(parts, 0), rng)


def _insert_twice(ctx, add, leaf, a, b, origin):
    """Insert a, then b (b's points in a's voxels: old centroids and new points share them, old first); compare after each."""
    from oracle import oracle as O
    ref = np.zeros((0, 4), np.float32)
    for cloud in (a, b):
        add(cloud)
        ref = vg.map_insert(ref, cloud, leaf, origin)
        got = ctx.map_download(0)
        exp = ref[O.cube_order(ref, origin)]
        assert _same(got, exp), (leaf, len(got), len(exp))
    return ref


@pytest.mark.parametrize("store", ["surf", "edge"])
@pytest.mark.parametrize("leaf", [0.05, 0.1, 0.2, 0.4])
def test_map_insert_block_faces(gpu_api, store, leaf):
    """Points on block faces and voxel faces through the surf insert (leaf planeRes) and the edge insert (leaf lineRes)."""
    rng = np.random.default_rng(int(leaf * 1000) + (store == "edge"))
    a = _block_face_cloud(leaf, rng)
    b = _xyzi(a[::3, :3], rng)
    if store == "surf":
        ctx = _ctx(gpu_api, plane_res=leaf)
        add = ctx.map_add_surf
    else:
        ctx = _ctx(gpu_api, plane_res=0.4, line_res=leaf)
        add = ctx.map_add_edge
    ref = _insert_twice(ctx, add, leaf, a, b, (10, 10, 5))
    assert len(ref) < len(a) + len(b)
    ctx.close()


@pytest.mark.parametrize("leaf", [0.05, 0.2])
def test_map_insert_far_from_the_world_origin(gpu_api, leaf):
    """A window 10 km from the world origin with the block archive on: the block-local voxel index of the insert at |x / leaf| up to
    2e5."""
    rng = np.random.default_rng(9)
    ctx = _ctx(gpu_api, plane_res=leaf)
    ctx.map_archive(1 << 20)
    ctx.map_set_origin([10000.0, 0.0, 0.0])
    origin = tuple(int(v) for v in ctx.map_origin())
    a = _block_face_cloud(leaf, rng, centre_x=10000.0)
    assert np.abs(a[:, 0]).min() > 9000
    b = _xyzi(a[::3, :3], rng)
    _insert_twice(ctx, ctx.map_add_surf, leaf, a, b, origin)
    ctx.close()


# ------------------------------------------------------------------------------------------------------------------ chain
def test_fallback_prefilter_chain(gpu_api):
    """A pre-filter that falls back leaves the verbatim cloud on the device: registering and inserting it from there gives the
    same bits as so_register and so_map_add_scan of that cloud."""
    case = get_case("cfg1")
    s = case["scan_xyzi"].copy()
    s[::1000, 0] = np.nan
    s[5::997, :3] *= np.float32(400.0)
    ctxs = []
    for _ in range(2):
        ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=262144, plane_res=0.2)
        ctx.map_set_points(case["map_xyzi"])
        ctxs.append(ctx)
    a, b = ctxs
    m, lr, pr, _ = a.scan_prefilter(s, 0.2, 0.2, False, download=False)
    assert m == len(s) and (lr, pr) == (np.float32(0.2), np.float32(0.2))
    ra = a.register_prefiltered(case["pose_prior"], 5, 2000)
    a.map_add_registered_scan(np.array(ra.pose))
    b.map_set_resolution(0.2, 0.2)
    rb = b.register(s, case["pose_prior"], 5, 2000)
    b.map_add_scan(s, np.array(rb.pose))
    assert np.array_equal(np.array(ra.pose), np.array(rb.pose)) and ra.n_iterations == rb.n_iterations and ra.status == rb.status
    assert np.array_equal(np.array(ra.cov), np.array(rb.cov))
    assert _same(a.map_download(0), b.map_download(0))
    for ctx in ctxs:
        ctx.close()

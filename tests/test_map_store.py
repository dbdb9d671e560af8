"""The map store's one pipeline (so_map.cu): filter stage + index stage on the paths no other test reaches -- a shift that rolls
off some blocks, an insert that opens more blocks than the index was sized for, rebuilds that change nothing, and a map too large
for the dense cell table."""
import numpy as np
import pytest

from conftest import get_case

pytestmark = pytest.mark.gpu

CAPACITY_MSG = "map spans too many 50 m blocks for the dense cell table (n_slots * nb^3 >= 2^31)"


def _gi(idx):
    g = idx.astype(np.int64)
    g[idx == 0xFFFFFFFF] = -1
    return g


def _cloud(rng, n, lo, hi):
    xyz = rng.uniform(lo, hi, size=(n, 3))
    return np.concatenate([xyz, rng.uniform(0, 255, size=(n, 1))], 1).astype(np.float32)


def _assert_knn_matches(ctx, oracle_mod, xyzi, origin, q):
    om = oracle_mod.OracleMap()
    om.set_origin(origin)
    om.set_points(xyzi)
    gi, gd = ctx.knn(q, 5, 0.0)
    oi, od, of = om.knn(q, 5, 0)
    assert of.any()
    assert np.array_equal(_gi(gi)[of], oi[of]) and np.array_equal(gd[of], od[of])
    assert (gi[~of] == 0xFFFFFFFF).all()
    return om


def test_shift_rolls_off_some_blocks(gpu_api, oracle_mod):
    """A shift that drops the blocks rolled off the grid and keeps the others: the store holds the points on the grid under the
    new origin, in their order, and its index answers k-NN exactly."""
    from superodom_b200 import synth
    rng = np.random.default_rng(21)
    xyzi = _cloud(rng, 300000, [-520.0, -40.0, -2.0], [520.0, 40.0, 6.0])
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=65536, plane_res=0.2)
    ctx.map_set_points(xyzi)
    ctx.map_shift([-450.0, 0.0, 0.0])
    origin = ctx.map_origin()
    assert list(origin) == [12, 10, 5]
    on_grid = synth.block_linear(synth.block_of(xyzi[:, :3], origin)) >= 0
    kept = xyzi[on_grid]
    assert 0 < len(kept) < len(xyzi) and ctx.map_size() == len(kept)
    got = ctx.map_download(0)
    assert got.shape == kept.shape and np.array_equal(got, kept[oracle_mod.cube_order(kept, origin)])
    q = kept[::40, :3] + rng.normal(0, 0.1, size=kept[::40, :3].shape).astype(np.float32)
    q = np.concatenate([q, xyzi[~on_grid][:500, :3]])                     # points of the dropped blocks: off the grid now
    _assert_knn_matches(ctx, oracle_mod, kept, origin, q)
    ctx.close()


def test_insert_past_the_slot_bound(gpu_api, oracle_mod):
    """An insert sizes its index for the store's blocks plus four new ones; one that opens more indexes again after growing the
    cell table.  Contents, k-NN and the 5x5x3 counts of every block equal the restatements."""
    rng = np.random.default_rng(22)
    ctx = gpu_api.Context(max_map_points=1 << 21, max_scan_points=65536, plane_res=0.2)
    a = _cloud(rng, 100000, [-20.0, -20.0, -2.0], [20.0, 20.0, 6.0])       # one block
    ctx.map_add_surf(a)
    ref = oracle_mod.map_insert_numpy(np.zeros((0, 4), np.float32), a, 0.2)
    b = _cloud(rng, 200000, [-160.0, -110.0, -2.0], [160.0, 110.0, 6.0])    # 7 x 5 blocks
    ctx.map_add_surf(b)
    ref2 = oracle_mod.map_insert_numpy(ref, b, 0.2)
    got = ctx.map_download(0)
    assert got.shape == ref2.shape and np.array_equal(got, ref2[oracle_mod.cube_order(ref2)])
    q = ref2[::30, :3] + rng.normal(0, 0.05, size=ref2[::30, :3].shape).astype(np.float32)
    om = _assert_knn_matches(ctx, oracle_mod, ref2, [10, 10, 5], q)
    for k in range(11):
        for j in range(21):
            for i in range(21):
                assert ctx.map_counts_5x5([i, j, k]) == om.counts_5x5([i, j, k]), (i, j, k)
    ctx.close()


def test_rebuild_without_changes_is_bit_equal(gpu_api):
    """Two rebuilds (to a resolution with another cell count per block and back) leave the store and its index as they were."""
    case = get_case("cfg1")
    ctx = gpu_api.Context(max_map_points=1 << 20, max_scan_points=65536, plane_res=0.2)
    ctx.map_set_points(case["map_xyzi"])
    q = case["map_xyzi"][::5, :3] + np.random.default_rng(23).normal(0, 0.1, size=case["map_xyzi"][::5, :3].shape).astype(np.float32)
    before = ctx.map_download(0), ctx.map_download(1, [10, 10, 5]), ctx.knn(q, 5, 0.0), ctx.knn(q, 5, 0.6)
    ctx.map_set_resolution(0.1, 0.4)                                       # nb 129 -> 91
    assert ctx.map_download(0).shape == before[0].shape
    ctx.map_set_resolution(0.1, 0.2)
    after = ctx.map_download(0), ctx.map_download(1, [10, 10, 5]), ctx.knn(q, 5, 0.0), ctx.knn(q, 5, 0.6)
    assert np.array_equal(after[0], before[0]) and np.array_equal(after[1], before[1])
    for (gi0, gd0), (gi1, gd1) in zip(before[2:], after[2:]):
        assert np.array_equal(gi0, gi1) and np.array_equal(gd0, gd1)
    ctx.close()


def _expect_capacity(gpu_api, call, *args):
    with pytest.raises(gpu_api.SuperOdomError) as e:
        call(*args)
    assert "(-3)" in str(e.value) and CAPACITY_MSG in str(e.value), str(e.value)


@pytest.mark.parametrize("how", ["map_set_points", "map_add_surf"])
def test_capacity_error_leaves_the_store_dirty(gpu_api, how):
    """One point in each of 304 blocks at planeRes 0.05 (nb = 192): 304 * 192^3 cells reach 2^31.  The call fails without growing
    the cell table for them, every later call that reads the map fails the same way, and a valid cloud recovers the store."""
    import torch
    gi, gj = np.meshgrid(np.arange(21), np.arange(21), indexing="ij")
    blocks = np.stack([gi.ravel(), gj.ravel()], 1)[:304]
    pts = np.zeros((304, 4), np.float32)
    pts[:, 0] = (blocks[:, 0] - 10) * 50.0
    pts[:, 1] = (blocks[:, 1] - 10) * 50.0
    ctx = gpu_api.Context(max_map_points=1 << 16, max_scan_points=4096, plane_res=0.05)
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info()[0]
    _expect_capacity(gpu_api, getattr(ctx, how), pts)
    _expect_capacity(gpu_api, ctx.map_download, 0)
    _expect_capacity(gpu_api, ctx.map_counts_5x5, [10, 10, 5])
    assert free0 - torch.cuda.mem_get_info()[0] < (4 << 30)             # 303 slots alone would take 8.6 GB
    small = pts[:3].copy()                                              # blocks (0, 0, 5), (0, 1, 5), (0, 2, 5): download order
    ctx.map_set_points(small)
    assert np.array_equal(ctx.map_download(0), small)
    assert ctx.map_counts_5x5([0, 2, 5]) == 3
    ctx.close()

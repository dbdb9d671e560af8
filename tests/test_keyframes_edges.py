"""so_map_from_keyframes at scale and at its edges, against the restatement in keyframe_map_numpy.py (as test_keyframes.py's
test_rebuild_equals_the_definition compares it): both stores, window and archive, bit for bit.

Code paths reached: k_kf_transform's binary search over a segment table of 320 entries with zero-length entries (keyframes without an
edge cloud) at the first, middle and last list positions, and an edge union with no point at all; duplicate ids in the list; points
on 50 m block faces and voxel faces; a rebuild that keeps nothing; and the block-box sort key at its limit: a 65 536 x 65 536 x 1 box
(bb = 32, whose decode divides by nx * ny = 2^32), the first box that needs 33 bits, and at a 0.02 m leaf the first box past
3 vb + bb = 63."""
import numpy as np
import pytest

import keyframe_map_numpy as KM
import loop_detection_numpy as LD
from test_keyframes import SO_ERR_CAPACITY, _ctx, _err, _merged, _reference, _rows

IDENT = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])


def _cloud(seed, n, half=15.0):
    rng = np.random.default_rng(seed)
    return np.c_[rng.uniform(-half, half, (n, 2)), rng.uniform(-2.0, 5.0, n), rng.uniform(0, 1, n)].astype(np.float32)


def _src(api, clouds, edges):
    """A context holding one keyframe per cloud (edge cloud or None), kept through a registration on its empty map."""
    ctx = _ctx(api)
    ctx.keyframe_reserve(max(sum(len(c) for c in clouds), 1), len(clouds))
    for c, e in zip(clouds, edges):
        ctx.register(c, IDENT, 1, 0, edge_xyzi=e)
        ctx.keyframe_add_registered(IDENT)
    return ctx


def _yaw(a):
    return np.array([0.0, 0.0, np.sin(a / 2), np.cos(a / 2)])


def _state(dst):
    return tuple(x.tobytes() for x in (dst.map_download(0), dst.map_download_all(0), dst.map_download_all(1))) + \
        tuple(dst.map_archive_info(s)[0] for s in (0, 1))


def _check(api, src, ids, poses, archive, stores=3, leaf=0.2, dst=None):
    """Rebuild into dst (a new context unless given) and compare it with the restatement -> (dst, surf window, edge window)."""
    if dst is None:
        dst = _ctx(api, max_map_points=1 << 22, plane_res=leaf)
        if archive:
            dst.map_archive(1 << 22)
    dst.map_from_keyframes(src, ids, poses, stores)
    origin = dst.map_origin()
    ws, arcs = _reference(src, ids, poses, 0, leaf, tuple(origin), archive)
    we, arce = _reference(src, ids, poses, 1, 0.1, tuple(origin), archive)
    if stores != 3:
        we, arce = np.zeros((0, 4), np.float32), {}
    assert dst.map_download(0).tobytes() == _merged(we, ws, origin).tobytes()
    for store, (w, a) in enumerate(((ws, arcs), (we, arce))):
        assert _rows(dst.map_download_all(store)).tobytes() == _rows(KM.download_all(w, a)).tobytes(), store
        assert dst.map_archive_info(store)[0] == sum(len(b) for b in a.values()), store
    return dst, ws, we


# ------------------------------------------------------------------------------------------------------------- 1. scale, empty segments
@pytest.fixture(scope="module")
def many(gpu_api):
    n = 320
    clouds = [_cloud(i, 120) for i in range(n)]
    edges = [None if i % 5 == 0 else _cloud(10000 + i, 40) for i in range(n)]
    src = _src(gpu_api, clouds, edges)
    assert src.keyframe_info()[0] == n and len(src.keyframe_download(0, 1)) == 0 and len(src.keyframe_download(1, 1)) > 0
    yield src, n
    src.close()


@pytest.mark.gpu
def test_scale_and_empty_edge_segments(gpu_api, many):
    src, n = many
    rng = np.random.default_rng(2)
    ids = rng.permutation(n).astype(np.int32)
    bare = [i for i in ids if i % 5 == 0]
    for pos, i in zip((0, n // 2, n - 1), bare[:3]):                    # keyframes without edges first, in the middle and last
        j = int(np.flatnonzero(ids == i)[0])
        ids[[pos, j]] = ids[[j, pos]]
    assert all(ids[p] % 5 == 0 for p in (0, n // 2, n - 1))
    # a trajectory over about 80 x 8 blocks: most of it leaves the window and goes to the archive
    t = np.c_[np.linspace(-2000.0, 2000.0, n), 200.0 * np.sin(np.linspace(0, 6, n)), np.zeros(n)]
    poses = np.c_[t, np.array([_yaw(a) for a in rng.uniform(-3, 3, n)])]
    dst, ws, we = _check(gpu_api, src, ids, poses, True)
    assert len(ws) > 2000 and len(we) > 500 and dst.map_archive_info(0)[1] > 50
    dst.close()
    # every selected keyframe without an edge cloud: an empty edge union
    near = np.c_[rng.uniform(-100, 100, (40, 2)), np.zeros(40), np.array([_yaw(a) for a in rng.uniform(-3, 3, 40)])]
    dst, ws, we = _check(gpu_api, src, np.array(bare[:40], np.int32), near, False)
    assert len(ws) > 1000 and len(we) == 0 and len(dst.map_download_all(1)) == 0
    dst.close()


# ------------------------------------------------------------------------------------------------------------- 2. duplicate ids
@pytest.mark.gpu
@pytest.mark.parametrize("archive", [False, True])
def test_duplicate_ids(gpu_api, archive):
    from scipy.spatial.transform import Rotation
    src = _src(gpu_api, [_cloud(i, 200) for i in range(6)], [_cloud(50 + i, 60) for i in range(6)])
    tilt = Rotation.from_euler("xyz", [0.2, -0.1, 0.4]).as_quat()
    ids = np.array([2, 5, 2, 0], np.int32)
    poses = np.array([np.r_[3.0, 1.0, 0.0, _yaw(0.3)], IDENT, np.r_[-40.0, 7.0, 0.5, tilt], np.r_[800.0 if archive else 20.0, 0, 0, _yaw(1)]])
    dst, ws, _ = _check(gpu_api, src, ids, poses, archive)
    once = _check(gpu_api, src, ids[1:], poses[1:], archive)
    assert len(ws) > len(once[1])                                       # both copies of keyframe 2 are in the union
    once[0].close()
    dst.close()
    # a self-rebuild: the last pose of keyframe 2 wins, and its descriptor is described again
    before = src.keyframe_descriptors(np.arange(6), exclude_recent=0)
    if archive:
        src.map_archive(1 << 22)
    _check(gpu_api, src, ids, poses, archive, dst=src)
    want = np.array([IDENT] * 6)
    want[[2, 5, 0]] = poses[[2, 1, 3]]
    assert np.array_equal(src.keyframe_poses(), want)
    _, st = src.loop_candidates(np.arange(6), 3, stats=True, exclude_recent=0)
    assert st["n_described"] == 2                                       # 2 and 0 moved; 5 kept its pose
    after = src.keyframe_descriptors(np.arange(6), exclude_recent=0)
    assert np.array_equal(after[[1, 3, 4, 5]], before[[1, 3, 4, 5]]) and not np.array_equal(after[2], before[2])
    lo, hi = LD.describe_bounds(src.keyframe_download(2, 0), poses[2], LD.Opts())     # described at the last pose
    assert np.all(lo <= after[2]) and np.all(after[2] <= hi)
    src.close()


# ------------------------------------------------------------------------------------------------------------- 3. faces
@pytest.mark.gpu
@pytest.mark.parametrize("archive", [False, True])
def test_points_on_block_and_voxel_faces(gpu_api, archive):
    """Points at x, y on 50 m block faces (25 + 50 k) and on 0.2 m voxel faces, moved by identity, 90 and 180 deg yaws and
    translations by multiples of the leaf and of the block."""
    ax = np.array([-25.0, 25.0, 75.0, 24.8, 25.2, 0.0, 0.2, 0.4, -0.2, -24.8, 49.8, 50.0], np.float32)
    g = np.stack(np.meshgrid(ax, ax, np.array([0.0, 0.2, -0.2, 24.8], np.float32), indexing="ij"), -1).reshape(-1, 3)
    cloud = np.c_[g, np.arange(len(g)) % 7].astype(np.float32)
    edge = cloud[::3].copy()
    src = _src(gpu_api, [cloud, cloud[::-1].copy()], [edge, None])
    ids = np.array([0, 1, 0, 0, 1, 0], np.int32)
    poses = np.array([IDENT, np.r_[0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0], np.r_[0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 1.0],
                      np.r_[50.0, -50.0, 0.0, 0, 0, 0, 1], np.r_[0.2 * 7, 0.2 * 3, 0.2, 0, 0, 0, 1], np.r_[25.0, 25.0, 0.0, _yaw(np.pi / 2)]])
    dst, ws, we = _check(gpu_api, src, ids, poses, archive)
    assert len(ws) > 500 and len(we) > 100
    dst.close()
    src.close()


# ------------------------------------------------------------------------------------------------------------- 4. nothing kept
@pytest.mark.gpu
def test_nothing_kept(gpu_api):
    src = _src(gpu_api, [_cloud(1, 200), _cloud(2, 200)], [_cloud(3, 50), None])
    dst = _ctx(gpu_api)
    dst.map_from_keyframes(src, [0, 1], [IDENT, IDENT], 3)
    assert dst.map_size() > 0 and len(dst.map_download_all(1)) > 0
    far = np.r_[1.0e4, -2.0e4, 0.0, 0, 0, 0, 1]                         # archive off, every point outside the window
    dst.map_from_keyframes(src, [0, 1], [far, far], 3)
    assert dst.map_size() == 0 and len(dst.map_download_all(0)) == 0 and len(dst.map_download_all(1)) == 0
    assert dst.map_archive_info(0)[0] == 0 and dst.map_archive_info(1)[0] == 0
    dst.close()
    src.close()


# ------------------------------------------------------------------------------------------------------------- 5. the block-box limit
def _corners(lo, hi):
    """Poses putting a small keyframe at the centres of world blocks lo and hi (x, y; z block 0)."""
    return np.array([np.r_[50.0 * lo[0], 50.0 * lo[1], 0.0, 0, 0, 0, 1], np.r_[50.0 * hi[0], 50.0 * hi[1], 0.0, 0, 0, 0, 1]])


@pytest.fixture(scope="module")
def small(gpu_api):
    src = _src(gpu_api, [_cloud(7, 300, half=10.0)], [_cloud(8, 100, half=10.0)])
    yield src
    src.close()


@pytest.mark.gpu
def test_block_box_of_2_to_the_32(gpu_api, small):
    """65 536 x 65 536 x 1 blocks (+-1 638 km): the largest box the key takes at 0.2 m; also 2^20 x 2^12 x 1."""
    ids = np.zeros(2, np.int32)
    for lo, hi in (((-32768, -32768), (32767, 32767)), ((-524288, -2048), (524287, 2047))):
        dst, ws, we = _check(gpu_api, small, ids, _corners(lo, hi), True)
        assert dst.map_archive_info(0)[1] == 2 and dst.map_archive_info(1)[1] == 2 and len(ws) == 0
        dst.close()


@pytest.mark.gpu
@pytest.mark.parametrize("leaf,lo,hi", [(0.2, (-32768, -32768), (32768, 32767)),     # 65 537 x 65 536: bb = 33
                                        (0.02, (-32768, -2048), (32767, 2047))])      # 2^28 blocks at vb = 12: 36 + 28 > 63
def test_block_box_past_the_key_is_refused(gpu_api, small, leaf, lo, hi):
    dst = _ctx(gpu_api, max_map_points=1 << 22, plane_res=leaf)
    dst.map_archive(1 << 22)
    near = np.array([np.r_[10.0, -5.0, 0.0, _yaw(0.5)], np.r_[5000.0, 0.0, 0.0, 0, 0, 0, 1]])   # one in the window, one archived
    dst.map_from_keyframes(small, [0, 0], near, 3)
    before = _state(dst)
    assert before[3] > 0
    assert _err(gpu_api, lambda: dst.map_from_keyframes(small, [0, 0], _corners(lo, hi), 3)) == SO_ERR_CAPACITY
    assert _state(dst) == before
    if leaf == 0.02:                                                   # half the box fits: 36 + 27 = 63
        _check(gpu_api, small, np.zeros(2, np.int32), _corners((-16384, -2048), (16383, 2047)), True, leaf=leaf, dst=dst)
    dst.close()

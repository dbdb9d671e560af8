"""The scan-order key carries a "dropped" bit (points a capped scan's decimation skips sort behind its survivors) only when a scan
of the chunk is capped.  Without one the bit is zero in every key, so leaving it out must give the very same order: the ordered
scan buffer (point, original index, place) and every result are compared byte for byte against SO_FORCE_DROP_BIT, which always
carries it."""
import numpy as np
import pytest

from conftest import get_case

SCAN = 28800                     # points of a cfg1 (VLP-16) scan


@pytest.fixture(scope="module")
def cfg1():
    case = get_case("cfg1")
    scans = [get_case("cfg1", i)["scan_xyzi"] for i in range(8)]
    priors = np.stack([get_case("cfg1", i)["pose_prior"] for i in range(8)])
    return case["map_xyzi"], scans, priors


def _run(api, monkeypatch, map_xyzi, scans, priors, force_drop_bit, max_surface_features=0, iters=3):
    if force_drop_bit:
        monkeypatch.setenv("SO_FORCE_DROP_BIT", "1")
    n_points = np.array([len(s) for s in scans], np.uint32)
    flat = np.ascontiguousarray(np.concatenate(scans, 0).astype(np.float32))
    ctx = api.Context(max_map_points=1 << 20, max_scan_points=int(n_points.max()), max_batch=len(scans), plane_res=0.2)
    ctx.map_set_points(map_xyzi)
    ctx.kernel_launches(reset=True)
    res = ctx.register_batch(flat, n_points, priors, iters, max_surface_features)
    launches = ctx.kernel_launches()
    order = ctx.ordered_scans(len(flat)).view(np.uint32)
    out = np.array([list(r.pose) + [r.status, r.n_iterations] + list(r.hist_obs) for r in res])
    ctx.close()
    monkeypatch.delenv("SO_FORCE_DROP_BIT", raising=False)
    return order, out, launches


def _check(api, monkeypatch, map_xyzi, scans, priors, **kw):
    ref_order, ref_out, ref_launches = _run(api, monkeypatch, map_xyzi, scans, priors, True, **kw)
    order, out, launches = _run(api, monkeypatch, map_xyzi, scans, priors, False, **kw)
    assert np.array_equal(order, ref_order)
    assert np.array_equal(out, ref_out)
    off = np.concatenate([[0], np.cumsum([len(s) for s in scans])])
    for s in range(len(scans)):          # every scan holds each of its original indices exactly once, at its own offset
        assert np.array_equal(np.sort(order[off[s]:off[s + 1], 3]), np.arange(len(scans[s]), dtype=np.uint32)), s
    return order, ref_launches, launches


@pytest.mark.gpu
@pytest.mark.parametrize("n_scans", [2, 8])
def test_uncapped_chunk(gpu_api, monkeypatch, cfg1, n_scans):
    map_xyzi, scans, priors = cfg1
    _, ref_launches, launches = _check(gpu_api, monkeypatch, map_xyzi, scans[:n_scans], priors[:n_scans])
    assert ref_launches - launches == 1          # one chunk: k_scan_finish has nothing to do and is not launched


@pytest.mark.gpu
def test_two_chunks_on_two_streams(gpu_api, monkeypatch, cfg1):
    map_xyzi, scans, priors = cfg1
    scans16 = scans + [s[::-1].copy() for s in scans]
    _check(gpu_api, monkeypatch, map_xyzi, scans16, np.concatenate([priors, priors]))


@pytest.mark.gpu
@pytest.mark.parametrize("max_surface_features", [0, 12000])
def test_mixed_scan_sizes(gpu_api, monkeypatch, cfg1, max_surface_features):
    # 12000: the long scans are capped and the short ones are not -- one chunk with both keeps the bit either way
    map_xyzi, scans, priors = cfg1
    lens = [SCAN, 9000, SCAN, 20000, 4500, SCAN, 700, 15000]
    mixed = [s[:n].copy() for s, n in zip(scans, lens)]
    _check(gpu_api, monkeypatch, map_xyzi, mixed, priors, max_surface_features=max_surface_features)


@pytest.mark.gpu
def test_key64(gpu_api, monkeypatch, cfg1):
    map_xyzi, scans, priors = cfg1
    order32 = _check(gpu_api, monkeypatch, map_xyzi, scans[:5], priors[:5])[0]
    monkeypatch.setenv("SO_FORCE_KEY64", "1")
    order64 = _check(gpu_api, monkeypatch, map_xyzi, scans[:5], priors[:5])[0]
    monkeypatch.delenv("SO_FORCE_KEY64")
    assert np.array_equal(order32, order64)


@pytest.mark.gpu
def test_off_map_points_sort_last(gpu_api, monkeypatch, cfg1):
    map_xyzi, scans, priors = cfg1
    rng = np.random.default_rng(7)
    far = []
    for s in scans[:5]:
        extra = s[rng.integers(0, len(s), 3000)].copy()
        extra[:, :3] += np.float32(5000.0)                   # far outside the map at any prior
        far.append(np.concatenate([extra[:1500], s, extra[1500:]]))
    order = _check(gpu_api, monkeypatch, map_xyzi, far, priors[:5])[0]
    n = len(far[0])
    for s in range(5):
        idx = order[s * n:(s + 1) * n, 3]
        off_map = (idx < 1500) | (idx >= 1500 + SCAN)
        assert off_map[-3000:].all() and not off_map[:-3000].any(), s

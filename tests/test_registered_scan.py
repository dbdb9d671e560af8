"""so_map_add_registered_scan inserts the scan the last single-scan registration left on the device, or refuses.

GPU: every call that overwrites the scan buffers without registering a scan to insert makes the insert fail with SO_ERR_ARG before
any device work, and the map stays as it was; calls that leave those buffers alone leave the insert as it was, in all three modes; a
context that never registered a scan inserts nothing."""
import numpy as np
import pytest

from test_optimized_undistortion import IDENTITY, _ctx, _moving_case

MODES = ["none", "approximated", "optimized"]


def _register(api, ctx, d, mode):
    """a single-scan registration of the mode -> the pose to insert at"""
    scan, prior = d["scan_xyzi"], d["prior"]
    if mode == "none":
        return np.array(ctx.register(scan, prior, 5, 2000).pose)
    if mode == "approximated":
        return np.array(ctx.register_undistort(scan, prior, api.undistort(d["pose_prev"], 0.1), 5, 2000).pose)
    return np.array(ctx.register_optimized(scan, prior, api.motion(0.1), 5, 2000).icp.pose)


def _overwriting_calls(api, d):
    """calls that overwrite d_scan or the registered scan's times and register nothing to insert"""
    scan, prior, n = d["scan_xyzi"], d["prior"], len(d["scan_xyzi"])
    plane_res = d["case"]["cfg"]["plane_res"]
    return {
        "so_scan_prefilter": lambda c: c.scan_prefilter(scan, 0.2, plane_res, auto_voxel_size=False, download=False),
        "so_scan_deskew": lambda c: c.scan_deskew(scan.copy(), 3, 0.0, [0.0, 1.0], [IDENTITY, IDENTITY]),
        "so_scan_extract_uniform": lambda c: c.scan_extract_uniform(scan, 3, 2, 0.5),
        "so_correspond": lambda c: c.correspond(scan, prior),
        "so_register_injected": lambda c: c.register_injected(scan, prior, 2, np.full((2, n, 5), -1, np.int64)),
        "so_register_batch_packed": lambda c: c.register_batch(scan, [n], prior[None], 5, 2000),
        "so_register_batch_strided": lambda c: c.register_batch(np.c_[scan, np.zeros(n, np.float32)], [n], prior[None], 5, 2000),
        "so_register_batch_edges": lambda c: c.register_batch_edges(scan, [n], scan[:64], [64], prior[None], 5, 2000),
        "so_register_batch_undistort": lambda c: c.register_batch_undistort(scan, [n], prior[None], [api.undistort(d["pose_prev"], 0.1)], 5, 2000),
        "so_register_batch_optimized": lambda c: c.register_batch_optimized(scan, [n], prior[None], [api.motion(0.1)], 5, 2000),
        "so_evaluate_optimized": lambda c: c.evaluate_optimized(scan, prior, IDENTITY, 0.1),
    }


def _leaving_calls(api, d):
    """calls that leave d_scan and the times alone; each may change the edge store, never the surf store"""
    import torch
    scan, prior = d["scan_xyzi"], d["prior"]
    n = len(scan)

    def batch_device(c):
        t = torch.from_numpy(scan).cuda()
        c.register_batch_device(t.data_ptr(), [n], prior[None], 5, 2000)
        torch.cuda.synchronize()

    def knn_device(c):
        q = torch.from_numpy(scan[:4096]).cuda()
        idx = torch.empty((len(q), 5), dtype=torch.int32, device="cuda")
        d2 = torch.empty((len(q), 5), dtype=torch.float32, device="cuda")
        c.knn_device(q.data_ptr(), len(q), 5, 0.0, idx.data_ptr(), d2.data_ptr())
        torch.cuda.synchronize()

    return {
        "so_register_batch_device": batch_device,
        "so_knn": lambda c: c.knn(scan[:4096, :3], 5, 0.0),
        "so_knn_device": knn_device,
        "so_map_add_edge": lambda c: c.map_add_edge(scan[:500]),
        "so_map_add_scan_edge": lambda c: c.map_add_scan_edge(scan[:500], prior),
        "so_undistort_points": lambda c: c.undistort_points(scan, prior, api.undistort(d["pose_prev"], 0.1)),
        "so_correspond_edge": lambda c: c.correspond_edge(scan[:256], prior),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_overwriting_call_makes_the_insert_fail(gpu_api, mode):
    d = _moving_case("cfg1", 5.0, 0.5)
    ctx = _ctx(gpu_api, d["case"], max_batch=2)
    for name, call in _overwriting_calls(gpu_api, d).items():
        pose = _register(gpu_api, ctx, d, mode)
        call(ctx)
        before = ctx.map_download()
        ctx.kernel_launches(reset=True)
        with pytest.raises(gpu_api.SuperOdomError, match=r"\(-1\).*so_map_add_registered_scan needs"):
            ctx.map_add_registered_scan(pose)
        assert ctx.kernel_launches() == 0, name
        assert ctx.map_size() == len(before) and np.array_equal(ctx.map_download(), before), name
    # a registration afterwards makes the insert work again
    pose = _register(gpu_api, ctx, d, mode)
    n0 = ctx.map_size()
    ctx.map_add_registered_scan(pose)
    assert ctx.map_size() > n0


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_call_that_leaves_the_scan_keeps_the_insert(gpu_api, mode):
    d = _moving_case("cfg1", 5.0, 0.5)
    for name, call in _leaving_calls(gpu_api, d).items():
        a, b = _ctx(gpu_api, d["case"], max_batch=2), _ctx(gpu_api, d["case"], max_batch=2)
        pa, pb = _register(gpu_api, a, d, mode), _register(gpu_api, b, d, mode)
        assert np.array_equal(pa, pb)
        call(a)
        a.map_add_registered_scan(pa)
        b.map_add_registered_scan(pb)
        call(b)
        assert np.array_equal(a.map_download(), b.map_download()), name
        a.close(), b.close()


@pytest.mark.gpu
def test_fresh_context_inserts_nothing(gpu_api):
    d = _moving_case("cfg1", 5.0, 0.5)
    ctx = _ctx(gpu_api, d["case"])
    n0 = ctx.map_size()
    ctx.kernel_launches(reset=True)
    ctx.map_add_registered_scan(d["prior"])
    assert ctx.map_size() == n0 and ctx.kernel_launches() == 0

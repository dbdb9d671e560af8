"""so_loop_edge_information (host only): equal to its restatement (tests/loop_edge_information_numpy.py) over random poses, all 64 flag
combinations and diagonal and general S; S byte for byte without flags; the frame checked on the pose graph's own residual
(pose_graph_numpy.edge_terms) independently of the restatement; argument errors; and a small graph in which the projected loop edge
leaves the flagged direction to the other edges."""
import ctypes as C
import math

import numpy as np
import pytest

import loop_edge_information_numpy as LE
import pose_graph_numpy as PG
import test_ceres_restatement as CR

SO_ERR_ARG = -1


def _api():
    from superodom_b200 import api
    return api


def _deg(api, flags_pos, pos_axes, flags_ori, ori_axes):
    d = api.DegeneracyResult()
    d.flags_pos, d.flags_ori = int(flags_pos), int(flags_ori)
    d.pos_axes[:] = [float(v) for v in np.asarray(pos_axes, float).ravel()]
    d.ori_axes[:] = [float(v) for v in np.asarray(ori_axes, float).ravel()]
    return d


def _raw(api, pose, d, S):
    """the C call as is -> (rc, out), out prefilled with a marker"""
    L = api.load_library()
    p = np.ascontiguousarray(pose, np.float64)
    s = np.ascontiguousarray(S, np.float64).reshape(36)
    out = np.full(36, 7.25)
    rc = L.so_loop_edge_information(api._p(p), C.byref(d), api._p(s), api._p(out))
    return rc, out


def _orthonormal(rng):
    q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    return q.T                                                           # rows: the eigenvectors


def _random_S(rng, general):
    if not general:
        return np.diag(np.r_[rng.uniform(1, 20, 3), rng.uniform(10, 200, 3)])
    return np.triu(rng.standard_normal((6, 6))) * 10 + np.diag(rng.uniform(5, 50, 6))


def test_equals_the_restatement():
    api = _api()
    rng = np.random.default_rng(31)
    worst = 0.0
    for k in range(24):
        pose = PG.rand_pose(rng, 20.0, 1.0)
        if k % 3 == 0:
            pose[3:] *= rng.uniform(0.5, 2.0)                            # not normalised: the rule normalises
        pa, oa = _orthonormal(rng), _orthonormal(rng)
        S = _random_S(rng, k % 2 == 1)
        for fp in range(8):
            for fo in range(8):
                rc, out = _raw(api, pose, _deg(api, fp, pa, fo, oa), S)
                assert rc == 0
                want = np.array(LE.edge_information(pose, fp, pa, fo, oa, S))
                assert out.tobytes() == want.tobytes(), (k, fp, fo)
                m = LE.matrix_form(pose, fp, pa, fo, oa, S).ravel()
                worst = max(worst, float(np.abs(out - m).max() / np.abs(S).max()))
    print(f"against the matrix form: max |difference| / max |S| = {worst:.3g}")
    assert worst <= 1e-14


def test_no_flags_is_S_byte_for_byte():
    api = _api()
    rng = np.random.default_rng(32)
    S = _random_S(rng, True)
    S.ravel()[[1, 7, 20]] = [-0.0, 5e-324, -1e300]
    for pose in (PG.rand_pose(rng), np.r_[1.0, 2.0, 3.0, 0.0, 0.0, 0.0, 3.0]):
        rc, out = _raw(api, pose, _deg(api, 0, _orthonormal(rng), 0, _orthonormal(rng)), S)
        assert rc == 0 and out.tobytes() == S.ravel().tobytes()
    got = api.loop_edge_information(PG.rand_pose(rng), api.DegeneracyResult(), S)
    assert got.tobytes() == S.tobytes()
    # out may alias S
    L = api.load_library()
    s = np.ascontiguousarray(S.ravel())
    p = PG.rand_pose(rng)
    d = _deg(api, 1, np.eye(3), 2, np.eye(3))
    want = _raw(api, p, d, S)[1]
    assert L.so_loop_edge_information(api._p(p), C.byref(d), api._p(s), api._p(s)) == 0 and s.tobytes() == want.tobytes()


def _residual(x_id, z, x_q):
    E = PG.to_array([PG.edge(0, 1, z, np.eye(6))])
    r, _, _ = PG.edge_terms(np.array([x_id, x_q]), E)
    return r[0]


def test_frame_on_the_graph_residual():
    """The edge (id, query, Z = X_id^-1 reg.pose) at X_q = Plus(reg.pose, eps u): |out r| is O(eps^2) along a flagged direction u
    (translation axes in the world frame, rotation axes on the right, as the registration steps) and O(eps) along an unflagged one."""
    api = _api()
    rng = np.random.default_rng(33)
    for k in range(20):
        x_id, reg = PG.rand_pose(rng, 10.0, 1.0), PG.rand_pose(rng, 10.0, 1.0)
        z = PG.compose(PG.inverse(x_id), reg)
        pa, oa = _orthonormal(rng), _orthonormal(rng)
        fp, fo = int(rng.integers(1, 8)), int(rng.integers(0, 8))
        S = _random_S(rng, k % 2 == 1)
        out = api.loop_edge_information(reg, _deg(api, fp, pa, fo, oa), S)
        r0 = _residual(x_id, z, reg)
        assert np.abs(r0).max() < 1e-12
        for blk, axes, flags in ((0, pa, fp), (1, oa, fo)):
            for j in range(3):
                u = np.zeros(6)
                u[3 * blk:3 * blk + 3] = axes[j]
                g = []
                for eps in (1e-3, 1e-4):
                    g.append(float(np.linalg.norm(out @ _residual(x_id, z, CR._plus(reg, eps * u)))) / eps)
                if flags >> j & 1:
                    assert g[0] < 1e-3 * np.abs(S).max() and g[1] < 0.2 * g[0] + 1e-9 * np.abs(S).max(), (k, blk, j, g)
                else:
                    assert g[0] > 0.3 and abs(g[1] / g[0] - 1.0) < 0.05, (k, blk, j, g)


def test_argument_errors():
    api = _api()
    rng = np.random.default_rng(34)
    pose, S = PG.rand_pose(rng), _random_S(rng, True)
    d = _deg(api, 1, np.eye(3), 1, np.eye(3))
    bad = []
    for k in range(7):
        p = pose.copy()
        p[k] = math.nan if k % 2 else math.inf
        bad.append((p, d, S))
    bad.append((np.r_[1.0, 2.0, 3.0, 0.0, 0.0, 0.0, 0.0], d, S))
    for v in (math.nan, -math.inf):
        s = S.copy()
        s[2, 4] = v
        bad.append((pose, d, s))
    for fp, fo in ((8, 0), (0, 8), (-1, 0), (0, -2)):
        bad.append((pose, _deg(api, fp, np.eye(3), fo, np.eye(3)), S))
    bad.append((pose, _deg(api, 1, np.r_[math.nan, 0, 0, 0, 1, 0, 0, 0, 1], 0, np.eye(3)), S))
    for p, dd, s in bad:
        rc, out = _raw(api, p, dd, s)
        assert rc == SO_ERR_ARG and np.all(out == 7.25)
        with pytest.raises(api.SuperOdomError):
            api.loop_edge_information(p, dd, s)
    L = api.load_library()
    p, s, out = np.ascontiguousarray(pose), np.ascontiguousarray(S.ravel()), np.zeros(36)
    for args in ((None, C.byref(d), api._p(s), api._p(out)), (api._p(p), None, api._p(s), api._p(out)),
                 (api._p(p), C.byref(d), None, api._p(out)), (api._p(p), C.byref(d), api._p(s), None)):
        assert L.so_loop_edge_information(*args) == SO_ERR_ARG


def test_projected_loop_edge_leaves_the_flagged_direction_to_the_graph():
    """Four nodes along x, odometry measured 3 % long along x and 0.05 m off in y per edge, and a loop edge 0 -> 3 measured from the
    truth but 2 m wrong along x, the way an alignment that held a corridor's axis gives it.  With x flagged the loop edge does not move
    x (the solution's x is the odometry's), and it still corrects y; the unprojected edge drags x."""
    api = _api()
    truth = np.array([[3.0 * k, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0] for k in range(4)])
    so = np.r_[[1 / 0.2] * 3, [1 / np.deg2rad(0.5)] * 3]
    odo = [PG.edge(k, k + 1, np.r_[3.09, 0.05, 0.0, 0.0, 0.0, 0.0, 1.0], so) for k in range(3)]
    est = [truth[0]]
    for e in odo:
        est.append(PG.compose(est[-1], e[2]))
    est = np.array(est)
    z = PG.compose(PG.inverse(truth[0]), truth[3])
    z[0] -= 2.0                                                          # the axis the alignment never measured
    reg = PG.compose(est[0], z)
    deg = _deg(api, 1, np.eye(3), 0, np.eye(3))                          # x flagged, in the world frame
    S = np.diag([1 / 0.1] * 3 + [1 / 0.01] * 3)
    Sp = api.loop_edge_information(reg, deg, S)
    assert np.array_equal(Sp[:, 0], np.zeros(6)) and np.array_equal(Sp[:, 1:], S[:, 1:])

    def solve(loop_S):
        edges = odo + ([PG.edge(0, 3, z, loop_S)] if loop_S is not None else [])
        prob = PG.PoseGraph(est, PG.to_array(edges))
        return prob.nodes(CR.solve_full(prob, prob.x0(), 50)["x"])
    X0, Xp, Xu = solve(None), solve(Sp), solve(S)
    assert np.allclose(X0, est, atol=1e-9)
    assert np.abs(Xp[:, 0] - X0[:, 0]).max() < 1e-4                     # x: the odometry's, to second order
    assert np.abs(Xp[:, 1] - truth[:, 1]).max() < 0.5 * np.abs(X0[:, 1] - truth[:, 1]).max()     # y: corrected
    assert np.abs(Xu[:, 0] - X0[:, 0]).max() > 0.5                       # the unprojected edge drags x


def test_entries_exported_and_shim_members_compile(tmp_path):
    import os
    import re
    import subprocess
    from superodom_b200 import api, build
    names = ("so_register_keyframes_degeneracy", "so_loop_verify_degeneracy", "so_loop_edge_information")
    lib = build.build()
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    for name in names:
        assert name in api.EXPORTS and re.search(rf"\b{name}\b", syms), name
    L = api.load_library()
    assert [len(getattr(L, n).argtypes) for n in names] == [8, 8, 4]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "shim.cpp"
    src.write_text("""#include "superodom_b200/LidarSlam.hpp"
namespace so = super_odometry::b200;
so_pose_edge first_edge(so::LidarSLAM& slam, so::LocalMap& scratch, const std::vector<so_loop_candidate>& c) {
    so_degeneracy d{};
    d.pos_threshold = 0.2; d.ori_threshold = 0.1; d.constrain = 1;
    const so::LidarSLAM::VerifiedLoops v = slam.verifyLoop(scratch, c, d);
    double S[36] = {};
    for (int k = 0; k < 6; ++k) S[7 * k] = k < 3 ? 10.0 : 100.0;
    return so::LidarSLAM::loopEdge(v.results.at(0), v.degeneracy.at(0), S, 10.0);
}
""")
    subprocess.check_call(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src)])

"""An out-and-back drive through the synthetic corridor (synth.make_corridor_scene) for degeneracy-aware loop verification: VLP-16
keyframes scanned at their true poses and stored at drifted ones, the loop candidate given explicitly, and the keyframe pose graph
solved with INTEGRATION.md's sigmas.  Shared by tests/test_loop_verify_degeneracy.py and scripts/bench_loop_verify_degeneracy.py.

The path: N_OUT keyframes 1 m apart along +x on the corridor's centre line, then as many back along -x, turned by pi, so that
keyframe QUERY (the last) lies at x = 0 and keyframe CAND at x = 2: a revisit 2 m along the corridor from the candidate, at the
relative heading pi (keyframe 0, at the query's own place, is the revisit without offset).  The stored poses drift by DRIFT per
keyframe (x along the corridor, y across it, yaw), in the world frame, so that odometry edges between them carry the drift and
keyframe 0 is exact."""
import functools

import numpy as np

N_OUT = 25
QUERY = 2 * N_OUT - 1
CAND = 2
DRIFT = (0.01, 0.015, 0.002)            # metres / keyframe along x and y, rad / keyframe in yaw
VLP16 = dict(el_res_deg=2.0, el_min_deg=-16.0, el_max_deg=16.0)
ODOM_SIGMA = (0.02, np.deg2rad(0.05))   # INTEGRATION.md, "Loop closure": odometry and loop sigmas (m, rad), loop Cauchy scale
LOOP_SIGMA = (0.1, 0.01)
LOOP_CAUCHY = 10.0


def _quat_z(yaw):
    return np.array([0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)])


def truth():
    out = [np.r_[float(i), 0.0, 0.0, _quat_z(0.0)] for i in range(N_OUT)]
    out += [np.r_[float(N_OUT - 1 - j), 0.0, 0.0, _quat_z(np.pi)] for j in range(N_OUT)]
    return np.array(out)


def drifted(tr):
    k = np.arange(len(tr))[:, None]
    yaw = np.array([heading(p) for p in tr]) + DRIFT[2] * k[:, 0]
    return np.c_[tr[:, :3] + k * np.array([DRIFT[0], DRIFT[1], 0.0]), np.array([_quat_z(a) for a in yaw])]


def heading(p):
    x, y, z, w = p[3:] / np.linalg.norm(p[3:])
    return float(np.arctan2(2 * (x * y + z * w), 1 - 2 * (y * y + z * z)))


def wrap(a):
    return (np.asarray(a) + np.pi) % (2 * np.pi) - np.pi


@functools.lru_cache(maxsize=None)
def scans(poles):
    from superodom_b200 import synth
    scene = synth.make_corridor_scene(poles=poles)
    return tuple(synth.make_scan(scene, "vlp16", p, 12000 + i, rmax=30.0) for i, p in enumerate(truth()))


def context(api, poles):
    """A context holding the keyframes at their drifted poses (registered against an empty map, which keeps the prior)."""
    tr = truth()
    ctx = api.Context(max_map_points=1 << 21, max_scan_points=1 << 18, plane_res=0.2, line_res=0.1)
    ctx.keyframe_reserve(len(tr) << 15, len(tr))
    for s, e in zip(scans(poles), drifted(tr)):
        ctx.register(s, e, 1, 0)
        ctx.keyframe_add_registered(e)
    return ctx


def candidate(api, query=QUERY, cand=CAND):
    c = np.zeros(1, api.LOOP_CANDIDATE_DTYPE)
    c[0]["query"], c[0]["id"], c[0]["yaw"] = query, cand, np.pi
    return c


def _compose(a, b):
    from scipy.spatial.transform import Rotation
    Ra = Rotation.from_quat(a[3:])
    return np.r_[a[:3] + Ra.apply(b[:3]), (Ra * Rotation.from_quat(b[3:])).as_quat()]


def _inverse(a):
    from scipy.spatial.transform import Rotation
    Ri = Rotation.from_quat(a[3:]).inv()
    return np.r_[-Ri.apply(a[:3]), Ri.as_quat()]


def loop_sqrt_info():
    return np.diag([1 / LOOP_SIGMA[0]] * 3 + [1 / LOOP_SIGMA[1]] * 3)


def solve(api, ctx, loop=None):
    """The keyframe graph from the drifted poses: odometry edges k -> k+1, and loop = (id, query, rel7, S) or None; keyframe 0 fixed.
    -> (poses [n, 7], per-keyframe errors against the truth: dict of x, y (m) and yaw (rad) arrays, the loop edge's rho')"""
    est = drifted(truth())
    so = np.diag([1 / ODOM_SIGMA[0]] * 3 + [1 / ODOM_SIGMA[1]] * 3)
    edges = [(k, k + 1, _compose(_inverse(est[k]), est[k + 1]), so, 0.0) for k in range(len(est) - 1)]
    if loop is not None:
        edges.append((loop[0], loop[1], np.asarray(loop[2], float), np.asarray(loop[3], float), LOOP_CAUCHY))
    X, _, w = ctx.pose_graph_solve(est, edges, weights=True)
    return X, errors(X), (float(w[-1]) if loop is not None else None)


def errors(X):
    tr = truth()
    return dict(x=np.abs(X[:, 0] - tr[:, 0]), y=np.abs(X[:, 1] - tr[:, 1]),
                yaw=np.abs(wrap(np.array([heading(p) for p in X]) - np.array([heading(p) for p in tr]))))


def along_error(rel7, cand=CAND):
    """The loop edge's error along the corridor: its x against the true relative pose's (in the candidate's frame)"""
    tr = truth()
    z = _compose(_inverse(tr[cand]), tr[QUERY])
    return float(rel7[0] - z[0])


def ratios(deg):
    """sqrt(i_min / i_max) of the translation and the rotation block of a so_degeneracy_result"""
    def r(v):
        return float(np.sqrt(max(v[0], 0.0) / v[2])) if v[2] > 0 else 0.0
    return r(deg.pos_info), r(deg.ori_info)

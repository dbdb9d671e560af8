"""Restatements for the multi-session entry points: the loop search over an id range (so_loop_candidates_range) and the pose graph
with a set of constant nodes (so_pose_graph_solve_constant), each built on the single-session restatement it generalises."""
import numpy as np

import loop_detection_numpy as LD
import pose_graph_numpy as PG


def search_range(descs, queries, k: int, begin: int, end: int):
    """LD.search with the eligible ids [begin, end) minus the query -> [(id, distance, shift, n_pairs, yaw)] * k per query."""
    nrm = [LD.norms(d) for d in descs]
    Ns = descs.shape[2]
    out = []
    for q in queries:
        rows = []
        for b in range(int(begin), int(end)):
            if b == int(q):
                continue
            d, s, n = LD.pair(descs[q], descs[b], nrm[q], nrm[b])
            rows.append((d, b, s, n))
        rows.sort(key=lambda t: (t[0], t[1]))
        best = [(b, d, s, n, LD.yaw_of(s, Ns)) for d, b, s, n in rows[:k]]
        out.append(best + [(-1, 1.0, 0, 0, 0.0)] * (k - len(best)))
    return out


class ConstantPoseGraph(PG.PoseGraph):
    """PG.PoseGraph with every node where constant[k] is set held at init[k] (SetParameterBlockConstant on each): x, its norm, the
    gradient and the Jacobian's columns cover the free nodes only."""

    def __init__(self, init, edges, constant):
        super().__init__(init, edges, 0)
        self.constant = np.asarray(constant, bool)
        assert self.constant.shape == (self.n,)
        self.free = np.nonzero(~self.constant)[0]
        self.col = np.full(self.n, -1)
        self.col[self.free] = np.arange(len(self.free))

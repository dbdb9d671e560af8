"""so_loop_edge_information (superodom_b200/csrc/so_verify_rule.h, loop_edge_information) restated in plain Python floats: the
same products and sums in the same order, so that the C function equals it bit for bit.  matrix_form states it as matrices (numpy),
for a check that does not share the order."""
import math

import numpy as np


def rotation(q):
    """R of quaternion {x, y, z, w}, normalised first, as the rule writes it"""
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    x, y, z, w = q[0] / n, q[1] / n, q[2] / n, q[3] / n
    return [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
            2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
            2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]


def edge_information(pose7, flags_pos, pos_axes, flags_ori, ori_axes, S):
    """-> out [36] (row-major), or None where the C function returns SO_ERR_ARG"""
    p = [float(v) for v in pose7]
    S = [float(v) for v in np.asarray(S, float).ravel()]
    pa = [float(v) for v in np.asarray(pos_axes, float).ravel()]
    oa = [float(v) for v in np.asarray(ori_axes, float).ravel()]
    if not all(math.isfinite(v) for v in p + S + pa + oa) or not (0 <= flags_pos <= 7 and 0 <= flags_ori <= 7):
        return None
    if not math.sqrt(p[3] * p[3] + p[4] * p[4] + p[5] * p[5] + p[6] * p[6]) > 0.0:
        return None
    if not flags_pos and not flags_ori:
        return list(S)
    R = rotation(p[3:])
    M = [0.0] * 36
    for i in range(6):
        M[7 * i] = 1.0
    for k in range(3):
        if flags_pos >> k & 1:
            u = pa[3 * k:3 * k + 3]
            a = [R[i] * u[0] + R[3 + i] * u[1] + R[6 + i] * u[2] for i in range(3)]
            for i in range(3):
                for j in range(3):
                    M[6 * i + j] -= a[i] * a[j]
        if flags_ori >> k & 1:
            b = oa[3 * k:3 * k + 3]
            for i in range(3):
                for j in range(3):
                    M[6 * (3 + i) + 3 + j] -= b[i] * b[j]
    out = [0.0] * 36
    for r in range(6):
        for c in range(6):
            v = 0.0
            for m in range(6):
                v += S[6 * r + m] * M[6 * m + c]
            out[6 * r + c] = v
    return out


def matrix_form(pose7, flags_pos, pos_axes, flags_ori, ori_axes, S):
    """S (I - blockdiag(A A^T, B B^T)), A = R^T [flagged translation axes], B = [flagged rotation axes], with numpy matrices"""
    R = np.array(rotation([float(v) for v in pose7[3:]])).reshape(3, 3)
    pa, oa = np.asarray(pos_axes, float).reshape(3, 3), np.asarray(ori_axes, float).reshape(3, 3)
    A = np.array([R.T @ pa[k] for k in range(3) if flags_pos >> k & 1]).reshape(-1, 3)
    B = np.array([oa[k] for k in range(3) if flags_ori >> k & 1]).reshape(-1, 3)
    P = np.zeros((6, 6))
    P[:3, :3] = A.T @ A
    P[3:, 3:] = B.T @ B
    return np.asarray(S, float).reshape(6, 6) @ (np.eye(6) - P)

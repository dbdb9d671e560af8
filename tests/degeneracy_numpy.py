"""Numpy restatement of the degeneracy analysis (DESIGN.md section 3), written apart from the device code.

H is the 6x6 normal matrix of a solve in tangent order (t, theta).  The information of each block is the Schur complement
    I_t = H_tt - H_tr H_rr^+ H_rt,   I_r = H_rr - H_rt H_tt^+ H_tr
with ^+ the pseudo-inverse under ceres::Covariance's cut (eigen-directions with sqrt(w_k / w_max) < 1e-7, or w_k <= 0, dropped).
Eigenpair k of a block (ascending) is flagged when i_k <= threshold^2 * max(i_max, 0).  B holds the unflagged eigenvectors,
translation ones first; with constrain and a flag the solve runs on B's columns."""
import numpy as np


def pinv_cut(A):
    w, V = np.linalg.eigh(A)
    inv = np.zeros(3)
    for k in range(3):
        ratio = np.sqrt(w[k] / w[2]) if (w[k] > 0 and w[2] > 0) else 0.0
        inv[k] = 0.0 if ratio < 1e-7 else 1.0 / w[k]
    return (V * inv) @ V.T


def block(A, C, other, thr):
    I = A - C @ pinv_cut(other) @ C.T
    I = 0.5 * (I + I.T)
    w, V = np.linalg.eigh(I)
    cut = thr * thr * max(w[2], 0.0)
    flags = sum(1 << k for k in range(3) if w[k] <= cut)
    return I, w, V.T.copy(), flags              # axes[k] = eigenvector k


def analysis(H, pos_threshold, ori_threshold, constrain=1):
    """-> dict(I_t, I_r, pos_info, pos_axes [3, 3], ori_info, ori_axes, flags_pos, flags_ori, B [6, m])."""
    H = np.asarray(H, np.float64)
    Htt, Htr, Hrr = H[:3, :3], H[:3, 3:], H[3:, 3:]
    It, wt, At, ft = block(Htt, Htr, Hrr, pos_threshold)
    Ir, wr, Ar, fr = block(Hrr, Htr.T, Htt, ori_threshold)
    if constrain and (ft | fr):
        cols = [np.concatenate([At[k], np.zeros(3)]) for k in range(3) if not (ft >> k) & 1]
        cols += [np.concatenate([np.zeros(3), Ar[k]]) for k in range(3) if not (fr >> k) & 1]
        B = np.array(cols).T.reshape(6, len(cols))
    else:
        B = np.eye(6)
    return dict(I_t=It, I_r=Ir, pos_info=wt, pos_axes=At, ori_info=wr, ori_axes=Ar, flags_pos=ft, flags_ori=fr, B=B)


def with_spectrum(rng, info_t, info_r, coupling=0.0, rot_t=None, rot_r=None):
    """A 6x6 H whose Schur complements have the prescribed eigenvalues: H = [[I_t + C P C^T, C], [C^T, H_rr]] with
    H_rr = R_r diag(info_r) R_r^T + C^T I_t^+ ... built from the block LDL form, so that I_t and I_r come out exactly as asked
    (up to rounding) when coupling = 0, and I_t when coupling != 0 (I_r is then whatever the coupling gives)."""
    def rot(r):
        if r is not None:
            return np.asarray(r, np.float64)
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        return q
    Rt, Rr = rot(rot_t), rot(rot_r)
    It = Rt @ np.diag(info_t) @ Rt.T
    Hrr = Rr @ np.diag(info_r) @ Rr.T
    C = coupling * rng.standard_normal((3, 3))
    Htt = It + C @ pinv_cut(Hrr) @ C.T
    H = np.zeros((6, 6))
    H[:3, :3], H[:3, 3:], H[3:, :3], H[3:, 3:] = Htt, C, C.T, Hrr
    return 0.5 * (H + H.T)


# ---------------------------------------------------------------------------------------------------------------- reduced solve
def solve_reduced(prob, x0, B, max_iterations=4, full=False):
    """Ceres' trust-region LM (restated in tests/test_ceres_restatement.py) on prob with the local parameterisation x [+] B y:
    Jacobian J B, Jacobi scaling and LM diagonal over B's m columns, model cost change of the reduced step, gradient max-norm
    through Plus(x, -B B^T g); x_norm and the parameter / function tolerances ambient.
    -> (x, iterations, successful_steps, unsuccessful_steps, termination) with the termination codes of that restatement; full: the
    dict of test_ceres_restatement.solve_full (costs, the final radius, decrease factor and gradient max-norm, decision margins)."""
    import test_ceres_restatement as CR
    r = CR.solve_full(prob, x0, max_iterations, B=B)
    return r if full else (r["x"], r["iterations"], r["successful"], r["unsuccessful"], r["termination"])


def register(ctx, scan, x0, pos_threshold, ori_threshold, iters, mf, a2, lm=4, constrain=1):
    """so_register_degeneracy's ICP loop restated: every iteration re-corresponds at x through the device's own search and fit
    (so_correspond), analyses H = J^T J of the corrected rows at x, solves on B's columns (or the ambient solve when nothing is
    flagged) and stops after a solve with one successful step or on the last iteration.
    -> (x, per-iteration (n_ok, lm steps, successful, termination, flagged translation, flagged rotation))"""
    import test_ceres_restatement as CR
    x = np.array(x0, float)
    its = []
    for _ in range(iters):
        corr, _, hr = ctx.correspond(scan, x, mf)
        ok = corr["w"] != 0.0
        prob = CR.Problem(scan[ok, :3].astype(np.float64), corr["n"][ok], corr["d"][ok], corr["w"][ok], a2)
        _, _, J = prob.linearise(x)
        a = analysis(J.T @ J, pos_threshold, ori_threshold, constrain)
        if a["B"].shape[1] < 6:
            x, it, succ, _, term = solve_reduced(prob, x, a["B"], lm)
        else:
            x, it, succ, _, term = CR.solve(prob, x, lm)
        its.append((int(hr[0]), it, succ, term, bin(a["flags_pos"]).count("1"), bin(a["flags_ori"]).count("1")))
        if succ == 1:
            break
    return x, its

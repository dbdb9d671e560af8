// so_undistort.cuh -- the warp of one point by a scan's motion D over dt (so_undistort.cu): the per-scan setup of D for mode APPROXIMATED
// (und_setup) and mode OPTIMIZED (motion_setup; so_motion.cu's solve reuses und_angle), then und_point.  Every product and sum is rounded
// on its own (no FMA contraction), so that the numpy restatements in tests/ restate the bits; only the FP64 acos / sin are the device's.
#pragma once
#include "so_ctx.cuh"

namespace so {

__device__ __forceinline__ void qmul_rn(const double a[4], const double b[4], double o[4]) {
    o[0] = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(a[3], b[0]), __dmul_rn(a[0], b[3])), __dmul_rn(a[1], b[2])), __dmul_rn(a[2], b[1]));
    o[1] = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(a[3], b[1]), __dmul_rn(a[1], b[3])), __dmul_rn(a[2], b[0])), __dmul_rn(a[0], b[2]));
    o[2] = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(a[3], b[2]), __dmul_rn(a[2], b[3])), __dmul_rn(a[0], b[1])), __dmul_rn(a[1], b[0]));
    o[3] = __dsub_rn(__dsub_rn(__dsub_rn(__dmul_rn(a[3], b[3]), __dmul_rn(a[0], b[0])), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}
// qrot of so_internal.cuh (v + 2w (q x v) + 2 q x (q x v)) with every operation rounded
__device__ __forceinline__ void qrot_rn(const double q[4], const double v[3], double o[3]) {
    double ux = __dsub_rn(__dmul_rn(q[1], v[2]), __dmul_rn(q[2], v[1]));
    double uy = __dsub_rn(__dmul_rn(q[2], v[0]), __dmul_rn(q[0], v[2]));
    double uz = __dsub_rn(__dmul_rn(q[0], v[1]), __dmul_rn(q[1], v[0]));
    ux = __dadd_rn(ux, ux); uy = __dadd_rn(uy, uy); uz = __dadd_rn(uz, uz);
    o[0] = __dadd_rn(__dadd_rn(v[0], __dmul_rn(q[3], ux)), __dsub_rn(__dmul_rn(q[1], uz), __dmul_rn(q[2], uy)));
    o[1] = __dadd_rn(__dadd_rn(v[1], __dmul_rn(q[3], uy)), __dsub_rn(__dmul_rn(q[2], ux), __dmul_rn(q[0], uz)));
    o[2] = __dadd_rn(__dadd_rn(v[2], __dmul_rn(q[3], uz)), __dsub_rn(__dmul_rn(q[0], uy), __dmul_rn(q[1], ux)));
}

// sh[7..8] from the normalised q_D in sh[0..3]: {theta, 1 / sin(theta)}; theta < 0 marks Eigen's linear branch (|d| >= 1 - eps,
// d = dot(identity, q_D) = q_D.w).
__device__ __forceinline__ void und_angle(double sh[9]) {
    const double ad = fabs(sh[3]);
    if (ad >= 1.0 - 2.220446049250313e-16) { sh[7] = -1.0; sh[8] = 0.0; }
    else { sh[7] = acos(ad); sh[8] = 1.0 / sin(sh[7]); }
}

// Per-scan part, once per CTA: sh = {q_D[4], t_D[3], theta, 1 / sin(theta)} of D = T_prev^-1 * T(x).
__device__ __forceinline__ void und_setup(const UndistortParams& P, const double x[7], double sh[9]) {
    double q[4];
    qmul_rn(P.q_prev_conj, x + 3, q);
    const double n2 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])), __dmul_rn(q[3], q[3]));
    const double s = 1.0 / sqrt(n2);
    for (int k = 0; k < 4; ++k) sh[k] = __dmul_rn(q[k], s);
    const double d[3] = {__dsub_rn(x[0], P.t_prev[0]), __dsub_rn(x[1], P.t_prev[1]), __dsub_rn(x[2], P.t_prev[2])};
    qrot_rn(P.q_prev_conj, d, sh + 4);
    und_angle(sh);
}

// sh = {q_D[4] normalised, t_D[3], theta, 1 / sin(theta)} of a motion D, rounded as und_setup rounds
__device__ __forceinline__ void motion_setup(const double D[7], double sh[9]) {
    const double n2 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(D[3], D[3]), __dmul_rn(D[4], D[4])), __dmul_rn(D[5], D[5])), __dmul_rn(D[6], D[6]));
    const double s = 1.0 / sqrt(n2);
    for (int k = 0; k < 4; ++k) sh[k] = __dmul_rn(D[3 + k], s);
    for (int k = 0; k < 3; ++k) sh[4 + k] = D[k];
    und_angle(sh);
}

__device__ __forceinline__ float4 und_point(const UndistortParams& P, const double sh[9], float4 p, float tau) {
    const double a = isfinite(tau) ? double(tau) / P.dt : 0.0;
    const double v[3] = {double(p.x), double(p.y), double(p.z)};
    double o[3] = {v[0], v[1], v[2]};
    if (P.rotation) {
        double s0, s1;
        if (sh[7] < 0.0) { s0 = __dsub_rn(1.0, a); s1 = a; }
        else {
            s0 = __dmul_rn(sin(__dmul_rn(__dsub_rn(1.0, a), sh[7])), sh[8]);
            s1 = __dmul_rn(sin(__dmul_rn(a, sh[7])), sh[8]);
        }
        if (sh[3] < 0.0) s1 = -s1;
        const double qi[4] = {__dadd_rn(__dmul_rn(s0, 0.0), __dmul_rn(s1, sh[0])), __dadd_rn(__dmul_rn(s0, 0.0), __dmul_rn(s1, sh[1])),
                              __dadd_rn(__dmul_rn(s0, 0.0), __dmul_rn(s1, sh[2])), __dadd_rn(s0, __dmul_rn(s1, sh[3]))};
        qrot_rn(qi, v, o);
    }
    return make_float4(float(__dadd_rn(o[0], __dmul_rn(a, sh[4]))), float(__dadd_rn(o[1], __dmul_rn(a, sh[5]))),
                       float(__dadd_rn(o[2], __dmul_rn(a, sh[6]))), p.w);
}

}  // namespace so

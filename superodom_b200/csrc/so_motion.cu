// so_motion.cu -- within-scan motion estimated by the registration itself: the reference's UndistortionMode::OPTIMIZED (LidarSlam.h:77-81,
// "both begin and end scan are optimized using registration of undistorted scan and map; scan is linearly undistorted between begin
// and end poses"; its branch of ComputePointInitAndFinalPose, LidarSlam.cpp:390-392, is empty upstream), sm_90a.
//
// Two pose7 parameter blocks per scan: T, the pose at tau = 0, and D, the motion over dt (the pose at tau = dt is T * D).  With
// alpha_i = double(tau_i) / dt (0 for a non-finite tau_i):
//   u_i(D) = qrot(slerp(identity, q_D, alpha_i), p_i) + alpha_i * t_D          (und_point's formula with D from the state)
//   r_i    = n_i . (R(q) u_i(D) + t) + d_i                                      under ScaledLoss(TukeyLoss), as so_register
// plus six rows of SE3AbsolutatePoseFactor on D (measurement D0, multiplier sqrt(n_ok * info_k)).  Each ICP iteration rounds u(D) to
// float and runs the unchanged search and fit at T on it (k_motion_warp -> d_scan_sorted); the solve evaluates u in double at the
// candidate D.  Both blocks use PoseLocalParameterization; the D rotation columns are the exact derivative
//   dr/d(dtheta_D) = alpha (p x b)^T J_r(alpha phi) J_r(phi)^-1,  b = R(q_alpha)^T R(q)^T n,  phi = Log(q_D) on the shortest path.
//   k_motion_warp        float(u(D)) of every active point into the ordered scan (w kept), like k_undistort
//   k_motion_eval<PH>    residual and 12-column row per correspondence, 91 per-CTA sums (78 + 12 + 1) through shared memory
//   k_motion_step<PH>    fixed-order cross-CTA sum, then the 12-parameter trust-region step; the 12x12 covariance at the end
//   k_motion_cloud       u(D_opt) of a contiguous cloud: the map insert after a single-scan registration
// With an edge cloud (so_register_optimized_edges): k_motion_warp_edges writes float(u_e(D)) for k_edge_fit's search and fit at T, and
//   k_motion_eval_edge<PH> adds the line rows' 91 per-CTA sums (three rows per line, motion_line_rows) into a partial buffer of their
//   own, which k_motion_step adds after the planes' in the same fixed order
#include <cmath>
#include <vector>

#include "so_trust_region.cuh"
#include "so_undistort.cuh"

namespace so {

// sh = {q_D[4] normalised, t_D[3], theta, 1 / sin(theta)} of a motion D, rounded as und_setup rounds
__device__ __forceinline__ void motion_setup(const double D[7], double sh[9]) {
    const double n2 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(D[3], D[3]), __dmul_rn(D[4], D[4])), __dmul_rn(D[5], D[5])), __dmul_rn(D[6], D[6]));
    const double s = 1.0 / sqrt(n2);
    for (int k = 0; k < 4; ++k) sh[k] = __dmul_rn(D[3 + k], s);
    for (int k = 0; k < 3; ++k) sh[4 + k] = D[k];
    und_angle(sh);
}

// ------------------------------------------------------------------------------------------------------------------ warp
__global__ void __launch_bounds__(kThreads) k_motion_warp(BatchView bv, float4* __restrict__ sorted, const float4* __restrict__ raw,
                                                          const float* __restrict__ times, const MotionState* __restrict__ ms) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    const uint32_t n = uint32_t(st->n_points);
    if (blockIdx.x * kThreads >= n) return;
    __shared__ double sh[9];
    if (threadIdx.x == 0) motion_setup(ms[s].D, sh);
    __syncthreads();
    UndistortParams P{};
    P.dt = ms[s].dt; P.on = 1; P.rotation = 1;
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const size_t base = size_t(bv.offset[s]), gi = base + i;
    const float w = sorted[gi].w;
    const size_t src = base + __float_as_uint(w);                        // original index (scan ordering)
    float4 o = und_point(P, sh, __ldg(&raw[src]), __ldg(&times[src]));
    o.w = w;
    sorted[gi] = o;
}

// The same warp for the edge cloud (so_register_optimized_edges): one thread per edge point, raw point, time and output at one index
__global__ void __launch_bounds__(kThreads) k_motion_warp_edges(BatchView bv, const uint32_t* __restrict__ eoffset, float4* __restrict__ out,
                                                                const float4* __restrict__ raw, const float* __restrict__ times,
                                                                const MotionState* __restrict__ ms) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    const uint32_t n = uint32_t(st->n_edge);
    if (blockIdx.x * kThreads >= n) return;
    __shared__ double sh[9];
    if (threadIdx.x == 0) motion_setup(ms[s].D, sh);
    __syncthreads();
    UndistortParams P{};
    P.dt = ms[s].dt; P.on = 1; P.rotation = 1;
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const size_t gi = size_t(eoffset[s]) + i;
    out[gi] = und_point(P, sh, __ldg(&raw[gi]), __ldg(&times[gi]));
}

struct MotionD { double v[7]; };
__global__ void __launch_bounds__(256) k_motion_cloud(float4* __restrict__ pts, const float* __restrict__ times, uint32_t n, MotionD D, double dt) {
    __shared__ double sh[9];
    if (threadIdx.x == 0) motion_setup(D.v, sh);
    __syncthreads();
    UndistortParams P{};
    P.dt = dt; P.on = 1; P.rotation = 1;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pts[i] = und_point(P, sh, pts[i], times[i]);
}

// ------------------------------------------------------------------------------------------------------------------ evaluation
__device__ __forceinline__ void cross3(const double a[3], const double b[3], double o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}

// per CTA: pose T, R(q), the motion's slerp setup, phi = Log(q_D) (shortest path), its angle, and c3(|phi|)
struct MotionCta { double T[7], R[9], sh[9], phi[3], th, c3, dt; };

__device__ __forceinline__ void motion_cta_setup(const double T[7], const double D[7], double dt, MotionCta& m) {
    for (int k = 0; k < 7; ++k) m.T[k] = T[k];
    qtoR(T + 3, m.R);
    double q[4];
    const double n = sqrt(D[3] * D[3] + D[4] * D[4] + D[5] * D[5] + D[6] * D[6]);
    for (int k = 0; k < 4; ++k) q[k] = D[3 + k] / n;
    for (int k = 0; k < 4; ++k) m.sh[k] = q[k];
    for (int k = 0; k < 3; ++k) m.sh[4 + k] = D[k];
    und_angle(m.sh);
    const double sg = q[3] < 0.0 ? -1.0 : 1.0;
    const double vn = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    m.th = 2.0 * atan2(vn, sg * q[3]);
    const double f = vn > 0.0 ? sg * m.th / vn : 0.0;
    for (int k = 0; k < 3; ++k) m.phi[k] = f * q[k];
    m.c3 = jrinv_coeff(m.th);
    m.dt = dt;
}

// One correspondence: the row sqrt(rho') [J (12), r] and rho / 2 (ScaledLoss(TukeyLoss) through Ceres' corrector, as accumulate())
__device__ __forceinline__ void motion_row(const MotionCta& m, const double nd[4], double wc, float4 p, float tau, double a2, double row[14]) {
    const double al = isfinite(tau) ? double(tau) / m.dt : 0.0;
    const double pv[3] = {double(p.x), double(p.y), double(p.z)};
    double s0, s1;                                                       // Eigen's slerp(identity, q_D, alpha)
    if (m.sh[7] < 0.0) { s0 = 1.0 - al; s1 = al; }
    else { s0 = sin((1.0 - al) * m.sh[7]) * m.sh[8]; s1 = sin(al * m.sh[7]) * m.sh[8]; }
    if (m.sh[3] < 0.0) s1 = -s1;
    const double qa[4] = {s1 * m.sh[0], s1 * m.sh[1], s1 * m.sh[2], s0 + s1 * m.sh[3]};
    double u[3];
    qrot(qa, pv, u);
    for (int k = 0; k < 3; ++k) u[k] += al * m.sh[4 + k];
    double pw[3];
    qrot(m.T + 3, u, pw);
    for (int k = 0; k < 3; ++k) pw[k] += m.T[k];
    const double r = nd[0] * pw[0] + nd[1] * pw[1] + nd[2] * pw[2] + nd[3];
    const double sr = r * r;
    double rho0, rho1;
    if (sr <= a2) { const double v = 1.0 - sr / a2, v2 = v * v; rho0 = a2 / 6.0 * (1.0 - v2 * v); rho1 = 0.5 * v2; }
    else { rho0 = a2 / 6.0; rho1 = 0.0; }
    rho0 *= wc; rho1 *= wc;
    const double* R = m.R;
    const double av[3] = {R[0] * nd[0] + R[3] * nd[1] + R[6] * nd[2], R[1] * nd[0] + R[4] * nd[1] + R[7] * nd[2],
                          R[2] * nd[0] + R[5] * nd[1] + R[8] * nd[2]};            // R^T n
    double J[12];
    J[0] = nd[0]; J[1] = nd[1]; J[2] = nd[2];
    cross3(u, av, J + 3);                                                // -n^T R [u]x
    for (int k = 0; k < 3; ++k) J[6 + k] = al * av[k];                   // alpha n^T R
    const double qc[4] = {-qa[0], -qa[1], -qa[2], qa[3]};
    double b[3], w[3], t1[3], t2[3];
    qrot(qc, av, b);                                                     // R(q_alpha)^T R^T n
    cross3(pv, b, w);                                                    // p x b
    // J_r(alpha phi)^T w = w + c1 (v x w) + c2 v x (v x w), v = alpha phi
    const double v[3] = {al * m.phi[0], al * m.phi[1], al * m.phi[2]};
    double c1, c2;
    jr_coeffs(fabs(al) * m.th, &c1, &c2);
    cross3(v, w, t1); cross3(v, t1, t2);
    for (int k = 0; k < 3; ++k) w[k] = w[k] + c1 * t1[k] + c2 * t2[k];
    // J_r(phi)^-T w = w - (phi x w) / 2 + c3 phi x (phi x w)
    cross3(m.phi, w, t1); cross3(m.phi, t1, t2);
    for (int k = 0; k < 3; ++k) J[9 + k] = al * (w[k] - 0.5 * t1[k] + m.c3 * t2[k]);
    const double sc = sqrt(rho1);
#pragma unroll
    for (int k = 0; k < 12; ++k) row[k] = sc * J[k];
    row[12] = sc * r;
    row[13] = 0.5 * rho0;
}

// One line correspondence (EdgeAnalyticCostFunction, lidarOptimization.cpp:12-47, at lp = R(q) u(D) + t): r = (lp - a) x (lp - b) / |a - b|,
// dr/dlp = skew(b - a) / |a - b|.  Row k is motion_row's 12 columns with n replaced by the k-th row of that matrix (the T columns
// are the reference's Jacobian at u(D), the D columns the plane row's chain rule); ScaledLoss(TukeyLoss) at a2 through Ceres'
// corrector for a 3-dimensional residual, as accumulate_edge: rows[k] = sqrt(rho') [J_k (12), r_k], *half_rho = rho / 2.
__device__ __forceinline__ void motion_line_rows(const MotionCta& m, const double a[3], const double bb[3], double wc, float4 p, float tau,
                                                 double a2, double rows[3][13], double* half_rho) {
    const double al = isfinite(tau) ? double(tau) / m.dt : 0.0;
    const double pv[3] = {double(p.x), double(p.y), double(p.z)};
    double s0, s1;                                                       // Eigen's slerp(identity, q_D, alpha)
    if (m.sh[7] < 0.0) { s0 = 1.0 - al; s1 = al; }
    else { s0 = sin((1.0 - al) * m.sh[7]) * m.sh[8]; s1 = sin(al * m.sh[7]) * m.sh[8]; }
    if (m.sh[3] < 0.0) s1 = -s1;
    const double qa[4] = {s1 * m.sh[0], s1 * m.sh[1], s1 * m.sh[2], s0 + s1 * m.sh[3]};
    double u[3];
    qrot(qa, pv, u);
    for (int k = 0; k < 3; ++k) u[k] += al * m.sh[4 + k];
    double pw[3];
    qrot(m.T + 3, u, pw);
    for (int k = 0; k < 3; ++k) pw[k] += m.T[k];
    const double de[3] = {a[0] - bb[0], a[1] - bb[1], a[2] - bb[2]};
    const double den = sqrt(de[0] * de[0] + de[1] * de[1] + de[2] * de[2]);
    const double x[3] = {pw[0] - a[0], pw[1] - a[1], pw[2] - a[2]}, y[3] = {pw[0] - bb[0], pw[1] - bb[1], pw[2] - bb[2]};
    const double r[3] = {(x[1] * y[2] - x[2] * y[1]) / den, (x[2] * y[0] - x[0] * y[2]) / den, (x[0] * y[1] - x[1] * y[0]) / den};
    const double sr = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    double rho0, rho1;
    if (sr <= a2) { const double v = 1.0 - sr / a2, v2 = v * v; rho0 = a2 / 6.0 * (1.0 - v2 * v); rho1 = 0.5 * v2; }
    else { rho0 = a2 / 6.0; rho1 = 0.0; }
    rho0 *= wc; rho1 *= wc;
    const double sc = sqrt(rho1);
    const double re[3] = {-de[0], -de[1], -de[2]};
    const double K[9] = {0, -re[2], re[1], re[2], 0, -re[0], -re[1], re[0], 0};     // skew(b - a)
    const double* R = m.R;
    const double qc[4] = {-qa[0], -qa[1], -qa[2], qa[3]};
    const double v[3] = {al * m.phi[0], al * m.phi[1], al * m.phi[2]};
    double c1, c2;
    jr_coeffs(fabs(al) * m.th, &c1, &c2);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double nd[3] = {K[3 * k] / den, K[3 * k + 1] / den, K[3 * k + 2] / den};
        const double av[3] = {R[0] * nd[0] + R[3] * nd[1] + R[6] * nd[2], R[1] * nd[0] + R[4] * nd[1] + R[7] * nd[2],
                              R[2] * nd[0] + R[5] * nd[1] + R[8] * nd[2]};        // R^T n_k
        double J[12];
        J[0] = nd[0]; J[1] = nd[1]; J[2] = nd[2];
        cross3(u, av, J + 3);
        for (int j = 0; j < 3; ++j) J[6 + j] = al * av[j];
        double b[3], w[3], t1[3], t2[3];
        qrot(qc, av, b);
        cross3(pv, b, w);
        cross3(v, w, t1); cross3(v, t1, t2);
        for (int j = 0; j < 3; ++j) w[j] = w[j] + c1 * t1[j] + c2 * t2[j];
        cross3(m.phi, w, t1); cross3(m.phi, t1, t2);
        for (int j = 0; j < 3; ++j) J[9 + j] = al * (w[j] - 0.5 * t1[j] + m.c3 * t2[j]);
        for (int j = 0; j < 12; ++j) rows[k][j] = sc * J[j];
        rows[k][12] = sc * r[k];
    }
    *half_rho = 0.5 * rho0;
}

constexpr int kRowStride = 14;
// Tiles of kThreads points (the per-CTA layout of k_evaluate: eval_pts(n) tiles per CTA, eval_ctas(n) CTAs per scan): every thread
// stages its row in shared memory, then thread e < 91 adds component e of the tile's 256 rows in index order.  One register
// accumulator per thread instead of 91.
template <int PHASE>
__global__ void __launch_bounds__(kThreads) k_motion_eval(BatchView bv, CorrBuf cb, const float4* __restrict__ raw, const float* __restrict__ times,
                                                          const MotionState* __restrict__ ms, double* __restrict__ partials, uint32_t stride) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PHASE) return;
    const uint32_t n = uint32_t(st->n_points);
    const int pts = eval_pts(n);
    if (blockIdx.x >= eval_ctas(n)) return;
    __shared__ MotionCta m;
    __shared__ double rows[kThreads * kRowStride];
    if (threadIdx.x == 0) motion_cta_setup(PHASE == PH_EVAL ? st->cand : st->x, PHASE == PH_EVAL ? ms[s].Dc : ms[s].D, ms[s].dt, m);
    const int e = threadIdx.x;
    int ei = 0, ej = 0;                                                  // component e: H(ei, ej) for e < 78, g(e - 78), cost
    if (e < 78) { int k = e; while (k >= 12 - ei) { k -= 12 - ei; ++ei; } ej = ei + k; }
    else if (e < 90) { ei = e - 78; ej = 12; }
    else { ei = 13; ej = -1; }
    double acc = 0.0;
    const size_t base = size_t(bv.offset[s]);
    __syncthreads();
#pragma unroll 1
    for (int r = 0; r < pts; ++r) {
        const uint32_t i = (blockIdx.x * uint32_t(pts) + uint32_t(r)) * kThreads + threadIdx.x;
        double row[14];
#pragma unroll
        for (int k = 0; k < 14; ++k) row[k] = 0.0;
        if (i < n) {
            const double wc = cb.w[base + i];
            if (wc != 0.0) {
                const double4 nd4 = cb.nd[base + i];
                const double nd[4] = {nd4.x, nd4.y, nd4.z, nd4.w};
                const size_t src = base + __float_as_uint(bv.scan[base + i].w);
                motion_row(m, nd, wc, __ldg(&raw[src]), __ldg(&times[src]), bv.tukey_a2, row);
            }
        }
#pragma unroll
        for (int k = 0; k < 14; ++k) rows[threadIdx.x * kRowStride + k] = row[k];
        __syncthreads();
        if (e < kMotionAcc) {
            if (ej >= 0) { for (int t = 0; t < kThreads; ++t) acc += rows[t * kRowStride + ei] * rows[t * kRowStride + ej]; }
            else { for (int t = 0; t < kThreads; ++t) acc += rows[t * kRowStride + ei]; }
        }
        __syncthreads();
    }
    if (e < kMotionAcc) partials[(size_t(s) * stride + blockIdx.x) * kMotionAcc + e] = acc;
}

// First edge-partial slot of chunk scan s (global scan first + s): edge clouds lie back to back, so slots s + eoffset / kThreads + b,
// b < ceil(n_edge / kThreads), never overlap and stay below the edge capacity's CTAs + max_batch
__device__ __forceinline__ size_t edge_slot(const uint32_t* eoffset, int s, uint32_t first) {
    return size_t(first) + size_t(s) + size_t(eoffset[s] / kThreads);
}

// The line rows of the edge cloud (so_register_optimized_edges): one edge point per thread from k_edge_fit's lines (EdgeBuf a / b, weight
// in a.w) and the raw edge point and time; the three rows of every point go through the same shared-memory reduction as k_motion_eval's
// one, row k of all the CTA's points before row k + 1.  91 sums per CTA into epartials.
template <int PHASE>
__global__ void __launch_bounds__(kThreads) k_motion_eval_edge(BatchView bv, EdgeBuf eb, const float4* __restrict__ raw, const float* __restrict__ times,
                                                               const MotionState* __restrict__ ms, double* __restrict__ epartials, uint32_t first) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PHASE) return;
    const uint32_t n = uint32_t(st->n_edge);
    if (blockIdx.x * kThreads >= n) return;
    __shared__ MotionCta m;
    __shared__ double rows[kThreads * kRowStride];
    if (threadIdx.x == 0) motion_cta_setup(PHASE == PH_EVAL ? st->cand : st->x, PHASE == PH_EVAL ? ms[s].Dc : ms[s].D, ms[s].dt, m);
    const int e = threadIdx.x;
    int ei = 0, ej = 0;
    if (e < 78) { int k = e; while (k >= 12 - ei) { k -= 12 - ei; ++ei; } ej = ei + k; }
    else if (e < 90) { ei = e - 78; ej = 12; }
    else { ei = 13; ej = -1; }
    __syncthreads();
    double lr[3][13], half = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int j = 0; j < 13; ++j) lr[k][j] = 0.0;
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i < n) {
        const size_t gi = size_t(eb.offset[s]) + i;
        const double4 a = eb.a[gi];
        if (a.w != 0.0) {                                                 // rejected points carry weight 0; NaN weights take part
            const double4 b = eb.b[gi];
            const double aa[3] = {a.x, a.y, a.z}, bb[3] = {b.x, b.y, b.z};
            motion_line_rows(m, aa, bb, a.w, __ldg(&raw[gi]), __ldg(&times[gi]), bv.tukey_a2_line, lr, &half);
        }
    }
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        for (int j = 0; j < 13; ++j) rows[threadIdx.x * kRowStride + j] = lr[k][j];
        rows[threadIdx.x * kRowStride + 13] = k == 0 ? half : 0.0;
        __syncthreads();
        if (e < kMotionAcc) {
            if (ej >= 0) { for (int t = 0; t < kThreads; ++t) acc += rows[t * kRowStride + ei] * rows[t * kRowStride + ej]; }
            else { for (int t = 0; t < kThreads; ++t) acc += rows[t * kRowStride + ei]; }
        }
        __syncthreads();
    }
    if (e < kMotionAcc) epartials[(edge_slot(eb.offset, s, first) + blockIdx.x) * kMotionAcc + e] = acc;
}

// ------------------------------------------------------------------------------------------------------------------ step
// The trust-region loop of so_trust_region.cuh over the 12 tangent columns of (T, D): Jacobi scaling and the LM diagonal over 12
// columns, x_norm and the step norm over the 14 ambient values, the gradient max-norm through Plus of both blocks, the prior rows
// on D.  Runs on one thread, on shared-memory copies of the two states.
__device__ __noinline__ void lm_continue(IcpState& st, MotionState& M, bool step_successful);

// SE3AbsolutatePoseFactor on D, multiplier sqrt(n_ok * info_k), measurement D0
__device__ __noinline__ void add_motion_prior(const MotionState& M, const double D[7], double a[kMotionAcc]) {
    add_se3_prior<12>(M.D0, M.sqrt_info, D, a);
}

// ||(x, D) - Plus((x, D), -g)||_inf over both blocks in one function (the larger of two grad_max_norm calls differs from it in the
// last bits of some solves' gmax)
__device__ __noinline__ double grad_max_norm(const IcpState& S, const MotionState& M) {
    double nt[6], nd[6], xp[7], dp[7];
    for (int j = 0; j < 6; ++j) { nt[j] = -M.g[j]; nd[j] = -M.g[6 + j]; }
    pose_plus(S.x, nt, xp);
    pose_plus(M.D, nd, dp);
    double m = 0.0;
    for (int i = 0; i < 7; ++i) m = fmax(m, fmax(fabs(S.x[i] - xp[i]), fabs(M.D[i] - dp[i])));
    return m;
}

struct TwoBlock {
    static constexpr int N = 12, kSums = kMotionAcc;
    // only with line rows (n_ok_edge > 0) does a non-finite first cost stop the registration; so_solve_optimized's caller-given
    // plane rows with a non-finite cost run the solve on
    static constexpr bool kAnyNonFinite = false;
    IcpState& st;
    MotionState& M;
    __device__ __forceinline__ double* scale() const { return M.scale; }
    __device__ __forceinline__ double* diag() const { return M.diag; }
    __device__ __forceinline__ void take(const double* acc) const {
        for (int k = 0; k < 78; ++k) M.H[k] = acc[k];
        for (int k = 0; k < 12; ++k) M.g[k] = acc[78 + k];
    }
    __device__ __forceinline__ void open_prior(double* acc, int n_ok) const {
        for (int k = 0; k < 6; ++k) M.sqrt_info[k] = sqrt(double(n_ok) * M.info[k]);
        add_motion_prior(M, M.D, acc);
    }
    __device__ __forceinline__ void prior_at_candidate(double* acc) const { add_motion_prior(M, M.Dc, acc); }
    __device__ __forceinline__ void init_scale() const { for (int j = 0; j < 12; ++j) M.scale[j] = 1.0 / (1.0 + sqrt(M.H[tri12(j, j)])); }
    __device__ __forceinline__ void scaled_system(double* Hs, double* gs) const {
        for (int i = 0; i < 12; ++i) {
            gs[i] = M.g[i] * M.scale[i];
            for (int j = 0; j < 12; ++j) Hs[i * 12 + j] = M.H[i <= j ? tri12(i, j) : tri12(j, i)] * M.scale[i] * M.scale[j];
        }
    }
    __device__ __forceinline__ void pad(double*) const {}
    __device__ __forceinline__ double x_norm2() const {      // pairwise in i, as step_norm2
        double xn = 0.0;
        for (int i = 0; i < 7; ++i) xn += st.x[i] * st.x[i] + M.D[i] * M.D[i];
        return xn;
    }
    __device__ __forceinline__ double step_norm2() const {
        double sn = 0.0;
        for (int i = 0; i < 7; ++i) { const double a = st.x[i] - st.cand[i], b = M.D[i] - M.Dc[i]; sn += a * a + b * b; }
        return sn;
    }
    __device__ __forceinline__ void accept() const { for (int i = 0; i < 7; ++i) { st.x[i] = st.cand[i]; M.D[i] = M.Dc[i]; } }
    __device__ __forceinline__ double gmax() const { return grad_max_norm(st, M); }
    __device__ __forceinline__ void candidate(const double* delta) const {
        pose_plus(st.x, delta, st.cand);
        pose_plus(M.D, delta + 6, M.Dc);
    }
    __device__ __forceinline__ void next(bool step_successful) const { lm_continue(st, M, step_successful); }
};

__device__ __noinline__ void lm_continue(IcpState& st, MotionState& M, bool step_successful) { tr_continue(TwoBlock{st, M}, step_successful); }
__device__ __noinline__ void lm_begin_solve(IcpState& st, MotionState& M, const double* acc_in, int n_ok) {
    tr_begin_solve(TwoBlock{st, M}, acc_in, n_ok, [&] { tr_start(TwoBlock{st, M}); });
}
__device__ __noinline__ void lm_after_eval(IcpState& st, MotionState& M, const double* acc_in) { tr_after_eval(TwoBlock{st, M}, acc_in); }

// ceres::Covariance{apply_loss_function, DENSE_SVD} over the 12 tangent columns on the CTA's first warp: cyclic Jacobi of H (each
// rotation's angle on lane 0, the rows of H on lanes 0-11, of the eigenvectors on lanes 12-23, the 2x2 block on lane 24), the
// pseudo-inverse dropping directions with s_i / s_max < sqrt(1e-14), and T's 6x6 block with EstimateRegistrationError's 3x3
// analyses into the scan's state, as covariance_and_errors_warp does for the 6-column solve.
struct Cov12 { double a[144], v[144], w[12], inv[12], t, c, s; int perm[12]; };

__device__ __noinline__ void cov12_warp(IcpState& S, const MotionState& M, Cov12& sc) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    for (int e = lane; e < 144; e += 32) {
        const int i = e / 12, j = e % 12;
        sc.a[e] = M.H[i <= j ? tri12(i, j) : tri12(j, i)];
        sc.v[e] = i == j ? 1.0 : 0.0;
    }
    __syncwarp();
#pragma unroll 1
    for (int sweep = 0; sweep < 30; ++sweep) {
        int stop = 0;
        if (lane == 0) {
            double off = 0.0, dia = 0.0;
            for (int p = 0; p < 12; ++p) { dia += sc.a[p * 12 + p] * sc.a[p * 12 + p]; for (int q = p + 1; q < 12; ++q) off += sc.a[p * 12 + q] * sc.a[p * 12 + q]; }
            stop = (off <= kJacobiOffTol * dia || off == 0.0) ? 1 : 0;
        }
        if (__shfl_sync(full, stop, 0)) break;
#pragma unroll 1
        for (int p = 0; p < 11; ++p) {
#pragma unroll 1
            for (int q = p + 1; q < 12; ++q) {
                if (lane == 0) {
                    const double apq = sc.a[p * 12 + q];
                    double t = 0.0;
                    if (apq != 0.0) {
                        const double dlt = sc.a[q * 12 + q] - sc.a[p * 12 + p], b2 = 2.0 * apq;
                        t = b2 / (fabs(dlt) + sqrt(dlt * dlt + b2 * b2));
                        if (dlt < 0.0) t = -t;
                    }
                    const double c = 1.0 / sqrt(t * t + 1.0);
                    sc.t = t; sc.c = c; sc.s = t * c;
                }
                __syncwarp();
                const double t = sc.t, c = sc.c, sn = sc.s;
                if (t != 0.0) {
                    const int r = lane < 12 ? lane : lane - 12;
                    const bool do_a = lane < 12 && r != p && r != q, do_v = lane >= 12 && lane < 24, do_d = lane == 24;
                    double n0 = 0.0, n1 = 0.0;
                    if (do_a) { const double arp = sc.a[r * 12 + p], arq = sc.a[r * 12 + q]; n0 = c * arp - sn * arq; n1 = sn * arp + c * arq; }
                    if (do_v) { const double vrp = sc.v[r * 12 + p], vrq = sc.v[r * 12 + q]; n0 = c * vrp - sn * vrq; n1 = sn * vrp + c * vrq; }
                    if (do_d) { const double apq = sc.a[p * 12 + q]; n0 = sc.a[p * 12 + p] - t * apq; n1 = sc.a[q * 12 + q] + t * apq; }
                    __syncwarp();
                    if (do_a) { sc.a[r * 12 + p] = sc.a[p * 12 + r] = n0; sc.a[r * 12 + q] = sc.a[q * 12 + r] = n1; }
                    if (do_v) { sc.v[r * 12 + p] = n0; sc.v[r * 12 + q] = n1; }
                    if (do_d) { sc.a[p * 12 + p] = n0; sc.a[q * 12 + q] = n1; sc.a[p * 12 + q] = 0.0; sc.a[q * 12 + p] = 0.0; }
                }
                __syncwarp();
            }
        }
    }
    if (lane == 0) {
        double w[12];
        int pm[12];
        for (int i = 0; i < 12; ++i) { w[i] = sc.a[i * 12 + i]; pm[i] = i; }
        for (int i = 0; i < 11; ++i)
            for (int j = i + 1; j < 12; ++j)
                if (w[j] < w[i]) { const double tw = w[i]; w[i] = w[j]; w[j] = tw; const int tp = pm[i]; pm[i] = pm[j]; pm[j] = tp; }
        const double lmax = w[11];
        bool cut = false;
        for (int i = 11; i >= 0; --i) {                                   // a cut direction cuts every smaller one
            const double ratio = (w[i] > 0.0 && lmax > 0.0) ? sqrt(w[i] / lmax) : 0.0;
            cut = cut || ratio < 1e-7;
            sc.inv[i] = cut ? 0.0 : 1.0 / w[i];
            sc.w[i] = w[i]; sc.perm[i] = pm[i];
        }
    }
    __syncwarp();
    for (int e = lane; e < 36; e += 32) {
        const int i = e / 6, j = e % 6;
        double t = 0.0;
        for (int k = 0; k < 12; ++k) t += sc.v[i * 12 + sc.perm[k]] * sc.inv[k] * sc.v[j * 12 + sc.perm[k]];
        S.cov[e] = t;
    }
    __syncwarp();
    registration_errors(S, lane);
}

// so_covariance (12 columns): cov12_warp on ms->H, in one 32-thread CTA and shared copies of both blocks as k_motion_step runs it
__global__ void __launch_bounds__(32) k_covariance12(IcpState* st, const MotionState* ms) {
    __shared__ IcpState s_st;
    __shared__ MotionState s_m;
    __shared__ Cov12 s_cov;
    cta_copy(&s_st, st);
    cta_copy(&s_m, ms);
    __syncthreads();
    cov12_warp(s_st, s_m, s_cov);
    __syncthreads();
    cta_copy(st, &s_st);
}

void launch_covariance12(IcpState* st, const MotionState* ms, cudaStream_t stream) { k_covariance12<<<1, 32, 0, stream>>>(st, ms); }

template <int AFTER>
__global__ void __launch_bounds__(128) k_motion_step(BatchView bv, MotionState* __restrict__ ms, const double* __restrict__ partials, uint32_t stride,
                                                      const double* __restrict__ epartials, const uint32_t* __restrict__ eoffset, uint32_t first) {
    const int s = blockIdx.x;
    IcpState* st = bv.st + s;
    if (st->phase != AFTER) return;
    __shared__ IcpState s_st;
    __shared__ MotionState s_m;
    __shared__ double s_sum[kMotionAcc];
    cta_copy(&s_st, st);
    cta_copy(&s_m, ms + s);
    if (threadIdx.x < kMotionAcc) {                                      // the scan's CTAs in index order
        const uint32_t np = eval_ctas(uint32_t(st->n_points));
        const double* base = partials + size_t(s) * stride * kMotionAcc + threadIdx.x;
        double v = 0.0;
        for (uint32_t b = 0; b < np; ++b) v += base[size_t(b) * kMotionAcc];
        const uint32_t ne = (uint32_t(st->n_edge) + kThreads - 1) / kThreads;          // the edge cloud's CTAs after the planes' (0: none)
        if (ne) {
            const double* eb = epartials + edge_slot(eoffset, s, first) * kMotionAcc + threadIdx.x;
            for (uint32_t b = 0; b < ne; ++b) v += eb[size_t(b) * kMotionAcc];
        }
        s_sum[threadIdx.x] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        IcpState& S = s_st;
        MotionState& M = s_m;
        if (AFTER == PH_CORR) {
            for (int k = 0; k < 9; ++k) S.hist_obs[k] = bv.hist[s * kHistStride + k];
            for (int k = 0; k < 7; ++k) S.hist_rej[k] = bv.hist[s * kHistStride + 9 + k];
            for (int k = 0; k < 7; ++k) S.hist_rej_line[k] = bv.hist[s * kHistStride + 16 + k];
            S.n_ok_edge = S.hist_rej_line[0];                            // 0 without an edge cloud
            const int n_ok = S.hist_rej[0] + S.n_ok_edge;                // features_corres.size(): planes plus lines
            for (int k = 0; k < kHistStride; ++k) bv.hist[s * kHistStride + k] = 0;
            if (M.stage) {                                               // so_evaluate_optimized: report the plane rows and stop
                for (int k = 0; k < 78; ++k) M.H[k] = s_sum[k];
                for (int k = 0; k < 12; ++k) M.g[k] = s_sum[78 + k];
                M.cost = s_sum[90]; S.n_ok = n_ok; S.n_iterations = 1; S.phase = PH_DONE;
            } else lm_begin_solve(S, M, s_sum, n_ok);
        } else lm_after_eval(S, M, s_sum);
    }
    __syncthreads();
    if (s_st.need_cov) {
        __shared__ Cov12 s_cov;
        if (threadIdx.x < 32) cov12_warp(s_st, s_m, s_cov);
        __syncthreads();
    }
    cta_copy(st, &s_st);
    cta_copy(ms + s, &s_m);
}

void launch_motion_warp(const BatchView& bv, float4* sorted, const float4* raw, const float* times, const MotionState* ms, uint32_t first,
                        uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const MotionEdges* me) {
    k_motion_warp<<<dim3(grid_x, n_scans), kThreads, 0, st>>>(bv, sorted, raw, times, ms + first);
    if (me && me->grid_e)
        k_motion_warp_edges<<<dim3(me->grid_e, n_scans), kThreads, 0, st>>>(bv, me->eb.offset, const_cast<float4*>(me->eb.scan), me->raw, me->times, ms + first);
}

void launch_motion_solve(int phase, const BatchView& bv, const CorrBuf& cb, const float4* raw, const float* times, MotionState* ms, uint32_t first,
                         double* partials, uint32_t stride, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const MotionEdges* me) {
    ms += first;
    const uint32_t gx = grid_x ? eval_grid(grid_x * kThreads) : 0;       // 0: every scan is empty; k_motion_step still ends their solves
    const uint32_t ge = me ? me->grid_e : 0;
    const uint32_t* eoff = me ? me->eb.offset : nullptr;
    double* ep = me ? me->partials : nullptr;
    if (phase == PH_CORR) {
        if (gx) k_motion_eval<PH_CORR><<<dim3(gx, n_scans), kThreads, 0, st>>>(bv, cb, raw, times, ms, partials, stride);
        if (ge) {
            launch_edge_fit(me->map, bv, me->eb, ge, n_scans, st);
            k_motion_eval_edge<PH_CORR><<<dim3(ge, n_scans), kThreads, 0, st>>>(bv, me->eb, me->raw, me->times, ms, ep, first);
        }
        k_motion_step<PH_CORR><<<n_scans, 128, 0, st>>>(bv, ms, partials, stride, ep, eoff, first);
    } else {
        if (gx) k_motion_eval<PH_EVAL><<<dim3(gx, n_scans), kThreads, 0, st>>>(bv, cb, raw, times, ms, partials, stride);
        if (ge) k_motion_eval_edge<PH_EVAL><<<dim3(ge, n_scans), kThreads, 0, st>>>(bv, me->eb, me->raw, me->times, ms, ep, first);
        k_motion_step<PH_EVAL><<<n_scans, 128, 0, st>>>(bv, ms, partials, stride, ep, eoff, first);
    }
}

int motion_tail(Ctx* c, float4* dst, const RegisteredScan& r) {
    if (!r.n) return SO_OK;
    MotionD D;
    for (int k = 0; k < 7; ++k) D.v[k] = r.D[k];
    timed_launch_begin(c);
    k_motion_cloud<<<(r.n + 255) / 256, 256, 0, c->stream>>>(dst, c->und.d_time, r.n, D, r.dt);
    timed_launch_end(c, 7);
    SO_CUDA_TRY(cudaGetLastError());
    return SO_OK;
}

int motion_edge_tail(Ctx* c, float4* dst, const RegisteredScan& r) {
    if (!r.n_edge) return SO_OK;
    MotionD D;
    for (int k = 0; k < 7; ++k) D.v[k] = r.D[k];
    timed_launch_begin(c);
    k_motion_cloud<<<(r.n_edge + 255) / 256, 256, 0, c->stream>>>(dst, c->und.d_etime, r.n_edge, D, r.dt);
    timed_launch_end(c, 7);
    SO_CUDA_TRY(cudaGetLastError());
    return SO_OK;
}


// ------------------------------------------------------------------------------------------------------------------ host side
int check_motion(const so_motion* m, const so_icp_opts* o) {
    if (!m || !o) return fail(SO_ERR_ARG, "bad args");
    if (!(std::isfinite(m->dt) && m->dt > 0.0)) return fail(SO_ERR_ARG, "so_motion.dt must be finite and > 0");
    if (!finite_pose(m->motion_prior)) return fail(SO_ERR_ARG, "so_motion.motion_prior must be finite with a non-zero quaternion");
    for (int k = 0; k < 6; ++k)
        if (!(std::isfinite(m->motion_info[k]) && m->motion_info[k] >= 0.0)) return fail(SO_ERR_ARG, "so_motion.motion_info must be finite and >= 0");
    if (o->use_pose_prior) return fail(SO_ERR_ARG, "use_pose_prior is not supported by so_register_optimized");
    return icp_opts_check(*o);
}

MotionState make_state(const so_motion& m) {
    MotionState M;
    std::memset(&M, 0, sizeof(M));
    const double* p = m.motion_prior;
    const double n = std::sqrt(p[3] * p[3] + p[4] * p[4] + p[5] * p[5] + p[6] * p[6]);
    for (int k = 0; k < 3; ++k) M.D0[k] = p[k];
    for (int k = 3; k < 7; ++k) M.D0[k] = p[k] / n;
    for (int k = 0; k < 7; ++k) M.D[k] = M.Dc[k] = M.D0[k];
    for (int k = 0; k < 6; ++k) M.info[k] = m.motion_info[k];
    M.dt = m.dt;
    return M;
}

int motion_reserve(Ctx* c, size_t n_points) {
    c->mot.stride = eval_grid(c->grid_x_cap * kThreads);
    int rc = c->mot.d_st.reserve(c->max_batch);
    if (!rc) rc = c->mot.d_partials.reserve(size_t(c->max_batch) * c->mot.stride * kMotionAcc);
    if (!rc) rc = c->und.d_time.reserve(std::max<size_t>(n_points, 1));
    return rc;
}

// The edge cloud's partials (edge_slot: at most the edge capacity's CTAs + max_batch slots), sized once, so that a captured schedule's
// pointer stays valid
int motion_edge_reserve(Ctx* c) {
    return c->mot.d_epartials.reserve((size_t(c->edge_grid_cap) + c->max_batch) * kMotionAcc);
}

// so_motion_result from the registration's result and the motion block: pose_end = T * D with T = pose_opt
void fill_motion(const so_icp_result& icp, const MotionState& M, so_motion_result* out) {
    out->icp = icp;
    for (int k = 0; k < 7; ++k) out->motion[k] = M.D[k];
    const double* T = icp.pose_opt;
    double t[3];
    qrot(T + 3, M.D, t);
    for (int k = 0; k < 3; ++k) out->pose_end[k] = T[k] + t[k];
    qmul(T + 3, M.D + 3, out->pose_end + 3);
}

}  // namespace so

using namespace so;

extern "C" {

// so_evaluate_optimized (edge == nullptr, n_edge == 0) and so_evaluate_optimized_edges
static int evaluate_optimized(so_ctx* ctx, const void* xyzi, size_t n, const void* edge, size_t n_edge, size_t stride, size_t ioff, size_t toff,
                              const double pose[7], const double motion[7], double dt, int32_t max_surface_features, double H[144], double g[12],
                              double* cost) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose || !motion || !xyzi || n == 0 || (!edge && n_edge) || stride < 12 || toff + 4 > stride || !finite_pose(pose))
        return fail(SO_ERR_ARG, "bad args");
    if (n_edge > c->edge_cap) return fail(SO_ERR_CAPACITY, "edge cloud larger than so_config.max_scan_points");
    so_motion m{};
    m.dt = dt;
    for (int k = 0; k < 7; ++k) m.motion_prior[k] = motion[k];
    so_icp_opts o{};
    o.max_icp_iters = 1; o.lm_max_iterations = 1; o.max_surface_features = max_surface_features; o.skip_map_checks = 1;
    int rc = check_motion(&m, &o);
    if (rc) return rc;
    if (n > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "scan larger than so_config.max_scan_points");
    MotionState M = make_state(m);
    M.stage = 1;
    const uint32_t nn = uint32_t(n);
    so_icp_result r;
    RegisterRequest q;                                                   // a stage evaluation leaves no registered scan and no pose row
    q.scans = xyzi; q.stride = stride; q.ioff = ioff; q.toff = toff; q.n_points = &nn; q.poses = pose; q.opts = &o;
    q.mode = UndistortionMode::OPTIMIZED; q.motion = &M; q.sink_rows = false; q.results = &r;
    const uint32_t ne = uint32_t(n_edge);
    if (ne) { q.edge = edge; q.n_edge = &ne; }
    rc = register_scans(c, q);
    if (rc) return rc;
    if (H) for (int i = 0; i < 12; ++i) for (int j = 0; j < 12; ++j) H[i * 12 + j] = M.H[i <= j ? tri12(i, j) : tri12(j, i)];
    if (g) for (int i = 0; i < 12; ++i) g[i] = M.g[i];
    if (cost) *cost = M.cost;
    return SO_OK;
}

int so_evaluate_optimized(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, size_t toff, const double pose[7],
                          const double motion[7], double dt, int32_t max_surface_features, double H[144], double g[12], double* cost) {
    return evaluate_optimized(ctx, xyzi, n, nullptr, 0, stride, ioff, toff, pose, motion, dt, max_surface_features, H, g, cost);
}

int so_evaluate_optimized_edges(so_ctx* ctx, const void* xyzi, size_t n, const void* edge, size_t n_edge, size_t stride, size_t ioff, size_t toff,
                                const double pose[7], const double motion[7], double dt, int32_t max_surface_features, double H[144],
                                double g[12], double* cost) {
    return evaluate_optimized(ctx, xyzi, n, edge, n_edge, stride, ioff, toff, pose, motion, dt, max_surface_features, H, g, cost);
}

}  // extern "C"

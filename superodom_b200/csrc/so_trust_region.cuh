#pragma once
// so_trust_region.cuh -- the device's trust-region solve, one loop for every parameter-block form.
//
// Restates ceres::Solve {max_num_iterations=4, DENSE_QR, defaults} of Ceres 2.0.0 as called at LidarSlam.cpp:230-240:
// TrustRegionMinimizer::Minimize, LevenbergMarquardtStrategy::ComputeStep/StepAccepted/StepRejected and the monotonic
// TrustRegionStepEvaluator, expressed on the robustified normal equations H = sum rho' J^T J, g = sum rho' J^T r
// (the QR of [J;D] that DENSE_QR performs solves exactly (H + D^2) y = g).  It runs on one thread of a step kernel, on shared-memory
// copies of the scan's states.  The loop (tr_begin_solve / tr_start / tr_continue / tr_after_eval) owns the control flow: the exit
// order and the ICP break rule (end_solve); every threshold, the step quality, the radius rule and the diagonal clamp come from
// so_trust_region_rule.h, which the pose graph's host loop shares.  A parameter-block policy P supplies what
// differs between the forms (so_icp.cu: Ambient and Reduced, six columns, and DegStart;
// so_motion.cu: TwoBlock, twelve):
//   N, kSums                     tangent columns; reduced sums per evaluation (upper triangle of H, g, cost)
//   kAnyNonFinite                whether any non-finite first cost stops the registration
//   scale() / diag()             the Jacobi scaling and the LM diagonal of the scaled system
//   take(acc)                    H and g from the sums;  init_scale(): the scaling at iteration 0
//   scaled_system(Hs, gs), pad(M)  the scaled system, and the LM matrix's padding (identity rows beyond the reduced columns)
//   x_norm2() / step_norm2()     squared norms over the ambient values;  gmax(): the gradient max-norm through Plus
//   candidate(delta), accept()   the scaled step into the candidate; the candidate into the iterate
//   open_prior(acc, n_ok) / prior_at_candidate(acc)  the prior rows at the iterate (solve start) and at the candidate
//   next(ok)                     the policy's __noinline__ entry of tr_continue
#include "so_internal.cuh"
#include "so_trust_region_rule.h"

namespace so {

// The registration's own termination code beside so_trust_region_rule.h's 0-5: a solve without rows
constexpr int kTermNoRows = 6;

// Copy of a state between global and shared memory by the CTA's threads, as 8-byte words
template <class T>
__device__ __forceinline__ void cta_copy(T* dst, const T* src) {
    static_assert(sizeof(T) % 8 == 0, "copied as 8-byte words");
    const unsigned long long* s = reinterpret_cast<const unsigned long long*>(src);
    unsigned long long* d = reinterpret_cast<unsigned long long*>(dst);
    for (uint32_t k = threadIdx.x; k < sizeof(T) / 8; k += blockDim.x) d[k] = s[k];
}

// Solve the SPD NxN system M y = r by Cholesky (M full row-major, destroyed).  Returns false on a non-positive pivot.  One reciprocal
// square root per column; every division by the pivot becomes a multiplication (the step this solves is compared with Ceres'
// QR-based one to ~1e-12 in any case: another algorithm, not another rounding).  N = 6 fully unrolled: every index is a compile-time
// constant, so the 36 + 18 values live in registers instead of a dynamically indexed local-memory array (the optimiser step is ONE
// thread's dependent FP64 chain; local-memory round trips were most of its 10-20 us).  N = 12 in loop form.
template <int N>
__device__ inline bool chol_solve(double* M, const double* r, double* y) {
    constexpr int U = N <= 6 ? N : 1;
    bool ok = true;
    double inv[N];
#pragma unroll U
    for (int j = 0; j < N; ++j) {
        double s = M[j * N + j];
#pragma unroll
        for (int k = 0; k < j; ++k) s -= M[j * N + k] * M[j * N + k];
        if (!(s > 0.0)) ok = false;
        const double il = rsqrt(s);
        inv[j] = il;
        M[j * N + j] = s * il;
#pragma unroll U
        for (int i = j + 1; i < N; ++i) {
            double t = M[i * N + j];
#pragma unroll
            for (int k = 0; k < j; ++k) t -= M[i * N + k] * M[j * N + k];
            M[i * N + j] = t * il;
        }
    }
    if (!ok) return false;
    double z[N];
#pragma unroll U
    for (int i = 0; i < N; ++i) {
        double t = r[i];
#pragma unroll
        for (int k = 0; k < i; ++k) t -= M[i * N + k] * z[k];
        z[i] = t * inv[i];
    }
#pragma unroll U
    for (int i = N - 1; i >= 0; --i) {
        double t = z[i];
#pragma unroll
        for (int k = i + 1; k < N; ++k) t -= M[k * N + i] * y[k];
        y[i] = t * inv[i];
    }
    return true;
}

// ||x - Plus(x, -g)||_inf of one pose block (TrustRegionMinimizer::EvaluateGradientAndJacobian)
inline __device__ __noinline__ double grad_max_norm(const double x[7], const double g[6]) {
    double neg[6], xp[7];
    _Pragma("unroll") for (int j = 0; j < 6; ++j) neg[j] = -g[j];
    pose_plus(x, neg, xp);
    double m = 0.0;
    _Pragma("unroll") for (int i = 0; i < 7; ++i) m = fmax(m, fabs(x[i] - xp[i]));
    return m;
}

// SE3AbsolutatePoseFactor (factor/SE3AbsolutatePoseFactor.cpp:9-51) at pose x: residual [p - p_meas ; 2 vec(q_meas^* q)] times
// sqrt_info (diagonal here), no loss function; local Jacobian [I 0; 0 (w I + [v]x)] of q_e = q_meas^* q (Utility::Qleft bottom-right
// block).  Adds its J^T J, J^T r and 1/2 r^T r to the reduced sums of an N-column solve whose last six columns are this block's:
// N = 6, the 28 sums of the pose; N = 12, the 91 sums of (T, D) at columns 6-11.
template <int N>
__device__ __forceinline__ void add_se3_prior(const double xm[7], const double sqrt_info[6], const double x[7], double* a) {
    constexpr int c0 = N - 6, g0 = N * (N + 1) / 2;
    const double qm[4] = {-xm[3], -xm[4], -xm[5], xm[6]};
    double e[4];
    qmul(qm, x + 3, e);
    double r[6] = {x[0] - xm[0], x[1] - xm[1], x[2] - xm[2], 2.0 * e[0], 2.0 * e[1], 2.0 * e[2]};
    double J[36];
    _Pragma("unroll") for (int i = 0; i < 36; ++i) J[i] = 0.0;
    J[0] = J[7] = J[14] = 1.0;
    J[3 * 6 + 3] = e[3];  J[3 * 6 + 4] = -e[2]; J[3 * 6 + 5] = e[1];
    J[4 * 6 + 3] = e[2];  J[4 * 6 + 4] = e[3];  J[4 * 6 + 5] = -e[0];
    J[5 * 6 + 3] = -e[1]; J[5 * 6 + 4] = e[0];  J[5 * 6 + 5] = e[3];
    _Pragma("unroll") for (int i = 0; i < 6; ++i) { r[i] *= sqrt_info[i]; _Pragma("unroll") for (int j = 0; j < 6; ++j) J[i * 6 + j] *= sqrt_info[i]; }
    _Pragma("unroll") for (int i = 0; i < 6; ++i) {
        _Pragma("unroll") for (int j = i; j < 6; ++j) {
            double t = 0.0;
            _Pragma("unroll") for (int k = 0; k < 6; ++k) t += J[k * 6 + i] * J[k * 6 + j];
            a[N == 6 ? tri(i, j) : tri12(c0 + i, c0 + j)] += t;
        }
        double t = 0.0; _Pragma("unroll") for (int k = 0; k < 6; ++k) t += J[k * 6 + i] * r[k];
        a[g0 + c0 + i] += t;
    }
    double sq = 0.0; _Pragma("unroll") for (int k = 0; k < 6; ++k) sq += r[k] * r[k];
    a[g0 + N] += 0.5 * sq;
}

// EstimateRegistrationError (LidarSlam.cpp:873-884) on S.cov: 3x3 eigen of the position (lane 0) / orientation (lane 1) blocks
__device__ __forceinline__ void registration_errors(IcpState& S, int lane) {
    if (lane < 2) {
        double M[9], E[9], e[3];
        const int o = lane * 3;
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) M[i * 3 + j] = S.cov[(i + o) * 6 + (j + o)];
        jacobi_eig<3, 20, true>(M, E, e);
        // the block is positive semi-definite: below a cut direction its smallest eigenvalue is zero and comes out as +-rounding,
        // read as 0 (the reference's sqrt of a negative rounding gives NaN; DESIGN.md section 3)
        const double err = sqrt(e[2]), inv_cond = sqrt(fmax(e[0], 0.0)) / sqrt(e[2]);
        if (lane == 0) { S.pos_err = err; S.pos_dir[0] = E[2]; S.pos_dir[1] = E[5]; S.pos_dir[2] = E[8]; S.pos_inv_cond = inv_cond; }
        else { S.ori_err_deg = err / M_PI * 180.0; S.ori_dir[0] = E[2]; S.ori_dir[1] = E[5]; S.ori_dir[2] = E[8]; S.ori_inv_cond = inv_cond; }
    }
    __syncwarp();
}

// End of one ceres::Solve == end of one ICP iteration (LidarSlam.cpp:134-146).
inline __device__ __noinline__ void end_solve(IcpState& st) {
    const int it = st.icp_iter;
    st.iter_n_surf[it] = st.n_ok - st.n_ok_edge;
    st.iter_n_edge[it] = st.n_ok_edge;
    rel_motion(st.x_iter_start, st.x, &st.iter_dtrans[it], &st.iter_drot[it]);      // recordIterationStats (:242-251)
    st.iter_lm_steps[it] = st.lm_iter;
    st.iter_lm_successful[it] = st.num_successful;
    st.iter_lm_termination[it] = st.termination;
    st.iter_cost[it] = st.cost;
    st.n_iterations = it + 1;
    // reference: ceres::Covariance CHECK-fails on an empty problem; we stop with a status.  use_prior is 0 in the two-block solve
    // (check_motion refuses use_pose_prior in OPTIMIZED): its prior rows on D alone do not make a problem.
    if (st.n_ok == 0 && !st.use_prior) {
        st.status = SO_STATUS_NO_CORRESPONDENCES; st.phase = PH_DONE; return;
    }
    if (st.num_successful == 1 || it == st.max_icp_iters - 1) {      // (:141)
        st.need_cov = 1;                          // first warp of the step kernel's CTA, right after this serial step
        st.phase = PH_DONE;
    } else {
        st.icp_iter = it + 1;
        st.phase = PH_CORR;
    }
}

// TrustRegionMinimizer loop from FinalizeIterationAndCheckIfMinimizerCanContinue up to the next cost evaluation
template <class P>
__device__ __forceinline__ void tr_continue(const P& p, bool step_successful) {
    constexpr int N = P::N;
    IcpState& st = p.st;
    for (;;) {
        tr_count(st, step_successful);
        if (tr_at_limit(st)) { st.termination = kTermIterations; end_solve(st); return; }
        if (tr_gradient_small(st)) { st.termination = kTermGradient; end_solve(st); return; }
        if (tr_radius_small(st)) { st.termination = kTermRadius; end_solve(st); return; }
        st.lm_iter++;
        step_successful = false;
        // LevenbergMarquardtStrategy::ComputeStep on the Jacobi-scaled system
        double Hs[N * N], gs[N];
        p.scaled_system(Hs, gs);
        if (!st.reuse_diagonal)
            _Pragma("unroll") for (int j = 0; j < N; ++j) p.diag()[j] = tr_lm_diagonal(Hs[j * N + j]);
        st.reuse_diagonal = 1;
        double M[N * N], y[N];
        _Pragma("unroll") for (int i = 0; i < N * N; ++i) M[i] = Hs[i];
        _Pragma("unroll") for (int j = 0; j < N; ++j) M[j * N + j] += p.diag()[j] / st.radius;       // lm_diagonal^2 = diagonal / radius
        p.pad(M);
        bool valid = chol_solve<N>(M, gs, y);
        double step[N], mcc = 0.0;
        if (valid) {
            _Pragma("unroll") for (int j = 0; j < N; ++j) { step[j] = -y[j]; valid = valid && isfinite(step[j]); }
            // model_cost_change = -(J step)'(f + J step / 2) = -step'gs - step'Hs step / 2
            double sg = 0.0, sHs = 0.0;
            _Pragma("unroll") for (int i = 0; i < N; ++i) { sg += step[i] * gs[i]; double t = 0.0; _Pragma("unroll") for (int j = 0; j < N; ++j) t += Hs[i * N + j] * step[j]; sHs += step[i] * t; }
            mcc = -sg - 0.5 * sHs;
        }
        if (!tr_step_valid(valid, mcc)) {       // HandleInvalidStep
            if (tr_invalid_step(st)) { st.termination = kTermInvalid; end_solve(st); return; }
            continue;
        }
        tr_valid_step(st);
        st.model_cost_change = mcc;
        double delta[N];
        _Pragma("unroll") for (int j = 0; j < N; ++j) delta[j] = step[j] * p.scale()[j];
        p.candidate(delta);
        st.phase = PH_EVAL;
        return;
    }
}

// IterationZero of a new solve, fed by the first evaluation's sums; start() takes the solve on from its first exits
template <class P, class F>
__device__ __forceinline__ void tr_begin_solve(const P& p, const double* acc_in, int n_ok, F start) {
    IcpState& st = p.st;
    double acc[P::kSums];
    _Pragma("unroll") for (int k = 0; k < P::kSums; ++k) acc[k] = acc_in[k];
    p.open_prior(acc, n_ok);
    p.take(acc);
    st.cost = acc[P::kSums - 1];
    st.n_ok = n_ok;
    _Pragma("unroll") for (int i = 0; i < 7; ++i) st.x_iter_start[i] = st.x[i];
    st.lm_iter = 0; st.num_successful = 0; st.num_unsuccessful = 0; st.consecutive_invalid = 0; st.termination = 0;
    if (n_ok == 0 && !st.use_prior) { st.termination = kTermNoRows; end_solve(st); return; }      // use_prior: see end_solve
    if ((P::kAnyNonFinite || st.n_ok_edge > 0) && !isfinite(st.cost)) {
        // A row's loss weight is not finite (ScaledLoss(TukeyLoss, w) with w = NaN: a line fit on an exactly collinear neighbourhood,
        // whose mean squared distance is rounding noise of either sign).  The reference CHECK-fails in ceres::Corrector here (Ceres
        // 2.0 corrector.cc: neither rho'' <= 0 nor rho' > 0 holds for NaN) and ends the process; the registration stops with a status
        // and the pose this ICP iteration started from (DESIGN.md section 3).
        const int it = st.icp_iter;
        st.iter_n_surf[it] = n_ok - st.n_ok_edge; st.iter_n_edge[it] = st.n_ok_edge; st.iter_cost[it] = st.cost;
        st.n_iterations = it + 1;
        st.status = SO_STATUS_INVALID_EVALUATION; st.phase = PH_DONE;
        return;
    }
    start();
}

// The rest of IterationZero: scaling, norms, radius, and the first step
template <class P>
__device__ __forceinline__ void tr_start(const P& p) {
    IcpState& st = p.st;
    p.init_scale();                                 // jacobi_scaling at iteration 0
    st.x_norm = sqrt(p.x_norm2());
    st.gmax = p.gmax();
    tr_iteration_zero(st);
    p.next(false);
}

// After the cost (and H, g) at the candidate are known
template <class P>
__device__ __forceinline__ void tr_after_eval(const P& p, const double* acc_in) {
    IcpState& st = p.st;
    double acc[P::kSums];
    _Pragma("unroll") for (int k = 0; k < P::kSums; ++k) acc[k] = acc_in[k];
    p.prior_at_candidate(acc);
    const double cand_cost = acc[P::kSums - 1];
    if (tr_parameter_small(st, p.step_norm2())) { st.termination = kTermParameter; end_solve(st); return; }
    const double cost_change = st.cost - cand_cost;
    if (tr_function_small(st, cost_change)) { st.termination = kTermFunction; end_solve(st); return; }
    const double rd = cost_change / st.model_cost_change;
    if (tr_step_rejected(rd)) {         // StepRejected
        tr_rejected(st);
        p.next(false);
    } else {                            // HandleSuccessfulStep
        p.accept();
        st.x_norm = sqrt(p.x_norm2());
        p.take(acc);
        st.cost = cand_cost;
        st.gmax = p.gmax();
        tr_accepted(st, rd);
        p.next(true);
    }
}

}  // namespace so

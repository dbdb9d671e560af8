// so_icp.cu -- sm_90a kernels of the per-scan ICP registration path.
//
//   k_scan_keys / k_scan_gather : order the scan by map cell once per registration (warp-coherent cell walks).
//   k_knn_scan   : per scan point -- pose transform, block lookup, radius-bounded 5-NN in the sorted hash grid
//                  (three-round select: bound, gather, refine); hands the five neighbours to k_fit.         [a5-a7]
//   k_fit        : 3x3 PCA + 5x3 column-pivoted QR plane fit with the reference's accept/reject gates, observability
//                  labels + histograms, fit weight; writes the correspondence record.                     [a8-a11]
//   k_evaluate   : per correspondence -- residual, 1x6 Jacobian, Tukey/Scaled robust weight at the matched pose (first
//                  evaluation of a solve) or at the LM candidate, warp/CTA-reduced in FP64 (21+6+1 accumulators). [a12-a13]
//   k_edge_fit / k_edge_evaluate : the edge / line branch (10-NN in the edge map, best-line selection, line factor).   [a19]
//   k_lm_step    : fixed-order cross-CTA reduction, then ONE thread per scan advances the device-resident state
//                  machine: Ceres' trust-region LM (step solve by 6x6 Cholesky, accept/reject, tolerances), the SE3 prior
//                  rows, the outer ICP convergence rule, and at the end the covariance pseudo-inverse + 3x3 eigen
//                  analysis.                                                                        [a3, a14-a16, a20]
//   k_loop_cond  : CUDA-graph WHILE condition of a chunk (any scan still iterating).
//   k_knn        : stand-alone k-NN (so_knn*), radius-bounded or exact with ring expansion.
//
// Reference citations are relative to /root/reference/super_odometry/.
#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>

#include "so_icp.cuh"
#include "so_knn.cuh"
#include "so_trust_region.cuh"

namespace so {

// ------------------------------------------------------------------------------------------------------------------
// CTA reduction of kAcc doubles per thread into partials[scan][cta][kAcc].  Fixed thread->point mapping and fixed
// reduction trees => run-to-run deterministic sums.  The cross-CTA sum and the optimiser step run in k_lm_step
// (keeping that scalar FP64 code out of the per-point kernels saves ~70 registers per thread in them).
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void reduce_to_partials(double acc[kAcc], const BatchView& bv, int s, uint32_t slot_offset = 0) {
    static_assert(kAcc <= 32, "one component per lane");
    __shared__ double s_red[kThreads / 32][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // Warp stage: a halving butterfly.  At distance o each lane keeps the half of its (padded to 32) components that matches
    // its lane bit, hands the other half to its partner and adds what it receives, so lane l ends up with the warp total of
    // component l after 16+8+4+2+1 = 31 FP64 shuffles -- the SHFL pipe (one warp-wide shuffle per clock per SM) was the
    // cost of the plain 28 x 5 butterfly.
    double v[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) v[k] = k < kAcc ? acc[k] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const bool up = (lane & o) != 0;
#pragma unroll
        for (int k = 0; k < o; ++k) {
            const double send = up ? v[k] : v[k + o];
            const double keep = up ? v[k + o] : v[k];
            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
    }
    s_red[warp][lane] = v[0];
    __syncthreads();
    if (threadIdx.x < kAcc) {
        double t = 0.0;
#pragma unroll
        for (int wv = 0; wv < kThreads / 32; ++wv) t += s_red[wv][threadIdx.x];
        bv.partials[(size_t(s) * bv.partial_stride + slot_offset + blockIdx.x) * kAcc + threadIdx.x] = t;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Device-resident optimiser state machine (runs on one thread of the last CTA): the trust-region loop of so_trust_region.cuh
// over the pose's six tangent columns.
// ------------------------------------------------------------------------------------------------------------------
// ceres::Covariance + EstimateRegistrationError at the end of a registration, on the 32 lanes of the CTA's first warp (S and sc in
// shared memory).  The 6x6 cyclic Jacobi (at most 30 sweeps, convergence test of jacobi_eig, FP64 angles) takes its rotations in
// ROUND-ROBIN order: five rounds of three pairs with disjoint indices -- (0,5)(1,4)(2,3) / (0,4)(3,5)(1,2) / (0,3)(2,4)(1,5) /
// (0,2)(1,3)(4,5) / (0,1)(2,5)(3,4).  The angle of a pair depends only on its own 2x2 block, which the other two rotations of the
// round do not touch, so the three angles of a round are computed by three lanes at once; each rotation then updates its 8
// off-diagonal entries, 12 eigenvector entries and 2x2 block on 15 lanes in one step instead of ~110 dependent FP64 instructions
// on one thread (on one thread the covariance was 38 of the ~50 us the last optimiser step of a registration took).
__constant__ int c_rr_p[15] = {0, 1, 2, 0, 3, 1, 0, 2, 1, 0, 1, 4, 0, 2, 3};
__constant__ int c_rr_q[15] = {5, 4, 3, 4, 5, 2, 3, 4, 5, 2, 3, 5, 1, 5, 4};
struct CovScratch { double a[36], v[36], w[6], inv[6], t[3], c[3], s[3]; int perm[6]; };

__device__ __noinline__ void covariance_and_errors_warp(IcpState& S, CovScratch& sc) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    for (int e = lane; e < 36; e += 32) {
        const int i = e / 6, j = e % 6;
        sc.a[e] = S.H[i <= j ? tri(i, j) : tri(j, i)];
        sc.v[e] = i == j ? 1.0 : 0.0;
    }
    __syncwarp();
#pragma unroll 1
    for (int sweep = 0; sweep < 30; ++sweep) {
        int stop = 0;
        if (lane == 0) {
            double off = 0.0, dia = 0.0;
#pragma unroll
            for (int p = 0; p < 6; ++p) {
                dia += sc.a[p * 6 + p] * sc.a[p * 6 + p];
#pragma unroll
                for (int q = p + 1; q < 6; ++q) off += sc.a[p * 6 + q] * sc.a[p * 6 + q];
            }
            stop = (off <= kJacobiOffTol * dia || off == 0.0) ? 1 : 0;
        }
        if (__shfl_sync(full, stop, 0)) break;
#pragma unroll 1
        for (int round = 0; round < 5; ++round) {
            if (lane < 3) {                                  // the three angles of the round (disjoint 2x2 blocks)
                const int p = c_rr_p[round * 3 + lane], q = c_rr_q[round * 3 + lane];
                // the angle in FP64: the update below (a_pp - t a_pq, a_qq + t a_pq, a_pq := 0) is exact only for the exact angle, and
                // an FP32 one left a backward error of 1e-7 |a_pq| per rotation -- cov off by ~1e-8 kappa(H) relative
                const double apq = sc.a[p * 6 + q];
                double t = 0.0;
                if (apq != 0.0) {
                    const double dlt = sc.a[q * 6 + q] - sc.a[p * 6 + p], b2 = 2.0 * apq;
                    t = b2 / (fabs(dlt) + sqrt(dlt * dlt + b2 * b2));
                    if (dlt < 0.0) t = -t;
                }
                const double c = rsqrt(t * t + 1.0);
                sc.t[lane] = t; sc.c[lane] = c; sc.s[lane] = t * c;
            }
            __syncwarp();
#pragma unroll 1
            for (int k = 0; k < 3; ++k) {
                const int p = c_rr_p[round * 3 + k], q = c_rr_q[round * 3 + k];
                const double t = sc.t[k], c = sc.c[k], sn = sc.s[k];
                if (t != 0.0) {                              // warp-uniform
                    // lanes 0..5: row r of a (r outside the pair); lanes 8..13: row r of v; lane 16: the 2x2 block
                    const int r = lane < 8 ? lane : lane - 8;
                    const bool do_a = lane < 6 && r != p && r != q, do_v = lane >= 8 && lane < 14, do_d = lane == 16;
                    double n0 = 0.0, n1 = 0.0;
                    if (do_a) { const double arp = sc.a[r * 6 + p], arq = sc.a[r * 6 + q]; n0 = c * arp - sn * arq; n1 = sn * arp + c * arq; }
                    if (do_v) { const double vrp = sc.v[r * 6 + p], vrq = sc.v[r * 6 + q]; n0 = c * vrp - sn * vrq; n1 = sn * vrp + c * vrq; }
                    if (do_d) { const double apq = sc.a[p * 6 + q]; n0 = sc.a[p * 6 + p] - t * apq; n1 = sc.a[q * 6 + q] + t * apq; }
                    __syncwarp();
                    if (do_a) { sc.a[r * 6 + p] = sc.a[p * 6 + r] = n0; sc.a[r * 6 + q] = sc.a[q * 6 + r] = n1; }
                    if (do_v) { sc.v[r * 6 + p] = n0; sc.v[r * 6 + q] = n1; }
                    if (do_d) { sc.a[p * 6 + p] = n0; sc.a[q * 6 + q] = n1; sc.a[p * 6 + q] = 0.0; sc.a[q * 6 + p] = 0.0; }
                    __syncwarp();
                }
            }
        }
    }
    if (lane == 0) {                                         // ascending order, as a column permutation
        double w[6];
        int pm[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) { w[i] = sc.a[i * 6 + i]; pm[i] = i; }
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
            for (int j = i + 1; j < 6; ++j)
                if (w[j] < w[i]) { const double tw = w[i]; w[i] = w[j]; w[j] = tw; const int tp = pm[i]; pm[i] = pm[j]; pm[j] = tp; }
#pragma unroll
        for (int i = 0; i < 6; ++i) { sc.w[i] = w[i]; sc.perm[i] = pm[i]; }
    }
    __syncwarp();
    {
        const int e0 = lane, e1 = lane + 32;
        const double v0 = sc.v[(e0 / 6) * 6 + sc.perm[e0 % 6]];
        const double v1 = e1 < 36 ? sc.v[(e1 / 6) * 6 + sc.perm[e1 % 6]] : 0.0;
        __syncwarp();
        sc.v[e0] = v0;
        if (e1 < 36) sc.v[e1] = v1;
    }
    __syncwarp();
    // ceres::Covariance{apply_loss_function, DENSE_SVD, null_space_rank=-1} in tangent space (LidarSlam.cpp:854-871):
    // pseudo-inverse of J^T J dropping singular directions with s_i/s_max < sqrt(1e-14) (covariance_impl.cc).
    {
        const double lmax = sc.w[5];
        const double wk = lane < 6 ? sc.w[lane] : 1.0;
        const double ratio = (wk > 0.0 && lmax > 0.0) ? sqrt(wk / lmax) : 0.0;
        const unsigned bad = __ballot_sync(full, lane < 6 && ratio < 1e-7);
        if (lane < 6) sc.inv[lane] = (bad >> lane) ? 0.0 : 1.0 / wk;     // a cut direction cuts every smaller one (descending singular values)
    }
    __syncwarp();
    for (int e = lane; e < 36; e += 32) {
        const int i = e / 6, j = e % 6;
        double t = 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) t += sc.v[i * 6 + k] * sc.inv[k] * sc.v[j * 6 + k];
        S.cov[e] = t;
    }
    __syncwarp();
    registration_errors(S, lane);
}

// Reduced system of a degeneracy-aware solve: Hr = B^T H B and gr = B^T g over the columns of B (zero beyond dg.m, so Hr and gr are
// zero-padded to 6).
__device__ __forceinline__ void reduced_system(const IcpState& st, const DegenState& dg, double Hr[36], double gr[6]) {
    double HB[36];
    _Pragma("unroll") for (int i = 0; i < 6; ++i)
        _Pragma("unroll") for (int k = 0; k < 6; ++k) {
            double t = 0.0;
            _Pragma("unroll") for (int j = 0; j < 6; ++j) t += st.H[i <= j ? tri(i, j) : tri(j, i)] * dg.B[j * 6 + k];
            HB[i * 6 + k] = t;
        }
    _Pragma("unroll") for (int k = 0; k < 6; ++k) {
        double t = 0.0;
        _Pragma("unroll") for (int i = 0; i < 6; ++i) t += dg.B[i * 6 + k] * st.g[i];
        gr[k] = t;
        _Pragma("unroll") for (int l = 0; l < 6; ++l) {
            double u = 0.0;
            _Pragma("unroll") for (int i = 0; i < 6; ++i) u += dg.B[i * 6 + k] * HB[i * 6 + l];
            Hr[k * 6 + l] = u;
        }
    }
}

// ||x - Plus(x, -B B^T g)||_inf: the gradient max-norm of the solve on B's columns.  (Not through grad_max_norm: a caller with a
// local-memory g would change the code of the ambient solve, whose callers all pass shared memory.)
__device__ __noinline__ double grad_max_norm_red(const double x[7], const double g[6], const DegenState& dg) {
    double gr[6], neg[6], xp[7];
    _Pragma("unroll") for (int k = 0; k < 6; ++k) { double t = 0.0; _Pragma("unroll") for (int i = 0; i < 6; ++i) t += dg.B[i * 6 + k] * g[i]; gr[k] = t; }
    _Pragma("unroll") for (int i = 0; i < 6; ++i) { double t = 0.0; _Pragma("unroll") for (int k = 0; k < 6; ++k) t += dg.B[i * 6 + k] * gr[k]; neg[i] = -t; }
    pose_plus(x, neg, xp);
    double m = 0.0;
    _Pragma("unroll") for (int i = 0; i < 7; ++i) m = fmax(m, fabs(x[i] - xp[i]));
    return m;
}

// Pseudo-inverse of a symmetric 3x3 with ceres::Covariance's cut rule (covariance_and_errors_warp): eigen-directions with
// sqrt(w_k / w_max) < 1e-7 or w_k <= 0 are dropped.
__device__ __forceinline__ void pinv3_cut(const double A[9], double P[9]) {
    double a[9], v[9], w[3];
    _Pragma("unroll") for (int i = 0; i < 9; ++i) a[i] = A[i];
    jacobi_eig<3, 20, true>(a, v, w);
    double inv[3];
    _Pragma("unroll") for (int k = 0; k < 3; ++k) {
        const double ratio = (w[k] > 0.0 && w[2] > 0.0) ? sqrt(w[k] / w[2]) : 0.0;
        inv[k] = ratio < 1e-7 ? 0.0 : 1.0 / w[k];
    }
    _Pragma("unroll") for (int i = 0; i < 3; ++i)
        _Pragma("unroll") for (int j = 0; j < 3; ++j) {
            double t = 0.0;
            _Pragma("unroll") for (int k = 0; k < 3; ++k) t += v[i * 3 + k] * inv[k] * v[j * 3 + k];
            P[i * 3 + j] = t;
        }
}

// Information of one block: the Schur complement I = A - C P C^T (P the cut pseudo-inverse of the other block), its eigenpairs
// (ascending) and the flagged ones (i_k <= thr2 * max(i_max, 0)).  C: the 3x3 coupling, rows this block, columns the other one.
__device__ __forceinline__ int block_information(const double A[9], const double C[9], const double Other[9], double thr2, double info[3], double axes[9]) {
    double P[9], CP[9], I[9], v[9];
    pinv3_cut(Other, P);
    _Pragma("unroll") for (int i = 0; i < 3; ++i)
        _Pragma("unroll") for (int j = 0; j < 3; ++j) {
            double t = 0.0;
            _Pragma("unroll") for (int k = 0; k < 3; ++k) t += C[i * 3 + k] * P[k * 3 + j];
            CP[i * 3 + j] = t;
        }
    _Pragma("unroll") for (int i = 0; i < 3; ++i)
        _Pragma("unroll") for (int j = i; j < 3; ++j) {
            double t = 0.0;
            _Pragma("unroll") for (int k = 0; k < 3; ++k) t += CP[i * 3 + k] * C[j * 3 + k];
            I[i * 3 + j] = I[j * 3 + i] = A[i * 3 + j] - t;      // symmetric by construction
        }
    jacobi_eig<3, 20, true>(I, v, info);
    int flags = 0;
    const double cut = thr2 * fmax(info[2], 0.0);
    _Pragma("unroll") for (int k = 0; k < 3; ++k) {
        _Pragma("unroll") for (int i = 0; i < 3; ++i) axes[k * 3 + i] = v[i * 3 + k];
        if (info[k] <= cut) flags |= 1 << k;
    }
    return flags;
}

// The degeneracy analysis of a solve (DESIGN.md section 3) on the normal matrix H (upper triangle, order t, theta): I_t and I_theta,
// their eigenpairs and flags, and B = the unflagged eigenvectors (translation ones first).  m = 6 unless constrain and something is
// flagged; B is then the identity.
__device__ __noinline__ void degeneracy_analysis(const double Hu[21], DegenState& dg) {
    double Htt[9], Htr[9], Hrt[9], Hrr[9];
    _Pragma("unroll") for (int i = 0; i < 3; ++i)
        _Pragma("unroll") for (int j = 0; j < 3; ++j) {
            Htt[i * 3 + j] = Hu[i <= j ? tri(i, j) : tri(j, i)];
            Hrr[i * 3 + j] = Hu[i <= j ? tri(i + 3, j + 3) : tri(j + 3, i + 3)];
            Htr[i * 3 + j] = Hu[tri(i, j + 3)];
            Hrt[j * 3 + i] = Hu[tri(i, j + 3)];
        }
    dg.flags_pos = block_information(Htt, Htr, Hrr, dg.pos_thr2, dg.pos_info, dg.pos_axes);
    dg.flags_ori = block_information(Hrr, Hrt, Htt, dg.ori_thr2, dg.ori_info, dg.ori_axes);
    _Pragma("unroll") for (int i = 0; i < 36; ++i) dg.B[i] = 0.0;
    const bool reduce = dg.constrain && (dg.flags_pos | dg.flags_ori);
    int m = 0;
    _Pragma("unroll") for (int k = 0; k < 6; ++k) {
        const bool pos = k < 3;
        const int e = pos ? k : k - 3;
        if (!reduce) { dg.B[k * 6 + k] = 1.0; ++m; continue; }
        if (((pos ? dg.flags_pos : dg.flags_ori) >> e) & 1) continue;
        const double* ax = (pos ? dg.pos_axes : dg.ori_axes) + 3 * e;
        _Pragma("unroll") for (int i = 0; i < 3; ++i) dg.B[(i + (pos ? 0 : 3)) * 6 + m] = ax[i];
        ++m;
    }
    dg.m = m;
}

__device__ __noinline__ void lm_continue(IcpState& st, bool step_successful);
__device__ __noinline__ void lm_continue_red(IcpState& st, const DegenState& dg, bool step_successful);

// The SE3 prior of addAbsolutePoseConstraints (LidarSlam.cpp:285-298) on the pose x, T_meas = T_w_initial_guess
__device__ __noinline__ void add_pose_prior(const IcpState& st, const double x[7], double a[kAcc]) {
    add_se3_prior<6>(st.x0, st.prior_sqrt_info, x, a);
}

// The six-column solve on the pose (x [+] delta): H, g, scale and diag in IcpState; the prior rows on x when use_prior
struct Ambient {
    static constexpr int N = 6, kSums = kAcc;
    static constexpr bool kAnyNonFinite = true;
    IcpState& st;
    __device__ __forceinline__ double* scale() const { return st.scale; }
    __device__ __forceinline__ double* diag() const { return st.diag; }
    __device__ __forceinline__ void take(const double* acc) const {
        _Pragma("unroll") for (int k = 0; k < 21; ++k) st.H[k] = acc[k];
        _Pragma("unroll") for (int k = 0; k < 6; ++k) st.g[k] = acc[21 + k];
    }
    __device__ __forceinline__ void open_prior(double* acc, int n_ok) const {
        if (st.use_prior) {
            // information diagonal (LidarSlam.cpp:287-294); sqrt by Eigen's unblocked LLT: the first non-positive pivot and everything
            // after it stay un-square-rooted
            const double vcf = double(st.prior_vcf);
            double info[6];
            const int m1 = max(50, int(n_ok * 0.1)), m2 = max(10, int(n_ok * 0.01));
            _Pragma("unroll") for (int a = 0; a < 3; ++a) info[a] = (1 - double(st.prior_unc[a])) * m1 * vcf;
            info[3] = info[4] = m2 * vcf;
            info[5] = max(5, int(n_ok * 0.001)) * 0;
            bool failed = false;
            _Pragma("unroll") for (int k = 0; k < 6; ++k) { if (!failed && info[k] <= 0.0) failed = true; st.prior_sqrt_info[k] = failed ? info[k] : sqrt(info[k]); }
            add_pose_prior(st, st.x, acc);
        }
    }
    __device__ __forceinline__ void prior_at_candidate(double* acc) const { if (st.use_prior) add_pose_prior(st, st.cand, acc); }
    __device__ __forceinline__ void init_scale() const {
        _Pragma("unroll") for (int j = 0; j < 6; ++j) st.scale[j] = 1.0 / (1.0 + sqrt(st.H[tri(j, j)]));
    }
    __device__ __forceinline__ void scaled_system(double* Hs, double* gs) const {
        _Pragma("unroll") for (int i = 0; i < 6; ++i) {
            gs[i] = st.g[i] * st.scale[i];
            _Pragma("unroll") for (int j = 0; j < 6; ++j) Hs[i * 6 + j] = st.H[i <= j ? tri(i, j) : tri(j, i)] * st.scale[i] * st.scale[j];
        }
    }
    __device__ __forceinline__ void pad(double*) const {}
    __device__ __forceinline__ double x_norm2() const {
        double xn = 0.0; _Pragma("unroll") for (int i = 0; i < 7; ++i) xn += st.x[i] * st.x[i];
        return xn;
    }
    __device__ __forceinline__ double step_norm2() const {
        double sn = 0.0; _Pragma("unroll") for (int i = 0; i < 7; ++i) { const double d = st.x[i] - st.cand[i]; sn += d * d; }
        return sn;
    }
    __device__ __forceinline__ void accept() const { _Pragma("unroll") for (int i = 0; i < 7; ++i) st.x[i] = st.cand[i]; }
    __device__ __forceinline__ double gmax() const { return grad_max_norm(st.x, st.g); }
    __device__ __forceinline__ void candidate(const double* delta) const { pose_plus(st.x, delta, st.cand); }
    __device__ __forceinline__ void next(bool step_successful) const { lm_continue(st, step_successful); }
};

// The degeneracy-aware solve on the m < 6 columns of dg.B (local parameterisation x [+] B y): Jacobi scaling, LM diagonal and model
// cost change of the reduced system, which is padded to 6 with identity rows and zero right-hand sides for chol_solve<6>
struct Reduced : Ambient {
    const DegenState& dg;
    __device__ __forceinline__ void init_scale() const {
        double Hr[36], gr[6];
        reduced_system(st, dg, Hr, gr);
        _Pragma("unroll") for (int j = 0; j < 6; ++j) st.scale[j] = 1.0 / (1.0 + sqrt(Hr[j * 6 + j]));
    }
    __device__ __forceinline__ void scaled_system(double* Hs, double* gs) const {
        double Hr[36], gr[6];
        reduced_system(st, dg, Hr, gr);
        _Pragma("unroll") for (int i = 0; i < 6; ++i) {
            gs[i] = gr[i] * st.scale[i];
            _Pragma("unroll") for (int j = 0; j < 6; ++j) Hs[i * 6 + j] = Hr[i * 6 + j] * st.scale[i] * st.scale[j];
        }
    }
    __device__ __forceinline__ void pad(double* M) const { _Pragma("unroll") for (int j = 0; j < 6; ++j) if (j >= dg.m) M[j * 6 + j] = 1.0; }
    __device__ __forceinline__ double gmax() const { return grad_max_norm_red(st.x, st.g, dg); }
    __device__ __forceinline__ void candidate(const double* delta) const {      // the ambient step B y
        double d6[6];
        _Pragma("unroll") for (int i = 0; i < 6; ++i) { double t = 0.0; _Pragma("unroll") for (int k = 0; k < 6; ++k) t += dg.B[i * 6 + k] * delta[k]; d6[i] = t; }
        pose_plus(st.x, d6, st.cand);
    }
    __device__ __forceinline__ void next(bool step_successful) const { lm_continue_red(st, dg, step_successful); }
};

// IterationZero's tail in the degeneracy-aware solve: on B's columns when the analysis left fewer than 6, else the ambient one
struct DegStart : Ambient {
    const DegenState& dg;
    bool red;
    __device__ __forceinline__ void init_scale() const { if (red) Reduced{{st}, dg}.init_scale(); else Ambient::init_scale(); }
    __device__ __forceinline__ double gmax() const { return red ? grad_max_norm_red(st.x, st.g, dg) : grad_max_norm(st.x, st.g); }
    __device__ __forceinline__ void next(bool step_successful) const { if (red) lm_continue_red(st, dg, step_successful); else lm_continue(st, step_successful); }
};

__device__ __noinline__ void lm_continue(IcpState& st, bool step_successful) { tr_continue(Ambient{st}, step_successful); }
__device__ __noinline__ void lm_continue_red(IcpState& st, const DegenState& dg, bool step_successful) { tr_continue(Reduced{{st}, dg}, step_successful); }

// IterationZero of a new solve, fed by k_fit's reduction
__device__ __noinline__ void lm_begin_solve(IcpState& st, const double* acc_in, int n_ok) {
    tr_begin_solve(Ambient{st}, acc_in, n_ok, [&] { tr_start(Ambient{st}); });
}
// ... of the degeneracy-aware solve: the analysis on H at x_iter_start, then the solve on B's columns when it has fewer than 6
// (otherwise exactly the ambient solve)
__device__ __noinline__ void lm_begin_solve_deg(IcpState& st, DegenState& dg, const double* acc_in, int n_ok) {
    tr_begin_solve(Ambient{st}, acc_in, n_ok, [&] {
        degeneracy_analysis(st.H, dg);
        dg.iter_n_flag_pos[st.icp_iter] = __popc(dg.flags_pos);
        dg.iter_n_flag_ori[st.icp_iter] = __popc(dg.flags_ori);
        tr_start(DegStart{{st}, dg, dg.m < 6});
    });
}

// After the cost (and H, g) at the candidate are known
__device__ __noinline__ void lm_after_eval(IcpState& st, const double* acc_in) { tr_after_eval(Ambient{st}, acc_in); }
// the degeneracy-aware solve's: on B's columns when it has fewer than 6, else the ambient step (its own copy: a third caller of
// lm_after_eval changes that function's code in the other kernels)
__device__ __noinline__ void lm_after_eval_deg(IcpState& st, const DegenState& dg, const double* acc_in) {
    if (dg.m < 6) tr_after_eval(Reduced{{st}, dg}, acc_in);
    else tr_after_eval(Ambient{st}, acc_in);
}

// ------------------------------------------------------------------------------------------------------------------
// residual + Jacobian + robust weight accumulation for one correspondence at pose (q, t) with rotation matrix R.
// SurfNormAnalyticCostFunction::Evaluate (lidarOptimization.cpp:55-80); ScaledLoss(TukeyLoss(a), w) through Ceres'
// Corrector: Tukey has rho'' <= 0, so residual and Jacobian are both scaled by sqrt(rho') (corrector.cc);
// TukeyLoss of Ceres 2.0.0: rho = a^2/6 (1-(1-s/a^2)^3), rho' = (1-s/a^2)^2 / 2 for s <= a^2.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void accumulate(double acc[kAcc], const double n[3], double d, double w, const double p[3],
                                           const double pw[3], const double R[9], double a2) {
    const double r = n[0] * pw[0] + n[1] * pw[1] + n[2] * pw[2] + d;
    const double s = r * r;
    double rho0, rho1;
    if (s <= a2) { const double v = 1.0 - s / a2, v2 = v * v; rho0 = a2 / 6.0 * (1.0 - v2 * v); rho1 = 0.5 * v2; }      // TukeyLoss::Evaluate divides (loss_function.cc)
    else { rho0 = a2 / 6.0; rho1 = 0.0; }
    rho0 *= w; rho1 *= w;
    // J = [ n^T , -n^T R [p]x ] ;  -a^T [p]x = p x a  with a = R^T n
    const double a0 = R[0] * n[0] + R[3] * n[1] + R[6] * n[2];
    const double a1 = R[1] * n[0] + R[4] * n[1] + R[7] * n[2];
    const double a2v = R[2] * n[0] + R[5] * n[1] + R[8] * n[2];
    const double J[6] = {n[0], n[1], n[2], p[1] * a2v - p[2] * a1, p[2] * a0 - p[0] * a2v, p[0] * a1 - p[1] * a0};
    int k = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        const double wi = rho1 * J[i];
#pragma unroll
        for (int j = i; j < 6; ++j) acc[k++] += wi * J[j];
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) acc[21 + i] += rho1 * J[i] * r;
    acc[27] += 0.5 * rho0;
}

// ICP iterations after the first: the previous iteration's five neighbours still exist, so the largest of their (exact)
// distances to the moved query bounds the new 5th-neighbour distance -- provided they lie in the block the query is in NOW
// (the search is block-local, LocalMap.h:488-507: after a pose update that carries the point across a 50 m block face the old
// neighbours belong to another block and bound nothing).  Returns the bound or -1 (no usable seed); *pos0: the previous nearest
// neighbour's position (in the query's block whenever the bound is returned).
__device__ __forceinline__ float seed_bound(const MapView& m, const QueryCell& qc, const NnBuf& nb, size_t gi, float qx, float qy, float qz, uint32_t* pos0 = nullptr) {
    const uint32_t cells = uint32_t(m.nb) * uint32_t(m.nb) * uint32_t(m.nb);
    const uint32_t lo = __ldg(&m.cell_start[uint32_t(qc.slot) * cells]), hi = __ldg(&m.cell_start[uint32_t(qc.slot) * cells + cells]);
    float u = 0.f;
    bool same_block = true;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const uint32_t pos = nb.pos[size_t(j) * nb.cap + gi];
        if (j == 0 && pos0) *pos0 = pos;
        same_block = same_block && pos >= lo && pos < hi;
        const float4 c = __ldg(&m.pts[same_block ? pos : lo]);
        const float dx = qx - c.x, dy = qy - c.y, dz = qz - c.z;
        u = fmaxf(u, float(double(dx) * double(dx) + double(dy) * double(dy) + double(dz) * double(dz)));
    }
    // use it only while it is about as tight as a freshly estimated bound would be (small pose update); after a large update
    // the cell-neighbourhood estimate of round 1 prunes better than a loose seed
    return (same_block && u <= 1.3f * nb.d5[gi]) ? u : -1.f;
}

// shouldProcessPoint (LidarSlam.cpp:353-359)
__device__ __forceinline__ bool should_process(uint32_t i, double rate) {
    if (rate < 0.0) return true;
    // explicit round-to-nearest operations: no FMA contraction, so that the host twin (so_api.cu: should_process_h, the decimated
    // upload of so_register) and the reference's x86 arithmetic select exactly the same points
    const double x = __dmul_rn(double(i), rate);
    const double rem = __dsub_rn(x, floor(x));            // == std::fmod(x, 1.0) for x >= 0: both are exact
    return !(__dadd_rn(rem, 0.001) > rate);
}

// ------------------------------------------------------------------------------------------------------------------
// Scan preparation (once per registration): order the scan points by the map cell they fall into at the PRIOR pose
// (scan_order_key: cell-linear, x fastest), so that the 32 lanes of a warp walk the same cell rows.  Pose updates inside one
// registration are a few cm against 0.39 m cells, so the order stays coherent for all ICP iterations.  The sorted copy carries
// the point's original index in .w (the reference's shouldProcessPoint() decimation is defined on the original index,
// LidarSlam.cpp:353-359).
// ------------------------------------------------------------------------------------------------------------------
// Key = (scan index inside the chunk) << cell_bits | cell; cells beyond the mask and off-map points sort last inside their scan.
// KeyT = uint32_t when cell_bits + scan bits fit (the usual case: 4 radix passes over 8-byte pairs instead of 5 over 12-byte ones).
// COMPACT: points that shouldProcessPoint (LidarSlam.cpp:353-359) drops get one more key bit above the cell and sort behind every
// survivor of their scan; k_scan_finish then shrinks the scan to its survivors (the decimation depends on the original index only,
// so it is decided once per registration and the ICP kernels run over max_surface_features points instead of the whole scan).
template <class KeyT, bool COMPACT>
__global__ void __launch_bounds__(kThreads) k_scan_keys(MapView m, BatchView bv, KeyT* __restrict__ keys, uint32_t* __restrict__ vals, int cell_bits) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    const uint32_t n = uint32_t(st->n_points);
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const size_t gi = size_t(bv.offset[s]) + i;
    if (COMPACT && !should_process(i, st->sampling_rate)) {
        keys[gi] = KeyT((KeyT(s) << (cell_bits + 1)) | (KeyT(1) << cell_bits));
        vals[gi] = uint32_t(gi);
        return;
    }
    const float4 sp = __ldg(&bv.scan[gi]);
    const double pin[3] = {double(sp.x), double(sp.y), double(sp.z)};
    double pf[3];
    qrot(st->x + 3, pin, pf);
    QueryCell qc;
    locate(m, float(pf[0] + st->x[0]), float(pf[1] + st->x[1]), float(pf[2] + st->x[2]), qc);
    const uint32_t cell = qc.slot >= 0 ? scan_order_key(m, qc) : 0xFFFFFFFFu;      // cell order (so_knn.cuh)
    const uint32_t mask = cell_bits >= 32 ? 0xFFFFFFFFu : ((1u << cell_bits) - 1u);
    keys[gi] = KeyT((KeyT(s) << (cell_bits + (COMPACT ? 1 : 0))) | KeyT(cell < mask ? cell : mask));
    vals[gi] = uint32_t(gi);
}

// After the sort of a COMPACT chunk: survivors of scan s = sorted keys of its range without the dropped bit (binary search);
// the scan shrinks to them and its decimation is switched off.
template <class KeyT>
__global__ void k_scan_finish(BatchView bv, const KeyT* __restrict__ sorted_keys, uint32_t pt_first, int cell_bits, uint32_t n_scans) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_scans) return;
    IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    const KeyT* k = sorted_keys + (bv.offset[s] - pt_first);
    uint32_t lo = 0, hi = uint32_t(st->n_points);
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((k[mid] >> cell_bits) & 1) hi = mid; else lo = mid + 1; }
    st->n_points = int32_t(lo);
    st->sampling_rate = -1.0;
}

template <class KeyT>
__global__ void __launch_bounds__(kThreads) k_scan_gather(const float4* __restrict__ in, const uint32_t* __restrict__ vals, const KeyT* __restrict__ keys,
                                                          const uint32_t* __restrict__ offset, size_t total, float4* __restrict__ out, int cell_bits) {
    const size_t j = size_t(blockIdx.x) * kThreads + threadIdx.x;
    if (j >= total) return;
    const uint32_t g = vals[j];
    const uint32_t s = uint32_t(keys[j] >> cell_bits);                 // cell_bits here = all key bits below the scan index
    const float4 p = __ldg(&in[g]);
    out[j] = make_float4(p.x, p.y, p.z, __uint_as_float(g - offset[s]));
}

// ------------------------------------------------------------------------------------------------------------------
// k_prepare_small: the whole scan preparation of a SMALL registration in one CTA per scan -- what k_scan_keys + a device-wide
// radix sort (4-5 launches whose fixed cost, ~35 us, is most of a latency-bound so_register) + k_scan_gather do for batches.
// Points that shouldProcessPoint (LidarSlam.cpp:353-359) drops are removed HERE, once (the decimation is a function of the
// original index only): the ICP kernels then run over the <= max_surface_features + 1 surviving points with sampling off.
// Deterministic: the survivors are compacted in index order (block scans), sorted by cell key with a stable block radix sort.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kSmallThreads = 1024, kSmallCap = kPrepareSmallCap;
static_assert(kSmallCap == kSmallThreads * 4, "k_prepare_small<4> covers kPrepareSmallCap survivors");
// ITEMS: survivors per thread in the sort (2 when they fit 2048 -- the shipped max_surface_features of 2000 -- else 4)
template <int ITEMS>
__global__ void __launch_bounds__(kSmallThreads) k_prepare_small(MapView m, BatchView bv, float4* __restrict__ out, int key_bits) {
    constexpr int kCap = kSmallThreads * ITEMS;
    using Sort = cub::BlockRadixSort<uint32_t, kSmallThreads, ITEMS, uint32_t>;
    using Scan = cub::BlockScan<uint32_t, kSmallThreads>;
    struct Compact { typename Scan::TempStorage scan; uint32_t idx[kCap]; };
    __shared__ union { typename Sort::TempStorage sort; Compact c; } s_tmp;      // the index list is consumed (into registers) before the sort starts
    uint32_t* s_idx = s_tmp.c.idx;
    __shared__ double s_pose[7];
    const int s = blockIdx.x;
    IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    if (threadIdx.x < 7) s_pose[threadIdx.x] = st->x[threadIdx.x];
    const uint32_t n = uint32_t(st->n_points);
    const double rate = st->sampling_rate;
    const size_t base = size_t(bv.offset[s]);
    // survivors, in index order: every thread owns a contiguous run of indices, ONE block scan places the runs
    const uint32_t per = (n + kSmallThreads - 1) / kSmallThreads, lo = min(n, threadIdx.x * per), hi = min(n, lo + per);
    uint32_t mine = 0;
    for (uint32_t i = lo; i < hi; ++i) mine += should_process(i, rate) ? 1u : 0u;
    uint32_t pos, total;
    Scan(s_tmp.c.scan).ExclusiveSum(mine, pos, total);
    for (uint32_t i = lo; i < hi && pos < uint32_t(kCap); ++i) if (should_process(i, rate)) s_idx[pos++] = i;
    __syncthreads();
    const uint32_t n_act = min(total, uint32_t(kCap));                  // the host chose this path only when the survivors fit
    uint32_t key[ITEMS], val[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        const uint32_t j = threadIdx.x * ITEMS + k;                     // blocked arrangement
        key[k] = 0xFFFFFFFFu; val[k] = 0xFFFFFFFFu;
        if (j < n_act) {
            const uint32_t i = s_idx[j];
            const float4 sp = __ldg(&bv.scan[base + i]);
            const double pin[3] = {double(sp.x), double(sp.y), double(sp.z)};
            double pf[3];
            qrot(s_pose + 3, pin, pf);
            QueryCell qc;
            locate(m, float(pf[0] + s_pose[0]), float(pf[1] + s_pose[1]), float(pf[2] + s_pose[2]), qc);
            const uint32_t mask = key_bits >= 32 ? 0xFFFFFFFFu : ((1u << key_bits) - 1u);
            const uint32_t cell = qc.slot >= 0 ? scan_order_key(m, qc) : 0xFFFFFFFFu;
            key[k] = cell < mask ? cell : mask;                          // off-map points sort last among the survivors, as in the batch path
            val[k] = i;
        }
    }
    __syncthreads();
    Sort(s_tmp.sort).Sort(key, val, 0, key_bits < 32 ? key_bits + 1 : 32);      // + 1: the padding keys (all ones) sort behind the mask
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        const uint32_t j = threadIdx.x * ITEMS + k;
        if (j < n_act) {
            const float4 p = __ldg(&bv.scan[base + val[k]]);
            out[base + j] = make_float4(p.x, p.y, p.z, __uint_as_float(val[k]));
        }
    }
    if (threadIdx.x == 0) { st->n_points = int32_t(n_act); st->sampling_rate = -1.0; }
}

// ------------------------------------------------------------------------------------------------------------------
// k_knn_scan: findNearestNeighbors (LidarSlam.cpp:720-747) for every processed scan point at the current pose: the select k-NN of
// so_knn.cuh, one query per thread, queries consecutive in scan order.  Light on registers (FP32 search, FP64 only for the pose
// transform and the exact d2 of real contenders) so that many warps per SM hide the latency of the cell walks.
// ------------------------------------------------------------------------------------------------------------------
// Queries per CTA, measured on an H100 80GB HBM3 (700 W limit, scripts/ab_knn.py, 64 cfg2 scans = 8.4 M queries per launch):
// 32 -> 1.08, 64 -> 1.05-1.07, 128 -> 1.07, 256 -> 1.11 ms per launch.  1024 / kKnnThreads CTAs per SM = 64 registers per thread.
constexpr int kKnnThreads = 64;
// GRAPH (the map has a neighbour graph, so_knn.cuh): a query the graph certifies is ranked from its anchor's row; any other goes to
// nb.queue with its round-1 bound, and k_knn_round2 runs round 2 for the queue.  Round 2 in this kernel would cost a warp its full
// length whenever one of its 32 lanes is not certified (at 82-91 % certified per lane almost every warp has one); the queue gathers
// those queries into warps of their own, in roughly the scan's cell order (each warp appends its lanes in order).
template <bool GRAPH>
__global__ void __launch_bounds__(kKnnThreads, 1024 / kKnnThreads) k_knn_scan(MapView m, BatchView bv, NnBuf nb) {
    const int s = blockIdx.y;
    IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    __shared__ double s_pose[7];
    __shared__ uint32_t s_buf[GRAPH ? 1 : kBufCap * kKnnThreads];
    if (threadIdx.x < 7) s_pose[threadIdx.x] = st->x[threadIdx.x];
    __syncthreads();
    const uint32_t n = uint32_t(st->n_points);
    const uint32_t i = blockIdx.x * kKnnThreads + threadIdx.x;
    if (blockIdx.x * kKnnThreads >= n) return;            // whole CTA past the end
    const bool in_range = i < n;
    const size_t gi = size_t(bv.offset[s]) + (in_range ? i : 0);
    const float4 sp = __ldg(&bv.scan[gi]);
    int pre = SO_MATCH_SKIPPED;
    TopK<5> tk;
    tk.init(m.bound_d2);
    bool searched = false, by_graph = false;
    float U = 0.f;
    if (in_range && should_process(__float_as_uint(sp.w), st->sampling_rate)) {
        const double pin[3] = {double(sp.x), double(sp.y), double(sp.z)};
        double pf[3];
        qrot(s_pose + 3, pin, pf);
        const float qx = float(pf[0] + s_pose[0]), qy = float(pf[1] + s_pose[1]), qz = float(pf[2] + s_pose[2]);
        QueryCell qc;
        locate(m, qx, qy, qz, qc);
        if (qc.slot < 0 || qc.nblock < 5) pre = SO_MATCH_NOT_ENOUGH_NEIGHBORS;
        else if (!GRAPH) {
            const float u_seed = st->icp_iter > 0 && nb.pre[gi] == SO_MATCH_SUCCESS ? seed_bound(m, qc, nb, gi, qx, qy, qz) : -1.f;
            knn_select<5, true>(BlockGrid(m, qc.slot), m, qc, qx, qy, qz, u_seed, m.bound_d2, s_buf, tk);
            pre = tk.count() < 5 ? SO_MATCH_NEIGHBORS_TOO_FAR : SO_MATCH_SUCCESS;       // d2[4] > 3*planeRes_ (:741-744)
        } else {
            // anchor of the graph certificate: the previous iteration's nearest neighbour when it seeds the bound, else the nearest
            // candidate round 1 saw
            uint32_t anchor = 0xFFFFFFFFu;
            const float u_seed = st->icp_iter > 0 && nb.pre[gi] == SO_MATCH_SUCCESS ? seed_bound(m, qc, nb, gi, qx, qy, qz, &anchor) : -1.f;
            U = knn_bound<5, true>(BlockGrid(m, qc.slot), m, qc, qx, qy, qz, u_seed, m.bound_d2, &anchor);
            searched = true;
            by_graph = anchor != 0xFFFFFFFFu && graph_certified(m, anchor, qx, qy, qz, U);
            if (by_graph) {
                knn_graph_rank<5>(m, anchor, qx, qy, qz, U, tk);
                pre = tk.count() < 5 ? SO_MATCH_NEIGHBORS_TOO_FAR : SO_MATCH_SUCCESS;
            }
        }
    }
    const bool defer = searched && !by_graph;
    if (GRAPH) {                                       // every lane of the warp is still here
        const int it = min(st->icp_iter, SO_MAX_ICP_ITERS - 1);
        const uint32_t lane = threadIdx.x & 31;
        const uint32_t dm = __ballot_sync(0xFFFFFFFFu, defer);
        if (dm) {
            const uint32_t lead = __ffs(dm) - 1;
            uint32_t base = 0;
            if (lane == lead) base = atomicAdd(&nb.qcount[s * SO_MAX_ICP_ITERS + it], uint32_t(__popc(dm)));
            base = __shfl_sync(0xFFFFFFFFu, base, lead);
            if (defer) {
                nb.queue[bv.offset[s] + base + __popc(dm & ((1u << lane) - 1u))] = uint32_t(gi);
                nb.d5[gi] = U;
            }
        }
        if (m.graph_stats) {                           // so_knn_graph_stats
            const uint32_t ns = __popc(__ballot_sync(0xFFFFFFFFu, searched)), ng = __popc(__ballot_sync(0xFFFFFFFFu, by_graph));
            if (lane == 0) { atomicAdd(&m.graph_stats[2 * it], ns); atomicAdd(&m.graph_stats[2 * it + 1], ng); }
        }
    }
    if (!in_range || defer) return;                    // a queued query's results come from k_knn_round2
    nb.pre[gi] = (unsigned char)pre;
    nb.d5[gi] = tk.d2[4];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const bool ok = tk.id[j] != 0xFFFFFFFFu;
        nb.pos[size_t(j) * nb.cap + gi] = ok ? tk.pos[j] : 0xFFFFFFFFu;
    }
}

// k_knn_round2: round 2 of the select search for the queries k_knn_scan<true> queued, one per thread in queue order, with the bound
// round 1 left in d5: the query, its cell and its bound are those k_knn_scan computed, so the result is the one it would have found.
__global__ void __launch_bounds__(kKnnThreads, 1024 / kKnnThreads) k_knn_round2(MapView m, BatchView bv, NnBuf nb) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    const uint32_t cnt = nb.qcount[s * SO_MAX_ICP_ITERS + min(st->icp_iter, SO_MAX_ICP_ITERS - 1)];
    if (blockIdx.x * kKnnThreads >= cnt) return;
    __shared__ double s_pose[7];
    __shared__ uint32_t s_buf[kBufCap * kKnnThreads];
    if (threadIdx.x < 7) s_pose[threadIdx.x] = st->x[threadIdx.x];
    __syncthreads();
    const uint32_t j = blockIdx.x * kKnnThreads + threadIdx.x;
    if (j >= cnt) return;
    const size_t gi = nb.queue[bv.offset[s] + j];
    const float U = nb.d5[gi];
    const float4 sp = __ldg(&bv.scan[gi]);
    const double pin[3] = {double(sp.x), double(sp.y), double(sp.z)};
    double pf[3];
    qrot(s_pose + 3, pin, pf);
    const float qx = float(pf[0] + s_pose[0]), qy = float(pf[1] + s_pose[1]), qz = float(pf[2] + s_pose[2]);
    QueryCell qc;
    locate(m, qx, qy, qz, qc);
    TopK<5> tk;
    tk.init(m.bound_d2);
    knn_gather<5>(BlockGrid(m, qc.slot), m, qc, qx, qy, qz, U, s_buf, tk);
    nb.pre[gi] = (unsigned char)(tk.count() < 5 ? SO_MATCH_NEIGHBORS_TOO_FAR : SO_MATCH_SUCCESS);
    nb.d5[gi] = tk.d2[4];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const bool ok = tk.id[k] != 0xFFFFFFFFu;
        nb.pos[size_t(k) * nb.cap + gi] = ok ? tk.pos[k] : 0xFFFFFFFFu;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// k_knn_scan_coop: the same search for SMALL registrations (a live scan after the shouldProcessPoint decimation: ~2 000 queries),
// one WARP per query.  With one query per thread such a launch is eight CTAs whose threads each walk ~3 800 dependent instructions
// (~20 us); here lane l < 25 takes row l of the 5 x 5 rows of the two-ring cube (the same pruning against the gate 3 * planeRes_
// as walk_cube), a warp scan flattens the rows' candidate spans, the lanes take the candidates 32 at a time -- FP32 filter, the
// reference's exact d2, a private top-5 -- and five warp arg-min rounds over (d2, id) merge the private lists.  The result is
// the exact block-local 5-NN in (d2, id) order with the same distances, i.e. bit-identical to k_knn_scan's, in ~700 instructions
// per warp spread over every SM.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kCoopWarps = kThreads / 32;
__global__ void __launch_bounds__(kThreads) k_knn_scan_coop(MapView m, BatchView bv, NnBuf nb) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    __shared__ double s_pose[7];
    __shared__ uint32_t s_scan[kCoopWarps][33], s_t[kCoopWarps][32];
    if (threadIdx.x < 7) s_pose[threadIdx.x] = st->x[threadIdx.x];
    __syncthreads();
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t n = uint32_t(st->n_points);
    const uint32_t i = blockIdx.x * kCoopWarps + warp;     // the warp's query
    if (i >= n) return;
    const size_t gi = size_t(bv.offset[s]) + i;
    const float4 sp = __ldg(&bv.scan[gi]);
    int pre = SO_MATCH_SKIPPED;
    TopK<5> tk;
    tk.init(m.bound_d2);
    if (should_process(__float_as_uint(sp.w), st->sampling_rate)) {
        const double pin[3] = {double(sp.x), double(sp.y), double(sp.z)};
        double pf[3];
        qrot(s_pose + 3, pin, pf);
        const float qx = float(pf[0] + s_pose[0]), qy = float(pf[1] + s_pose[1]), qz = float(pf[2] + s_pose[2]);
        QueryCell qc;
        locate(m, qx, qy, qz, qc);
        if (qc.slot < 0 || qc.nblock < 5) pre = SO_MATCH_NOT_ENOUGH_NEIGHBORS;
        else {
            const BlockGrid g(m, qc.slot);
            const int nbc = m.nb, R = m.R;
            const float cs = m.cs, U = m.bound_d2 * 1.000004f, Um = U * 1.0001f;
            // ---- lane l: row (oz, oy) of the cube, its candidate span
            uint32_t t = 0, len = 0;
            const int side = 2 * R + 1;
            if (lane < side * side) {                      // R <= 2 by construction of the grid (cells >= half the search radius)
                const int oz = lane / side - R, oy = lane % side - R;
                const int zz = qc.c[2] + oz, yy = qc.c[1] + oy, cx = qc.c[0];
                const float fx = qc.f[0], gx = cs - fx;
                const float lz = axis_gap(oz, qc.f[2], cs - qc.f[2], cs), ly = axis_gap(oy, qc.f[1], cs - qc.f[1], cs);
                const float lb = fmaf(ly, ly, lz * lz);
                if (zz >= 0 && zz < nbc && yy >= 0 && yy < nbc && lb <= Um) {
                    const bool l1 = cx >= 1 && fmaf(fx, fx, lb) <= Um;
                    const bool l2 = l1 && R >= 2 && cx >= 2 && fmaf(fx + cs, fx + cs, lb) <= Um;
                    const bool r1 = cx + 1 < nbc && fmaf(gx, gx, lb) <= Um;
                    const bool r2 = r1 && R >= 2 && cx + 2 < nbc && fmaf(gx + cs, gx + cs, lb) <= Um;
                    uint32_t end;
                    g.row(zz, yy, cx - int(l1) - int(l2), cx + int(r1) + int(r2), t, end);
                    len = end - t;
                }
            }
            // ---- exclusive scan of the span lengths: candidate c of the flattened list sits in the row whose prefix interval holds c
            uint32_t incl = len;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(full, incl, o); if (lane >= o) incl += v; }
            const uint32_t total = __shfl_sync(full, incl, 31);
            s_scan[warp][lane] = incl - len;
            s_t[warp][lane] = t;
            if (lane == 0) s_scan[warp][32] = total;
            __syncwarp();
            for (uint32_t c = lane; c < total; c += 32) {
                int lo = 0;                                // largest row with prefix <= c (empty rows share a prefix: the search lands past them)
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) if (s_scan[warp][lo + o] <= c) lo += o;
                const uint32_t e = s_t[warp][lo] + (c - s_scan[warp][lo]);
                const float4 cand = g.load(e);
                if (approx_d2(cand, qx, qy, qz) <= U) tk.offer(exact_d2(cand, qx, qy, qz), __float_as_uint(cand.w), e);
            }
            // ---- merge: five rounds of warp arg-min over the heads of the private lists
            TopK<5> out;
            out.init(m.bound_d2);
            int head = 0;
#pragma unroll
            for (int j = 0; j < 5; ++j) {
                float hd = m.bound_d2; uint32_t hi = 0xFFFFFFFFu, hp = 0;
#pragma unroll
                for (int k = 0; k < 5; ++k) if (k == head) { hd = tk.d2[k]; hi = tk.id[k]; hp = tk.pos[k]; }
                if (head >= 5) { hd = FLT_MAX; hi = 0xFFFFFFFFu; }
                const uint32_t dbits = hi != 0xFFFFFFFFu ? __float_as_uint(hd) : 0xFFFFFFFFu;      // d2 >= 0: the bit pattern orders like the value
                const uint32_t dmin = __reduce_min_sync(full, dbits);
                if (dmin == 0xFFFFFFFFu) break;            // fewer than five within the gate (warp-uniform)
                const uint32_t imin = __reduce_min_sync(full, dbits == dmin ? hi : 0xFFFFFFFFu);
                const bool win = dbits == dmin && hi == imin;      // ids are unique: exactly one lane
                const int src = __ffs(__ballot_sync(full, win)) - 1;
                out.d2[j] = __uint_as_float(dmin); out.id[j] = imin; out.pos[j] = __shfl_sync(full, hp, src);
                if (win) ++head;
            }
            tk = out;
            pre = tk.count() < 5 ? SO_MATCH_NEIGHBORS_TOO_FAR : SO_MATCH_SUCCESS;       // d2[4] > 3*planeRes_ (:741-744)
        }
    }
    if (lane == 0) { nb.pre[gi] = (unsigned char)pre; nb.d5[gi] = tk.d2[4]; }
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        if (lane == j) {
            const bool ok = tk.id[j] != 0xFFFFFFFFu;
            nb.pos[size_t(j) * nb.cap + gi] = ok ? tk.pos[j] : 0xFFFFFFFFu;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// k_knn_inject: test hook behind so_register_injected -- the neighbour SEARCH of k_knn_scan replaced by caller-supplied
// neighbour ids (ids[it][original point index][5], map point ids in so_map_set_points order, 0xFFFFFFFF = no result), everything
// after it (the NEIGHBORS_TOO_FAR gate on the 5th distance, LidarSlam.cpp:741-744, the hand-off to k_fit) unchanged.  Feeding it
// the neighbour sets of the reference's own octree (oracle knn_mode 2) isolates the one known deviation of this library from the
// reference path: exact in-block k-NN instead of the octree's data-dependent misses (flann/octree.h:383-385,984-1001).
// ------------------------------------------------------------------------------------------------------------------
// Position of map point `id` (coordinates c) in the sorted map: locate() bins a point exactly as the index build does (k_keys,
// k_keys_dev: the same double expressions), so the point lies in the cell its own coordinates locate and one scan of that cell
// finds it.  0xFFFFFFFF when the index does not hold it (outside the grid).
__device__ __forceinline__ uint32_t sorted_pos_of(const MapView& m, const float4 c, uint32_t id) {
    QueryCell qc;
    locate(m, c.x, c.y, c.z, qc);
    if (qc.slot < 0) return 0xFFFFFFFFu;
    const uint32_t key = scan_order_key(m, qc);
    for (uint32_t t = __ldg(&m.cell_start[key]), e = __ldg(&m.cell_start[key + 1]); t < e; ++t)
        if (__float_as_uint(__ldg(&m.pts[t]).w) == id) return t;
    return 0xFFFFFFFFu;
}

__global__ void __launch_bounds__(kThreads) k_knn_inject(MapView m, const float4* __restrict__ by_id, uint32_t n_map, BatchView bv, NnBuf nb,
                                                         const uint32_t* __restrict__ ids, int n_trace_iters) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    __shared__ double s_pose[7];
    if (threadIdx.x < 7) s_pose[threadIdx.x] = st->x[threadIdx.x];
    __syncthreads();
    const uint32_t n = uint32_t(st->n_points);
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const size_t gi = size_t(bv.offset[s]) + i;
    const float4 sp = __ldg(&bv.scan[gi]);
    const uint32_t orig = __float_as_uint(sp.w);
    int pre = SO_MATCH_SKIPPED;
    float d5 = m.bound_d2;
    uint32_t pos[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) pos[j] = 0xFFFFFFFFu;
    if (should_process(orig, st->sampling_rate)) {
        pre = SO_MATCH_NOT_ENOUGH_NEIGHBORS;
        const int it = st->icp_iter;
        if (it < n_trace_iters) {
            const uint32_t* p = ids + (size_t(it) * uint32_t(st->n_input) + orig) * 5;      // the trace is laid out over the scan as uploaded
            bool ok = true;
#pragma unroll
            for (int j = 0; j < 5; ++j) ok = ok && p[j] < n_map;
            // k_fit takes positions in the sorted map; a neighbour the index does not hold counts as no result
#pragma unroll
            for (int j = 0; j < 5; ++j) {
                if (ok) pos[j] = sorted_pos_of(m, __ldg(&by_id[p[j]]), p[j]);
                ok = ok && pos[j] != 0xFFFFFFFFu;
            }
            if (ok) {
                const double pin[3] = {double(sp.x), double(sp.y), double(sp.z)};
                double pf[3];
                qrot(s_pose + 3, pin, pf);
                const float qx = float(pf[0] + s_pose[0]), qy = float(pf[1] + s_pose[1]), qz = float(pf[2] + s_pose[2]);
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    const float4 c = __ldg(&by_id[p[j]]);
                    const float dx = qx - c.x, dy = qy - c.y, dz = qz - c.z;
                    d5 = float(double(dx) * double(dx) + double(dy) * double(dy) + double(dz) * double(dz));
                }
                pre = double(d5) > double(m.bound_d2) ? SO_MATCH_NEIGHBORS_TOO_FAR : SO_MATCH_SUCCESS;      // pointSearchSqDis[4] > 3*planeRes_ (:741-744)
            }
        }
    }
    nb.pre[gi] = (unsigned char)pre;
    nb.d5[gi] = d5;
    // positions only for a full neighbour set: the stage outputs (cb.nn) of a rejected point carry no ids on this path
#pragma unroll
    for (int j = 0; j < 5; ++j) nb.pos[size_t(j) * nb.cap + gi] = pre == SO_MATCH_SUCCESS ? pos[j] : 0xFFFFFFFFu;
}

// ------------------------------------------------------------------------------------------------------------------
// k_fit: the rest of LidarSLAM::ComputePlaneDistanceParameters (LidarSlam.cpp:536-572) for every scan point, from the
// neighbours k_knn_scan handed over: fit_point() below + the per-scan histograms.  The first residual/Jacobian evaluation of
// the following ceres::Solve is a separate k_evaluate<PH_CORR> launch, which keeps this kernel at 64 registers.
// ------------------------------------------------------------------------------------------------------------------
// Shared-memory load the compiler may not replace by the value stored earlier: k_fit keeps its neighbours' FP64 coordinates
// in shared memory rather than live in registers across the eigen-solve.
__device__ __forceinline__ double ld_shared_again(const double* p) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(uint32_t(__cvta_generic_to_shared(p))));
    return v;
}

// The rest of LidarSLAM::ComputePlaneDistanceParameters (LidarSlam.cpp:536-572) for one scan point whose k-NN outcome is
// `status`: PCA, plane fit, gates, observability labels, fit weight; writes the correspondence record and counts the
// histograms.  FP64 throughout.  k_knn_scan hands over the neighbours' positions (nb.pos) and the points are gathered from the
// sorted map: it fits in L2 (16 MB at the bench shape) and the queries are cell-ordered, so neighbouring lanes mostly load the
// same points.  The fit reads them three more times
// after the mean (scatter, QR, plane distances) and does not hold them in 30 FP64 registers across the eigen-solve: the first
// pass widens each coordinate once and parks it in shared memory (nbd[(3 j + k) * kFitThreads], this thread's column), and the
// later passes load it from there instead of re-reading and widening afresh (float -> double conversions run at a quarter of
// the FP64 rate).
__device__ __forceinline__ void fit_point(const MapView& m, const CorrBuf& cb, const NnBuf& nb, size_t gi, size_t ri, const float4 sp, const double* s_pose,
                                          int status, double* nbd, int* s_hist) {
    auto nbr_d = [&](int j, double& x, double& y, double& z) {
        x = ld_shared_again(nbd + (3 * j + 0) * kFitThreads); y = ld_shared_again(nbd + (3 * j + 1) * kFitThreads); z = ld_shared_again(nbd + (3 * j + 2) * kFitThreads);
    };
    cb.p[ri * 3 + 0] = sp.x; cb.p[ri * 3 + 1] = sp.y; cb.p[ri * 3 + 2] = sp.z;
    int o0 = 0, o1 = 0, o2 = 0;
    double xq[3] = {0, 0, 0}, wq = 0.0;
    if (status == SO_MATCH_SUCCESS) {
                    // ComputePointInitAndFinalPose (:382-400): pInit = double(p), pFinal = T_w_lidar * pInit
        const double pin[3] = {double(sp.x), double(sp.y), double(sp.z)};
        double pf[3];
        qrot(s_pose + 3, pin, pf);
        pf[0] += s_pose[0]; pf[1] += s_pose[1]; pf[2] += s_pose[2];
        const float qx = float(pf[0]), qy = float(pf[1]), qz = float(pf[2]);
        // computePCAForFeature (:749-790) + utils::ComputePCA (superodom_utils.h:143-151)
        double mean[3] = {0, 0, 0};
#pragma unroll
        for (int j = 0; j < 5; ++j) {
            const float4 c = __ldg(&m.pts[__ldg(&nb.pos[size_t(j) * nb.cap + gi])]);
            const double x = double(c.x), y = double(c.y), z = double(c.z);
            nbd[(3 * j + 0) * kFitThreads] = x; nbd[(3 * j + 1) * kFitThreads] = y; nbd[(3 * j + 2) * kFitThreads] = z;
            mean[0] += x; mean[1] += y; mean[2] += z;
            if (cb.nn) {
                const float dx = qx - c.x, dy = qy - c.y, dz = qz - c.z;
                cb.nn[gi * 5 + j] = __float_as_uint(c.w);
                cb.nn_d2[gi * 5 + j] = float(double(dx) * double(dx) + double(dy) * double(dy) + double(dz) * double(dz));
            }
        }
        // mean /= 5, as utils::ComputePCA divides (superodom_utils.h:146): the eigenvalue gates below read it.  The division by
        // the reciprocal 0.2 = RN(1/5) gives the same bits (div_rcp): a sum of five floats is +0 (exact through div_rcp) or in
        // [2^-149, 2^131], inside div_rcp_ok's range.
        mean[0] = div_rcp(mean[0], 5.0, 0.2); mean[1] = div_rcp(mean[1], 5.0, 0.2); mean[2] = div_rcp(mean[2], 5.0, 0.2);
        double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int j = 0; j < 5; ++j) {
            double x, y, z;
            nbr_d(j, x, y, z);
            const double c0 = x - mean[0], c1 = y - mean[1], c2 = z - mean[2];
            S[0] += c0 * c0; S[1] += c0 * c1; S[2] += c0 * c2; S[4] += c1 * c1; S[5] += c1 * c2; S[8] += c2 * c2;
        }
        S[3] = S[1]; S[6] = S[2]; S[7] = S[5];
        const double sxx = S[0], sxy = S[1], sxz = S[2], syy = S[4], syz = S[5], szz = S[8];
        // SelfAdjointEigenSolver<Matrix3d> (utils::ComputePCA, superodom_utils.h:150): eigenvalues by the closed form, the smallest
        // eigenvector from its eigenvalue, then the smallest eigenvalue once more as the Rayleigh quotient of that vector (full
        // double precision where the lambda0 < 1e-6 gate reads it)
        double ev[3], no[3];
        sym3_eigenvalues(sxx, sxy, sxz, syy, syz, szz, ev);
        eigvec3_from_value(sxx, sxy, sxz, syy, syz, szz, ev[0], no);
        ev[0] = no[0] * (sxx * no[0] + sxy * no[1] + sxz * no[2]) + no[1] * (sxy * no[0] + syy * no[1] + syz * no[2]) +
                no[2] * (sxz * no[0] + syz * no[1] + szz * no[2]);
        ev[1] = (sxx + syy + szz) - ev[0] - ev[2];
        if (ev[0] < 1e-6 || ev[1] / ev[2] < 0.1) status = SO_MATCH_BAD_PCA_STRUCTURE;      // the reference's quotient, literally (:772)
        else {
            // What FeatureObservabilityAnalysis (:574-693) needs from the PCA -- the oriented normal (:553-561) and the
            // planarity -- is reduced to four floats here, ahead of the register-hungry QR.
            float nf[3], cr[3], planar_sq;
            {
                if (pf[0] * no[0] + pf[1] * no[1] + pf[2] * no[2] < 0) { no[0] = -no[0]; no[1] = -no[1]; no[2] = -no[2]; }
                const double l1 = sqrt(ev[2]), l2 = sqrt(ev[1]), l3 = sqrt(ev[0]);
                const double planar_2 = (l2 - l3) / l1;
                planar_sq = float(planar_2 * planar_2);
                nf[0] = float(no[0]); nf[1] = float(no[1]); nf[2] = float(no[2]);
                cr[0] = __fmul_rn(qy, nf[2]) - __fmul_rn(qz, nf[1]);
                cr[1] = __fmul_rn(qz, nf[0]) - __fmul_rn(qx, nf[2]);
                cr[2] = __fmul_rn(qx, nf[1]) - __fmul_rn(qy, nf[0]);
            }
            // computePlaneQualityMetrics (:792-844)
            double x[3];
            {
                double A[5][3], b[5];
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    nbr_d(j, A[j][0], A[j][1], A[j][2]);
                    b[j] = -1.0;
                }
                colpiv_qr_solve_5x3(A, b, x);
            }
            if (!(isfinite(x[0]) && isfinite(x[1]) && isfinite(x[2]))) status = SO_MATCH_INVALID_NUMERICAL;
            else {
                // negative_OA_dot_norm and the normalised normal (:812-816), as every reader of the record decodes them from x
                double pn[3], dd;
                plane_of_solution(x[0], x[1], x[2], pn, dd);
                const double maxd = double(m.plane_res) / 2.0;
                double msum = 0.0;
                bool ok = true;
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    double cx, cy, cz;
                    nbr_d(j, cx, cy, cz);
                    const double dist = fabs(pn[0] * cx + pn[1] * cy + pn[2] * cz + dd);
                    if (ok && dist > maxd) ok = false;
                    msum += dist;
                }
                if (!ok) status = SO_MATCH_MSE_TOO_LARGE;
                else {
                    const double mean_dist = div_rcp_ok(msum, 5.0) ? div_rcp(msum, 5.0, 0.2) : msum / 5.0;
                    const float fq[4] = {float(s_pose[3]), float(s_pose[4]), float(s_pose[5]), float(s_pose[6])};
                    float rcq[3], trq[3];          // rotation scores +rc_a / -rc_a, translation scores; indexed by constants only
#pragma unroll
                    for (int a = 0; a < 3; ++a) {
                        // computeRotatedAxes (:624-638): float quaternion * e_a, no FMA contraction (host code is plain IEEE)
                        const float v0 = a == 0 ? 1.f : 0.f, v1 = a == 1 ? 1.f : 0.f, v2 = a == 2 ? 1.f : 0.f;
                        float ux = __fsub_rn(__fmul_rn(fq[1], v2), __fmul_rn(fq[2], v1));
                        float uy = __fsub_rn(__fmul_rn(fq[2], v0), __fmul_rn(fq[0], v2));
                        float uz = __fsub_rn(__fmul_rn(fq[0], v1), __fmul_rn(fq[1], v0));
                        ux = __fadd_rn(ux, ux); uy = __fadd_rn(uy, uy); uz = __fadd_rn(uz, uz);
                        const float ax = __fadd_rn(__fadd_rn(v0, __fmul_rn(fq[3], ux)), __fsub_rn(__fmul_rn(fq[1], uz), __fmul_rn(fq[2], uy)));
                        const float ay = __fadd_rn(__fadd_rn(v1, __fmul_rn(fq[3], uy)), __fsub_rn(__fmul_rn(fq[2], ux), __fmul_rn(fq[0], uz)));
                        const float az = __fadd_rn(__fadd_rn(v2, __fmul_rn(fq[3], uz)), __fsub_rn(__fmul_rn(fq[0], uy), __fmul_rn(fq[1], ux)));
                        // Eigen's unrolled 3-vector dot associates as a0*b0 + (a1*b1 + a2*b2)
                        const float rc = __fadd_rn(__fmul_rn(cr[0], ax), __fadd_rn(__fmul_rn(cr[1], ay), __fmul_rn(cr[2], az)));
                        rcq[a] = rc;
                        const float dn = __fadd_rn(__fmul_rn(nf[0], ax), __fadd_rn(__fmul_rn(nf[1], ay), __fmul_rn(nf[2], az)));
                        trq[a] = __fmul_rn(planar_sq, fabsf(dn));
                    }
                    // top-2 rotation labels and top-1 translation label of a stable descending sort (:654-679).  The six rotation
                    // scores are {+rc_a, -rc_a}, a = 0..2, so the largest is +|rc_a| of the axis with the largest magnitude (first axis
                    // on ties, as the stable sort keeps index order; index 2a for rc_a >= 0, 2a+1 below) and the runner-up the same
                    // among the other two axes -- unless every score is zero (or the winner's is NaN), when index order decides: 0, 1.
                    // (Scores picked by selects, not by a computed index: an array indexed at run time lives in local memory.)
                    const float m0 = fabsf(rcq[0]), m1 = fabsf(rcq[1]), m2 = fabsf(rcq[2]);
                    int a0 = 0; float mb = m0;
                    if (m1 > mb) { a0 = 1; mb = m1; }
                    if (m2 > mb) { a0 = 2; mb = m2; }
                    const int b0 = a0 == 0 ? 1 : 0, b1 = a0 == 2 ? 1 : 2;             // the other two axes, ascending
                    const float mb0 = a0 == 0 ? m1 : m0, mb1 = a0 == 2 ? m1 : m2;
                    const int a1 = mb1 > mb0 ? b1 : b0;
                    const float rc_a0 = a0 == 0 ? rcq[0] : (a0 == 1 ? rcq[1] : rcq[2]), rc_a1 = a1 == 0 ? rcq[0] : (a1 == 1 ? rcq[1] : rcq[2]);
                    const int r0 = 2 * a0 + (rc_a0 < 0.f ? 1 : 0);
                    const int r1 = (mb > 0.f) ? 2 * a1 + (rc_a1 < 0.f ? 1 : 0) : 1;
                    int t0 = 0;
                    float tb = trq[0];
                    if (trq[1] > tb) { t0 = 1; tb = trq[1]; }
                    if (trq[2] > tb) t0 = 2;
                    o0 = r0; o1 = r1; o2 = 6 + t0;
                    xq[0] = x[0]; xq[1] = x[1]; xq[2] = x[2];
                    // fitQualityCoeff = 1 - sqrt(meanDist / (3*planeRes_)) (:568); the map's inv_bound_d2 is RN(1 / bound_d2)
                    const double bd2 = double(m.bound_d2);
                    wq = 1.0 - sqrt(div_rcp_ok(mean_dist, bd2) ? div_rcp(mean_dist, bd2, m.inv_bound_d2) : mean_dist / bd2);
                    status = SO_MATCH_SUCCESS;
                }
            }
        }
    } else if (cb.nn) {
#pragma unroll
        for (int j = 0; j < 5; ++j) {
            const uint32_t pos = nb.pos[size_t(j) * nb.cap + gi];
            cb.nn[gi * 5 + j] = pos != 0xFFFFFFFFu ? __float_as_uint(__ldg(&m.pts[pos]).w) : 0xFFFFFFFFu;
            cb.nn_d2[gi * 5 + j] = 0.f;
        }
    }
    if (status != SO_MATCH_SKIPPED) {
        if (status == SO_MATCH_SUCCESS) { atomicAdd(&s_hist[o0], 1); atomicAdd(&s_hist[o1], 1); atomicAdd(&s_hist[o2], 1); }
        atomicAdd(&s_hist[9 + status], 1);
    }
    cb.x[ri * 3 + 0] = xq[0]; cb.x[ri * 3 + 1] = xq[1]; cb.x[ri * 3 + 2] = xq[2];
    cb.w[ri] = wq;
    cb.flags[gi] = make_uchar4((unsigned char)status, (unsigned char)o0, (unsigned char)o1, (unsigned char)o2);
}

__global__ void __launch_bounds__(kFitThreads, kFitMinBlocks) k_fit(MapView m, BatchView bv, CorrBuf cb, NnBuf nb) {
    const int s = blockIdx.y;
    IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    __shared__ double s_pose[7];
    __shared__ int s_hist[16];
    __shared__ double s_nbd[15 * kFitThreads];      // the five neighbours in FP64, one column per thread (15 x 8 B x 256 = 30 KB)
    if (threadIdx.x < 7) s_pose[threadIdx.x] = st->x[threadIdx.x];
    if (threadIdx.x < 16) s_hist[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t n = uint32_t(st->n_points);
#pragma unroll 1
    for (int rr = 0; rr < kFitPts; ++rr) {          // kFitPts points per thread
        const uint32_t i = (blockIdx.x * kFitPts + rr) * kFitThreads + threadIdx.x;
        const size_t gi = size_t(bv.offset[s]) + i;
        if (i < n) fit_point(m, cb, nb, gi, corr_first(cb.first + s, bv.offset[s]) + i, __ldg(&bv.scan[gi]), s_pose, int(nb.pre[gi]),
                             s_nbd + threadIdx.x, s_hist);
    }
    __syncthreads();
    if (threadIdx.x < 16 && s_hist[threadIdx.x]) atomicAdd(&bv.hist[s * kHistStride + threadIdx.x], s_hist[threadIdx.x]);
}

// ------------------------------------------------------------------------------------------------------------------
// k_evaluate: robustified normal equations at the candidate pose over the stored correspondences.
// kEvalPts points per thread (strided by the CTA width, so loads stay coalesced) before the one warp/CTA reduction.
// ------------------------------------------------------------------------------------------------------------------
template <int PHASE, bool ND>
__device__ __forceinline__ void evaluate_body(const BatchView& bv, const CorrBuf& cb, int s) {
    constexpr int X = kCorrX<ND>;
    IcpState* st = bv.st + s;
    __shared__ double s_pose[7];
    __shared__ double s_R[9];
    // PH_EVAL: the LM candidate; PH_CORR: the first evaluation of a new solve, at the pose k_fit just matched at
    if (threadIdx.x < 7) s_pose[threadIdx.x] = PHASE == PH_EVAL ? st->cand[threadIdx.x] : st->x[threadIdx.x];
    __syncthreads();
    if (threadIdx.x == 0) qtoR(s_pose + 3, s_R);
    __syncthreads();
    const uint32_t n = uint32_t(st->n_points);
    const size_t base = corr_first(cb.first + s, bv.offset[s]);
    double acc[kAcc];
#pragma unroll
    for (int k = 0; k < kAcc; ++k) acc[k] = 0.0;
    // Software-pipelined: the three loads of point r+1 are issued (unconditionally, so they do not chain behind the weight)
    // before the FP64 work of point r, which keeps two points' worth of the record stream in flight per thread.
    const int pts = eval_pts(n);
    if (blockIdx.x >= eval_ctas(n)) return;                // the grid covers the largest scan of the chunk
    const uint32_t i0 = blockIdx.x * uint32_t(pts) * kThreads + threadIdx.x;
    double w_n = 0.0, x_n[X] = {};
    float p_n[3] = {0.f, 0.f, 0.f};
    auto load = [&](uint32_t i) {
        w_n = cb.w[base + i];
#pragma unroll
        for (int k = 0; k < X; ++k) x_n[k] = cb.x[(base + i) * X + k];
#pragma unroll
        for (int k = 0; k < 3; ++k) p_n[k] = cb.p[(base + i) * 3 + k];
    };
    if (i0 < n) load(i0);
#pragma unroll 1
    for (int r = 0; r < pts; ++r) {
        const double w = w_n;
        double xr[X];
#pragma unroll
        for (int k = 0; k < X; ++k) xr[k] = x_n[k];
        const double pin[3] = {double(p_n[0]), double(p_n[1]), double(p_n[2])};
        const uint32_t inext = i0 + (r + 1) * kThreads;
        w_n = 0.0;
        if (r + 1 < pts && inext < n) load(inext);
        if (w != 0.0) {
            double pw[3];
            qrot(s_pose + 3, pin, pw);
            pw[0] += s_pose[0]; pw[1] += s_pose[1]; pw[2] += s_pose[2];
            double nn[3], d;
            corr_plane<ND>(xr, nn, d);
            accumulate(acc, nn, d, w, pin, pw, s_R, bv.tukey_a2);
        }
    }
    reduce_to_partials(acc, bv, s);
}

// ---- mbarrier / bulk-copy primitives (PTX ISA: mbarrier, cp.async.bulk) ----------------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(arrivals) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "SO_MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra SO_MBAR_DONE;\n"
        "bra SO_MBAR_WAIT;\n"
        "SO_MBAR_DONE:\n"
        "}\n" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
// 1-D TMA: `bytes` (multiple of 16) from global to shared memory, completion counted on the mbarrier
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_global, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst_smem)),
                 "l"(src_global), "r"(bytes), "r"(smem_addr(bar))
                 : "memory");
}

// The same evaluation with the record staged by the TMA engine.  A CTA's points are eval_pts(n) consecutive tiles of kThreads points,
// and a tile is three spans of the record (the QR solution 24 B/pt or {n, d} 32 B/pt, weight 8 B/pt, scan point 12 B/pt): one
// elected thread enqueues three cp.async.bulk copies per tile into a kEvalStages-deep shared-memory ring, each stage completing on its
// own mbarrier; every thread then takes its own point from the stage (thread -> point mapping, arithmetic and reduction are those of
// evaluate_body: results are bit-identical).  kEvalStages tiles (33 KB) are in flight per CTA whatever the threads are doing, instead
// of the one software-prefetched point per thread that 2 CTAs per SM leave room for.  Every scan's record starts on a tile of its own
// (so_corr_tiles.h), so every span is 16 B-aligned and a scan's ragged last tile is copied whole: the slots past its last point are
// the scan's own and are not read.
constexpr int kEvalStages = 3;
template <bool ND>
struct __align__(128) EvalStage { double x[kCorrX<ND> * kThreads]; double w[kThreads]; float p[3 * kThreads]; };

template <int PHASE, bool ND>
__device__ __forceinline__ void evaluate_body_tma(const BatchView& bv, const CorrBuf& cb, int s) {
    constexpr int X = kCorrX<ND>;
    constexpr uint32_t kStageBytes = uint32_t(X * sizeof(double) + sizeof(double) + 3 * sizeof(float)) * kThreads;
    IcpState* st = bv.st + s;
    __shared__ double s_pose[7];
    __shared__ double s_R[9];
    __shared__ EvalStage<ND> s_stage[kEvalStages];
    __shared__ unsigned long long s_bar[kEvalStages];
    const uint32_t n = uint32_t(st->n_points);
    const int pts = eval_pts(n);
    if (blockIdx.x >= eval_ctas(n)) return;                // the grid covers the largest scan of the chunk
    if (threadIdx.x < 7) s_pose[threadIdx.x] = PHASE == PH_EVAL ? st->cand[threadIdx.x] : st->x[threadIdx.x];
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < kEvalStages; ++k) mbar_init(&s_bar[k], 1);
    }
    __syncthreads();
    const size_t base = corr_first(cb.first + s, bv.offset[s]);
    const uint32_t cta0 = blockIdx.x * uint32_t(pts) * kThreads;
    // tiles [0, tiles) of this CTA hold points (the last one may be ragged), later ones are empty
    const int tiles = int(min(uint32_t(pts), (n - min(n, cta0) + kThreads - 1) / kThreads));
    auto issue = [&](int r) {                              // thread 0 only
        EvalStage<ND>& sg = s_stage[r % kEvalStages];
        unsigned long long* bar = &s_bar[r % kEvalStages];
        const size_t g = base + cta0 + size_t(r) * kThreads;
        mbar_arrive_expect_tx(bar, kStageBytes);
        bulk_copy_g2s(sg.x, cb.x + g * X, uint32_t(X * sizeof(double)) * kThreads, bar);
        bulk_copy_g2s(sg.w, cb.w + g, uint32_t(sizeof(double)) * kThreads, bar);
        bulk_copy_g2s(sg.p, cb.p + g * 3, uint32_t(3 * sizeof(float)) * kThreads, bar);
    };
    if (threadIdx.x == 0) {
        for (int r = 0; r < kEvalStages && r < tiles; ++r) issue(r);
        qtoR(s_pose + 3, s_R);
    }
    __syncthreads();
    double acc[kAcc];
#pragma unroll
    for (int k = 0; k < kAcc; ++k) acc[k] = 0.0;
#pragma unroll 1
    for (int r = 0; r < tiles; ++r) {
        const uint32_t i = cta0 + uint32_t(r) * kThreads + threadIdx.x;
        const EvalStage<ND>& sg = s_stage[r % kEvalStages];
        mbar_wait(&s_bar[r % kEvalStages], uint32_t(r / kEvalStages) & 1u);
        const double w = i < n ? sg.w[threadIdx.x] : 0.0;
        double xr[X];
#pragma unroll
        for (int k = 0; k < X; ++k) xr[k] = sg.x[threadIdx.x * X + k];
        const double pin[3] = {double(sg.p[threadIdx.x * 3 + 0]), double(sg.p[threadIdx.x * 3 + 1]), double(sg.p[threadIdx.x * 3 + 2])};
        __syncthreads();                                   // every thread holds its point: the stage may be refilled
        if (threadIdx.x == 0 && r + kEvalStages < tiles) {
            // the stage was just read through the generic proxy and is rewritten through the async (TMA) proxy:
            // the two are ordered only by a proxy fence
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            issue(r + kEvalStages);
        }
        if (w != 0.0) {
            double pw[3];
            qrot(s_pose + 3, pin, pw);
            pw[0] += s_pose[0]; pw[1] += s_pose[1]; pw[2] += s_pose[2];
            double nn[3], d;
            corr_plane<ND>(xr, nn, d);
            accumulate(acc, nn, d, w, pin, pw, s_R, bv.tukey_a2);
        }
    }
    reduce_to_partials(acc, bv, s);
}

template <int PHASE, bool ND>
__global__ void __launch_bounds__(kThreads, 2) k_evaluate(BatchView bv, CorrBuf cb) {
    const int s = blockIdx.y;
    if (bv.st[s].phase != PHASE) return;
    evaluate_body_tma<PHASE, ND>(bv, cb, s);
}

// ------------------------------------------------------------------------------------------------------------------
// Edge / line branch (a19; dormant upstream because featureExtraction emits an empty edge cloud, featureExtraction.cpp:429-436).
// k_edge_fit: LidarSLAM::ComputeLineDistanceParameters (LidarSlam.cpp:402-435) for every edge point -- exact 10-NN in the
// point's block of the EDGE map, LocalMap::nearestKSearchSpecificEdgePoint's best-line-by-inliers selection in float
// (LocalMap.h:377-474), PCA of the selected points, the line gates and processLineResults (:438-493) -- plus the first
// evaluation of EdgeAnalyticCostFunction (lidarOptimization.cpp:12-47) for the following solve.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void accumulate_edge(double acc[kAcc], const double a[3], const double b[3], double w, const double p[3],
                                                const double lp[3], const double R[9], double a2_line) {
    const double u[3] = {lp[0] - a[0], lp[1] - a[1], lp[2] - a[2]}, v[3] = {lp[0] - b[0], lp[1] - b[1], lp[2] - b[2]};
    const double de[3] = {a[0] - b[0], a[1] - b[1], a[2] - b[2]};
    const double den = sqrt(de[0] * de[0] + de[1] * de[1] + de[2] * de[2]);
    const double r[3] = {(u[1] * v[2] - u[2] * v[1]) / den, (u[2] * v[0] - u[0] * v[2]) / den, (u[0] * v[1] - u[1] * v[0]) / den};
    const double s = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    double rho0, rho1;
    if (s <= a2_line) { const double t = 1.0 - s / a2_line, t2 = t * t; rho0 = a2_line / 6.0 * (1.0 - t2 * t); rho1 = 0.5 * t2; }
    else { rho0 = a2_line / 6.0; rho1 = 0.0; }
    rho0 *= w; rho1 *= w;
    // J = skew(b - a) [I, -R [p]x] / |a - b|
    const double re[3] = {-de[0], -de[1], -de[2]};
    const double K[9] = {0, -re[2], re[1], re[2], 0, -re[0], -re[1], re[0], 0};
    const double Sp[9] = {0, -p[2], p[1], p[2], 0, -p[0], -p[1], p[0], 0};
    double J[18];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
        J[i * 6 + j] = K[i * 3 + j] / den;
        double t = 0.0;
        for (int k = 0; k < 3; ++k) { double rs = 0.0; for (int l = 0; l < 3; ++l) rs += R[k * 3 + l] * Sp[l * 3 + j]; t += K[i * 3 + k] * (-rs); }
        J[i * 6 + 3 + j] = t / den;
    }
    int kk = 0;
    for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { acc[kk++] += rho1 * (J[i] * J[j] + J[6 + i] * J[6 + j] + J[12 + i] * J[12 + j]); }
    for (int i = 0; i < 6; ++i) acc[21 + i] += rho1 * (J[i] * r[0] + J[6 + i] * r[1] + J[12 + i] * r[2]);
    acc[27] += 0.5 * rho0;
}

__global__ void __launch_bounds__(kThreads) k_edge_fit(MapView m, BatchView bv, EdgeBuf eb, uint32_t partial_offset) {
    const int s = blockIdx.y;
    IcpState* st = bv.st + s;
    if (st->phase != PH_CORR || st->n_edge == 0) return;
    __shared__ double s_pose[7];
    __shared__ double s_R[9];
    __shared__ int s_hist[8];
    __shared__ uint32_t s_buf[kBufCap * kThreads];
    if (threadIdx.x < 7) s_pose[threadIdx.x] = st->x[threadIdx.x];
    if (threadIdx.x < 8) s_hist[threadIdx.x] = 0;
    __syncthreads();
    if (threadIdx.x == 0) qtoR(s_pose + 3, s_R);
    __syncthreads();
    const uint32_t n = uint32_t(st->n_edge);
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    double acc[kAcc];
#pragma unroll
    for (int k = 0; k < kAcc; ++k) acc[k] = 0.0;
    if (i < n) {
        const size_t gi = size_t(eb.offset[s]) + i;
        const float4 sp = __ldg(&eb.scan[gi]);
        const double pin[3] = {double(sp.x), double(sp.y), double(sp.z)};
        double pf[3];
        qrot(s_pose + 3, pin, pf);
        pf[0] += s_pose[0]; pf[1] += s_pose[1]; pf[2] += s_pose[2];
        const float qx = float(pf[0]), qy = float(pf[1]), qz = float(pf[2]);
        int status = SO_MATCH_NOT_ENOUGH_NEIGHBORS;
        double ea[3] = {0, 0, 0}, ebb[3] = {0, 0, 0}, wq = 0.0;
        int nsel = 0;
        uint32_t selmask = 0;
        TopK<10> tk;
        tk.init(FLT_MAX);
        QueryCell qc;
        locate(m, qx, qy, qz, qc);
        // "<10 points in the block": the reference indexes with size_t(-1) (LocalMap.h:404-419); treated as NOT_ENOUGH_NEIGHBORS
        if (qc.slot >= 0 && qc.nblock >= 10) {
            knn_search<10>(BlockGrid(m, qc.slot), m, qc, qx, qy, qz, 0.f, s_buf, tk);
            float P[10][3];
#pragma unroll
            for (int j = 0; j < 10; ++j) { const float4 c = __ldg(&m.pts[tk.pos[j]]); P[j][0] = c.x; P[j][1] = c.y; P[j][2] = c.z; }
            // best line through the closest point by inlier count: float arithmetic in Eigen's evaluation order, no FMA contraction
            const float thr = __fmul_rn(0.2f, 0.2f);
            int best_n = 0;
            for (int pi = 1; pi < 10; ++pi) {
                float dx = __fsub_rn(P[pi][0], P[0][0]), dy = __fsub_rn(P[pi][1], P[0][1]), dz = __fsub_rn(P[pi][2], P[0][2]);
                const float z2 = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
                if (z2 > 0.f) { const float sq = __fsqrt_rn(z2); dx = __fdiv_rn(dx, sq); dy = __fdiv_rn(dy, sq); dz = __fdiv_rn(dz, sq); }
                uint32_t mask = 0; int cnt = 0;
                for (int ci = 1; ci < 10; ++ci) {
                    bool ok;
                    if (ci == pi) ok = true;
                    else {
                        const float vx = __fsub_rn(P[ci][0], P[0][0]), vy = __fsub_rn(P[ci][1], P[0][1]), vz = __fsub_rn(P[ci][2], P[0][2]);
                        const float cx = __fsub_rn(__fmul_rn(vy, dz), __fmul_rn(vz, dy)), cy = __fsub_rn(__fmul_rn(vz, dx), __fmul_rn(vx, dz)),
                                    cz = __fsub_rn(__fmul_rn(vx, dy), __fmul_rn(vy, dx));
                        ok = __fadd_rn(__fmul_rn(cx, cx), __fadd_rn(__fmul_rn(cy, cy), __fmul_rn(cz, cz))) < thr;
                    }
                    if (ok) { mask |= 1u << ci; ++cnt; }
                }
                if (cnt > best_n) { best_n = cnt; selmask = mask; }
            }
            selmask |= 1u;                                               // the closest point is always kept, first
            nsel = __popc(selmask);
            const int last = 31 - __clz(selmask);
            if (nsel < 4) status = SO_MATCH_NOT_ENOUGH_NEIGHBORS;                                 // validateNeighborSearch (:495-512)
            else if (tk.d2[last] > __fmul_rn(3.f, m.plane_res)) status = SO_MATCH_NEIGHBORS_TOO_FAR;   // MapView::plane_res holds lineRes_ for the edge map
            else {
                // PCA of the selected points (computePCAForFeature, EdgeFeature branch, :749-790)
                double mean[3] = {0, 0, 0};
                for (int j = 0; j < 10; ++j) if (selmask >> j & 1) { mean[0] += double(P[j][0]); mean[1] += double(P[j][1]); mean[2] += double(P[j][2]); }
                mean[0] /= double(nsel); mean[1] /= double(nsel); mean[2] /= double(nsel);
                double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
                for (int j = 0; j < 10; ++j) if (selmask >> j & 1) {
                    const double c0 = double(P[j][0]) - mean[0], c1 = double(P[j][1]) - mean[1], c2 = double(P[j][2]) - mean[2];
                    S[0] += c0 * c0; S[1] += c0 * c1; S[2] += c0 * c2; S[4] += c1 * c1; S[5] += c1 * c2; S[8] += c2 * c2;
                }
                S[3] = S[1]; S[6] = S[2]; S[7] = S[5];
                double V[9], ev[3];
                jacobi_eig<3, 12>(S, V, ev);
                if (!(isfinite(ev[0]) && isfinite(ev[1]) && isfinite(ev[2]))) status = SO_MATCH_INVALID_NUMERICAL;
                else if (ev[2] < 4.0 * ev[1]) status = SO_MATCH_BAD_PCA_STRUCTURE;
                else {
                    double dir[3] = {V[2], V[5], V[8]};                     // processLineResults (:438-493)
                    const double dn = sqrt(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
                    dir[0] /= dn; dir[1] /= dn; dir[2] /= dn;
                    const double lim = double(__fmul_rn(3.f, m.plane_res));
                    double msd = 0.0;
                    bool ok = isfinite(dir[0]) && isfinite(dir[1]) && isfinite(dir[2]);
                    if (!ok) status = SO_MATCH_INVALID_NUMERICAL;
                    else {
                        for (int j = 0; j < 10; ++j) if (selmask >> j & 1) {
                            const double c[3] = {double(P[j][0]) - mean[0], double(P[j][1]) - mean[1], double(P[j][2]) - mean[2]};
                            double sd = 0.0;
                            for (int a2 = 0; a2 < 3; ++a2) {
                                double Ac = 0.0;
                                for (int b2 = 0; b2 < 3; ++b2) Ac += ((a2 == b2 ? 1.0 : 0.0) - dir[a2] * dir[b2]) * c[b2];
                                sd += c[a2] * Ac;
                            }
                            if (ok && sd > lim) ok = false;
                            msd += sd;
                        }
                        if (!ok) status = SO_MATCH_MSE_TOO_LARGE;
                        else {
                            msd /= double(nsel);
                            wq = 1.0 - sqrt(msd / lim);
                            for (int a2 = 0; a2 < 3; ++a2) { ea[a2] = 0.1 * dir[a2] + mean[a2]; ebb[a2] = -0.1 * dir[a2] + mean[a2]; }
                            status = SO_MATCH_SUCCESS;
                            accumulate_edge(acc, ea, ebb, wq, pin, pf, s_R, bv.tukey_a2_line);
                        }
                    }
                }
            }
        }
        atomicAdd(&s_hist[status], 1);
        eb.a[gi] = make_double4(ea[0], ea[1], ea[2], wq);
        eb.b[gi] = make_double4(ebb[0], ebb[1], ebb[2], 0.0);
        eb.flags[gi] = make_uchar4((unsigned char)status, (unsigned char)nsel, 0, 0);
        if (eb.nn) {
#pragma unroll
            for (int j = 0; j < 10; ++j) eb.nn[gi * 10 + j] = tk.id[j];
            eb.selmask[gi] = selmask;
        }
    }
    __syncthreads();
    if (threadIdx.x < 7 && s_hist[threadIdx.x]) atomicAdd(&bv.hist[s * kHistStride + 16 + threadIdx.x], s_hist[threadIdx.x]);
    reduce_to_partials(acc, bv, s, partial_offset);
}

__global__ void __launch_bounds__(kThreads) k_edge_evaluate(BatchView bv, EdgeBuf eb, uint32_t partial_offset) {
    const int s = blockIdx.y;
    IcpState* st = bv.st + s;
    if (st->phase != PH_EVAL || st->n_edge == 0) return;
    __shared__ double s_pose[7];
    __shared__ double s_R[9];
    if (threadIdx.x < 7) s_pose[threadIdx.x] = st->cand[threadIdx.x];
    __syncthreads();
    if (threadIdx.x == 0) qtoR(s_pose + 3, s_R);
    __syncthreads();
    const uint32_t n = uint32_t(st->n_edge);
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    double acc[kAcc];
#pragma unroll
    for (int k = 0; k < kAcc; ++k) acc[k] = 0.0;
    if (i < n) {
        const size_t gi = size_t(eb.offset[s]) + i;
        const double4 a = eb.a[gi];
        if (a.w != 0.0) {
            const double4 b = eb.b[gi];
            const float4 sp = __ldg(&eb.scan[gi]);
            const double pin[3] = {double(sp.x), double(sp.y), double(sp.z)};
            double lp[3];
            qrot(s_pose + 3, pin, lp);
            lp[0] += s_pose[0]; lp[1] += s_pose[1]; lp[2] += s_pose[2];
            const double aa[3] = {a.x, a.y, a.z}, bb[3] = {b.x, b.y, b.z};
            accumulate_edge(acc, aa, bb, a.w, pin, lp, s_R, bv.tukey_a2_line);
        }
    }
    reduce_to_partials(acc, bv, s, partial_offset);
}

// ------------------------------------------------------------------------------------------------------------------
// k_lm_step: one CTA per scan.  Sums the per-CTA partials of the preceding k_fit (AFTER == PH_CORR) or k_evaluate
// (AFTER == PH_EVAL) in a fixed order, then one thread advances the optimiser / ICP state machine.
// ------------------------------------------------------------------------------------------------------------------
// Called by >= 128 threads of one CTA (all of them: it synchronises the CTA); the first 128 do the work.  DEG: the step of the
// degeneracy-aware registration, with the scan's DegenState (dg: the chunk's array) beside its IcpState.
template <int AFTER, bool DEG = false>
__device__ __forceinline__ void lm_step_body(const BatchView& bv, int s, uint32_t n_partials, uint32_t edge_partial_offset, DegenState* dg = nullptr) {
    IcpState* st = bv.st + s;
    __shared__ double s_red[4][kAcc];
    __shared__ double s_sum[kAcc];
    const int comp = threadIdx.x & 31, sub = threadIdx.x >> 5;
    double v = 0.0;
    if (comp < kAcc && sub < 4) {
        const double* base = bv.partials + size_t(s) * bv.partial_stride * kAcc;
        const uint32_t np = eval_ctas(uint32_t(st->n_points));
        // __ldcg: straight from L2 -- in k_evaluate_lm the rows were written by other CTAs of the same launch
        for (uint32_t b = sub; b < np && b < n_partials; b += 4) v += __ldcg(&base[size_t(b) * kAcc + comp]);
        const uint32_t ne = (uint32_t(st->n_edge) + kThreads - 1) / kThreads;          // edge branch partials (0 when no edge cloud)
        for (uint32_t b = sub; b < ne; b += 4) v += __ldcg(&base[size_t(edge_partial_offset + b) * kAcc + comp]);
        s_red[sub][comp] = v;
    }
    // The serial step works on a SHARED-MEMORY copy of the scan's state: through the global pointer every field access of the
    // one working thread was a dependent L2 round trip (the step took 5-12 us, the covariance 40 us); the copy in and out is two
    // coalesced passes of the CTA.
    __shared__ IcpState s_st;
    cta_copy(&s_st, st);
    DegenState* sdg = nullptr;                             // the DegenState's shared copy, the same way
    if constexpr (DEG) {
        __shared__ DegenState s_dg;
        sdg = &s_dg;
        cta_copy(sdg, dg + s);
    }
    __syncthreads();
    if (threadIdx.x < kAcc) s_sum[threadIdx.x] = (s_red[0][threadIdx.x] + s_red[1][threadIdx.x]) + (s_red[2][threadIdx.x] + s_red[3][threadIdx.x]);
    __syncthreads();
    if (threadIdx.x == 0) {
        IcpState& S = s_st;
        if (AFTER == PH_CORR) {
            // histograms of this ICP iteration (ResetDistanceParameters + processPlannerFeatures, :847-852,:336-341)
            for (int k = 0; k < 9; ++k) S.hist_obs[k] = bv.hist[s * kHistStride + k];
            for (int k = 0; k < 7; ++k) S.hist_rej[k] = bv.hist[s * kHistStride + 9 + k];
            for (int k = 0; k < 7; ++k) S.hist_rej_line[k] = bv.hist[s * kHistStride + 16 + k];
            S.n_ok_edge = S.hist_rej_line[0];
            const int n_ok = S.hist_rej[0] + S.n_ok_edge;       // features_corres.size(): edges + planes
            for (int k = 0; k < kHistStride; ++k) bv.hist[s * kHistStride + k] = 0;
            if (S.max_icp_iters < 0) {          // stage mode (so_correspond): stop here
                for (int k = 0; k < 21; ++k) S.H[k] = s_sum[k];
                for (int k = 0; k < 6; ++k) S.g[k] = s_sum[21 + k];
                S.cost = s_sum[27]; S.n_ok = n_ok; S.phase = PH_DONE;
            } else if constexpr (DEG) lm_begin_solve_deg(S, *sdg, s_sum, n_ok);
            else lm_begin_solve(S, s_sum, n_ok);
        } else {
            if (S.max_icp_iters < 0) {          // stage mode (so_evaluate): report and stop
                for (int k = 0; k < 21; ++k) S.H[k] = s_sum[k];
                for (int k = 0; k < 6; ++k) S.g[k] = s_sum[21 + k];
                S.cost = s_sum[27]; S.phase = PH_DONE;
            } else if constexpr (DEG) lm_after_eval_deg(S, *sdg, s_sum);
            else lm_after_eval(S, s_sum);
        }
    }
    __syncthreads();
    if (s_st.need_cov) {                                   // the registration just ended (CTA-uniform)
        __shared__ CovScratch s_cov;
        if (threadIdx.x < 32) covariance_and_errors_warp(s_st, s_cov);      // need_cov stays set: the state is re-initialised per registration
        __syncthreads();
    }
    cta_copy(st, &s_st);
    if constexpr (DEG) cta_copy(dg + s, sdg);
}

template <int AFTER>
__global__ void __launch_bounds__(128) k_lm_step(BatchView bv, uint32_t n_partials, uint32_t edge_partial_offset) {
    const int s = blockIdx.x;
    if (bv.st[s].phase != AFTER) return;
    lm_step_body<AFTER>(bv, s, n_partials, edge_partial_offset);
}

// k_lm_step of the degeneracy-aware registration (so_register_degeneracy*); dg: the chunk's DegenState array
template <int AFTER>
__global__ void __launch_bounds__(128) k_lm_step_deg(BatchView bv, uint32_t n_partials, uint32_t edge_partial_offset, DegenState* __restrict__ dg) {
    const int s = blockIdx.x;
    if (bv.st[s].phase != AFTER) return;
    lm_step_body<AFTER, true>(bv, s, n_partials, edge_partial_offset, dg);
}

// so_degeneracy_analysis: degeneracy_analysis on st->H, one thread
__global__ void k_degeneracy_analysis(const IcpState* __restrict__ st, DegenState* __restrict__ dg) { degeneracy_analysis(st->H, *dg); }
uint32_t launch_degeneracy_analysis(const IcpState* st, DegenState* dg, cudaStream_t stream) { k_degeneracy_analysis<<<1, 1, 0, stream>>>(st, dg); return 1; }

// so_covariance (6 columns): the covariance step that ends a registration, on st->H, in one 32-thread CTA and a shared copy of the
// state as lm_step_body runs it
__global__ void __launch_bounds__(32) k_covariance(IcpState* st) {
    __shared__ IcpState s_st;
    __shared__ CovScratch s_cov;
    cta_copy(&s_st, st);
    __syncthreads();
    covariance_and_errors_warp(s_st, s_cov);
    __syncthreads();
    cta_copy(st, &s_st);
}

uint32_t launch_covariance(IcpState* st, cudaStream_t stream) { k_covariance<<<1, 32, 0, stream>>>(st); return 1; }


// ------------------------------------------------------------------------------------------------------------------
// k_evaluate_lm: k_evaluate with the optimiser step of k_lm_step folded in -- the CTA that finishes LAST (ticket counter, after a
// device-scope fence) sums the partial rows in their fixed order and advances the state machine.  Same arithmetic in the same
// order as the two-kernel form, one launch less per cost evaluation: used when a registration is launch-latency bound (one or
// two scans in flight, no edge cloud), where the ~190 registers of the serial step cost no occupancy that matters.
// ------------------------------------------------------------------------------------------------------------------
template <int PHASE, bool ND>
__global__ void __launch_bounds__(kThreads, 1) k_evaluate_lm(BatchView bv, CorrBuf cb, uint32_t* __restrict__ counters) {
    const int s = blockIdx.y;
    if (bv.st[s].phase != PHASE) return;
    evaluate_body<PHASE, ND>(bv, cb, s);
    __shared__ uint32_t s_ticket;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_ticket = atomicAdd(&counters[s], 1u);
    __syncthreads();
    if (s_ticket != gridDim.x - 1) return;
    if (threadIdx.x == 0) counters[s] = 0;               // ready for the next launch
    __threadfence();
    lm_step_body<PHASE>(bv, s, gridDim.x, bv.edge_partial_offset);
}

// Loop condition of the CUDA-graph WHILE node that wraps one ICP iteration: keep iterating while any scan of the
// batch is still registering (LidarSlam.cpp:119-148 runs this loop on the host, one scan at a time).
__global__ void k_loop_cond(const IcpState* __restrict__ st, uint32_t n_scans, cudaGraphConditionalHandle handle) {
    int active = 0;
    for (uint32_t s = threadIdx.x; s < n_scans; s += 32) active |= (st[s].phase != PH_DONE);
    active = __any_sync(0xffffffffu, active);
    if (threadIdx.x == 0) cudaGraphSetConditional(handle, active ? 1u : 0u);
}

// ------------------------------------------------------------------------------------------------------------------
// k_knn: LocalMap::nearestKSearchSurf for a batch of world-frame queries (so_knn / so_knn_device)
// ------------------------------------------------------------------------------------------------------------------
// cell-order key of every query (so_knn* orders large query sets first, for the same reason scans are ordered)
__global__ void __launch_bounds__(kThreads) k_query_keys(MapView m, const float4* __restrict__ q, size_t nq, uint32_t* __restrict__ keys,
                                                         uint32_t* __restrict__ vals) {
    const size_t i = size_t(blockIdx.x) * kThreads + threadIdx.x;
    if (i >= nq) return;
    const float4 p = __ldg(&q[i]);
    QueryCell qc;
    locate(m, p.x, p.y, p.z, qc);
    keys[i] = qc.slot >= 0 ? scan_order_key(m, qc) : 0xFFFFFFFFu;
    vals[i] = uint32_t(i);
}

// kKnnThreads queries per CTA; `order` (optional): the queries in cell order, thread j takes the j-th of them.
template <int K>
__global__ void __launch_bounds__(kKnnThreads) k_knn(MapView m, const float4* __restrict__ q, const uint32_t* __restrict__ order, size_t nq,
                                                     float max_d2, uint32_t* __restrict__ idx, float* __restrict__ d2) {
    __shared__ uint32_t s_buf[kBufCap * kKnnThreads];
    const size_t j0 = size_t(blockIdx.x) * kKnnThreads;
    if (j0 >= nq) return;
    const size_t j = j0 + threadIdx.x;
    const bool in_range = j < nq;
    const size_t i = in_range ? (order ? size_t(order[j]) : j) : 0;        // thread j handles the j-th query in cell order, answers in caller order
    const float4 p = __ldg(&q[i]);
    TopK<K> tk;
    tk.init(max_d2 > 0.f ? max_d2 : FLT_MAX);
    QueryCell qc;
    qc.slot = -1; qc.nblock = 0; qc.c[0] = qc.c[1] = qc.c[2] = 0; qc.f[0] = qc.f[1] = qc.f[2] = 0.f;
    if (in_range) locate(m, p.x, p.y, p.z, qc);
    if (in_range && qc.slot >= 0) knn_search<K>(BlockGrid(m, qc.slot), m, qc, p.x, p.y, p.z, max_d2, s_buf, tk);
    if (!in_range) return;
#pragma unroll
    for (int jj = 0; jj < K; ++jj) {
        const bool ok = tk.id[jj] != 0xFFFFFFFFu;
        idx[i * K + jj] = tk.id[jj];
        d2[i * K + jj] = ok ? tk.d2[jj] : 0.f;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Replay plumbing (SURVEY 8e, K8): one row of 8 doubles per scan -- the optimiser's pose {tx,ty,tz,qx,qy,qz,qw} (so_icp_result.pose_opt)
// and status + 256 * n_iterations -- into a caller-owned device buffer, so that the NCCL gather of a sharded replay reads device
// memory on the compute stream instead of waiting for a host round trip.
__global__ void k_pack_poses(const IcpState* __restrict__ st, uint32_t n_scans, double* __restrict__ rows) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_scans) return;
#pragma unroll
    for (int k = 0; k < 7; ++k) rows[size_t(s) * 8 + k] = st[s].x[k];
    rows[size_t(s) * 8 + 7] = double(st[s].status + 256 * st[s].n_iterations);
}

// ------------------------------------------------------------------------------------------------------------------
// host-side launchers
// ------------------------------------------------------------------------------------------------------------------
// keys: the 64-bit key buffer; with key32 it is used as an array of uint32_t (same point indexing)
uint32_t launch_scan_keys(const MapView& m, const BatchView& bv, uint64_t* keys, uint32_t* vals, uint32_t grid_x, uint32_t n_scans, int cell_bits, bool key32,
                          bool compact, cudaStream_t st) {
    const dim3 g(grid_x, n_scans);
    uint32_t* k32 = reinterpret_cast<uint32_t*>(keys);
    if (key32) { if (compact) k_scan_keys<uint32_t, true><<<g, kThreads, 0, st>>>(m, bv, k32, vals, cell_bits); else k_scan_keys<uint32_t, false><<<g, kThreads, 0, st>>>(m, bv, k32, vals, cell_bits); }
    else { if (compact) k_scan_keys<uint64_t, true><<<g, kThreads, 0, st>>>(m, bv, keys, vals, cell_bits); else k_scan_keys<uint64_t, false><<<g, kThreads, 0, st>>>(m, bv, keys, vals, cell_bits); }
    return 1;
}
uint32_t launch_scan_finish(const BatchView& bv, const uint64_t* sorted_keys, size_t first, uint32_t pt_first, int cell_bits, bool key32, uint32_t n_scans, cudaStream_t st) {
    if (key32) k_scan_finish<uint32_t><<<(n_scans + 63) / 64, 64, 0, st>>>(bv, reinterpret_cast<const uint32_t*>(sorted_keys) + first, pt_first, cell_bits, n_scans);
    else k_scan_finish<uint64_t><<<(n_scans + 63) / 64, 64, 0, st>>>(bv, sorted_keys + first, pt_first, cell_bits, n_scans);
    return 1;
}
uint32_t launch_prepare_small(const MapView& m, const BatchView& bv, float4* out, uint32_t n_scans, int key_bits, uint32_t max_kept, cudaStream_t st) {
    if (max_kept <= 2u * kSmallThreads) k_prepare_small<2><<<n_scans, kSmallThreads, 0, st>>>(m, bv, out, key_bits);
    else k_prepare_small<4><<<n_scans, kSmallThreads, 0, st>>>(m, bv, out, key_bits);
    return 1;
}
uint32_t launch_scan_gather(const float4* in, const uint32_t* vals, const uint64_t* keys, size_t first, const uint32_t* offset, size_t total, float4* out,
                            int cell_bits, bool key32, cudaStream_t st) {
    const uint32_t grid = uint32_t((total + kThreads - 1) / kThreads);
    if (key32) k_scan_gather<uint32_t><<<grid, kThreads, 0, st>>>(in, vals + first, reinterpret_cast<const uint32_t*>(keys) + first, offset, total, out, cell_bits);
    else k_scan_gather<uint64_t><<<grid, kThreads, 0, st>>>(in, vals + first, keys + first, offset, total, out, cell_bits);
    return 1;
}
// The correspondence stage of one ICP iteration is launch_match (search + fit of every scan point), then launch_first_eval (first
// evaluation of the new solve, the edge kernel when an edge cloud is present, and the optimiser's iteration zero).
// medge / eb / grid_e: edge branch (grid_e == 0: idle); k_lm_step sums the partials of both branches.
uint32_t launch_match(const MapView& m, const BatchView& bv, const CorrBuf& cb, const NnBuf& nb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, int part) {
    if (!grid_x) return 0;
    uint32_t n = 0;
    if (part != 2) {
        if (bv.coop_knn) { k_knn_scan_coop<<<dim3(grid_x * (kThreads / kCoopWarps), n_scans), kThreads, 0, st>>>(m, bv, nb); n = 1; }
        else if (m.graph && nb.queue) {
            k_knn_scan<true><<<dim3(grid_x * (kThreads / kKnnThreads), n_scans), kKnnThreads, 0, st>>>(m, bv, nb);
            k_knn_round2<<<dim3(grid_x * (kThreads / kKnnThreads), n_scans), kKnnThreads, 0, st>>>(m, bv, nb);
            n = 2;
        } else { k_knn_scan<false><<<dim3(grid_x * (kThreads / kKnnThreads), n_scans), kKnnThreads, 0, st>>>(m, bv, nb); n = 1; }
    }
    const uint32_t gf = (grid_x * kThreads + kFitPts * kFitThreads - 1) / (kFitPts * kFitThreads);
    if (part != 1) { k_fit<<<dim3(gf, n_scans), kFitThreads, 0, st>>>(m, bv, cb, nb); n++; }
    return n;
}
uint32_t launch_inject(const MapView& m, const float4* by_id, uint32_t n_map, const BatchView& bv, const NnBuf& nb, const uint32_t* ids, int n_trace_iters,
                       uint32_t grid_x, uint32_t n_scans, cudaStream_t st) {
    if (!grid_x) return 0;
    k_knn_inject<<<dim3(grid_x, n_scans), kThreads, 0, st>>>(m, by_id, n_map, bv, nb, ids, n_trace_iters);
    return 1;
}
uint32_t launch_first_eval(const BatchView& bv, const CorrBuf& cb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const MapView* medge, const EdgeBuf* eb,
                           uint32_t grid_e, DegenState* dg) {
    const uint32_t gp = grid_x ? eval_grid(grid_x * kThreads) : 0;
    if (bv.counters && gp && !grid_e && !dg) {
        (cb.given ? k_evaluate_lm<PH_CORR, true> : k_evaluate_lm<PH_CORR, false>)<<<dim3(gp, n_scans), kThreads, 0, st>>>(bv, cb, bv.counters);
        return 1;
    }
    if (gp) (cb.given ? k_evaluate<PH_CORR, true> : k_evaluate<PH_CORR, false>)<<<dim3(gp, n_scans), kThreads, 0, st>>>(bv, cb);
    if (grid_e) k_edge_fit<<<dim3(grid_e, n_scans), kThreads, 0, st>>>(*medge, bv, *eb, bv.edge_partial_offset);
    if (dg) k_lm_step_deg<PH_CORR><<<n_scans, 128, 0, st>>>(bv, gp, bv.edge_partial_offset, dg);
    else k_lm_step<PH_CORR><<<n_scans, 128, 0, st>>>(bv, gp, bv.edge_partial_offset);
    return (gp ? 1 : 0) + (grid_e ? 1 : 0) + 1;
}
uint32_t launch_edge_fit(const MapView& medge, const BatchView& bv, const EdgeBuf& eb, uint32_t grid_e, uint32_t n_scans, cudaStream_t st) {
    if (!grid_e) return 0;
    k_edge_fit<<<dim3(grid_e, n_scans), kThreads, 0, st>>>(medge, bv, eb, bv.edge_partial_offset);
    return 1;
}
uint32_t launch_evaluate(const BatchView& bv, const CorrBuf& cb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const EdgeBuf* eb, uint32_t grid_e,
                         DegenState* dg) {
    const uint32_t gx = grid_x ? eval_grid(grid_x * kThreads) : 0;
    if (bv.counters && gx && !grid_e && !dg) {
        (cb.given ? k_evaluate_lm<PH_EVAL, true> : k_evaluate_lm<PH_EVAL, false>)<<<dim3(gx, n_scans), kThreads, 0, st>>>(bv, cb, bv.counters);
        return 1;
    }
    if (gx) (cb.given ? k_evaluate<PH_EVAL, true> : k_evaluate<PH_EVAL, false>)<<<dim3(gx, n_scans), kThreads, 0, st>>>(bv, cb);
    if (grid_e) k_edge_evaluate<<<dim3(grid_e, n_scans), kThreads, 0, st>>>(bv, *eb, bv.edge_partial_offset);
    if (dg) k_lm_step_deg<PH_EVAL><<<n_scans, 128, 0, st>>>(bv, gx, bv.edge_partial_offset, dg);
    else k_lm_step<PH_EVAL><<<n_scans, 128, 0, st>>>(bv, gx, bv.edge_partial_offset);
    return (gx ? 1 : 0) + (grid_e ? 1 : 0) + 1;
}
uint32_t launch_loop_cond(const BatchView& bv, uint32_t n_scans, cudaGraphConditionalHandle handle, cudaStream_t st) {
    k_loop_cond<<<1, 32, 0, st>>>(bv.st, n_scans, handle);
    return 1;
}
uint32_t launch_pack_poses(const IcpState* st, uint32_t n_scans, double* rows, cudaStream_t stream) {
    k_pack_poses<<<(n_scans + 63) / 64, 64, 0, stream>>>(st, n_scans, rows);
    return 1;
}
void launch_query_keys(const MapView& m, const float4* q, size_t nq, uint32_t* keys, uint32_t* vals, cudaStream_t st) {
    k_query_keys<<<uint32_t((nq + kThreads - 1) / kThreads), kThreads, 0, st>>>(m, q, nq, keys, vals);
}
template <int K>
static void launch_knn_k(const MapView& m, const float4* q, const uint32_t* order, size_t nq, float max_d2, uint32_t* idx, float* d2, cudaStream_t st) {
    k_knn<K><<<uint32_t((nq + kKnnThreads - 1) / kKnnThreads), kKnnThreads, 0, st>>>(m, q, order, nq, max_d2, idx, d2);
}
int launch_knn(const MapView& m, const float4* q, const uint32_t* order, size_t nq, int k, float max_d2, uint32_t* idx, float* d2, cudaStream_t st) {
    switch (k) {
        case 1: launch_knn_k<1>(m, q, order, nq, max_d2, idx, d2, st); break;
        case 2: launch_knn_k<2>(m, q, order, nq, max_d2, idx, d2, st); break;
        case 3: launch_knn_k<3>(m, q, order, nq, max_d2, idx, d2, st); break;
        case 4: launch_knn_k<4>(m, q, order, nq, max_d2, idx, d2, st); break;
        case 5: launch_knn_k<5>(m, q, order, nq, max_d2, idx, d2, st); break;
        case 6: launch_knn_k<6>(m, q, order, nq, max_d2, idx, d2, st); break;
        case 7: launch_knn_k<7>(m, q, order, nq, max_d2, idx, d2, st); break;
        case 8: launch_knn_k<8>(m, q, order, nq, max_d2, idx, d2, st); break;
        default: return -1;
    }
    return 0;
}

}  // namespace so

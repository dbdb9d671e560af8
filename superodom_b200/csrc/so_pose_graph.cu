// so_pose_graph.cu -- sparse SE(3) pose-graph least squares on the device (so_pose_graph_solve), sm_90a, FP64.
//
// The problem and its trust-region rules: include/superodom_b200.h and DESIGN.md section 4, "Pose graph".  The rules are those of
// so_trust_region.cuh (DESIGN.md section 3), restated here on the host: that loop runs on one thread over a dense system in shared
// memory, this one over kernels and a control block read back once per trust-region trial.
//   k_pg_edges     one thread per edge: E = Z^-1 X_i^-1 X_j, r, the Cauchy weight, the corrected Jacobians, the edge's blocks
//                  A_ii, A_jj, A_ij, its gradient parts and 1/2 rho
//   k_pg_nodes     one thread per node: its incident edges' blocks summed in incidence order (ascending edge id), the chain block
//                  (k, k+1), the gradient max-norm through Plus and |x_k|^2; the Jacobi scaling at iteration 0
//   k_pg_reduce    one CTA: cost, gmax and |x|^2 in a fixed order into the control block
//   k_pg_trial     cooperative, across the grid: the damped, scaled system, its block-tridiagonal preconditioner factored by block
//                  cyclic reduction (one thread per block row of a level), PCG to kPcgTol with grid-wide barriers between its phases,
//                  the model cost change, the candidate by Plus and the step norm
// No float atomics: every sum runs in an order fixed by the graph, so results are bit-identical run to run.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "so_ctx.cuh"
#include "so_trust_region.cuh"

#include <cooperative_groups.h>

namespace so {

namespace cg = cooperative_groups;

// PCG stops when r'M^-1 r <= kPcgTol^2 r0'M^-1 r0 (DESIGN.md, "Pose graph": the measurement behind the value), or after kPcgMaxIter
constexpr double kPcgTol = 1e-10;
constexpr int kPcgMaxIter = 1000;
constexpr int kTrialThreads = 256;

struct PgEdgeBlk { double aii[36], ajj[36], aij[36], gi[6], gj[6]; };
struct PgCtl {
    double cost[2], gmax[2], xnorm2[2];            // per linearisation set (k_pg_reduce)
    double mcc, step_norm2;                        // the last trial (k_pg_trial)
    int32_t valid, pcg_iters;
};

// ------------------------------------------------------------------------------------------------------------------ 6x6 blocks
__device__ __forceinline__ void mm6(const double* A, const double* B, double* C) {        // C = A B
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) { double t = 0.0; for (int k = 0; k < 6; ++k) t += A[i * 6 + k] * B[k * 6 + j]; C[i * 6 + j] = t; }
}
__device__ __forceinline__ void mv6_add(const double* A, const double* x, double* y, double sgn) {    // y += sgn A x
    for (int i = 0; i < 6; ++i) { double t = 0.0; for (int k = 0; k < 6; ++k) t += A[i * 6 + k] * x[k]; y[i] += sgn * t; }
}
__device__ __forceinline__ void mtv6_add(const double* A, const double* x, double* y) {               // y += A^T x
    for (int i = 0; i < 6; ++i) { double t = 0.0; for (int k = 0; k < 6; ++k) t += A[k * 6 + i] * x[k]; y[i] += t; }
}

// ------------------------------------------------------------------------------------------------------------------ linearisation
__global__ void __launch_bounds__(128) k_pg_edges(const so_pose_edge* __restrict__ E, uint32_t m, const double* __restrict__ x,
                                                  PgEdgeBlk* __restrict__ blk, double* __restrict__ ecost, double* __restrict__ wout) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    const so_pose_edge& ed = E[e];
    const double* xi = x + 7 * size_t(ed.i);
    const double* xj = x + 7 * size_t(ed.j);
    const double qzc[4] = {-ed.z[3], -ed.z[4], -ed.z[5], ed.z[6]}, qic[4] = {-xi[3], -xi[4], -xi[5], xi[6]};
    double qa[4], qE[4], a[3], tE[3];
    qmul(qzc, qic, qa);
    qmul(qa, xj + 3, qE);
    const double dt[3] = {xj[0] - xi[0], xj[1] - xi[1], xj[2] - xi[2]};
    qrot(qic, dt, a);                                                     // a = R_i^T (t_j - t_i)
    const double at[3] = {a[0] - ed.z[0], a[1] - ed.z[1], a[2] - ed.z[2]};
    qrot(qzc, at, tE);                                                    // t_E = R_z^T (a - t_z)
    // Log(R_E): angle in [0, pi]
    const double sg = qE[3] < 0.0 ? -1.0 : 1.0;
    const double vn = sqrt(qE[0] * qE[0] + qE[1] * qE[1] + qE[2] * qE[2]);
    const double th = 2.0 * atan2(vn, sg * qE[3]);
    const double f = vn > 0.0 ? sg * th / vn : 0.0;
    const double phi[3] = {f * qE[0], f * qE[1], f * qE[2]};
    const double c3 = jrinv_coeff(th);
    // J_r^-1(phi) = I + [phi]x / 2 + c3 [phi]x^2
    const double P[9] = {0, -phi[2], phi[1], phi[2], 0, -phi[0], -phi[1], phi[0], 0};
    double Jinv[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            double p2 = 0.0;
            for (int k = 0; k < 3; ++k) p2 += P[r * 3 + k] * P[k * 3 + c];
            Jinv[r * 3 + c] = (r == c ? 1.0 : 0.0) + 0.5 * P[r * 3 + c] + c3 * p2;
        }
    double Rz[9], Ri[9], Rj[9];
    qtoR(ed.z + 3, Rz); qtoR(xi + 3, Ri); qtoR(xj + 3, Rj);
    // raw Jacobians in the tangent of Plus at 0 (world-frame translation, right-perturbed rotation), rows [t_E ; phi]
    double RzRi[9], RjRi[9], Ax[9], RA[9], JR[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            double t = 0.0, u = 0.0;
            for (int k = 0; k < 3; ++k) { t += Rz[k * 3 + r] * Ri[c * 3 + k]; u += Rj[k * 3 + r] * Ri[k * 3 + c]; }
            RzRi[r * 3 + c] = t;                                          // R_z^T R_i^T
            RjRi[r * 3 + c] = u;                                          // R_j^T R_i
        }
    const double ax[9] = {0, -a[2], a[1], a[2], 0, -a[0], -a[1], a[0], 0};
    for (int r = 0; r < 9; ++r) Ax[r] = ax[r];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            double t = 0.0, u = 0.0;
            for (int k = 0; k < 3; ++k) { t += Rz[k * 3 + r] * Ax[k * 3 + c]; u += Jinv[r * 3 + k] * RjRi[k * 3 + c]; }
            RA[r * 3 + c] = t;                                            // R_z^T [a]x
            JR[r * 3 + c] = u;                                            // J_r^-1 R_j^T R_i
        }
    double Ji[36], Jj[36];
    for (int k = 0; k < 36; ++k) { Ji[k] = 0.0; Jj[k] = 0.0; }
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            Ji[r * 6 + c] = -RzRi[r * 3 + c];
            Ji[r * 6 + 3 + c] = RA[r * 3 + c];
            Ji[(3 + r) * 6 + 3 + c] = -JR[r * 3 + c];
            Jj[r * 6 + c] = RzRi[r * 3 + c];
            Jj[(3 + r) * 6 + 3 + c] = Jinv[r * 3 + c];
        }
    const double rr[6] = {tE[0], tE[1], tE[2], phi[0], phi[1], phi[2]};
    // S applied to r and both Jacobians
    double res[6], SJi[36], SJj[36];
    for (int r = 0; r < 6; ++r) {
        double t = 0.0;
        for (int k = 0; k < 6; ++k) t += ed.sqrt_info[r * 6 + k] * rr[k];
        res[r] = t;
        for (int c = 0; c < 6; ++c) {
            double u = 0.0, v = 0.0;
            for (int k = 0; k < 6; ++k) { u += ed.sqrt_info[r * 6 + k] * Ji[k * 6 + c]; v += ed.sqrt_info[r * 6 + k] * Jj[k * 6 + c]; }
            SJi[r * 6 + c] = u; SJj[r * 6 + c] = v;
        }
    }
    double s = 0.0;
    for (int r = 0; r < 6; ++r) s += res[r] * res[r];
    double rho = s, rho1 = 1.0;
    if (ed.cauchy > 0.0) {                                                // ceres::CauchyLoss(c): b = c^2, 1 / b
        const double b = ed.cauchy * ed.cauchy, ib = 1.0 / b;
        const double sum = 1.0 + s * ib;
        rho = b * log(sum);
        rho1 = fmax(DBL_MIN, 1.0 / sum);
    }
    // ceres::Corrector with rho'' <= 0: r and J both scaled by sqrt(rho'); the products below are rho' J^T J and rho' J^T r
    PgEdgeBlk& B = blk[e];
    for (int r = 0; r < 6; ++r) {
        for (int c = 0; c < 6; ++c) {
            double tii = 0.0, tjj = 0.0, tij = 0.0;
            for (int k = 0; k < 6; ++k) {
                tii += SJi[k * 6 + r] * SJi[k * 6 + c];
                tjj += SJj[k * 6 + r] * SJj[k * 6 + c];
                tij += SJi[k * 6 + r] * SJj[k * 6 + c];
            }
            B.aii[r * 6 + c] = rho1 * tii; B.ajj[r * 6 + c] = rho1 * tjj; B.aij[r * 6 + c] = rho1 * tij;
        }
        double gi = 0.0, gj = 0.0;
        for (int k = 0; k < 6; ++k) { gi += SJi[k * 6 + r] * res[k]; gj += SJj[k * 6 + r] * res[k]; }
        B.gi[r] = rho1 * gi; B.gj[r] = rho1 * gj;
    }
    ecost[e] = 0.5 * rho;
    wout[e] = rho1;
}

struct PgNodeArgs {
    const so_pose_edge* E; const int32_t* inc; const PgEdgeBlk* blk; const double* x;
    double *H, *C, *g, *scale, *part;                                    // part: [n][2] gmax, |x_k|^2 (0 for the fixed node)
    uint32_t n; int32_t fixed, init;
};

__global__ void __launch_bounds__(128) k_pg_nodes(PgNodeArgs a) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= a.n) return;
    const bool fixed = int32_t(k) == a.fixed, next_fixed = int32_t(k) + 1 == a.fixed;
    double H[36], C[36], g[6];
    for (int t = 0; t < 36; ++t) { H[t] = 0.0; C[t] = 0.0; }
    for (int t = 0; t < 6; ++t) g[t] = 0.0;
    if (!fixed) {
        for (int32_t q = a.inc[k]; q < a.inc[k + 1]; ++q) {
            const int32_t e = a.inc[a.n + 1 + q];
            const PgEdgeBlk& B = a.blk[e];
            const int32_t i = a.E[e].i, j = a.E[e].j;
            if (i == int32_t(k)) {
                for (int t = 0; t < 36; ++t) H[t] += B.aii[t];
                for (int t = 0; t < 6; ++t) g[t] += B.gi[t];
                if (j == int32_t(k) + 1 && !next_fixed) for (int t = 0; t < 36; ++t) C[t] += B.aij[t];
            } else {
                for (int t = 0; t < 36; ++t) H[t] += B.ajj[t];
                for (int t = 0; t < 6; ++t) g[t] += B.gj[t];
                if (i == int32_t(k) + 1 && !next_fixed)                   // A_{k,k+1} = A_ij^T with i = k + 1, j = k
                    for (int r = 0; r < 6; ++r) for (int c = 0; c < 6; ++c) C[r * 6 + c] += B.aij[c * 6 + r];
            }
        }
    }
    for (int t = 0; t < 36; ++t) { a.H[36 * size_t(k) + t] = H[t]; a.C[36 * size_t(k) + t] = C[t]; }
    for (int t = 0; t < 6; ++t) a.g[6 * size_t(k) + t] = g[t];
    if (a.init)                                                           // Jacobi scaling: 1 / (1 + |column of J|)
        for (int t = 0; t < 6; ++t) a.scale[6 * size_t(k) + t] = fixed ? 1.0 : 1.0 / (1.0 + sqrt(H[t * 7]));
    const double* xk = a.x + 7 * size_t(k);
    double x2 = 0.0;
    for (int t = 0; t < 7; ++t) x2 += xk[t] * xk[t];
    a.part[2 * size_t(k)] = fixed ? 0.0 : grad_max_norm(xk, g);
    a.part[2 * size_t(k) + 1] = fixed ? 0.0 : x2;
}

// Fixed-order reductions of one CTA: threads stride over the items, then a tree in shared memory
template <int T>
__device__ __forceinline__ double cta_sum(double v, double* sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = T / 2; o > 0; o >>= 1) {
        if (int(threadIdx.x) < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    const double r = sh[0];
    __syncthreads();
    return r;
}
template <int T>
__device__ __forceinline__ double cta_max(double v, double* sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = T / 2; o > 0; o >>= 1) {
        if (int(threadIdx.x) < o) sh[threadIdx.x] = fmax(sh[threadIdx.x], sh[threadIdx.x + o]);
        __syncthreads();
    }
    const double r = sh[0];
    __syncthreads();
    return r;
}

constexpr int kReduceThreads = 1024;
__global__ void __launch_bounds__(kReduceThreads) k_pg_reduce(const double* __restrict__ ecost, uint32_t m, const double* __restrict__ part,
                                                               uint32_t n, PgCtl* ctl, int set) {
    __shared__ double sh[kReduceThreads];
    double c = 0.0, gm = 0.0, x2 = 0.0;
    for (uint32_t e = threadIdx.x; e < m; e += kReduceThreads) c += ecost[e];
    for (uint32_t k = threadIdx.x; k < n; k += kReduceThreads) { gm = fmax(gm, part[2 * k]); x2 += part[2 * k + 1]; }
    c = cta_sum<kReduceThreads>(c, sh);
    gm = cta_max<kReduceThreads>(gm, sh);
    x2 = cta_sum<kReduceThreads>(x2, sh);
    if (threadIdx.x == 0) { ctl->cost[set] = c; ctl->gmax[set] = gm; ctl->xnorm2[set] = x2; }
}

// ------------------------------------------------------------------------------------------------------------------ the trial
// k_pg_trial is a cooperative kernel: every phase is spread over the grid (one thread per vector element, node or block row of a
// cyclic-reduction level) and the phases are separated by grid-wide barriers, so the PCG loop and its stopping test stay on the
// device.  Reductions are fixed-order: a tree per CTA, then every thread adds the CTA partials in CTA order, so every thread holds
// the same value and every loop decision is uniform across the grid.
struct PgTrialArgs {
    const so_pose_edge* E; const int32_t* inc; const PgEdgeBlk* blk;
    const double *x, *H, *C, *g;                                          // the iterate's set
    double* xc;                                                           // the candidate, into the other set
    double *scale, *diag, *dd;
    double *b, *y, *r, *z, *p, *q;
    double *crD, *crL, *crU, *crB;
    double* red;                                                          // [2][gridDim.x] CTA partials of the grid reductions
    PgCtl* ctl;
    uint32_t n; int32_t fixed, reuse_diagonal;
    double radius;
};

__device__ __forceinline__ uint32_t gtid() { return blockIdx.x * blockDim.x + threadIdx.x; }
__device__ __forceinline__ uint32_t gstride() { return gridDim.x * blockDim.x; }
__device__ __forceinline__ void gsync() { cg::this_grid().sync(); }

// Sum (max = false) or maximum (max = true) of v over the grid.  The partials alternate between the two halves of red: a half is
// written again only after the barrier of the reduction in between, which every thread reaches after reading it.
__device__ __noinline__ double grid_reduce(double v, bool max, double* sh, double* red, int& slot) {
    v = max ? cta_max<kTrialThreads>(v, sh) : cta_sum<kTrialThreads>(v, sh);
    double* r = red + size_t(slot) * gridDim.x;
    slot ^= 1;
    if (threadIdx.x == 0) r[blockIdx.x] = v;
    gsync();
    double s = 0.0;
    for (uint32_t k = 0; k < gridDim.x; ++k) s = max ? fmax(s, r[k]) : s + r[k];
    return s;
}

// q = (Hs + D^2) p over every node: its block, the chain blocks to k - 1 and k + 1, and the off-chain edges in incidence order
__device__ __noinline__ void pg_matvec(const PgTrialArgs& a, const double* p, double* q) {
    for (uint32_t k = gtid(); k < a.n; k += gstride()) {
        double y[6] = {0, 0, 0, 0, 0, 0}, sp[6];
        if (int32_t(k) == a.fixed) { for (int t = 0; t < 6; ++t) q[6 * k + t] = p[6 * k + t]; continue; }
        for (int t = 0; t < 6; ++t) sp[t] = a.scale[6 * k + t] * p[6 * k + t];
        mv6_add(a.H + 36 * size_t(k), sp, y, 1.0);
        if (k > 0) {
            for (int t = 0; t < 6; ++t) sp[t] = a.scale[6 * (k - 1) + t] * p[6 * (k - 1) + t];
            mtv6_add(a.C + 36 * size_t(k - 1), sp, y);
        }
        if (k + 1 < a.n) {
            for (int t = 0; t < 6; ++t) sp[t] = a.scale[6 * (k + 1) + t] * p[6 * (k + 1) + t];
            mv6_add(a.C + 36 * size_t(k), sp, y, 1.0);
        }
        for (int32_t w = a.inc[k]; w < a.inc[k + 1]; ++w) {
            const int32_t e = a.inc[a.n + 1 + w];
            const int32_t i = a.E[e].i, j = a.E[e].j;
            if (i - j == 1 || j - i == 1) continue;                       // in the chain blocks
            const int32_t o = i == int32_t(k) ? j : i;
            if (o == a.fixed) continue;
            for (int t = 0; t < 6; ++t) sp[t] = a.scale[6 * o + t] * p[6 * o + t];
            if (i == int32_t(k)) mv6_add(a.blk[e].aij, sp, y, 1.0);
            else mtv6_add(a.blk[e].aij, sp, y);
        }
        for (int t = 0; t < 6; ++t) q[6 * k + t] = a.scale[6 * k + t] * y[t] + a.dd[6 * k + t] * p[6 * k + t];
    }
}

// Cyclic-reduction storage: level l holds rows i = r 2^l, r < m_l = ceil(n / 2^l), at compact offset off_l + r
struct CrLevels {
    uint32_t m[33], off[33];
    int levels;                                                           // levels with m > 1; the last level (m == 1) follows
};
__device__ __forceinline__ CrLevels cr_levels(uint32_t n) {
    CrLevels L;
    uint32_t mm = n, off = 0;
    int l = 0;
    for (; mm > 1; ++l) { L.m[l] = mm; L.off[l] = off; off += mm; mm = (mm + 1) / 2; }
    L.m[l] = 1; L.off[l] = off;
    L.levels = l;
    return L;
}

// D^-1 of an SPD 6x6 by chol_solve<6> on the unit vectors; false on a non-positive pivot
__device__ __noinline__ bool inv6(const double* D, double* Dinv) {
    bool ok = true;
    for (int c = 0; c < 6; ++c) {
        double M[36], e[6], col[6];
        for (int t = 0; t < 36; ++t) M[t] = D[t];
        for (int t = 0; t < 6; ++t) e[t] = t == c ? 1.0 : 0.0;
        ok = chol_solve<6>(M, e, col) && ok;
        for (int t = 0; t < 6; ++t) Dinv[t * 6 + c] = col[t];
    }
    return ok;
}

// Factor: eliminated (odd) rows keep D^-1 (in crD), L, U; kept (even) rows keep W- = L D-^-1 and W+ = U D+^-1 (in crL, crU) and pass
// D' = D - W- U- - W+ L+, L' = -W- L-, U' = -W+ U+ to the next level.  The last level's single row keeps D^-1.  One thread per block
// row of a level.  Returns this thread's pivot failures (the caller reduces them over the grid).
__device__ __noinline__ double cr_factor(const PgTrialArgs& a, const CrLevels& L) {
    double bad = 0.0;
    for (int l = 0; l < L.levels; ++l) {
        const uint32_t m = L.m[l], o = L.off[l], o1 = L.off[l + 1];
        for (uint32_t r = 2 * gtid() + 1; r < m; r += 2 * gstride()) {
            double D[36], Di[36];
            for (int t = 0; t < 36; ++t) D[t] = a.crD[36 * size_t(o + r) + t];
            if (!inv6(D, Di)) bad = 1.0;
            for (int t = 0; t < 36; ++t) a.crD[36 * size_t(o + r) + t] = Di[t];
        }
        gsync();
        for (uint32_t r = 2 * gtid(); r < m; r += 2 * gstride()) {
            double D[36], W[36], T[36];                                   // L', U' go straight to the next level's slot
            const size_t d = 36 * size_t(o1 + r / 2);
            for (int t = 0; t < 36; ++t) D[t] = a.crD[36 * size_t(o + r) + t];
            if (r > 0) {
                mm6(a.crL + 36 * size_t(o + r), a.crD + 36 * size_t(o + r - 1), W);                // W- = L D-^-1
                mm6(W, a.crU + 36 * size_t(o + r - 1), T);
                for (int t = 0; t < 36; ++t) D[t] -= T[t];
                if (r >= 2) { mm6(W, a.crL + 36 * size_t(o + r - 1), T); for (int t = 0; t < 36; ++t) a.crL[d + t] = -T[t]; }
                else for (int t = 0; t < 36; ++t) a.crL[d + t] = 0.0;
                for (int t = 0; t < 36; ++t) a.crL[36 * size_t(o + r) + t] = W[t];
            } else {
                for (int t = 0; t < 36; ++t) a.crL[d + t] = 0.0;
            }
            if (r + 1 < m) {
                mm6(a.crU + 36 * size_t(o + r), a.crD + 36 * size_t(o + r + 1), W);                // W+ = U D+^-1
                mm6(W, a.crL + 36 * size_t(o + r + 1), T);
                for (int t = 0; t < 36; ++t) D[t] -= T[t];
                if (r + 2 < m) { mm6(W, a.crU + 36 * size_t(o + r + 1), T); for (int t = 0; t < 36; ++t) a.crU[d + t] = -T[t]; }
                else for (int t = 0; t < 36; ++t) a.crU[d + t] = 0.0;
                for (int t = 0; t < 36; ++t) a.crU[36 * size_t(o + r) + t] = W[t];
            } else {
                for (int t = 0; t < 36; ++t) a.crU[d + t] = 0.0;
            }
            for (int t = 0; t < 36; ++t) a.crD[d + t] = D[t];
        }
        gsync();
    }
    if (gtid() == 0) {
        double D[36], Di[36];
        const size_t d = 36 * size_t(L.off[L.levels]);
        for (int t = 0; t < 36; ++t) D[t] = a.crD[d + t];
        if (!inv6(D, Di)) bad = 1.0;
        for (int t = 0; t < 36; ++t) a.crD[d + t] = Di[t];
    }
    gsync();
    return bad;
}

// z = M^-1 v: one reduce sweep down the levels and one back-substitute sweep up them, one thread per block row of a level
__device__ __noinline__ void cr_apply(const PgTrialArgs& a, const CrLevels& L, const double* v, double* z) {
    for (uint32_t i = gtid(); i < 6 * a.n; i += gstride()) a.crB[i] = v[i];
    gsync();
    for (int l = 0; l < L.levels; ++l) {
        const uint32_t m = L.m[l], o = L.off[l], o1 = L.off[l + 1];
        for (uint32_t r = 2 * gtid(); r < m; r += 2 * gstride()) {
            double b[6];
            for (int t = 0; t < 6; ++t) b[t] = a.crB[6 * size_t(o + r) + t];
            if (r > 0) mv6_add(a.crL + 36 * size_t(o + r), a.crB + 6 * size_t(o + r - 1), b, -1.0);
            if (r + 1 < m) mv6_add(a.crU + 36 * size_t(o + r), a.crB + 6 * size_t(o + r + 1), b, -1.0);
            for (int t = 0; t < 6; ++t) a.crB[6 * size_t(o1 + r / 2) + t] = b[t];
        }
        gsync();
    }
    if (gtid() == 0) {
        const size_t o = L.off[L.levels];
        double b[6], x[6] = {0, 0, 0, 0, 0, 0};
        for (int t = 0; t < 6; ++t) b[t] = a.crB[6 * o + t];
        mv6_add(a.crD + 36 * o, b, x, 1.0);
        for (int t = 0; t < 6; ++t) a.crB[6 * o + t] = x[t];
    }
    gsync();
    for (int l = L.levels - 1; l >= 0; --l) {
        const uint32_t m = L.m[l], o = L.off[l], o1 = L.off[l + 1];
        for (uint32_t r = gtid(); r < m; r += gstride()) {
            double x[6];
            if (!(r & 1)) {
                for (int t = 0; t < 6; ++t) x[t] = a.crB[6 * size_t(o1 + r / 2) + t];
            } else {
                double b[6];
                for (int t = 0; t < 6; ++t) { b[t] = a.crB[6 * size_t(o + r) + t]; x[t] = 0.0; }
                mv6_add(a.crL + 36 * size_t(o + r), a.crB + 6 * size_t(o1 + (r - 1) / 2), b, -1.0);
                if (r + 1 < m) mv6_add(a.crU + 36 * size_t(o + r), a.crB + 6 * size_t(o1 + (r + 1) / 2), b, -1.0);
                mv6_add(a.crD + 36 * size_t(o + r), b, x, 1.0);
            }
            for (int t = 0; t < 6; ++t) a.crB[6 * size_t(o + r) + t] = x[t];
        }
        gsync();
    }
    for (uint32_t i = gtid(); i < 6 * a.n; i += gstride()) z[i] = a.crB[i];
    gsync();
}

__device__ __forceinline__ double grid_dot(const double* u, const double* v, uint32_t len, double* sh, double* red, int& slot) {
    double s = 0.0;
    for (uint32_t i = gtid(); i < len; i += gstride()) s += u[i] * v[i];
    return grid_reduce(s, false, sh, red, slot);
}

// One trust-region trial (LevenbergMarquardtStrategy::ComputeStep with PCG as the linear solver, then the candidate)
__global__ void __launch_bounds__(kTrialThreads) k_pg_trial(PgTrialArgs a) {
    __shared__ double sh[kTrialThreads];
    int slot = 0;
    const uint32_t n = a.n, len = 6 * n;
    // the LM diagonal of the scaled system (kept after a rejected step), and the damping diag / radius
    for (uint32_t i = gtid(); i < len; i += gstride()) {
        const uint32_t k = i / 6, t = i % 6;
        if (!a.reuse_diagonal) {
            const double s = a.scale[i];
            a.diag[i] = int32_t(k) == a.fixed ? 1.0 : fmin(fmax(s * s * a.H[36 * size_t(k) + t * 7], 1e-6), 1e32);
        }
        a.dd[i] = a.diag[i] / a.radius;
        a.b[i] = int32_t(k) == a.fixed ? 0.0 : a.scale[i] * a.g[i];       // gs
        a.y[i] = 0.0;
        a.r[i] = a.b[i];
    }
    gsync();
    // level 0 of the preconditioner: the block-tridiagonal part of Hs + D^2 (identity row, zero coupling at the fixed node)
    for (uint32_t k = gtid(); k < n; k += gstride()) {
        const double* s = a.scale + 6 * size_t(k);
        double* D = a.crD + 36 * size_t(k);
        double* Lo = a.crL + 36 * size_t(k);
        double* Up = a.crU + 36 * size_t(k);
        const bool fx = int32_t(k) == a.fixed;
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) {
                D[r * 6 + c] = fx ? (r == c ? 1.0 : 0.0) : s[r] * a.H[36 * size_t(k) + r * 6 + c] * s[c] + (r == c ? a.dd[6 * k + r] : 0.0);
                Lo[r * 6 + c] = (fx || k == 0) ? 0.0 : s[r] * a.C[36 * size_t(k - 1) + c * 6 + r] * a.scale[6 * (k - 1) + c];
                Up[r * 6 + c] = (fx || k + 1 >= n) ? 0.0 : s[r] * a.C[36 * size_t(k) + r * 6 + c] * a.scale[6 * (k + 1) + c];
            }
    }
    gsync();
    const CrLevels L = cr_levels(n);
    // a non-positive pivot anywhere (a direction no edge observes, at a damping rounding cannot resolve) invalidates the step for
    // every thread alike: the flag is reduced over the grid before it decides anything
    bool ok = grid_reduce(cr_factor(a, L), true, sh, a.red, slot) == 0.0;
    // PCG from y = 0
    cr_apply(a, L, a.r, a.z);
    for (uint32_t i = gtid(); i < len; i += gstride()) a.p[i] = a.z[i];
    double rz = grid_dot(a.r, a.z, len, sh, a.red, slot);                 // its barrier also orders the copy into p
    const double stop = kPcgTol * kPcgTol * rz;
    int it = 0;
    while (ok && rz > stop && it < kPcgMaxIter) {                         // rz, ok: the same in every thread
        pg_matvec(a, a.p, a.q);
        gsync();
        const double pq = grid_dot(a.p, a.q, len, sh, a.red, slot);
        if (!(pq > 0.0)) { ok = false; break; }
        const double alpha = rz / pq;
        for (uint32_t i = gtid(); i < len; i += gstride()) { a.y[i] += alpha * a.p[i]; a.r[i] -= alpha * a.q[i]; }
        gsync();
        cr_apply(a, L, a.r, a.z);
        const double rz1 = grid_dot(a.r, a.z, len, sh, a.red, slot);
        const double beta = rz1 / rz;
        for (uint32_t i = gtid(); i < len; i += gstride()) a.p[i] = a.z[i] + beta * a.p[i];
        gsync();
        rz = rz1;
        ++it;
    }
    // step = -y; model_cost_change = -step'gs - step'Hs step / 2 = y'gs - (y'(Hs + D^2)y - y'D^2 y) / 2
    pg_matvec(a, a.y, a.q);
    gsync();
    double fin = 1.0, ydy = 0.0, yg = 0.0, yay = 0.0;
    for (uint32_t i = gtid(); i < len; i += gstride()) {
        const double v = a.y[i];
        if (!isfinite(v)) fin = 0.0;
        ydy += a.dd[i] * v * v; yg += v * a.b[i]; yay += v * a.q[i];
    }
    fin = grid_reduce(1.0 - fin, true, sh, a.red, slot);
    ydy = grid_reduce(ydy, false, sh, a.red, slot);
    yg = grid_reduce(yg, false, sh, a.red, slot);
    yay = grid_reduce(yay, false, sh, a.red, slot);
    // the candidate: Plus(x_k, -y_k * scale_k) on the free nodes, and |x - candidate|^2
    double sn = 0.0;
    for (uint32_t k = gtid(); k < n; k += gstride()) {
        const double* xk = a.x + 7 * size_t(k);
        double* ck = a.xc + 7 * size_t(k);
        if (int32_t(k) == a.fixed) { for (int t = 0; t < 7; ++t) ck[t] = xk[t]; continue; }
        double d[6], o[7];
        for (int t = 0; t < 6; ++t) d[t] = -a.y[6 * k + t] * a.scale[6 * k + t];
        pose_plus(xk, d, o);
        for (int t = 0; t < 7; ++t) { ck[t] = o[t]; sn += (xk[t] - o[t]) * (xk[t] - o[t]); }
    }
    sn = grid_reduce(sn, false, sh, a.red, slot);
    if (gtid() == 0) {
        a.ctl->mcc = yg - 0.5 * (yay - ydy);
        a.ctl->step_norm2 = sn;
        a.ctl->valid = ok && fin == 0.0;
        a.ctl->pcg_iters = it;
    }
}

// ------------------------------------------------------------------------------------------------------------------ host
static bool finite_quat(const double* p) {
    for (int k = 0; k < 7; ++k) if (!std::isfinite(p[k])) return false;
    return p[3] * p[3] + p[4] * p[4] + p[5] * p[5] + p[6] * p[6] > 0.0;
}

static int graph_check(size_t n, const so_pose_edge* edges, size_t m, const so_pose_graph_opts& o) {
    if (n < 2) return fail(SO_ERR_ARG, "so_pose_graph: at least two nodes");
    if (n >= (size_t(1) << 27) || m >= (size_t(1) << 28)) return fail(SO_ERR_ARG, "so_pose_graph: too many nodes or edges");
    if (m && !edges) return fail(SO_ERR_ARG, "so_pose_graph: NULL edges");
    if (o.fixed < 0 || size_t(o.fixed) >= n) return fail(SO_ERR_ARG, "so_pose_graph: fixed node out of range");
    if (o.max_iterations < 0) return fail(SO_ERR_ARG, "so_pose_graph: max_iterations < 0");
    std::vector<int32_t> parent(n);
    for (size_t k = 0; k < n; ++k) parent[k] = int32_t(k);
    auto root = [&](int32_t v) { while (parent[v] != v) { parent[v] = parent[parent[v]]; v = parent[v]; } return v; };
    for (size_t e = 0; e < m; ++e) {
        const so_pose_edge& E = edges[e];
        const std::string at = " (edge " + std::to_string(e) + ")";
        if (E.i < 0 || E.j < 0 || size_t(E.i) >= n || size_t(E.j) >= n) return fail(SO_ERR_ARG, "so_pose_graph: edge node id out of range" + at);
        if (E.i == E.j) return fail(SO_ERR_ARG, "so_pose_graph: edge with i == j" + at);
        if (!finite_quat(E.z)) return fail(SO_ERR_ARG, "so_pose_graph: edge measurement z not finite or with a zero-norm quaternion" + at);
        for (int k = 0; k < 36; ++k)
            if (!std::isfinite(E.sqrt_info[k])) return fail(SO_ERR_ARG, "so_pose_graph: sqrt_info not finite" + at);
        if (!std::isfinite(E.cauchy) || E.cauchy < 0.0) return fail(SO_ERR_ARG, "so_pose_graph: cauchy must be finite and >= 0" + at);
        parent[root(E.i)] = root(E.j);
    }
    const int32_t rf = root(o.fixed);
    for (size_t k = 0; k < n; ++k)
        if (root(int32_t(k)) != rf) return fail(SO_ERR_ARG, "so_pose_graph: node " + std::to_string(k) + " is not connected to the fixed node");
    return SO_OK;
}

static void pg_defaults(so_pose_graph_opts* o) { o->fixed = 0; o->max_iterations = 50; }

static int pg_reserve(Ctx* c, size_t n, size_t m) {
    Ctx::Pg& g = c->pg;
    size_t T = 0;
    for (size_t mm = n; ; mm = (mm + 1) / 2) { T += mm; if (mm == 1) break; }
    int rc = g.d_edges.reserve(m);
    if (!rc) rc = g.d_inc.reserve(n + 1 + 2 * m);
    for (int s = 0; s < 2 && !rc; ++s) {
        rc = g.d_x[s].reserve(7 * n);
        if (!rc) rc = g.d_blk[s].reserve(std::max<size_t>(m, 1));
        if (!rc) rc = g.d_ecost[s].reserve(std::max<size_t>(m, 1));
        if (!rc) rc = g.d_w[s].reserve(std::max<size_t>(m, 1));
        if (!rc) rc = g.d_H[s].reserve(36 * n);
        if (!rc) rc = g.d_C[s].reserve(36 * n);
        if (!rc) rc = g.d_g[s].reserve(6 * n);
    }
    if (!rc) rc = g.d_scale.reserve(6 * n);
    if (!rc) rc = g.d_diag.reserve(6 * n);
    if (!rc) rc = g.d_dd.reserve(6 * n);
    if (!rc) rc = g.d_vec.reserve(6 * 6 * n);
    if (!rc) rc = g.d_crD.reserve(36 * T);
    if (!rc) rc = g.d_crL.reserve(36 * T);
    if (!rc) rc = g.d_crU.reserve(36 * T);
    if (!rc) rc = g.d_crB.reserve(6 * T);
    if (!rc && !g.max_blocks) {                                       // co-resident CTAs of the cooperative trial kernel
        int dev = 0, sms = 0, per_sm = 0, coop = 0;
        SO_CUDA_TRY(cudaGetDevice(&dev));
        SO_CUDA_TRY(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
        if (!coop) return fail(SO_ERR_CUDA, "so_pose_graph_solve: the device has no cooperative launch");
        SO_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        SO_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pg_trial, kTrialThreads, 0));
        if (per_sm < 1) return fail(SO_ERR_CUDA, "so_pose_graph_solve: the trial kernel does not fit on a multiprocessor");
        g.max_blocks = sms * per_sm;
    }
    if (!rc) rc = g.d_red.reserve(2 * size_t(std::max(g.max_blocks, 1)));
    if (!rc) rc = g.d_ctl.reserve(1);
    if (!rc) rc = g.h_ctl.reserve(1);
    if (!rc && !(cudaEvent_t)g.ev[0]) { rc = g.ev[0].create(); if (!rc) rc = g.ev[1].create(); }
    return rc;
}

// The linearisation of set s at d_x[s]: edges, nodes, the fixed-order reductions into ctl
static void pg_linearise(Ctx* c, uint32_t n, uint32_t m, int32_t fixed, int s, bool init, double* part) {
    Ctx::Pg& g = c->pg;
    if (m) k_pg_edges<<<(m + 127) / 128, 128, 0, c->stream>>>(g.d_edges, m, g.d_x[s], g.d_blk[s], g.d_ecost[s], g.d_w[s]);
    PgNodeArgs na{g.d_edges, g.d_inc, g.d_blk[s], g.d_x[s], g.d_H[s], g.d_C[s], g.d_g[s], g.d_scale, part, n, fixed, init ? 1 : 0};
    k_pg_nodes<<<(n + 127) / 128, 128, 0, c->stream>>>(na);
    k_pg_reduce<<<1, kReduceThreads, 0, c->stream>>>(g.d_ecost[s], m, part, n, g.d_ctl, s);
    c->launches += m ? 3 : 2;
}

static int pg_solve(Ctx* c, const double* init7, uint32_t n, const so_pose_edge* edges, uint32_t m, const so_pose_graph_opts& o,
                    double* out7, double* weights, so_pose_graph_result* res) {
    Ctx::Pg& g = c->pg;
    int rc = pg_reserve(c, n, m);
    if (rc) return rc;
    // every quaternion normalised; the incidence lists by a counting sort over the edges in id order
    std::vector<double> x(init7, init7 + 7 * size_t(n));
    for (uint32_t k = 0; k < n; ++k) {
        double* q = x.data() + 7 * size_t(k) + 3;
        const double s = 1.0 / std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        for (int t = 0; t < 4; ++t) q[t] *= s;
    }
    std::vector<so_pose_edge> E(edges, edges + m);
    for (so_pose_edge& e : E) {
        const double s = 1.0 / std::sqrt(e.z[3] * e.z[3] + e.z[4] * e.z[4] + e.z[5] * e.z[5] + e.z[6] * e.z[6]);
        for (int t = 3; t < 7; ++t) e.z[t] *= s;
    }
    std::vector<int32_t> inc(n + 1 + 2 * size_t(m), 0);
    for (const so_pose_edge& e : E) { inc[e.i + 1]++; inc[e.j + 1]++; }
    for (uint32_t k = 0; k < n; ++k) inc[k + 1] += inc[k];
    {
        std::vector<int32_t> at(inc.begin(), inc.begin() + n);
        for (uint32_t e = 0; e < m; ++e) { inc[n + 1 + at[E[e].i]++] = int32_t(e); inc[n + 1 + at[E[e].j]++] = int32_t(e); }
    }
    double* part = g.d_vec + 5 * 6 * size_t(n);                          // q's slot doubles as the node partials of a linearisation
    SO_CUDA_TRY(cudaEventRecord(g.ev[0], c->stream));
    if (m) SO_CUDA_TRY(cudaMemcpyAsync(g.d_edges, E.data(), m * sizeof(so_pose_edge), cudaMemcpyHostToDevice, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(g.d_inc, inc.data(), inc.size() * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(g.d_x[0], x.data(), x.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    count_h2d(c, m * sizeof(so_pose_edge) + inc.size() * sizeof(int32_t) + x.size() * sizeof(double));
    int cur = 0;
    pg_linearise(c, n, m, o.fixed, cur, true, part);
    SO_CUDA_TRY(cudaGetLastError());
    PgCtl& h = *g.h_ctl;
    SO_CUDA_TRY(cudaMemcpyAsync(g.h_ctl, g.d_ctl, sizeof(PgCtl), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    // TrustRegionMinimizer: the rules of so_trust_region.cuh (tr_start, tr_continue, tr_after_eval), restated over the kernels above
    so_pose_graph_result r{};
    double cost = h.cost[cur], gmax = h.gmax[cur], x_norm = std::sqrt(h.xnorm2[cur]);
    r.initial_cost = cost;
    double radius = 1e4, decrease = 2.0;
    bool reuse = false, step_ok = false;
    int invalid = 0, term = 0;
    PgTrialArgs ta{};
    ta.E = g.d_edges; ta.inc = g.d_inc;
    ta.scale = g.d_scale; ta.diag = g.d_diag; ta.dd = g.d_dd;
    double* v = g.d_vec;
    const size_t len = 6 * size_t(n);
    ta.b = v; ta.y = v + len; ta.r = v + 2 * len; ta.z = v + 3 * len; ta.p = v + 4 * len; ta.q = v + 5 * len;
    ta.crD = g.d_crD; ta.crL = g.d_crL; ta.crU = g.d_crU; ta.crB = g.d_crB;
    ta.ctl = g.d_ctl; ta.n = n; ta.fixed = o.fixed; ta.red = g.d_red;
    // one thread per node, at most the co-resident CTAs; a function of n and the device only, so the reductions' order is fixed
    const uint32_t blocks = std::max<uint32_t>(1, std::min<uint32_t>(uint32_t(g.max_blocks), (n + kTrialThreads - 1) / kTrialThreads));
    for (;;) {
        if (step_ok) r.successful++; else r.unsuccessful++;
        if (r.iterations >= o.max_iterations) { term = 0; break; }
        if (gmax <= 1e-10) { term = 1; break; }
        if (radius <= 1e-32) { term = 4; break; }
        r.iterations++;
        step_ok = false;
        ta.blk = g.d_blk[cur]; ta.x = g.d_x[cur]; ta.H = g.d_H[cur]; ta.C = g.d_C[cur]; ta.g = g.d_g[cur];
        ta.xc = g.d_x[1 - cur];
        ta.reuse_diagonal = reuse ? 1 : 0;
        ta.radius = radius;
        reuse = true;
        {
            void* args[] = {&ta};
            SO_CUDA_TRY(cudaLaunchCooperativeKernel((const void*)k_pg_trial, dim3(blocks), dim3(kTrialThreads), args, 0, c->stream));
        }
        c->launches++;
        pg_linearise(c, n, m, o.fixed, 1 - cur, false, part);            // the candidate in full: an accepted step needs no second pass
        SO_CUDA_TRY(cudaGetLastError());
        SO_CUDA_TRY(cudaMemcpyAsync(g.h_ctl, g.d_ctl, sizeof(PgCtl), cudaMemcpyDeviceToHost, c->stream));
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
        r.pcg_iterations += uint64_t(h.pcg_iters);
        const double mcc = h.mcc;
        if (!h.valid || !(mcc > 0.0)) {                                   // HandleInvalidStep
            if (++invalid >= 5) { term = 5; break; }
            radius *= 0.5;
            continue;
        }
        invalid = 0;
        const double cand_cost = h.cost[1 - cur];
        if (std::sqrt(h.step_norm2) <= 1e-8 * (x_norm + 1e-8)) { term = 2; break; }       // ParameterToleranceReached
        const double change = cost - cand_cost;
        if (std::fabs(change) <= 1e-6 * cost) { term = 3; break; }                          // FunctionToleranceReached
        const double rd = change / mcc;
        if (rd > 1e-3) {                                                  // HandleSuccessfulStep
            cur = 1 - cur;
            cost = cand_cost; gmax = h.gmax[cur]; x_norm = std::sqrt(h.xnorm2[cur]);
            const double t = 2.0 * rd - 1.0;
            radius = std::fmin(1e16, radius / std::fmax(1.0 / 3.0, 1.0 - t * t * t));
            decrease = 2.0; reuse = false;
            step_ok = true;
        } else {                                                          // StepRejected
            radius = radius / decrease; decrease *= 2.0; reuse = true;
        }
    }
    SO_CUDA_TRY(cudaMemcpyAsync(x.data(), g.d_x[cur], x.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (weights && m) SO_CUDA_TRY(cudaMemcpyAsync(weights, g.d_w[cur], m * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaEventRecord(g.ev[1], c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    count_d2h(c, x.size() * sizeof(double) + (weights ? m * sizeof(double) : 0));
    float ms = 0.f;
    SO_CUDA_TRY(cudaEventElapsedTime(&ms, g.ev[0], g.ev[1]));
    std::memcpy(out7, x.data(), x.size() * sizeof(double));
    r.termination = term;
    r.final_cost = cost; r.gmax = gmax; r.radius = radius;
    r.time_ms = ms;
    if (res) *res = r;
    return SO_OK;
}

}  // namespace so

// =================================================================================================== C ABI
using namespace so;

extern "C" {

void so_pose_graph_opts_defaults(so_pose_graph_opts* opts) { if (opts) pg_defaults(opts); }

int so_pose_graph_check(size_t n_nodes, const so_pose_edge* edges, size_t n_edges, const so_pose_graph_opts* opts) {
    so_pose_graph_opts o;
    pg_defaults(&o);
    if (opts) o = *opts;
    return graph_check(n_nodes, edges, n_edges, o);
}

int so_pose_graph_solve(so_ctx* ctx, const double* init7, size_t n_nodes, const so_pose_edge* edges, size_t n_edges,
                        const so_pose_graph_opts* opts, double* out7, double* edge_weights, so_pose_graph_result* result) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !init7 || !out7) return fail(SO_ERR_ARG, "so_pose_graph_solve: NULL ctx, init7 or out7");
    so_pose_graph_opts o;
    pg_defaults(&o);
    if (opts) o = *opts;
    { int rc = graph_check(n_nodes, edges, n_edges, o); if (rc) return rc; }
    for (size_t k = 0; k < n_nodes; ++k)
        if (!finite_quat(init7 + 7 * k)) return fail(SO_ERR_ARG, "so_pose_graph_solve: init pose " + std::to_string(k) + " not finite or with a zero-norm quaternion");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    return pg_solve(c, init7, uint32_t(n_nodes), edges, uint32_t(n_edges), o, out7, edge_weights, result);
}

}  // extern "C"

// =============================================================================
// so_oracle.cpp -- CPU ORACLE for the SuperOdom per-scan ICP registration path.
//
// TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may load this library.  The product
// (superodom_b200/) never links, imports or calls it.
//
// What it is: a line-by-line restatement, in dependency-free C++17, of the
// reference's LidarSLAM::performLocalizationAndMapping path
//   /root/reference/super_odometry/src/LidarProcess/LidarSlam.cpp:107-152 (+ callees)
// plus the third-party arithmetic that path calls and that is NOT vendored in
// /root/reference:
//   * Ceres Solver 2.0.0 (apt libceres-dev on osrf/ros:humble, Dockerfile:4,43):
//     trust-region Levenberg-Marquardt minimizer, DENSE_QR, TukeyLoss, ScaledLoss,
//     loss Corrector, Covariance(DENSE_SVD) -- restated from the published
//     algorithm (ceres-solver 2.0.0: internal/ceres/trust_region_minimizer.cc,
//     levenberg_marquardt_strategy.cc, trust_region_step_evaluator.cc,
//     dense_qr_solver.cc, corrector.cc, loss_function.cc, covariance_impl.cc).
//   * Eigen 3.4.0: SelfAdjointEigenSolver<Matrix3d>, colPivHouseholderQr,
//     Quaternion ops -- restated (results are algorithm-independent to ~1e-15).
//   * tf2 Matrix3x3::getRPY / Quaternion::setRPY (MannualYawCorrection).
//
// PARITY PINNING: the reference ships no tests, golden vectors or fixtures
// (SURVEY.md section 4) => the Ceres/Eigen side of this oracle is "parity unpinned".
// The k-NN side IS pinned: when built with -DSO_ORACLE_WITH_REF_OCTREE (the
// oracle/_ref build, see oracle/Makefile) the reference's own
// include/super_odometry/flann/{octree.h,nanoflann.h} are compiled verbatim from
// /root/reference and used as knn mode 2; tests compare modes 0/1/2.
// =============================================================================
#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <memory>
#include <thread>
#include <vector>

#ifdef SO_ORACLE_WITH_REF_OCTREE
#include "super_odometry/flann/octree.h"   // verbatim reference header (via -I/root/reference/...)
#endif

namespace orc {

// ----------------------------------------------------------------------------- constants
// LocalMap.h:131-138
static constexpr int kW = 21, kH = 21, kD = 11, kNumBlocks = kW * kH * kD;
static constexpr double kBlock = 50.0, kHalfBlock = 25.0;

// LidarSlam.h:85-94 MatchingResult
enum { SUCCESS = 0, NOT_ENOUGH_NEIGHBORS = 1, NEIGHBORS_TOO_FAR = 2, BAD_PCA_STRUCTURE = 3,
       INVALID_NUMERICAL = 4, MSE_TOO_LARGE = 5, UNKNOWN = 6, N_REJ = 7 };

struct Pt { float x, y, z; };

// ----------------------------------------------------------------------------- small linear algebra
// Symmetric eigen decomposition, n<=6: Householder tridiagonalisation + implicit QL (the
// same family of algorithm as Eigen::SelfAdjointEigenSolver).  a is row-major n*n (symmetric),
// on return w ascending, v row-major with eigenvectors in COLUMNS (v[i*n+k] = component i of vector k).
static void sym_eig(int n, const double* a_in, double* w, double* v) {
    double a[36], d[6], e[6];
    for (int i = 0; i < n * n; ++i) a[i] = a_in[i];
    auto A = [&](int i, int j) -> double& { return a[i * n + j]; };
    // tred2
    for (int i = n - 1; i > 0; --i) {
        int l = i - 1;
        double h = 0.0, scale = 0.0;
        if (l > 0) {
            for (int k = 0; k <= l; ++k) scale += std::fabs(A(i, k));
            if (scale == 0.0) e[i] = A(i, l);
            else {
                for (int k = 0; k <= l; ++k) { A(i, k) /= scale; h += A(i, k) * A(i, k); }
                double f = A(i, l);
                double g = (f >= 0.0 ? -std::sqrt(h) : std::sqrt(h));
                e[i] = scale * g; h -= f * g; A(i, l) = f - g; f = 0.0;
                for (int j = 0; j <= l; ++j) {
                    A(j, i) = A(i, j) / h;
                    g = 0.0;
                    for (int k = 0; k <= j; ++k) g += A(j, k) * A(i, k);
                    for (int k = j + 1; k <= l; ++k) g += A(k, j) * A(i, k);
                    e[j] = g / h; f += e[j] * A(i, j);
                }
                double hh = f / (h + h);
                for (int j = 0; j <= l; ++j) {
                    f = A(i, j); e[j] = g = e[j] - hh * f;
                    for (int k = 0; k <= j; ++k) A(j, k) -= (f * e[k] + g * A(i, k));
                }
            }
        } else e[i] = A(i, l);
        d[i] = h;
    }
    d[0] = 0.0; e[0] = 0.0;
    for (int i = 0; i < n; ++i) {
        int l = i - 1;
        if (d[i] != 0.0) {
            for (int j = 0; j <= l; ++j) {
                double g = 0.0;
                for (int k = 0; k <= l; ++k) g += A(i, k) * A(k, j);
                for (int k = 0; k <= l; ++k) A(k, j) -= g * A(k, i);
            }
        }
        d[i] = A(i, i); A(i, i) = 1.0;
        for (int j = 0; j <= l; ++j) A(j, i) = A(i, j) = 0.0;
    }
    // tqli
    for (int i = 1; i < n; ++i) e[i - 1] = e[i];
    e[n - 1] = 0.0;
    for (int l = 0; l < n; ++l) {
        int iter = 0, m;
        do {
            for (m = l; m < n - 1; ++m) {
                double dd = std::fabs(d[m]) + std::fabs(d[m + 1]);
                if (std::fabs(e[m]) <= std::numeric_limits<double>::epsilon() * dd) break;
            }
            if (m != l) {
                if (iter++ == 60) break;
                double g = (d[l + 1] - d[l]) / (2.0 * e[l]);
                double r = std::hypot(g, 1.0);
                g = d[m] - d[l] + e[l] / (g + (g >= 0.0 ? std::fabs(r) : -std::fabs(r)));
                double s = 1.0, c = 1.0, p = 0.0;
                int i;
                for (i = m - 1; i >= l; --i) {
                    double f = s * e[i], b = c * e[i];
                    e[i + 1] = (r = std::hypot(f, g));
                    if (r == 0.0) { d[i + 1] -= p; e[m] = 0.0; break; }
                    s = f / r; c = g / r; g = d[i + 1] - p;
                    r = (d[i] - g) * s + 2.0 * c * b;
                    d[i + 1] = g + (p = s * r); g = c * r - b;
                    for (int k = 0; k < n; ++k) {
                        f = A(k, i + 1);
                        A(k, i + 1) = s * A(k, i) + c * f;
                        A(k, i) = c * A(k, i) - s * f;
                    }
                }
                if (r == 0.0 && i >= l) continue;
                d[l] -= p; e[l] = g; e[m] = 0.0;
            }
        } while (m != l);
    }
    // sort ascending
    int idx[6];
    for (int i = 0; i < n; ++i) idx[i] = i;
    std::sort(idx, idx + n, [&](int x, int y) { return d[x] < d[y]; });
    for (int k = 0; k < n; ++k) {
        w[k] = d[idx[k]];
        for (int i = 0; i < n; ++i) v[i * n + k] = A(i, idx[k]);
    }
}

// Eigen::ColPivHouseholderQR<Matrix<double,5,3>>::solve restated (Eigen 3.4 ColPivHouseholderQR.h):
// greedy max-remaining-column-norm pivoting, Householder reflectors, rank by |R_ii| > maxpivot*eps*3,
// minimum-norm-on-truncation solve.  A row-major [m x 3], b [m].  Returns x[3].
static void colpiv_qr_solve(int m, const double* A_in, const double* b_in, double* x) {
    const int n = 3;
    double A[8 * 3], b[8];
    for (int i = 0; i < m * n; ++i) A[i] = A_in[i];
    for (int i = 0; i < m; ++i) b[i] = b_in[i];
    int perm[3] = {0, 1, 2};
    double maxpivot = 0.0;
    int nonzero_pivots = n;
    double rdiag[3] = {0, 0, 0};
    double colnorm2[3];
    for (int j = 0; j < n; ++j) { double s = 0; for (int i = 0; i < m; ++i) s += A[i * n + j] * A[i * n + j]; colnorm2[j] = s; }
    double maxn = std::max(colnorm2[0], std::max(colnorm2[1], colnorm2[2]));
    const double thresh_helper = maxn * std::numeric_limits<double>::epsilon() * std::numeric_limits<double>::epsilon() / double(m);
    for (int k = 0; k < n; ++k) {
        // remaining column norms (recomputed exactly; Eigen down-dates, same pivot choice up to rounding)
        int piv = k; double best = -1.0;
        for (int j = k; j < n; ++j) {
            double s = 0; for (int i = k; i < m; ++i) s += A[i * n + j] * A[i * n + j];
            if (s > best) { best = s; piv = j; }
        }
        if (nonzero_pivots == n && best < thresh_helper * double(m - k)) nonzero_pivots = k;
        if (piv != k) { for (int i = 0; i < m; ++i) std::swap(A[i * n + k], A[i * n + piv]); std::swap(perm[k], perm[piv]); }
        // Householder on column k, rows k..m-1 (Eigen makeHouseholderInPlace)
        double c0 = A[k * n + k];
        double tail2 = 0; for (int i = k + 1; i < m; ++i) tail2 += A[i * n + k] * A[i * n + k];
        double beta, tau;
        double ess[8];
        if (tail2 <= std::numeric_limits<double>::min()) {
            tau = 0.0; beta = c0;
            for (int i = k + 1; i < m; ++i) ess[i] = 0.0;
        } else {
            beta = std::sqrt(c0 * c0 + tail2);
            if (c0 >= 0.0) beta = -beta;
            for (int i = k + 1; i < m; ++i) ess[i] = A[i * n + k] / (c0 - beta);
            tau = (beta - c0) / beta;
        }
        // apply H = I - tau * v v^T (v = [1; ess]) to remaining columns and to b
        for (int j = k + 1; j < n; ++j) {
            double s = A[k * n + j];
            for (int i = k + 1; i < m; ++i) s += ess[i] * A[i * n + j];
            s *= tau;
            A[k * n + j] -= s;
            for (int i = k + 1; i < m; ++i) A[i * n + j] -= s * ess[i];
        }
        {
            double s = b[k];
            for (int i = k + 1; i < m; ++i) s += ess[i] * b[i];
            s *= tau;
            b[k] -= s;
            for (int i = k + 1; i < m; ++i) b[i] -= s * ess[i];
        }
        A[k * n + k] = beta;
        for (int i = k + 1; i < m; ++i) A[i * n + k] = 0.0;
        rdiag[k] = beta;
        if (std::fabs(beta) > maxpivot) maxpivot = std::fabs(beta);
    }
    // rank (ColPivHouseholderQR::rank with default threshold eps*diagonalSize)
    const double premult = std::fabs(maxpivot) * std::numeric_limits<double>::epsilon() * double(std::min(m, n));
    int rank = 0;
    for (int i = 0; i < nonzero_pivots; ++i) rank += (std::fabs(rdiag[i]) > premult);
    double y[3] = {0, 0, 0};
    for (int i = rank - 1; i >= 0; --i) {
        double s = b[i];
        for (int j = i + 1; j < rank; ++j) s -= A[i * n + j] * y[j];
        y[i] = s / A[i * n + i];
    }
    for (int i = 0; i < n; ++i) x[perm[i]] = (i < rank ? y[i] : 0.0);
}

// Unpivoted Householder QR least squares (Eigen::HouseholderQR::solve as used by Ceres
// DenseQRSolver, dense_qr_solver.cc): min || A y - b ||, A column-major [m x n] (destroyed).
// If R_out != nullptr the n x n upper-triangular factor is written row-major.
static void householder_ls(int m, int n, double* A, double* b, double* y, double* R_out) {
    auto a = [&](int i, int j) -> double& { return A[size_t(j) * m + i]; };
    for (int k = 0; k < n; ++k) {
        double c0 = a(k, k), tail2 = 0.0;
        for (int i = k + 1; i < m; ++i) tail2 += a(i, k) * a(i, k);
        double beta, tau;
        if (tail2 <= std::numeric_limits<double>::min()) { tau = 0.0; beta = c0; for (int i = k + 1; i < m; ++i) a(i, k) = 0.0; }
        else {
            beta = std::sqrt(c0 * c0 + tail2); if (c0 >= 0.0) beta = -beta;
            const double inv = 1.0 / (c0 - beta);
            for (int i = k + 1; i < m; ++i) a(i, k) *= inv;
            tau = (beta - c0) / beta;
        }
        for (int j = k + 1; j < n; ++j) {
            double s = a(k, j);
            for (int i = k + 1; i < m; ++i) s += a(i, k) * a(i, j);
            s *= tau; a(k, j) -= s;
            for (int i = k + 1; i < m; ++i) a(i, j) -= s * a(i, k);
        }
        if (b) {
            double s = b[k];
            for (int i = k + 1; i < m; ++i) s += a(i, k) * b[i];
            s *= tau; b[k] -= s;
            for (int i = k + 1; i < m; ++i) b[i] -= s * a(i, k);
        }
        a(k, k) = beta;
    }
    if (R_out) for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) R_out[i * n + j] = (j >= i ? a(i, j) : 0.0);
    if (y) for (int i = n - 1; i >= 0; --i) {
        double s = b[i];
        for (int j = i + 1; j < n; ++j) s -= a(i, j) * y[j];
        y[i] = s / a(i, i);
    }
}

// One-sided Jacobi SVD of a small square matrix R (row-major n x n): R = U S V^T.
// Returns singular values descending in s and V (row-major, vectors in columns).
static void jacobi_svd(int n, const double* R, double* s, double* V) {
    double U[36];
    for (int i = 0; i < n * n; ++i) U[i] = R[i];
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) V[i * n + j] = (i == j);
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < n - 1; ++p) for (int q = p + 1; q < n; ++q) {
            double alpha = 0, beta = 0, gamma = 0;
            for (int i = 0; i < n; ++i) { alpha += U[i * n + p] * U[i * n + p]; beta += U[i * n + q] * U[i * n + q]; gamma += U[i * n + p] * U[i * n + q]; }
            if (gamma == 0.0) continue;
            off = std::max(off, std::fabs(gamma) / std::sqrt(alpha * beta));
            double zeta = (beta - alpha) / (2.0 * gamma);
            double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
            double c = 1.0 / std::sqrt(1.0 + t * t), sn = c * t;
            for (int i = 0; i < n; ++i) {
                double up = U[i * n + p], uq = U[i * n + q];
                U[i * n + p] = c * up - sn * uq; U[i * n + q] = sn * up + c * uq;
                double vp = V[i * n + p], vq = V[i * n + q];
                V[i * n + p] = c * vp - sn * vq; V[i * n + q] = sn * vp + c * vq;
            }
        }
        if (off < 1e-15) break;
    }
    double sv[6]; int idx[6];
    for (int j = 0; j < n; ++j) { double t = 0; for (int i = 0; i < n; ++i) t += U[i * n + j] * U[i * n + j]; sv[j] = std::sqrt(t); idx[j] = j; }
    std::sort(idx, idx + n, [&](int a, int b) { return sv[a] > sv[b]; });
    double Vs[36];
    for (int k = 0; k < n; ++k) { s[k] = sv[idx[k]]; for (int i = 0; i < n; ++i) Vs[i * n + k] = V[i * n + idx[k]]; }
    for (int i = 0; i < n * n; ++i) V[i] = Vs[i];
}

// ----------------------------------------------------------------------------- quaternion / pose (pose7 = tx,ty,tz,qx,qy,qz,qw; LidarSlam.cpp:7-9)
struct Quat { double x, y, z, w; };
static inline Quat qmul(const Quat& a, const Quat& b) {   // Eigen quaternion product
    return Quat{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
                a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
                a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x,
                a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
static inline Quat qnormalized(const Quat& q) {
    double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    if (n2 > 0) { double s = 1.0 / std::sqrt(n2); return Quat{q.x * s, q.y * s, q.z * s, q.w * s}; }
    return q;
}
static inline Quat qconj(const Quat& q) { return Quat{-q.x, -q.y, -q.z, q.w}; }
// Eigen QuaternionBase::_transformVector: v + 2w (q x v) + 2 q x (q x v)
static inline void qrot(const Quat& q, const double v[3], double out[3]) {
    double ux = q.y * v[2] - q.z * v[1], uy = q.z * v[0] - q.x * v[2], uz = q.x * v[1] - q.y * v[0];
    ux += ux; uy += uy; uz += uz;
    out[0] = v[0] + q.w * ux + (q.y * uz - q.z * uy);
    out[1] = v[1] + q.w * uy + (q.z * ux - q.x * uz);
    out[2] = v[2] + q.w * uz + (q.x * uy - q.y * ux);
}
static inline void qtoR(const Quat& q, double R[9]) {   // Eigen toRotationMatrix
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
// PoseLocalParameterization::Plus (pose_local_parameterization.cpp:7-22) + Utility::deltaQ (utility.h:11-24)
static inline void pose_plus(const double x[7], const double d[6], double out[7]) {
    out[0] = x[0] + d[0]; out[1] = x[1] + d[1]; out[2] = x[2] + d[2];
    Quat q{x[3], x[4], x[5], x[6]}, dq{d[3] / 2.0, d[4] / 2.0, d[5] / 2.0, 1.0};
    Quat r = qnormalized(qmul(q, dq));
    out[3] = r.x; out[4] = r.y; out[5] = r.z; out[6] = r.w;
}
// relative motion a^-1 * b -> (|t|, angle) as used by recordIterationStats / updateOptimizationStats
// (LidarSlam.cpp:198-210,242-251; Twist.h:172-187)
static inline void rel_motion(const double a[7], const double b[7], double* trans, double* rot) {
    Quat qa{a[3], a[4], a[5], a[6]}, qb{b[3], b[4], b[5], b[6]};
    Quat qi = qconj(qa);
    double dt[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, t[3];
    qrot(qi, dt, t);
    Quat r = qmul(qi, qb);
    *trans = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    *rot = 2.0 * std::atan2(std::sqrt(r.x * r.x + r.y * r.y + r.z * r.z), r.w);
}

// ----------------------------------------------------------------------------- map
static inline int block_coord(double v_plus_half, int origin) {     // LocalMap.h:488-497
    int c = int(v_plus_half / kBlock) + origin;
    if (v_plus_half < 0) c--;
    return c;
}
static inline int block_of(float x, float y, float z, const int o[3]) {
    int i = block_coord(double(x) + kHalfBlock, o[0]);
    int j = block_coord(double(y) + kHalfBlock, o[1]);
    int k = block_coord(double(z) + kHalfBlock, o[2]);
    if (!(i >= 0 && i < kW && j >= 0 && j < kH && k >= 0 && k < kD)) return -1;
    return i + kW * j + kW * kH * k;
}

// octree.h:95-102: float diff, std::pow(float,int) -> double, sum in double, return float
static inline float l2_ref(const Pt& a, const Pt& b) {
    float d1 = a.x - b.x, d2 = a.y - b.y, d3 = a.z - b.z;
    return float(double(d1) * double(d1) + double(d2) * double(d2) + double(d3) * double(d3));
}

// KNNResult (nanoflann.h:72-155) restated: ascending, stable for ties (first seen first).
struct Knn {
    int k, count = 0; int64_t* idx; float* d;
    Knn(int k_, int64_t* i_, float* d_) : k(k_), idx(i_), d(d_) { d[k - 1] = std::numeric_limits<float>::max(); }
    inline void add(float dist, int64_t id) {
        int i;
        for (i = count; i > 0; --i) {
            if (d[i - 1] > dist) { if (i < k) { d[i] = d[i - 1]; idx[i] = idx[i - 1]; } }
            else break;
        }
        if (i < k) { d[i] = dist; idx[i] = id; }
        if (count < k) count++;
    }
    inline float worst() const { return d[k - 1]; }
    inline bool full() const { return count == k; }
};

struct BlockData {
    std::vector<Pt> pts;            // block cloud in insertion order (psurf_pc_)
    std::vector<int64_t> gid;       // index into the caller's input array
    // acceleration grid for mode 0 (exact): cells of edge `cs` over the block's bbox
    float bmin[3]; int dim[3]; float cs = 1.0f;
    std::vector<uint32_t> cell_start; std::vector<uint32_t> cell_pts;
#ifdef SO_ORACLE_WITH_REF_OCTREE
    std::unique_ptr<nanoflann::Octree<Pt, std::vector<Pt>>> octree;
#endif
    void build_grid() {
        const size_t n = pts.size();
        float mn[3] = {pts[0].x, pts[0].y, pts[0].z}, mx[3] = {pts[0].x, pts[0].y, pts[0].z};
        for (auto& p : pts) { mn[0] = std::min(mn[0], p.x); mn[1] = std::min(mn[1], p.y); mn[2] = std::min(mn[2], p.z);
                              mx[0] = std::max(mx[0], p.x); mx[1] = std::max(mx[1], p.y); mx[2] = std::max(mx[2], p.z); }
        cs = 0.5f; size_t nc = 1;
        for (int a = 0; a < 3; ++a) { bmin[a] = mn[a]; dim[a] = int((mx[a] - mn[a]) / cs) + 1; nc *= size_t(dim[a]); }
        cell_start.assign(nc + 1, 0); cell_pts.resize(n);
        std::vector<uint32_t> c(n);
        for (size_t i = 0; i < n; ++i) { c[i] = cell_of(pts[i]); cell_start[c[i] + 1]++; }
        for (size_t i = 0; i < nc; ++i) cell_start[i + 1] += cell_start[i];
        std::vector<uint32_t> cur(cell_start.begin(), cell_start.end() - 1);
        for (size_t i = 0; i < n; ++i) cell_pts[cur[c[i]]++] = uint32_t(i);   // ascending index inside a cell
    }
    inline void cell_xyz(const Pt& p, int c[3]) const {
        c[0] = std::min(dim[0] - 1, std::max(0, int((p.x - bmin[0]) / cs)));
        c[1] = std::min(dim[1] - 1, std::max(0, int((p.y - bmin[1]) / cs)));
        c[2] = std::min(dim[2] - 1, std::max(0, int((p.z - bmin[2]) / cs)));
    }
    inline uint32_t cell_of(const Pt& p) const { int c[3]; cell_xyz(p, c); return uint32_t((c[2] * dim[1] + c[1]) * dim[0] + c[0]); }
};

struct Map {
    int origin[3] = {kW / 2, kH / 2, kD / 2};     // LocalMap() ctor: (10,10,5)
    std::vector<std::unique_ptr<BlockData>> blocks;   // surf clouds: kNumBlocks entries, null if empty
    std::vector<std::unique_ptr<BlockData>> eblocks;  // edge clouds (pedge_pc_ / pkdtree_edge_from_block_)
    Map() : blocks(kNumBlocks), eblocks(kNumBlocks) {}
};

// Exact k-NN inside one block with tie-break (d2, index) ascending == brute force scanning the block
// cloud in index order with KNNResult semantics.
static bool knn_exact(const BlockData& B, const Pt& q, int k, int64_t* idx, float* d2) {
    const size_t n = B.pts.size();
    std::vector<std::pair<float, uint32_t>> cand;
    int c[3]; B.cell_xyz(q, c);
    // distance from q to its (clamped) cell -- q may lie outside the block bbox
    for (int ring = 0;; ++ring) {
        const int lo[3] = {c[0] - ring, c[1] - ring, c[2] - ring}, hi[3] = {c[0] + ring, c[1] + ring, c[2] + ring};
        for (int z = std::max(0, lo[2]); z <= std::min(B.dim[2] - 1, hi[2]); ++z)
            for (int y = std::max(0, lo[1]); y <= std::min(B.dim[1] - 1, hi[1]); ++y)
                for (int x = std::max(0, lo[0]); x <= std::min(B.dim[0] - 1, hi[0]); ++x) {
                    if (ring > 0 && x != lo[0] && x != hi[0] && y != lo[1] && y != hi[1] && z != lo[2] && z != hi[2]) continue;
                    const uint32_t cid = uint32_t((z * B.dim[1] + y) * B.dim[0] + x);
                    for (uint32_t t = B.cell_start[cid]; t < B.cell_start[cid + 1]; ++t) {
                        const uint32_t i = B.cell_pts[t];
                        cand.emplace_back(l2_ref(q, B.pts[i]), i);
                    }
                }
        const bool covers_all = lo[0] <= 0 && lo[1] <= 0 && lo[2] <= 0 && hi[0] >= B.dim[0] - 1 && hi[1] >= B.dim[1] - 1 && hi[2] >= B.dim[2] - 1;
        if (int(cand.size()) >= k || covers_all) {
            std::sort(cand.begin(), cand.end());
            if (covers_all) break;
            // every unvisited point is farther than the visited shell's inner boundary
            const double kth = int(cand.size()) >= k ? double(cand[k - 1].first) : std::numeric_limits<double>::infinity();
            double reach = std::numeric_limits<double>::infinity();   // min distance from q to outside of visited box
            const float qq[3] = {q.x, q.y, q.z};
            for (int a = 0; a < 3; ++a) {
                if (lo[a] > 0) reach = std::min(reach, double(qq[a]) - (double(B.bmin[a]) + double(lo[a]) * double(B.cs)));
                if (hi[a] < B.dim[a] - 1) reach = std::min(reach, (double(B.bmin[a]) + double(hi[a] + 1) * double(B.cs)) - double(qq[a]));
            }
            if (reach > 0 && kth < reach * reach * 0.999) break;
        }
    }
    (void)n;
    for (int j = 0; j < k; ++j) {
        if (j < int(cand.size())) { idx[j] = cand[j].second; d2[j] = cand[j].first; }
        else { idx[j] = 0; d2[j] = 0.f; }       // unfilled slots keep index 0 / dist 0 (LocalMap.h:516-517)
    }
    return int(cand.size()) >= k;
}
static bool knn_brute(const BlockData& B, const Pt& q, int k, int64_t* idx, float* d2) {
    for (int j = 0; j < k; ++j) { idx[j] = 0; d2[j] = 0.f; }
    Knn r(k, idx, d2);
    for (size_t i = 0; i < B.pts.size(); ++i) r.add(l2_ref(q, B.pts[i]), int64_t(i));
    return r.full();
}

// LocalMap::nearestKSearchSurf (LocalMap.h:481-525).  mode 0 exact(grid) 1 brute 2 reference octree.
// idx are BLOCK-LOCAL indices; *blk receives the block or nullptr.
static bool nearest_k_surf(const Map& M, const Pt& q, int k, int mode, int64_t* idx, float* d2, const BlockData** blk) {
    *blk = nullptr;
    const int b = block_of(q.x, q.y, q.z, M.origin);
    if (b < 0) return false;
    const BlockData* B = M.blocks[b].get();
    if (!B) return false;                 // pkdtree_surf_from_block_ == nullptr
    *blk = B;
    if (mode == 2) {
#ifdef SO_ORACLE_WITH_REF_OCTREE
        std::vector<size_t> ind(k, 0);
        std::vector<float> dd(k, 0.f);
        B->octree->template knnNeighbors<nanoflann::L2Distance<Pt>>(q, size_t(k), ind.data(), dd.data());
        for (int j = 0; j < k; ++j) { idx[j] = int64_t(ind[j]); d2[j] = dd[j]; }
        return true;
#else
        return false;
#endif
    }
    if (mode == 1) knn_brute(*B, q, k, idx, d2); else knn_exact(*B, q, k, idx, d2);
    return true;
}

// ----------------------------------------------------------------------------- correspondence (SURVEY Appendix A)
struct Corr {
    double p[3];        // Xvalue = pInit
    double n[3];        // NormDir (QR normal, unit, unflipped)
    double d;           // negative_OA_dot_norm
    double w;           // residualCoefficient
    double eigval[3];   // PCA eigenvalues ascending
    double mean_dist;   // "meanSquareDist" (mean abs distance)
    int64_t nn[5];      // neighbour ids (caller's input index)
    float nn_d2[5];
    int32_t status;     // MatchingResult; -1 = skipped by sampling
    int32_t obs[3];     // observability labels histogrammed (LidarSlam.cpp:336-339)
};

// LidarSLAM::ComputePlaneDistanceParameters (LidarSlam.cpp:514-572)
static void plane_correspondence(const Map& M, const float* sp, const double pose[7], float planeRes, int knn_mode, Corr& out) {
    std::memset(&out, 0, sizeof(out));
    for (int j = 0; j < 5; ++j) out.nn[j] = -1;
    // ComputePointInitAndFinalPose (:382-400): pInit = double(p); pFinal = T_w_lidar * pInit
    const Quat q{pose[3], pose[4], pose[5], pose[6]};
    const double pin[3] = {double(sp[0]), double(sp[1]), double(sp[2])};
    double pf[3]; qrot(q, pin, pf); pf[0] += pose[0]; pf[1] += pose[1]; pf[2] += pose[2];
    out.p[0] = pin[0]; out.p[1] = pin[1]; out.p[2] = pin[2];
    const double square_max_dist = double(3 * planeRes);      // :526, float product widened
    // findNearestNeighbors (:720-747)
    Pt qf{float(pf[0]), float(pf[1]), float(pf[2])};
    int64_t idx[5]; float d2[5]; const BlockData* B;
    bool found = nearest_k_surf(M, qf, 5, knn_mode, idx, d2, &B);
    // "<k points in the block" -> NOT_ENOUGH_NEIGHBORS (SURVEY Appendix C; reference would use index-0 duplicates)
    if (!found || B->pts.size() < 5) { out.status = NOT_ENOUGH_NEIGHBORS; return; }
    for (int j = 0; j < 5; ++j) { out.nn[j] = B->gid[idx[j]]; out.nn_d2[j] = d2[j]; }
    if (double(d2[4]) > square_max_dist) { out.status = NEIGHBORS_TOO_FAR; return; }
    // computePCAForFeature (:749-790) + utils::ComputePCA (superodom_utils.h:143-151)
    double m[5][3], mean[3] = {0, 0, 0};
    for (int j = 0; j < 5; ++j) { const Pt& a = B->pts[idx[j]]; m[j][0] = a.x; m[j][1] = a.y; m[j][2] = a.z; }
    for (int j = 0; j < 5; ++j) for (int a = 0; a < 3; ++a) mean[a] += m[j][a];
    for (int a = 0; a < 3; ++a) mean[a] /= 5.0;
    double S[9] = {0};
    for (int j = 0; j < 5; ++j) {
        const double c[3] = {m[j][0] - mean[0], m[j][1] - mean[1], m[j][2] - mean[2]};
        for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) S[a * 3 + b] += c[a] * c[b];
    }
    double ev[3], V[9];
    sym_eig(3, S, ev, V);
    out.eigval[0] = ev[0]; out.eigval[1] = ev[1]; out.eigval[2] = ev[2];
    if (ev[0] < 1e-6 || ev[1] / ev[2] < 0.1) { out.status = BAD_PCA_STRUCTURE; return; }
    // computePlaneQualityMetrics (:792-844)
    double A[15], bneg[5] = {-1, -1, -1, -1, -1}, nrm[3];
    for (int j = 0; j < 5; ++j) for (int a = 0; a < 3; ++a) A[j * 3 + a] = m[j][a];
    colpiv_qr_solve(5, A, bneg, nrm);
    if (!(std::isfinite(nrm[0]) && std::isfinite(nrm[1]) && std::isfinite(nrm[2]))) { out.status = INVALID_NUMERICAL; return; }
    const double nn = std::sqrt(nrm[0] * nrm[0] + nrm[1] * nrm[1] + nrm[2] * nrm[2]);
    const double d = 1.0 / nn;
    nrm[0] /= nn; nrm[1] /= nn; nrm[2] /= nn;
    double mean_dist = 0.0;
    const double max_point_distance = planeRes / 2.0;
    for (int j = 0; j < 5; ++j) {
        const double dist = std::fabs(nrm[0] * m[j][0] + nrm[1] * m[j][1] + nrm[2] * m[j][2] + d);
        if (dist > max_point_distance) { out.status = MSE_TOO_LARGE; return; }
        mean_dist += dist;
    }
    mean_dist /= 5.0;
    // normal direction check (:553-561) on the PCA normal
    double nobs[3] = {V[0], V[3], V[6]};
    if (pf[0] * nobs[0] + pf[1] * nobs[1] + pf[2] * nobs[2] < 0) { nobs[0] = -nobs[0]; nobs[1] = -nobs[1]; nobs[2] = -nobs[2]; }
    // FeatureObservabilityAnalysis (:574-693)
    const double l1 = std::sqrt(ev[2]), l2 = std::sqrt(ev[1]), l3 = std::sqrt(ev[0]);
    const double planar_2 = (l2 - l3) / l1;
    const float nf[3] = {float(nobs[0]), float(nobs[1]), float(nobs[2])};
    const float ptf[3] = {float(pf[0]), float(pf[1]), float(pf[2])};          // pcl::PointNormal is float
    const float cross[3] = {ptf[1] * nf[2] - ptf[2] * nf[1], ptf[2] * nf[0] - ptf[0] * nf[2], ptf[0] * nf[1] - ptf[1] * nf[0]};
    // computeRotatedAxes (:624-638): float quaternion * unit axes (Eigen _transformVector in float)
    const float qx = float(pose[3]), qy = float(pose[4]), qz = float(pose[5]), qw = float(pose[6]);
    float axes[3][3];
    for (int a = 0; a < 3; ++a) {
        const float v[3] = {a == 0 ? 1.f : 0.f, a == 1 ? 1.f : 0.f, a == 2 ? 1.f : 0.f};
        float ux = qy * v[2] - qz * v[1], uy = qz * v[0] - qx * v[2], uz = qx * v[1] - qy * v[0];
        ux += ux; uy += uy; uz += uz;
        axes[a][0] = v[0] + qw * ux + (qy * uz - qz * uy);
        axes[a][1] = v[1] + qw * uy + (qz * ux - qx * uz);
        axes[a][2] = v[2] + qw * uz + (qx * uy - qy * ux);
    }
    float rotq[6], trq[3];
    for (int a = 0; a < 3; ++a) {
        // Eigen's unrolled 3-vector dot associates as a0*b0 + (a1*b1 + a2*b2); result stored in a double member
        const double rc = double(cross[0] * axes[a][0] + (cross[1] * axes[a][1] + cross[2] * axes[a][2]));
        rotq[2 * a] = float(rc); rotq[2 * a + 1] = float(-rc);
    }
    const float planar_sq = float(planar_2 * planar_2);
    for (int a = 0; a < 3; ++a) trq[a] = float(double(planar_sq * std::fabs(nf[0] * axes[a][0] + (nf[1] * axes[a][1] + nf[2] * axes[a][2]))));
    // std::sort descending on <= 16 elements == insertion sort == stable: top-2 rot labels, top-1 trans label
    int r0 = 0; for (int i = 1; i < 6; ++i) if (rotq[i] > rotq[r0]) r0 = i;
    int r1 = -1; for (int i = 0; i < 6; ++i) { if (i == r0) continue; if (r1 < 0 || rotq[i] > rotq[r1]) r1 = i; }
    int t0 = 0; for (int i = 1; i < 3; ++i) if (trq[i] > trq[t0]) t0 = i;
    out.obs[0] = r0; out.obs[1] = r1; out.obs[2] = 6 + t0;
    // setPlaneResults (:695-708)
    out.n[0] = nrm[0]; out.n[1] = nrm[1]; out.n[2] = nrm[2]; out.d = d;
    out.mean_dist = mean_dist;
    out.w = 1.0 - std::sqrt(mean_dist / square_max_dist);      // :568
    out.status = SUCCESS;
}

// ----------------------------------------------------------------------------- edge / line branch (dormant upstream: the edge cloud is always empty)
struct EdgeCorr {
    double p[3];        // Xvalue = pInit
    double a[3], b[3];  // corres = (mean + 0.1 dir, mean - 0.1 dir)
    double w;           // residualCoefficient
    int64_t nn[10];     // the 10 nearest edge points (caller's input index)
    int32_t sel[10];    // positions in nn[] of the points kept by the best-line selection (closest first), -1 padded
    int32_t n_sel;
    int32_t status;
};

// LocalMap::nearestKSearchSpecificEdgePoint (LocalMap.h:377-474) + ComputeLineDistanceParameters (LidarSlam.cpp:402-435)
// + processLineResults (:438-493).
static void line_correspondence(const Map& M, const float* sp, const double pose[7], float lineRes, int knn_mode, EdgeCorr& out) {
    std::memset(&out, 0, sizeof(out));
    for (int j = 0; j < 10; ++j) { out.nn[j] = -1; out.sel[j] = -1; }
    const Quat q{pose[3], pose[4], pose[5], pose[6]};
    const double pin[3] = {double(sp[0]), double(sp[1]), double(sp[2])};
    double pf[3]; qrot(q, pin, pf); pf[0] += pose[0]; pf[1] += pose[1]; pf[2] += pose[2];
    out.p[0] = pin[0]; out.p[1] = pin[1]; out.p[2] = pin[2];
    const Pt qf{float(pf[0]), float(pf[1]), float(pf[2])};
    const int bl = block_of(qf.x, qf.y, qf.z, M.origin);
    const BlockData* B = bl >= 0 ? M.eblocks[bl].get() : nullptr;
    // "<k points in the block": the reference indexes with size_t(-1) (UB, LocalMap.h:404-419); treated as NOT_ENOUGH_NEIGHBORS
    if (!B || B->pts.size() < 10) { out.status = NOT_ENOUGH_NEIGHBORS; return; }
    int64_t idx[10]; float d2[10];
    if (knn_mode == 1) knn_brute(*B, qf, 10, idx, d2); else knn_exact(*B, qf, 10, idx, d2);
    for (int j = 0; j < 10; ++j) out.nn[j] = B->gid[idx[j]];
    // best line through the closest point by inlier count (float arithmetic, Eigen's evaluation order)
    const Pt& P1 = B->pts[idx[0]];
    const float thr = 0.2f * 0.2f;                       // LocalizationLineMaxDistInlier^2 (LidarSlam.h:280), static_cast<float>
    int best = -1; size_t best_n = 0; bool best_in[10] = {false};
    for (int pi = 1; pi < 10; ++pi) {
        const Pt& P2 = B->pts[idx[pi]];
        float dx = P2.x - P1.x, dy = P2.y - P1.y, dz = P2.z - P1.z;
        const float z2 = dx * dx + (dy * dy + dz * dz);                        // Vector3f::squaredNorm
        if (z2 > 0.f) { const float s = std::sqrt(z2); dx /= s; dy /= s; dz /= s; }   // normalized(): zero vector stays zero
        bool in[10] = {false}; size_t cnt = 0;
        for (int ci = 1; ci < 10; ++ci) {
            bool ok;
            if (ci == pi) ok = true;
            else {
                const Pt& Pc = B->pts[idx[ci]];
                const float vx = Pc.x - P1.x, vy = Pc.y - P1.y, vz = Pc.z - P1.z;
                const float cx = vy * dz - vz * dy, cy = vz * dx - vx * dz, cz = vx * dy - vy * dx;
                ok = (cx * cx + (cy * cy + cz * cz)) < thr;
            }
            in[ci] = ok; cnt += ok;
        }
        if (cnt > best_n) { best_n = cnt; best = pi; for (int ci = 0; ci < 10; ++ci) best_in[ci] = in[ci]; }
    }
    (void)best;
    int sel[10], ns = 0;
    sel[ns++] = 0;
    for (int ci = 1; ci < 10; ++ci) if (best_in[ci]) sel[ns++] = ci;
    out.n_sel = ns;
    for (int j = 0; j < ns; ++j) out.sel[j] = sel[j];
    // validateNeighborSearch (:495-512)
    if (ns < 4) { out.status = NOT_ENOUGH_NEIGHBORS; return; }
    if (d2[sel[ns - 1]] > 3 * lineRes) { out.status = NEIGHBORS_TOO_FAR; return; }      // float compare
    // computePCAForFeature, EdgeFeature branch (:749-790)
    double m[10][3], mean[3] = {0, 0, 0};
    for (int j = 0; j < ns; ++j) { const Pt& a = B->pts[idx[sel[j]]]; m[j][0] = a.x; m[j][1] = a.y; m[j][2] = a.z; }
    for (int j = 0; j < ns; ++j) for (int a = 0; a < 3; ++a) mean[a] += m[j][a];
    for (int a = 0; a < 3; ++a) mean[a] /= double(ns);
    double S[9] = {0};
    for (int j = 0; j < ns; ++j) {
        const double c[3] = {m[j][0] - mean[0], m[j][1] - mean[1], m[j][2] - mean[2]};
        for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) S[a * 3 + b] += c[a] * c[b];
    }
    double ev[3], V[9];
    sym_eig(3, S, ev, V);
    if (!(std::isfinite(ev[0]) && std::isfinite(ev[1]) && std::isfinite(ev[2]))) { out.status = INVALID_NUMERICAL; return; }
    if (ev[2] < 4.0 * ev[1]) { out.status = BAD_PCA_STRUCTURE; return; }                 // LocalizationMinmumLineNeighborRejection * ev1
    // processLineResults (:438-493)
    double dir[3] = {V[2], V[5], V[8]};
    const double dn = std::sqrt(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
    dir[0] /= dn; dir[1] /= dn; dir[2] /= dn;
    double A[9];
    for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) A[a * 3 + b] = (a == b ? 1.0 : 0.0) - dir[a] * dir[b];
    for (int i = 0; i < 9; ++i) if (!std::isfinite(A[i])) { out.status = INVALID_NUMERICAL; return; }
    double msd = 0.0;
    const double lim = double(3 * lineRes);
    for (int j = 0; j < ns; ++j) {
        const double c[3] = {m[j][0] - mean[0], m[j][1] - mean[1], m[j][2] - mean[2]};
        double Ac[3]; for (int a = 0; a < 3; ++a) Ac[a] = A[a * 3] * c[0] + A[a * 3 + 1] * c[1] + A[a * 3 + 2] * c[2];
        const double sd = c[0] * Ac[0] + c[1] * Ac[1] + c[2] * Ac[2];
        if (sd > lim) { out.status = MSE_TOO_LARGE; return; }
        msd += sd;
    }
    msd /= double(ns);
    out.w = 1.0 - std::sqrt(msd / lim);
    for (int a = 0; a < 3; ++a) { out.a[a] = 0.1 * dir[a] + mean[a]; out.b[a] = -0.1 * dir[a] + mean[a]; }
    out.status = SUCCESS;
}

// EdgeAnalyticCostFunction::Evaluate (lidarOptimization.cpp:12-47): r = ((lp-a) x (lp-b)) / |a-b|, J = skew(b-a) [I, -R [p]x] / |a-b|
static inline void edge_residual(const EdgeCorr& c, const double x[7], const double R[9], double r[3], double J[18]) {
    Quat q{x[3], x[4], x[5], x[6]};
    double lp[3]; qrot(q, c.p, lp); lp[0] += x[0]; lp[1] += x[1]; lp[2] += x[2];
    const double u[3] = {lp[0] - c.a[0], lp[1] - c.a[1], lp[2] - c.a[2]}, v[3] = {lp[0] - c.b[0], lp[1] - c.b[1], lp[2] - c.b[2]};
    const double de[3] = {c.a[0] - c.b[0], c.a[1] - c.b[1], c.a[2] - c.b[2]};
    const double den = std::sqrt(de[0] * de[0] + de[1] * de[1] + de[2] * de[2]);
    r[0] = (u[1] * v[2] - u[2] * v[1]) / den; r[1] = (u[2] * v[0] - u[0] * v[2]) / den; r[2] = (u[0] * v[1] - u[1] * v[0]) / den;
    if (!J) return;
    const double re[3] = {-de[0], -de[1], -de[2]};      // b - a
    const double K[9] = {0, -re[2], re[1], re[2], 0, -re[0], -re[1], re[0], 0};     // skew(re)
    // dp_by_so3 = [I, -R skew(p)]
    const double* p = c.p;
    const double Sp[9] = {0, -p[2], p[1], p[2], 0, -p[0], -p[1], p[0], 0};
    double RS[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double t = 0; for (int k = 0; k < 3; ++k) t += R[i * 3 + k] * Sp[k * 3 + j]; RS[i * 3 + j] = -t; }
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
        J[i * 6 + j] = K[i * 3 + j] / den;
        double t = 0; for (int k = 0; k < 3; ++k) t += K[i * 3 + k] * RS[k * 3 + j];
        J[i * 6 + 3 + j] = t / den;
    }
}

// shouldProcessPoint (LidarSlam.cpp:346-359)
static inline bool should_process(size_t i, double rate) {
    if (rate < 0.0) return true;
    double rem = std::fmod(double(i) * rate, 1.0);
    return !(rem + 0.001 > rate);
}

// processPlannerFeatures (:323-344) over the whole scan; corr[i].status = -1 for points skipped by sampling.
static void correspond_all(const Map& M, const float* scan, size_t n, size_t stride, const double pose[7], float planeRes,
                           int max_surface_features, int knn_mode, int n_threads, Corr* corr, int32_t hist_obs[9], int32_t hist_rej[7]) {
    double rate = -1.0;
    if (max_surface_features > 0 && n > size_t(max_surface_features)) rate = 1.0 * max_surface_features / double(n);
    auto work = [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; ++i) {
            if (!should_process(i, rate)) { std::memset(&corr[i], 0, sizeof(Corr)); corr[i].status = -1; continue; }
            plane_correspondence(M, scan + i * stride, pose, planeRes, knn_mode, corr[i]);
        }
    };
    if (n_threads <= 1) work(0, n);
    else {
        std::vector<std::thread> th;
        size_t chunk = (n + n_threads - 1) / n_threads;
        for (int t = 0; t < n_threads; ++t) { size_t lo = t * chunk, hi = std::min(n, lo + chunk); if (lo < hi) th.emplace_back(work, lo, hi); }
        for (auto& t : th) t.join();
    }
    for (int i = 0; i < 9; ++i) hist_obs[i] = 0;
    for (int i = 0; i < 7; ++i) hist_rej[i] = 0;
    for (size_t i = 0; i < n; ++i) {
        if (corr[i].status < 0) continue;
        if (corr[i].status == SUCCESS) { hist_obs[corr[i].obs[0]]++; hist_obs[corr[i].obs[1]]++; hist_obs[corr[i].obs[2]]++; }
        hist_rej[corr[i].status]++;
    }
}

// ----------------------------------------------------------------------------- residual / loss (Ceres 2.0.0 semantics)
// SE3AbsolutatePoseFactor (factor/SE3AbsolutatePoseFactor.{h,cpp}) as added by addAbsolutePoseConstraints
// (LidarSlam.cpp:285-298): 6 residuals [p - p_meas ; 2 vec(q_meas^* q)] premultiplied by sqrt_information, no loss function.
// The information matrix is diagonal; sqrt_information = LLT(information).matrixL().transpose() -- Eigen's unblocked LLT
// stops at the first non-positive pivot and leaves that and all later diagonal entries as they were (NOT square-rooted).
struct PosePrior {
    bool on = false;
    double meas[7];
    double sqrt_info[6];
    void set_information(const double info[6]) {
        bool failed = false;
        for (int k = 0; k < 6; ++k) {
            if (!failed && info[k] <= 0.0) failed = true;
            sqrt_info[k] = failed ? info[k] : std::sqrt(info[k]);
        }
    }
    // residual (6) and local Jacobian (6x6, row-major) at pose x
    void eval(const double x[7], double r[6], double J[36]) const {
        const Quat qm{meas[3], meas[4], meas[5], meas[6]}, q{x[3], x[4], x[5], x[6]};
        const Quat e = qmul(qconj(qm), q);
        r[0] = x[0] - meas[0]; r[1] = x[1] - meas[1]; r[2] = x[2] - meas[2];
        r[3] = 2.0 * e.x; r[4] = 2.0 * e.y; r[5] = 2.0 * e.z;
        for (int i = 0; i < 36; ++i) J[i] = 0.0;
        J[0] = J[7] = J[14] = 1.0;
        // Utility::Qleft(q_meas^* q).bottomRightCorner<3,3>() = w I + [v]x   (utils/utility.h:47-55)
        J[3 * 6 + 3] = e.w;  J[3 * 6 + 4] = -e.z; J[3 * 6 + 5] = e.y;
        J[4 * 6 + 3] = e.z;  J[4 * 6 + 4] = e.w;  J[4 * 6 + 5] = -e.x;
        J[5 * 6 + 3] = -e.y; J[5 * 6 + 4] = e.x;  J[5 * 6 + 5] = e.w;
        for (int i = 0; i < 6; ++i) { r[i] *= sqrt_info[i]; for (int j = 0; j < 6; ++j) J[i * 6 + j] *= sqrt_info[i]; }
    }
};

// addAbsolutePoseConstraints (LidarSlam.cpp:285-298): the information diagonal from features_corres.size() = good
static void set_pose_prior(PosePrior& P, const double meas[7], int good, float visual_confidence_factor, const float prior_uncertainty[3]) {
    const double vcf = double(visual_confidence_factor);
    double info[6];
    for (int a = 0; a < 3; ++a) info[a] = (1 - double(prior_uncertainty[a])) * std::max(50, int(good * 0.1)) * vcf;
    info[3] = info[4] = std::max(10, int(good * 0.01)) * vcf;
    info[5] = std::max(5, int(good * 0.001)) * 0;
    P.on = true;
    std::memcpy(P.meas, meas, sizeof(P.meas));
    P.set_information(info);
}

struct Evaluator {
    std::vector<const EdgeCorr*> edges; // accepted edge correspondences (added BEFORE the planes, LidarSlam.cpp:304-307)
    double a2_line = 0;                 // Tukey a^2 for edges, a = double(sqrtf(3*lineRes)) (LidarSlam.cpp:263)
    std::vector<const Corr*> blocks;    // accepted correspondences in scan order
    PosePrior prior;                    // optional 6 extra residual rows (after the plane blocks, as the reference adds it)
    double a2;                          // Tukey a^2, a = double(sqrtf(3*planeRes)) (LidarSlam.cpp:271)
    // TukeyLoss::Evaluate (ceres 2.0.0 loss_function.cc) wrapped by ScaledLoss(w)
    inline void rho(double s, double w, double r[3]) const { rho_a(s, w, a2, r); }
    size_t rows() const { return blocks.size() + 3 * edges.size() + (prior.on ? 6 : 0); }
    bool empty() const { return blocks.empty() && edges.empty() && !prior.on; }
    static inline void rho_a(double s, double w, double a2, double r[3]) {
        if (s <= a2) { const double v = 1.0 - s / a2, v2 = v * v; r[0] = a2 / 6.0 * (1.0 - v2 * v); r[1] = 0.5 * v2; r[2] = -1.0 / a2 * v; }
        else { r[0] = a2 / 6.0; r[1] = 0.0; r[2] = 0.0; }
        r[0] *= w; r[1] *= w; r[2] *= w;
    }
    // SurfNormAnalyticCostFunction::Evaluate (lidarOptimization.cpp:55-80): residual only
    static inline double residual(const Corr& c, const double x[7]) {
        Quat q{x[3], x[4], x[5], x[6]};
        double pw[3]; qrot(q, c.p, pw);
        pw[0] += x[0]; pw[1] += x[1]; pw[2] += x[2];
        return c.n[0] * pw[0] + c.n[1] * pw[1] + c.n[2] * pw[2] + c.d;
    }
    // cost only: 0.5 * sum rho[0]  (ResidualBlock::Evaluate, residual_block.cc)
    double cost(const double x[7]) const {
        double c = 0.0;
        for (const Corr* b : blocks) { double r = residual(*b, x), rr[3]; rho(r * r, b->w, rr); c += 0.5 * rr[0]; }
        for (const EdgeCorr* e : edges) { double r[3], rr[3]; edge_residual(*e, x, nullptr, r, nullptr); rho_a(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], e->w, a2_line, rr); c += 0.5 * rr[0]; }
        if (prior.on) { double r[6], J[36]; prior.eval(x, r, J); double sq = 0; for (int i = 0; i < 6; ++i) sq += r[i] * r[i]; c += 0.5 * sq; }
        return c;
    }
    // full: corrected residuals, corrected local Jacobian (column-major n x 6), gradient, cost.
    // Tukey has rho'' <= 0 everywhere => Corrector takes the "rho[2] <= 0" branch: both r and J scaled by sqrt(rho') (corrector.cc).
    void full(const double x[7], double* cost_out, std::vector<double>& res, std::vector<double>& J, double g[6]) const {
        const size_t np = blocks.size(), ne = edges.size();
        const size_t n = np + 3 * ne + (prior.on ? 6 : 0);          // rows: planes, then 3 per edge, then the prior (order is immaterial to the sums)
        res.resize(n); J.resize(n * 6);
        Quat q{x[3], x[4], x[5], x[6]};
        double R[9]; qtoR(q, R);
        double c = 0.0;
        for (int j = 0; j < 6; ++j) g[j] = 0.0;
        if (prior.on) {
            double r[6], Jp[36]; prior.eval(x, r, Jp);
            for (int i = 0; i < 6; ++i) {
                res[np + 3 * ne + i] = r[i]; c += 0.5 * r[i] * r[i];
                for (int j = 0; j < 6; ++j) { J[size_t(j) * n + np + 3 * ne + i] = Jp[i * 6 + j]; g[j] += Jp[i * 6 + j] * r[i]; }
            }
        }
        for (size_t e = 0; e < ne; ++e) {
            double r[3], Je[18], rr[3];
            edge_residual(*edges[e], x, R, r, Je);
            rho_a(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], edges[e]->w, a2_line, rr);
            c += 0.5 * rr[0];
            const double sc = std::sqrt(rr[1]);
            for (int i = 0; i < 3; ++i) {
                r[i] *= sc;
                for (int j = 0; j < 6; ++j) { Je[i * 6 + j] *= sc; J[size_t(j) * n + np + 3 * e + i] = Je[i * 6 + j]; g[j] += Je[i * 6 + j] * r[i]; }
                res[np + 3 * e + i] = r[i];
            }
        }
        for (size_t i = 0; i < np; ++i) {
            const Corr& b = *blocks[i];
            double r = residual(b, x);
            // J = [ n^T , -n^T R [p]x ] ; -a^T[p]x = p x a with a = R^T n
            const double a[3] = {R[0] * b.n[0] + R[3] * b.n[1] + R[6] * b.n[2], R[1] * b.n[0] + R[4] * b.n[1] + R[7] * b.n[2], R[2] * b.n[0] + R[5] * b.n[1] + R[8] * b.n[2]};
            double Jr[6] = {b.n[0], b.n[1], b.n[2], b.p[1] * a[2] - b.p[2] * a[1], b.p[2] * a[0] - b.p[0] * a[2], b.p[0] * a[1] - b.p[1] * a[0]};
            double rr[3]; rho(r * r, b.w, rr);
            c += 0.5 * rr[0];
            const double s = std::sqrt(rr[1]);
            r *= s;
            for (int j = 0; j < 6; ++j) { Jr[j] *= s; J[size_t(j) * n + i] = Jr[j]; g[j] += Jr[j] * r; }
            res[i] = r;
        }
        *cost_out = c;
    }
};

struct SolveSummary {
    int num_successful_steps = 0, num_unsuccessful_steps = 0, iterations = 0, termination = 0; double initial_cost = 0, final_cost = 0;
    double radius = 0, decrease_factor = 0, gmax = 0;      // the trust-region state the loop ended in
};
// termination: 0 NO_CONVERGENCE(max iters) 1 gradient tol 2 parameter tol 3 function tol 4 radius 5 invalid steps 6 no residuals
//              7 non-finite cost at the start (the reference aborts)

// ceres::Solve with options {max_num_iterations=4, DENSE_QR} (LidarSlam.cpp:230-240), everything else default:
// TrustRegionMinimizer::Minimize + LevenbergMarquardtStrategy + TrustRegionStepEvaluator(monotonic).  NC tangent columns: NC / 6 pose7
// blocks, each with PoseLocalParameterization (Plus block by block; x_norm, the step norm and the gradient max-norm over all of them).
// E: rows(), empty(), cost(x) and full(x, ...) with a column-major rows() x NC Jacobian.
template <int NC, class Eval>
static SolveSummary ceres_solve_t(const Eval& E, double* params, int max_num_iterations) {
    constexpr int NX = NC / 6 * 7;
    SolveSummary S;
    if (E.empty()) { S.termination = 6; return S; }
    const size_t n = E.rows();      // residual rows
    const double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
    const double min_relative_decrease = 1e-3, min_lm_diagonal = 1e-6, max_lm_diagonal = 1e32;
    const double max_radius = 1e16, min_radius = 1e-32;
    const int max_consecutive_invalid = 5;
    double x[NX]; std::memcpy(x, params, sizeof(x));
    double x_norm = 0; for (int i = 0; i < NX; ++i) x_norm += x[i] * x[i]; x_norm = std::sqrt(x_norm);
    double x_cost; std::vector<double> res, J; double g[NC];
    double scale[NC];
    auto plus = [](const double* xx, const double* d, double* out) { for (int b = 0; b < NC / 6; ++b) pose_plus(xx + 7 * b, d + 6 * b, out + 7 * b); };
    auto grad_max_norm = [&](const double* xx, const double* gg) {
        double neg[NC]; for (int j = 0; j < NC; ++j) neg[j] = -gg[j];
        double xp[NX]; plus(xx, neg, xp);
        double m = 0; for (int i = 0; i < NX; ++i) m = std::max(m, std::fabs(xx[i] - xp[i]));
        return m;
    };
    auto scale_columns = [&]() { for (int j = 0; j < NC; ++j) { double* c = &J[size_t(j) * n]; for (size_t i = 0; i < n; ++i) c[i] *= scale[j]; } };
    // IterationZero
    E.full(x, &x_cost, res, J, g);
    // a non-finite loss weight (ScaledLoss(TukeyLoss, w), w = NaN) makes the cost NaN: Ceres 2.0 CHECK-fails in the Corrector of that
    // residual block (corrector.cc: neither rho'' <= 0 nor rho' > 0 holds) and ends the process; reported as termination 7
    if (!std::isfinite(x_cost)) { S.termination = 7; S.initial_cost = S.final_cost = x_cost; return S; }
    for (int j = 0; j < NC; ++j) { double s = 0; const double* c = &J[size_t(j) * n]; for (size_t i = 0; i < n; ++i) s += c[i] * c[i]; scale[j] = 1.0 / (1.0 + std::sqrt(s)); }
    scale_columns();
    double gmax = grad_max_norm(x, g);
    S.initial_cost = x_cost;
    double radius = 1e4, decrease_factor = 2.0; bool reuse_diagonal = false; double diagonal[NC];
    int iteration = 0, consecutive_invalid = 0; bool step_successful = false;
    double best[NX]; std::memcpy(best, x, sizeof(x));
    std::vector<double> Aaug, baug;
    for (;;) {
        // FinalizeIterationAndCheckIfMinimizerCanContinue
        if (step_successful) { ++S.num_successful_steps; std::memcpy(best, x, sizeof(x)); } else ++S.num_unsuccessful_steps;
        if (iteration >= max_num_iterations) { S.termination = 0; break; }
        if (gmax <= gradient_tolerance) { S.termination = 1; break; }
        if (radius <= min_radius) { S.termination = 4; break; }
        ++iteration; step_successful = false;
        // LevenbergMarquardtStrategy::ComputeStep
        if (!reuse_diagonal) for (int j = 0; j < NC; ++j) { double s = 0; const double* c = &J[size_t(j) * n]; for (size_t i = 0; i < n; ++i) s += c[i] * c[i]; diagonal[j] = std::min(std::max(s, min_lm_diagonal), max_lm_diagonal); }
        double lm[NC]; for (int j = 0; j < NC; ++j) lm[j] = std::sqrt(diagonal[j] / radius);
        const int m = int(n) + NC;
        Aaug.assign(size_t(m) * NC, 0.0); baug.assign(m, 0.0);
        for (int j = 0; j < NC; ++j) { std::memcpy(&Aaug[size_t(j) * m], &J[size_t(j) * n], n * sizeof(double)); Aaug[size_t(j) * m + n + j] = lm[j]; }
        std::memcpy(baug.data(), res.data(), n * sizeof(double));
        double y[NC]; householder_ls(m, NC, Aaug.data(), baug.data(), y, nullptr);
        bool finite = true; for (int j = 0; j < NC; ++j) finite = finite && std::isfinite(y[j]);
        reuse_diagonal = true;
        double step[NC]; for (int j = 0; j < NC; ++j) step[j] = -y[j];
        // model_cost_change = -(J step)'(f + J step / 2)
        double mcc = 0.0;
        if (finite) for (size_t i = 0; i < n; ++i) { double mr = 0; for (int j = 0; j < NC; ++j) mr += J[size_t(j) * n + i] * step[j]; mcc -= mr * (res[i] + mr / 2.0); }
        if (!finite || !(mcc > 0.0)) {   // HandleInvalidStep
            if (++consecutive_invalid >= max_consecutive_invalid) { S.termination = 5; break; }
            radius *= 0.5; reuse_diagonal = true; continue;
        }
        consecutive_invalid = 0;
        double delta[NC]; for (int j = 0; j < NC; ++j) delta[j] = step[j] * scale[j];
        double cand[NX]; plus(x, delta, cand);
        const double cand_cost = E.cost(cand);
        // ParameterToleranceReached
        double sn = 0; for (int i = 0; i < NX; ++i) sn += (x[i] - cand[i]) * (x[i] - cand[i]); sn = std::sqrt(sn);
        if (sn <= parameter_tolerance * (x_norm + parameter_tolerance)) { S.termination = 2; break; }
        // FunctionToleranceReached
        const double cost_change = x_cost - cand_cost;
        if (std::fabs(cost_change) <= function_tolerance * x_cost) { S.termination = 3; break; }
        const double relative_decrease = cost_change / mcc;       // monotonic TrustRegionStepEvaluator
        if (relative_decrease > min_relative_decrease) {          // HandleSuccessfulStep
            std::memcpy(x, cand, sizeof(x));
            x_norm = 0; for (int i = 0; i < NX; ++i) x_norm += x[i] * x[i]; x_norm = std::sqrt(x_norm);
            E.full(x, &x_cost, res, J, g); scale_columns();
            gmax = grad_max_norm(x, g);
            step_successful = true;
            radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * relative_decrease - 1.0, 3));
            radius = std::min(max_radius, radius); decrease_factor = 2.0; reuse_diagonal = false;
        } else {
            radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true;
        }
    }
    S.iterations = iteration; S.final_cost = x_cost;
    S.radius = radius; S.decrease_factor = decrease_factor; S.gmax = gmax;
    // parameters_ hold the best (last accepted, monotonic) iterate
    if (S.termination == 2 || S.termination == 3) { /* tolerance returns skip Finalize; best already == x (last accepted) */ std::memcpy(best, x, sizeof(x)); }
    std::memcpy(params, best, sizeof(best));
    return S;
}
static SolveSummary ceres_solve(const Evaluator& E, double params[7], int max_num_iterations = 4) { return ceres_solve_t<6>(E, params, max_num_iterations); }

// The two-block problem of so_register_optimized (DESIGN.md section 3), for ceres_solve_t<12>: pose7 blocks T (the pose at tau = 0)
// and D (the motion over dt).  Plane row i, alpha_i = tau_i / dt (0 for a non-finite tau_i):
//   u_i = qrot(slerp(identity, q_D, alpha_i), p_i) + alpha_i t_D,   r_i = n_i . (qrot(q_T, u_i) + t_T) + d_i
// under ScaledLoss(TukeyLoss(a), w_i) through the Corrector, as Evaluator's plane rows; then SE3AbsolutatePoseFactor on D (measurement
// D0, row k times sqrt(n_rows * info_k), no loss).  Columns: T's translation and rotation, D's translation and rotation under
// PoseLocalParameterization.  D's rotation columns are the exact derivative: a right perturbation delta of q_D moves
// Log(q_D) = phi by J_r(phi)^-1 delta, so slerp's exp(alpha phi) by J_r(alpha phi) alpha J_r(phi)^-1 delta, and the row is
//   alpha (p x b)^T J_r(alpha phi) J_r(phi)^-1,   b = R(q_alpha)^T R(q_T)^T n,   phi on the shortest path,
// with J_r(v) = I - (1 - cos th) / th^2 [v]x + (th - sin th) / th^3 [v]x^2 and J_r(v)^-1 = I + [v]x / 2 + (1 / th^2 - (1 + cos th) /
// (2 th sin th)) [v]x^2 (th = |v|) built as 3x3 matrices, their coefficients' Taylor series to th^4 below th = 1e-2.
struct MotionEvaluator {
    struct Row { double p[3], n[3], d, w, alpha; };
    std::vector<Row> planes;
    PosePrior prior;                    // on D, on always; sqrt_info = sqrt(n_rows * info)
    double a2;
    size_t rows() const { return planes.size() + 6; }
    bool empty() const { return planes.empty(); }     // no correspondences: the registration's termination 6

    static void mat_coeffs(double th, double* c1, double* c2, double* c3) {
        const double t2 = th * th;
        if (th < 1e-2) {
            *c1 = 0.5 - t2 / 24.0 + t2 * t2 / 720.0;
            *c2 = 1.0 / 6.0 - t2 / 120.0 + t2 * t2 / 5040.0;
            *c3 = 1.0 / 12.0 + t2 / 720.0 + t2 * t2 / 30240.0;
        } else {
            *c1 = (1.0 - std::cos(th)) / t2;
            *c2 = (th - std::sin(th)) / (t2 * th);
            *c3 = 1.0 / t2 - (1.0 + std::cos(th)) / (2.0 * th * std::sin(th));
        }
    }
    // I + a [v]x + b [v]x^2, row-major
    static void jmat(const double v[3], double a, double b, double M[9]) {
        const double K[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                double k2 = 0.0;
                for (int k = 0; k < 3; ++k) k2 += K[i * 3 + k] * K[k * 3 + j];
                M[i * 3 + j] = (i == j ? 1.0 : 0.0) + a * K[i * 3 + j] + b * k2;
            }
    }
    struct Setup { Quat qT, qD; double R[9], tT[3], tD[3], phi[3], th, Jinv[9]; bool linear; double s_theta, theta; };
    static Setup setup(const double* x) {
        Setup S;
        S.qT = Quat{x[3], x[4], x[5], x[6]};
        qtoR(S.qT, S.R);
        S.qD = qnormalized(Quat{x[10], x[11], x[12], x[13]});
        for (int k = 0; k < 3; ++k) { S.tT[k] = x[k]; S.tD[k] = x[7 + k]; }
        const double absd = std::fabs(S.qD.w);                 // Eigen's slerp(identity, q_D, .): dot = q_D.w
        S.linear = absd >= 1.0 - std::numeric_limits<double>::epsilon();
        S.theta = S.linear ? 0.0 : std::acos(absd);
        S.s_theta = std::sin(S.theta);
        const Quat q = S.qD.w < 0.0 ? Quat{-S.qD.x, -S.qD.y, -S.qD.z, -S.qD.w} : S.qD;
        const double vn = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
        S.th = 2.0 * std::atan2(vn, q.w);
        const double f = vn > 0.0 ? S.th / vn : 0.0;
        S.phi[0] = f * q.x; S.phi[1] = f * q.y; S.phi[2] = f * q.z;
        double c1, c2, c3;
        mat_coeffs(S.th, &c1, &c2, &c3);
        jmat(S.phi, 0.5, c3, S.Jinv);
        return S;
    }
    static Quat slerp_alpha(const Setup& S, double al) {
        double s0, s1;
        if (S.linear) { s0 = 1.0 - al; s1 = al; }
        else { s0 = std::sin((1.0 - al) * S.theta) / S.s_theta; s1 = std::sin(al * S.theta) / S.s_theta; }
        if (S.qD.w < 0.0) s1 = -s1;
        return Quat{s1 * S.qD.x, s1 * S.qD.y, s1 * S.qD.z, s0 + s1 * S.qD.w};
    }
    // residual of one row, with u and q_alpha for the Jacobian
    static double residual(const Setup& S, const Row& r, double u[3], Quat* qa) {
        *qa = slerp_alpha(S, r.alpha);
        qrot(*qa, r.p, u);
        for (int k = 0; k < 3; ++k) u[k] += r.alpha * S.tD[k];
        double pw[3];
        qrot(S.qT, u, pw);
        return r.n[0] * (pw[0] + S.tT[0]) + r.n[1] * (pw[1] + S.tT[1]) + r.n[2] * (pw[2] + S.tT[2]) + r.d;
    }
    double cost(const double* x) const {
        const Setup S = setup(x);
        double c = 0.0;
        for (const Row& r : planes) { double u[3], rr[3]; Quat qa; const double e = residual(S, r, u, &qa); Evaluator::rho_a(e * e, r.w, a2, rr); c += 0.5 * rr[0]; }
        double rp[6], Jp[36]; prior.eval(x + 7, rp, Jp);
        for (int i = 0; i < 6; ++i) c += 0.5 * rp[i] * rp[i];
        return c;
    }
    void full(const double* x, double* cost_out, std::vector<double>& res, std::vector<double>& J, double g[12]) const {
        const size_t np = planes.size(), n = rows();
        res.assign(n, 0.0); J.assign(n * 12, 0.0);
        for (int j = 0; j < 12; ++j) g[j] = 0.0;
        const Setup S = setup(x);
        double c = 0.0;
        for (size_t i = 0; i < np; ++i) {
            const Row& r = planes[i];
            double u[3]; Quat qa;
            const double e = residual(S, r, u, &qa);
            const double a[3] = {S.R[0] * r.n[0] + S.R[3] * r.n[1] + S.R[6] * r.n[2], S.R[1] * r.n[0] + S.R[4] * r.n[1] + S.R[7] * r.n[2],
                                 S.R[2] * r.n[0] + S.R[5] * r.n[1] + S.R[8] * r.n[2]};                      // R(q_T)^T n
            double b[3];
            qrot(qconj(qa), a, b);
            const double w[3] = {r.p[1] * b[2] - r.p[2] * b[1], r.p[2] * b[0] - r.p[0] * b[2], r.p[0] * b[1] - r.p[1] * b[0]};     // p x b
            const double v[3] = {r.alpha * S.phi[0], r.alpha * S.phi[1], r.alpha * S.phi[2]};
            double c1, c2, c3, Jr[9], M[9];
            mat_coeffs(std::fabs(r.alpha) * S.th, &c1, &c2, &c3);
            jmat(v, -c1, c2, Jr);
            for (int k = 0; k < 3; ++k) for (int l = 0; l < 3; ++l) { double t = 0.0; for (int m = 0; m < 3; ++m) t += Jr[k * 3 + m] * S.Jinv[m * 3 + l]; M[k * 3 + l] = t; }
            double row[12] = {r.n[0], r.n[1], r.n[2], u[1] * a[2] - u[2] * a[1], u[2] * a[0] - u[0] * a[2], u[0] * a[1] - u[1] * a[0],
                              r.alpha * a[0], r.alpha * a[1], r.alpha * a[2], 0, 0, 0};
            for (int l = 0; l < 3; ++l) row[9 + l] = r.alpha * (w[0] * M[l] + w[1] * M[3 + l] + w[2] * M[6 + l]);
            double rr[3]; Evaluator::rho_a(e * e, r.w, a2, rr);
            c += 0.5 * rr[0];
            const double sc = std::sqrt(rr[1]);
            res[i] = e * sc;
            for (int j = 0; j < 12; ++j) { J[size_t(j) * n + i] = row[j] * sc; g[j] += row[j] * sc * res[i]; }
        }
        double rp[6], Jp[36]; prior.eval(x + 7, rp, Jp);
        for (int i = 0; i < 6; ++i) {
            res[np + i] = rp[i]; c += 0.5 * rp[i] * rp[i];
            for (int j = 0; j < 6; ++j) { J[size_t(6 + j) * n + np + i] = Jp[i * 6 + j]; g[6 + j] += Jp[i * 6 + j] * rp[i]; }
        }
        *cost_out = c;
    }
};

// ceres::Covariance{apply_loss_function, DENSE_SVD, null_space_rank=-1} in tangent space (LidarSlam.cpp:854-871;
// covariance_impl.cc ComputeCovarianceValuesUsingDenseSVD): V diag(1/s^2) V^T with s_i/s_0 < sqrt(1e-14) truncated.
static void ceres_covariance(const Evaluator& E, const double x[7], double cov[36]) {
    const size_t n = E.blocks.size() + 3 * E.edges.size() + (E.prior.on ? 6 : 0);
    std::vector<double> res, J; double g[6], c;
    E.full(x, &c, res, J, g);
    double R[36]; householder_ls(int(n), 6, J.data(), nullptr, nullptr, R);
    double s[6], V[36]; jacobi_svd(6, R, s, V);
    const double min_ratio = std::sqrt(1e-14);
    double inv2[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 6; ++i) { if (s[i] / s[0] < min_ratio) break; inv2[i] = 1.0 / (s[i] * s[i]); }
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) { double t = 0; for (int k = 0; k < 6; ++k) t += V[i * 6 + k] * inv2[k] * V[j * 6 + k]; cov[i * 6 + j] = t; }
}

// tf2 Matrix3x3(q).getRPY + Quaternion::setRPY round trip (LidarSlam.cpp:891-913)
static void manual_yaw_correction(const double last[7], double T[7], double yaw_ratio) {
    double tn, rn; rel_motion(last, T, &tn, &rn);
    const float translation_norm = float(tn);
    const double x = T[3], y = T[4], z = T[5], w = T[6];
    const double d = x * x + y * y + z * z + w * w, s = 2.0 / d;
    const double xs = x * s, ys = y * s, zs = z * s, wx = w * xs, wy = w * ys, wz = w * zs, xx = x * xs, xy = x * ys, xz = x * zs, yy = y * ys, yz = y * zs, zz = z * zs;
    const double m00 = 1.0 - (yy + zz), m10 = xy + wz, m20 = xz - wy, m21 = yz + wx, m22 = 1.0 - (xx + yy);
    const double m01 = xy - wz, m02 = xz + wy;
    double roll, pitch, yaw;
    if (std::fabs(m20) >= 1) {      // tf2 Matrix3x3::getEulerYPR gimbal-lock branch
        yaw = 0;
        if (m20 < 0) { pitch = M_PI / 2.0; roll = std::atan2(m01, m02); }
        else { pitch = -M_PI / 2.0; roll = std::atan2(-m01, -m02); }
    } else {
        pitch = -std::asin(m20);
        roll = std::atan2(m21 / std::cos(pitch), m22 / std::cos(pitch));
        yaw = std::atan2(m10 / std::cos(pitch), m00 / std::cos(pitch));
    }
    const double cyaw = yaw + double(translation_norm) * yaw_ratio * M_PI / 180;
    const double hy = cyaw * 0.5, hp = pitch * 0.5, hr = roll * 0.5;
    const double cy = std::cos(hy), sy = std::sin(hy), cp = std::cos(hp), sp = std::sin(hp), cr = std::cos(hr), sr = std::sin(hr);
    Quat q{sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy};
    q = qnormalized(q);
    T[3] = q.x; T[4] = q.y; T[5] = q.z; T[6] = q.w;
}

}  // namespace orc

// ============================================================================= C API (ctypes)
// Which source this library was compiled from (oracle.py reads it out of the file): a library left from another version of this
// file, e.g. a prebuilt _ref/ that cannot be rebuilt where the reference tree is absent, is then not loaded.
#ifndef SO_ORACLE_SOURCE_ID
#define SO_ORACLE_SOURCE_ID "unknown"
#endif
__attribute__((used)) static const char kOracleSourceId[] = "so_oracle source id " SO_ORACLE_SOURCE_ID ";";

extern "C" {

#define ORC_MAX_ICP_ITERS 32

typedef struct {
    float plane_res;            // localMap.planeRes_
    int32_t max_icp_iters;      // LocalizationICPMaxIter
    int32_t max_surface_features;   // OptSet.max_surface_features (0 = uncapped)
    int32_t lm_max_iterations;  // 4 (LidarSlam.cpp:232)
    int32_t knn_mode;           // 0 exact-in-block, 1 brute force, 2 verbatim reference octree
    int32_t n_threads;          // threads for the per-point loop (1 = faithful to the reference)
    float yaw_ratio;            // OptSet.yaw_ratio (0 in all shipped calibrations)
    int32_t skip_map_checks;    // 0: shiftMap + hasEnoughFeatures as the reference does
    int32_t use_pose_prior;     // shouldAddAbsolutePoseConstraints(): VIO_ODOM && isDegenerate && Visual_confidence_factor != 0
    float visual_confidence_factor;
    float prior_uncertainty[3]; // lidarOdomUncer.uncertainty_{x,y,z} (from the previous scan's histogram)
    float line_res;             // localMap.lineRes_ (edge branch)
} orc_opts;

typedef struct {
    double pose[7];             // T_w_lidar after MannualYawCorrection
    double pose_opt[7];         // optimiser output before the RPY round trip
    int32_t status;             // 0 ok, 1 not enough map features (pose = prior), 2 no correspondences
    int32_t n_iterations;
    int32_t iter_n_surf[ORC_MAX_ICP_ITERS];
    int32_t iter_n_edge[ORC_MAX_ICP_ITERS];
    double iter_dtrans[ORC_MAX_ICP_ITERS];
    double iter_drot[ORC_MAX_ICP_ITERS];
    int32_t iter_lm_steps[ORC_MAX_ICP_ITERS];
    int32_t iter_lm_successful[ORC_MAX_ICP_ITERS];
    int32_t iter_lm_termination[ORC_MAX_ICP_ITERS];
    double iter_cost[ORC_MAX_ICP_ITERS];
    int32_t hist_obs[9];
    int32_t hist_reject_plane[7];
    int32_t hist_reject_line[7];
    double cov[36];
    double pos_err, pos_dir[3], pos_inv_cond;
    double ori_err_deg, ori_dir[3], ori_inv_cond;
    double total_translation, total_rotation, translation_from_last, rotation_from_last;
    int32_t map_surf_5x5, map_edge_5x5, scan_surf_num, scan_edge_num;
    int32_t pos_in_localmap[3];
    int32_t pad_;
    double time_ms;             // whole ICP loop wall time (stats.time_elapsed, LidarSlam.cpp:118,199-200)
    double time_knn_ms;         // share spent in correspond_all
} orc_result;

typedef orc::Corr orc_corr;
typedef orc::EdgeCorr orc_edge_corr;

int orc_has_ref_octree(void) {
#ifdef SO_ORACLE_WITH_REF_OCTREE
    return 1;
#else
    return 0;
#endif
}
size_t orc_sizeof_corr(void) { return sizeof(orc_corr); }
size_t orc_sizeof_result(void) { return sizeof(orc_result); }
size_t orc_sizeof_edge_corr(void) { return sizeof(orc_edge_corr); }

void* orc_map_create(void) { return new orc::Map(); }
void orc_map_destroy(void* m) { delete static_cast<orc::Map*>(m); }
void orc_map_set_origin(void* m, const int32_t o[3]) { auto* M = static_cast<orc::Map*>(m); M->origin[0] = o[0]; M->origin[1] = o[1]; M->origin[2] = o[2]; }
void orc_map_get_origin(void* m, int32_t o[3]) { auto* M = static_cast<orc::Map*>(m); o[0] = M->origin[0]; o[1] = M->origin[1]; o[2] = M->origin[2]; }

// Replace the map's surf points with xyzi (world frame), binned by LocalMap.h:594-612 under the current origin.
// No voxel filtering (callers pass an already-filtered cloud; the filter itself is orc_voxel_filter).
int64_t orc_map_set_points(void* m, const float* xyzi, size_t n, size_t stride_floats, int build_ref_octree) {
    auto* M = static_cast<orc::Map*>(m);
    for (auto& b : M->blocks) b.reset();
    int64_t kept = 0;
    for (size_t i = 0; i < n; ++i) {
        const float* p = xyzi + i * stride_floats;
        int b = orc::block_of(p[0], p[1], p[2], M->origin);
        if (b < 0) continue;
        if (!M->blocks[b]) M->blocks[b].reset(new orc::BlockData());
        M->blocks[b]->pts.push_back(orc::Pt{p[0], p[1], p[2]});
        M->blocks[b]->gid.push_back(int64_t(i));
        ++kept;
    }
    for (auto& b : M->blocks) if (b) {
        b->build_grid();
#ifdef SO_ORACLE_WITH_REF_OCTREE
        if (build_ref_octree) { b->octree.reset(new nanoflann::Octree<orc::Pt, std::vector<orc::Pt>>()); b->octree->initialize(b->pts); }
#endif
    }
    (void)build_ref_octree;
    return kept;
}

// Same for the edge clouds (pedge_pc_): already line-res filtered points, binned under the current origin.
int64_t orc_map_set_edge_points(void* m, const float* xyzi, size_t n, size_t stride_floats) {
    auto* M = static_cast<orc::Map*>(m);
    for (auto& b : M->eblocks) b.reset();
    int64_t kept = 0;
    for (size_t i = 0; i < n; ++i) {
        const float* p = xyzi + i * stride_floats;
        int b = orc::block_of(p[0], p[1], p[2], M->origin);
        if (b < 0) continue;
        if (!M->eblocks[b]) M->eblocks[b].reset(new orc::BlockData());
        M->eblocks[b]->pts.push_back(orc::Pt{p[0], p[1], p[2]});
        M->eblocks[b]->gid.push_back(int64_t(i));
        ++kept;
    }
    for (auto& b : M->eblocks) if (b) b->build_grid();
    return kept;
}

int orc_correspond_edge(void* m, const float* scan_xyzi, size_t n, size_t stride_floats, const double pose[7], float line_res, int knn_mode,
                        orc_edge_corr* out, int32_t hist_rej_line[7]) {
    auto* M = static_cast<orc::Map*>(m);
    for (int i = 0; i < 7; ++i) hist_rej_line[i] = 0;
    for (size_t i = 0; i < n; ++i) { orc::line_correspondence(*M, scan_xyzi + i * stride_floats, pose, line_res, knn_mode, out[i]); hist_rej_line[out[i].status]++; }
    return 0;
}

// LocalMap::shiftMap (LocalMap.h:169-287): returns the sensor block; origin may change, blocks that roll off are dropped.
// Because block membership is a pure function of (world coordinate, origin), rolling == re-binning under the new origin.
void orc_map_shift(void* m, const double t[3], int32_t out_ijk[3]) {
    auto* M = static_cast<orc::Map*>(m);
    int c[3];
    for (int a = 0; a < 3; ++a) c[a] = orc::block_coord(t[a] + orc::kHalfBlock, M->origin[a]);
    const int dims[3] = {orc::kW, orc::kH, orc::kD};
    int shift[3] = {0, 0, 0};
    for (int a = 0; a < 3; ++a) {
        while (c[a] < 3) { c[a]++; shift[a]++; }
        while (c[a] >= dims[a] - 3) { c[a]--; shift[a]--; }
    }
    if (shift[0] || shift[1] || shift[2]) {
        std::vector<std::unique_ptr<orc::BlockData>> nb(orc::kNumBlocks);
        for (int k = 0; k < orc::kD; ++k) for (int j = 0; j < orc::kH; ++j) for (int i = 0; i < orc::kW; ++i) {
            int ni = i + shift[0], nj = j + shift[1], nk = k + shift[2];
            if (ni < 0 || ni >= orc::kW || nj < 0 || nj >= orc::kH || nk < 0 || nk >= orc::kD) continue;
            nb[ni + orc::kW * nj + orc::kW * orc::kH * nk] = std::move(M->blocks[i + orc::kW * j + orc::kW * orc::kH * k]);
        }
        M->blocks.swap(nb);
        std::vector<std::unique_ptr<orc::BlockData>> ne(orc::kNumBlocks);
        for (int k = 0; k < orc::kD; ++k) for (int j = 0; j < orc::kH; ++j) for (int i = 0; i < orc::kW; ++i) {
            int ni = i + shift[0], nj = j + shift[1], nk = k + shift[2];
            if (ni < 0 || ni >= orc::kW || nj < 0 || nj >= orc::kH || nk < 0 || nk >= orc::kD) continue;
            ne[ni + orc::kW * nj + orc::kW * orc::kH * nk] = std::move(M->eblocks[i + orc::kW * j + orc::kW * orc::kH * k]);
        }
        M->eblocks.swap(ne);
        for (int a = 0; a < 3; ++a) M->origin[a] += shift[a];
    }
    out_ijk[0] = c[0]; out_ijk[1] = c[1]; out_ijk[2] = c[2];
}

// get5x5LocalMapFeatureSize (LocalMap.h:291-318), surf only
int32_t orc_map_counts_5x5(void* m, const int32_t ijk[3]) {
    auto* M = static_cast<orc::Map*>(m);
    int n = 0;
    for (int i = ijk[0] - 2; i <= ijk[0] + 2; ++i) for (int j = ijk[1] - 2; j <= ijk[1] + 2; ++j) for (int k = ijk[2] - 1; k <= ijk[2] + 1; ++k)
        if (i >= 0 && i < orc::kW && j >= 0 && j < orc::kH && k >= 0 && k < orc::kD) { auto& b = M->blocks[i + orc::kW * j + orc::kW * orc::kH * k]; if (b) n += int(b->pts.size()); }
    return n;
}

int32_t orc_map_edge_counts_5x5(void* m, const int32_t ijk[3]) {
    auto* M = static_cast<orc::Map*>(m);
    int n = 0;
    for (int i = ijk[0] - 2; i <= ijk[0] + 2; ++i) for (int j = ijk[1] - 2; j <= ijk[1] + 2; ++j) for (int k = ijk[2] - 1; k <= ijk[2] + 1; ++k)
        if (i >= 0 && i < orc::kW && j >= 0 && j < orc::kH && k >= 0 && k < orc::kD) { auto& b = M->eblocks[i + orc::kW * j + orc::kW * orc::kH * k]; if (b) n += int(b->pts.size()); }
    return n;
}

// Batch k-NN through LocalMap::nearestKSearchSurf; idx = caller input index (or -1), found[i] = search ran.
int orc_knn(void* m, const float* q_xyz, size_t nq, size_t stride_floats, int k, int mode, int64_t* idx, float* d2, uint8_t* found) {
    auto* M = static_cast<orc::Map*>(m);
    if (k > 16) return -1;
    for (size_t i = 0; i < nq; ++i) {
        const float* p = q_xyz + i * stride_floats;
        int64_t li[16]; float ld[16]; const orc::BlockData* B;
        bool f = orc::nearest_k_surf(*M, orc::Pt{p[0], p[1], p[2]}, k, mode, li, ld, &B);
        found[i] = f ? 1 : 0;
        for (int j = 0; j < k; ++j) {
            if (f && size_t(li[j]) < B->pts.size()) { idx[i * k + j] = B->gid[li[j]]; d2[i * k + j] = ld[j]; }
            else { idx[i * k + j] = -1; d2[i * k + j] = 0.f; }
        }
        if (f && int(B->pts.size()) < k) for (int j = int(B->pts.size()); j < k; ++j) idx[i * k + j] = -1;
    }
    return 0;
}

int orc_correspond(void* m, const float* scan_xyzi, size_t n, size_t stride_floats, const double pose[7], float plane_res,
                   int max_surface_features, int knn_mode, int n_threads, orc_corr* out, int32_t hist_obs[9], int32_t hist_rej[7]) {
    orc::correspond_all(*static_cast<orc::Map*>(m), scan_xyzi, n, stride_floats, pose, plane_res, max_surface_features, knn_mode, n_threads, out, hist_obs, hist_rej);
    return 0;
}

// H = sum rho' J^T J (row-major 6x6), g = sum rho' J^T r, cost = 1/2 sum rho, over status==0 correspondences.
int orc_evaluate(const orc_corr* corr, size_t n, const double pose[7], float plane_res, double H[36], double g[6], double* cost, int64_t* n_ok) {
    orc::Evaluator E; const double a = double(std::sqrt(3 * plane_res)); E.a2 = a * a;
    for (size_t i = 0; i < n; ++i) if (corr[i].status == orc::SUCCESS) E.blocks.push_back(&corr[i]);
    std::vector<double> res, J; E.full(pose, cost, res, J, g);
    const size_t m = E.blocks.size();
    for (int a1 = 0; a1 < 6; ++a1) for (int b1 = 0; b1 < 6; ++b1) { double s = 0; for (size_t i = 0; i < m; ++i) s += J[a1 * m + i] * J[b1 * m + i]; H[a1 * 6 + b1] = s; }
    *n_ok = int64_t(m);
    return 0;
}

// One ceres::Solve on fixed correspondences (stage parity for the LM state machine).  prior_meas (optional): the SE3 prior rows with
// that measurement, their information from the accepted correspondences as a registration computes it.
// costs: initial and final cost, then the final radius, decrease factor and gradient max-norm.
int orc_solve(const orc_corr* corr, size_t n, double pose[7], float plane_res, int lm_max_iterations, const double* prior_meas,
              float visual_confidence_factor, const float* prior_uncertainty, int32_t summary[4], double costs[5]) {
    orc::Evaluator E; const double a = double(std::sqrt(3 * plane_res)); E.a2 = a * a;
    for (size_t i = 0; i < n; ++i) if (corr[i].status == orc::SUCCESS) E.blocks.push_back(&corr[i]);
    if (prior_meas) orc::set_pose_prior(E.prior, prior_meas, int(E.blocks.size()), visual_confidence_factor, prior_uncertainty);
    orc::SolveSummary S = orc::ceres_solve(E, pose, lm_max_iterations);
    summary[0] = S.num_successful_steps; summary[1] = S.num_unsuccessful_steps; summary[2] = S.iterations; summary[3] = S.termination;
    costs[0] = S.initial_cost; costs[1] = S.final_cost; costs[2] = S.radius; costs[3] = S.decrease_factor; costs[4] = S.gmax;
    return 0;
}

// The two-block solve of so_register_optimized (MotionEvaluator) on n given rows {p, tau, n, d, w} from T and D (D's quaternion normalised
// first); T and D are overwritten with the result.  summary and costs as orc_solve.
int orc_solve_optimized(const double* p, const float* tau, const double* nrm, const double* d, const double* w, size_t n, double T[7],
                        double D[7], double dt, const double D0[7], const double info[6], float plane_res, int lm_max_iterations,
                        int32_t summary[4], double costs[5]) {
    orc::MotionEvaluator E; const double a = double(std::sqrt(3 * plane_res)); E.a2 = a * a;
    for (size_t i = 0; i < n; ++i) {
        orc::MotionEvaluator::Row r;
        for (int k = 0; k < 3; ++k) { r.p[k] = p[3 * i + k]; r.n[k] = nrm[3 * i + k]; }
        r.d = d[i]; r.w = w[i];
        r.alpha = std::isfinite(tau[i]) ? double(tau[i]) / dt : 0.0;
        E.planes.push_back(r);
    }
    E.prior.on = true;
    std::memcpy(E.prior.meas, D0, sizeof(E.prior.meas));
    for (int k = 0; k < 6; ++k) E.prior.sqrt_info[k] = std::sqrt(double(n) * info[k]);
    double x[14];
    std::memcpy(x, T, 7 * sizeof(double));
    const double qn = std::sqrt(D[3] * D[3] + D[4] * D[4] + D[5] * D[5] + D[6] * D[6]);
    for (int k = 0; k < 7; ++k) x[7 + k] = k < 3 ? D[k] : D[k] / qn;
    orc::SolveSummary S = orc::ceres_solve_t<12>(E, x, lm_max_iterations);
    std::memcpy(T, x, 7 * sizeof(double));
    std::memcpy(D, x + 7, 7 * sizeof(double));
    summary[0] = S.num_successful_steps; summary[1] = S.num_unsuccessful_steps; summary[2] = S.iterations; summary[3] = S.termination;
    costs[0] = S.initial_cost; costs[1] = S.final_cost; costs[2] = S.radius; costs[3] = S.decrease_factor; costs[4] = S.gmax;
    return 0;
}

int orc_covariance(const orc_corr* corr, size_t n, const double pose[7], float plane_res, double cov[36]) {
    orc::Evaluator E; const double a = double(std::sqrt(3 * plane_res)); E.a2 = a * a;
    for (size_t i = 0; i < n; ++i) if (corr[i].status == orc::SUCCESS) E.blocks.push_back(&corr[i]);
    if (E.blocks.empty()) return 1;
    orc::ceres_covariance(E, pose, cov);
    return 0;
}

// small-linear-algebra hooks so tests can pin them against numpy
void orc_sym_eig(int n, const double* a, double* w, double* v) { orc::sym_eig(n, a, w, v); }
void orc_colpiv_qr_solve(int m, const double* A, const double* b, double* x) { orc::colpiv_qr_solve(m, A, b, x); }
void orc_pose_plus(const double x[7], const double d[6], double out[7]) { orc::pose_plus(x, d, out); }
void orc_yaw_round_trip(const double last[7], double T[7], double yaw_ratio) { orc::manual_yaw_correction(last, T, yaw_ratio); }

// Optional per-ICP-iteration neighbour trace of the next orc_register* call on this thread: ids[it][i][0..4] = the five neighbour
// ids (caller's map index) findNearestNeighbors returned for scan point i in ICP iteration it, -1 where no search result exists
// (skipped by sampling, off-grid, block with < 5 points).  Lets a test feed the reference octree's own neighbour sets into the
// GPU fit / solve stages (tests/test_gpu_parity.py::test_injected_reference_octree_neighbours_*).
static thread_local int64_t* g_nn_trace = nullptr;
static thread_local size_t g_nn_trace_n = 0;
static thread_local int g_nn_trace_iters = 0;
void orc_set_nn_trace(int64_t* buf, size_t n_points, int max_iters) { g_nn_trace = buf; g_nn_trace_n = n_points; g_nn_trace_iters = max_iters; }

// LidarSLAM::Localization, initialization==true branch -> performLocalizationAndMapping (LidarSlam.cpp:30-51,107-171),
// without the map insert at the end (transformAndAddToMap is a "next" row; use orc_voxel_filter + orc_map_set_points).
int orc_register_full(void* m, const float* scan_xyzi, size_t n, const float* edge_xyzi, size_t n_edge, size_t stride_floats,
                      const double pose_in[7], const orc_opts* opt, orc_result* out) {
    using namespace orc;
    auto* M = static_cast<Map*>(m);
    std::memset(out, 0, sizeof(*out));
    double T[7], T0[7], last_T[7];
    std::memcpy(T, pose_in, sizeof(T)); std::memcpy(T0, pose_in, sizeof(T)); std::memcpy(last_T, pose_in, sizeof(T));   // initializeState (:53-57)
    std::memcpy(out->pose, T, sizeof(T)); std::memcpy(out->pose_opt, T, sizeof(T));
    out->scan_surf_num = int32_t(n); out->scan_edge_num = int32_t(n_edge);
    // prepareOptimizationState (:361-369)
    int32_t ijk[3];
    if (!opt->skip_map_checks) orc_map_shift(m, T, ijk);
    else for (int a = 0; a < 3; ++a) ijk[a] = block_coord(T[a] + kHalfBlock, M->origin[a]);
    out->pos_in_localmap[0] = ijk[0]; out->pos_in_localmap[1] = ijk[1]; out->pos_in_localmap[2] = ijk[2];
    out->map_surf_5x5 = orc_map_counts_5x5(m, ijk);
    out->map_edge_5x5 = orc_map_edge_counts_5x5(m, ijk);
    if (!(out->map_surf_5x5 > 50)) { out->status = 1; return 1; }       // hasEnoughFeatures (:379-381)
    const int max_iters = std::min<int>(opt->max_icp_iters, ORC_MAX_ICP_ITERS);
    std::vector<Corr> corr(n);
    std::vector<EdgeCorr> ecorr(n_edge);
    Evaluator E; { const double a = double(std::sqrt(3 * opt->plane_res)); E.a2 = a * a; const double al = double(std::sqrt(3 * opt->line_res)); E.a2_line = al * al; }   // TukeyLoss(std::sqrt(3*planeRes_)) float sqrt (:271)
    auto t0 = std::chrono::steady_clock::now();
    double knn_ms = 0;
    bool have_cov = false;
    for (int it = 0; it < max_iters; ++it) {
        auto tk = std::chrono::steady_clock::now();
        // processEdgeFeatures (:310-321): every edge point, no decimation
        for (int k = 0; k < 7; ++k) out->hist_reject_line[k] = 0;
        E.edges.clear();
        for (size_t i = 0; i < n_edge; ++i) {
            line_correspondence(*M, edge_xyzi + i * stride_floats, T, opt->line_res, opt->knn_mode == 1 ? 1 : 0, ecorr[i]);
            out->hist_reject_line[ecorr[i].status]++;
            if (ecorr[i].status == SUCCESS) E.edges.push_back(&ecorr[i]);
        }
        correspond_all(*M, scan_xyzi, n, stride_floats, T, opt->plane_res, opt->max_surface_features, opt->knn_mode, opt->n_threads, corr.data(), out->hist_obs, out->hist_reject_plane);
        knn_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tk).count();
        if (g_nn_trace && it < g_nn_trace_iters && g_nn_trace_n == n)
            for (size_t i = 0; i < n; ++i) for (int j = 0; j < 5; ++j) g_nn_trace[(size_t(it) * n + i) * 5 + j] = corr[i].status < 0 ? -1 : corr[i].nn[j];
        E.blocks.clear();
        for (size_t i = 0; i < n; ++i) if (corr[i].status == SUCCESS) E.blocks.push_back(&corr[i]);
        E.prior.on = false;
        if (opt->use_pose_prior)                                  // position = T_w_initial_guess
            set_pose_prior(E.prior, T0, int(E.blocks.size() + E.edges.size()), opt->visual_confidence_factor, opt->prior_uncertainty);
        double prev[7]; std::memcpy(prev, T, sizeof(T));
        double params[7]; std::memcpy(params, T, sizeof(T));     // pose_parameters were set in prepareOptimizationState and by the previous solve
        SolveSummary S = ceres_solve(E, params, opt->lm_max_iterations);
        std::memcpy(T, params, sizeof(T));                       // T_w_lidar <- T_w_curr/Q_w_curr (:135-136)
        out->iter_n_surf[it] = int32_t(E.blocks.size()); out->iter_n_edge[it] = int32_t(E.edges.size());
        rel_motion(prev, T, &out->iter_dtrans[it], &out->iter_drot[it]);
        out->iter_lm_steps[it] = S.iterations; out->iter_lm_successful[it] = S.num_successful_steps; out->iter_lm_termination[it] = S.termination; out->iter_cost[it] = S.final_cost;
        out->n_iterations = it + 1;
        if (S.termination == 7) {                                 // SO_STATUS_INVALID_EVALUATION: no step, no covariance
            out->iter_lm_steps[it] = out->iter_lm_successful[it] = out->iter_lm_termination[it] = 0;
            out->status = 3;
            break;
        }
        if (S.num_successful_steps == 1 || it == max_iters - 1) {     // (:141-146)
            if (!E.blocks.empty() || !E.edges.empty()) {
                ceres_covariance(E, T, out->cov); have_cov = true;
            }
            break;
        }
    }
    if (have_cov) {     // EstimateRegistrationError (:873-884)
        double P[9], O[9], w[3], V[9];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { P[i * 3 + j] = out->cov[i * 6 + j]; O[i * 3 + j] = out->cov[(i + 3) * 6 + (j + 3)]; }
        sym_eig(3, P, w, V);
        out->pos_err = std::sqrt(w[2]); out->pos_dir[0] = V[2]; out->pos_dir[1] = V[5]; out->pos_dir[2] = V[8];
        out->pos_inv_cond = std::sqrt(w[0]) / std::sqrt(w[2]);
        sym_eig(3, O, w, V);
        out->ori_err_deg = std::sqrt(w[2]) / M_PI * 180.; out->ori_dir[0] = V[2]; out->ori_dir[1] = V[5]; out->ori_dir[2] = V[8];
        out->ori_inv_cond = std::sqrt(w[0]) / std::sqrt(w[2]);
    } else if (out->n_iterations > 0 && out->iter_n_surf[out->n_iterations - 1] == 0 && out->iter_n_edge[out->n_iterations - 1] == 0) out->status = 2;
    std::memcpy(out->pose_opt, T, sizeof(T));
    // performPostOptimizationProcessing (:155-171)
    manual_yaw_correction(last_T, T, double(opt->yaw_ratio));
    out->time_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    out->time_knn_ms = knn_ms;
    rel_motion(T0, T, &out->total_translation, &out->total_rotation);
    rel_motion(last_T, T, &out->translation_from_last, &out->rotation_from_last);
    std::memcpy(out->pose, T, sizeof(T));
    return out->status;
}

int orc_register(void* m, const float* scan_xyzi, size_t n, size_t stride_floats, const double pose_in[7], const orc_opts* opt, orc_result* out) {
    return orc_register_full(m, scan_xyzi, n, nullptr, 0, stride_floats, pose_in, opt, out);
}

// EstimateLidarUncertainty (LidarSlam.cpp:915-964) from a 9-bin observability histogram
// ------------------------------------------------------------------------------------------------------------------
// Scan preparation in front of the path (SURVEY 8f row 2): featureExtraction::removePointDistortion and
// featureExtraction::uniformFeatureExtraction, restated with the Eigen 3.4.0 operations they go through.
// ------------------------------------------------------------------------------------------------------------------
namespace orc_prep {
struct Q { double w, x, y, z; };
struct T { Q q; double p[3]; };

static Q q_normalized(Q a) {
    const double n = std::sqrt(a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w);
    return {a.w / n, a.x / n, a.y / n, a.z / n};
}
// Eigen::QuaternionBase::toRotationMatrix (Quaternion.h)
static void q_to_R(const Q& q, double R[9]) {
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y,
                 tzz = tz * q.z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
// Eigen::internal::quaternionbase_assign_impl<Other,3,3>::run (rotation matrix -> quaternion)
static Q R_to_q(const double m[9]) {
    Q q;
    double t = m[0] + m[4] + m[8];
    if (t > 0) {
        t = std::sqrt(t + 1.0);
        q.w = 0.5 * t;
        t = 0.5 / t;
        q.x = (m[7] - m[5]) * t; q.y = (m[2] - m[6]) * t; q.z = (m[3] - m[1]) * t;
    } else {
        int i = 0;
        if (m[4] > m[0]) i = 1;
        if (m[8] > m[i * 4]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(m[i * 4] - m[j * 4] - m[k * 4] + 1.0);
        double v[3];
        v[i] = 0.5 * t;
        t = 0.5 / t;
        q.w = (m[k * 3 + j] - m[j * 3 + k]) * t;
        v[j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
        v[k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
        q.x = v[0]; q.y = v[1]; q.z = v[2];
    }
    return q;
}
// Eigen::QuaternionBase::_transformVector
static void q_rot(const Q& q, const double v[3], double out[3]) {
    double uv[3] = {q.y * v[2] - q.z * v[1], q.z * v[0] - q.x * v[2], q.x * v[1] - q.y * v[0]};
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    out[0] = v[0] + q.w * uv[0] + (q.y * uv[2] - q.z * uv[1]);
    out[1] = v[1] + q.w * uv[1] + (q.z * uv[0] - q.x * uv[2]);
    out[2] = v[2] + q.w * uv[2] + (q.x * uv[1] - q.y * uv[0]);
}
// Eigen::QuaternionBase::slerp
static Q q_slerp(const Q& a, double t, const Q& b) {
    const double one = 1.0 - std::numeric_limits<double>::epsilon();
    const double d = a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
    const double absD = std::fabs(d);
    double s0, s1;
    if (absD >= one) { s0 = 1.0 - t; s1 = t; }
    else {
        const double theta = std::acos(absD), sinTheta = std::sin(theta);
        s0 = std::sin((1.0 - t) * theta) / sinTheta;
        s1 = std::sin(t * theta) / sinTheta;
    }
    if (d < 0) s1 = -s1;
    return {s0 * a.w + s1 * b.w, s0 * a.x + s1 * b.x, s0 * a.y + s1 * b.y, s0 * a.z + s1 * b.z};
}
// Twist::inverse (Twist.h:172-179)
static T t_inverse(const T& a) {
    T r;
    r.q = {a.q.w, -a.q.x, -a.q.y, -a.q.z};
    double R[9];
    q_to_R(r.q, R);
    for (int i = 0; i < 3; ++i) r.p[i] = -(R[i * 3] * a.p[0] + R[i * 3 + 1] * a.p[1] + R[i * 3 + 2] * a.p[2]);
    return r;
}
// Twist::operator*(Twist) (Twist.h:181-185): through Eigen::Transform (normalised rotations), back to a normalised quaternion
static T t_mul(const T& a, const T& b) {
    double Ra[9], Rb[9], R[9];
    q_to_R(q_normalized(a.q), Ra);
    q_to_R(q_normalized(b.q), Rb);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i * 3 + j] = Ra[i * 3] * Rb[j] + Ra[i * 3 + 1] * Rb[3 + j] + Ra[i * 3 + 2] * Rb[6 + j];
    T r;
    for (int i = 0; i < 3; ++i) r.p[i] = Ra[i * 3] * b.p[0] + Ra[i * 3 + 1] * b.p[1] + Ra[i * 3 + 2] * b.p[2] + a.p[i];
    r.q = q_normalized(R_to_q(R));
    return r;
}
static T from7(const double* p) { return T{{p[6], p[3], p[4], p[5]}, {p[0], p[1], p[2]}}; }
static void to7(const T& t, double* p) { p[0] = t.p[0]; p[1] = t.p[1]; p[2] = t.p[2]; p[3] = t.q.x; p[4] = t.q.y; p[5] = t.q.z; p[6] = t.q.w; }

// getInterpolatedPoseAtTime (featureExtraction.cpp:256-276): std::map::upper_bound over the sample times; the `< 0.0001`
// rewind; first sample as is when nothing precedes; else slerp + lerp.  *past_end is set where the reference would
// dereference end() (it relies on synchronize_measurements, :187-196, to make that impossible); the last interval is used.
static T interpolate(const double* times, const double* poses, size_t ns, bool imu_only, double ts, bool* past_end) {
    size_t after = size_t(std::upper_bound(times, times + ns, ts) - times);
    if (after == ns) { if (past_end) *past_end = true; after = ns - 1; }
    if (times[after] < 0.0001) after = 0;
    auto extract = [&](size_t i) {
        T t = from7(poses + 7 * i);
        if (imu_only) t.p[0] = t.p[1] = t.p[2] = 0.0;      // Imu::Ptr: rotation only (:232-236)
        return t;
    };
    if (after == 0) return extract(0);
    const size_t before = after - 1;
    const double ratio = (ts - times[before]) / (times[after] - times[before]);
    const T a = extract(before), b = extract(after);
    T r;
    r.q = q_slerp(a.q, ratio, b.q);
    for (int i = 0; i < 3; ++i) r.p[i] = (1 - ratio) * a.p[i] + ratio * b.p[i];
    return r;
}
}  // namespace orc_prep

// featureExtraction::removePointDistortion<BufferType> (featureExtraction.cpp:222-314).  pts: n points of `stride_floats`
// floats, x,y,z first, per-point time (seconds since lidar_start_time) at float index time_idx; rewritten in place.
// sample_poses: n_samples x {tx,ty,tz,qx,qy,qz,qw}.  start_pose_out = {t_w_original_l, q_w_original_l}.
// Returns the number of points whose time lay past the last sample (undefined behaviour upstream).
int64_t orc_deskew(float* pts, size_t n, size_t stride_floats, size_t time_idx, double lidar_start_time, const double* sample_times,
                   const double* sample_poses, size_t n_samples, int imu_only, const double T_i_l7[7], double start_pose_out[7]) {
    using namespace orc_prep;
    if (n_samples == 0) return -1;
    const bool imu = imu_only != 0;
    const T Til = from7(T_i_l7), Tli = t_inverse(Til);                      // parameter.cpp:192-193
    const T start = interpolate(sample_times, sample_poses, n_samples, imu, lidar_start_time, nullptr);
    const T Two = start;                                                     // T_w_original(start.rot, start.pos)
    const T Two_sensor = imu ? t_mul(Two, Til) : Two;
    to7(Two_sensor, start_pose_out);
    const T Two_inv = t_inverse(Two);
    int64_t past = 0;
    for (size_t i = 0; i < n; ++i) {
        float* p = pts + i * stride_floats;
        if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
        const double point_time = p[time_idx] + lidar_start_time;           // float + double
        bool pe = false;
        const T Twc = interpolate(sample_times, sample_poses, n_samples, imu, point_time, &pe);
        past += pe;
        const T Toc = t_mul(Two_inv, Twc);
        const T Tf = imu ? t_mul(t_mul(Tli, Toc), Til) : Toc;
        const double v[3] = {double(p[0]), double(p[1]), double(p[2])};
        double r[3];
        q_rot(Tf.q, v, r);
        p[0] = float(r[0] + Tf.p[0]); p[1] = float(r[1] + Tf.p[1]); p[2] = float(r[2] + Tf.p[2]);
    }
    return past;
}

// featureExtraction::uniformFeatureExtraction (featureExtraction.cpp:504-525): every skip_num-th point from index 1 whose
// predecessor differs -- `|dx| > 1e-7 || |dy| > 1e-7 || (|dz| > 1e-7 && r^2 > block_range^2)`, exactly that precedence --
// becomes {x, y, z, intensity = time}.  int_abs != 0 evaluates the unqualified abs() as ::abs(int), which is what the
// expression means in a translation unit where only <cmath>/<cstdlib> (not <math.h>/<stdlib.h>) declared abs.
int64_t orc_extract_uniform(const float* pts, size_t n, size_t stride_floats, size_t time_idx, int skip_num, float block_range, int int_abs,
                            float* out_xyzi, size_t cap) {
    if (skip_num <= 0) return -1;
    int64_t m = 0;
    for (size_t i = 1; i < n; i += size_t(skip_num)) {
        const float* p = pts + i * stride_floats;
        const float* q = p - stride_floats;
        const float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
        double ax, ay, az;
        if (int_abs) {
            // int(NaN / inf / |d| >= 2^31) is undefined upstream; such a difference counts as "no difference" here and on the GPU
            auto ia = [](float d) { return (std::isfinite(d) && std::fabs(d) < 2147483648.0f) ? double(std::abs(int(d))) : 0.0; };
            ax = ia(dx); ay = ia(dy); az = ia(dz);
        }
        else { ax = std::fabs(dx); ay = std::fabs(dy); az = std::fabs(dz); }
        const float r2 = p[0] * p[0] + p[1] * p[1] + p[2] * p[2];
        if (ax > 1e-7 || ay > 1e-7 || (az > 1e-7 && r2 > block_range * block_range)) {
            if (size_t(m) < cap) { float* o = out_xyzi + 4 * m; o[0] = p[0]; o[1] = p[1]; o[2] = p[2]; o[3] = p[time_idx]; }
            ++m;
        }
    }
    return m;
}

void orc_lidar_uncertainty(const int32_t h[9], double u[6]) {
    const double tt = double(h[6]) + double(h[7]) + double(h[8]);
    const double tr = double(h[0]) + h[1] + h[2] + h[3] + h[4] + h[5];
    u[0] = std::min(double(h[6]) / tt * 3, 1.0); u[1] = std::min(double(h[7]) / tt * 3, 1.0); u[2] = std::min(double(h[8]) / tt * 3, 1.0);
    u[3] = std::min((double(h[0]) + h[1]) / tr * 3, 1.0); u[4] = std::min((double(h[2]) + h[3]) / tr * 3, 1.0); u[5] = std::min((double(h[4]) + h[5]) / tr * 3, 1.0);
    if (tt == 0 || tr == 0) for (int i = 0; i < 6; ++i) u[i] = 0;
}

}  // extern "C"

// so_scan.cu -- scan preparation in front of the registration path (SURVEY 8f row 2), sm_90a:
//   k_deskew          featureExtraction::removePointDistortion<BufferType> (src/FeatureExtraction/featureExtraction.cpp:222-314)
//   k_uniform_flags / k_uniform_scatter
//                     featureExtraction::uniformFeatureExtraction (:504-525)
// Both are one thread per point over float4 {x, y, z, time} clouds in d_scan / d_scan_sorted; HBM-bound streaming work
// (32 B per point for the deskew; 16 B in + 4 B flag + 16 B out per kept point for the extraction).
#include <cub/cub.cuh>

#include "so_ctx.cuh"

namespace so {

// Eigen::QuaternionBase::slerp (xyzw); the caller normalises (Twist::transform() does, Twist.h:78-83).
__device__ __forceinline__ void slerp_xyzw(const double a[4], double t, const double b[4], double o[4]) {
    const double one = 1.0 - 2.220446049250313e-16;
    const double d = a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3];
    const double ad = fabs(d);
    double s0, s1;
    if (ad >= one) { s0 = 1.0 - t; s1 = t; }
    else {
        const double th = acos(ad), inv = 1.0 / sin(th);
        s0 = sin((1.0 - t) * th) * inv;
        s1 = sin(t * th) * inv;
    }
    if (d < 0) s1 = -s1;
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = s0 * a[k] + s1 * b[k];
}

__device__ __forceinline__ void normalize4(double q[4]) {
    const double s = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    q[0] *= s; q[1] *= s; q[2] *= s; q[3] *= s;
}

// One thread per point.  T_final = T_w_original^-1 * T_w_current (conjugated by the IMU-lidar extrinsic for IMU samples,
// :300-306).  The reference composes through 3x3 matrices and converts back to a quaternion at every product; the same
// rigid motions are composed here as quaternions (identical to ~1e-15 before the result is rounded to float).
__global__ void __launch_bounds__(256) k_deskew(float4* __restrict__ pts, uint32_t n, DeskewParams P) {
    extern __shared__ double s_times[];
    for (uint32_t k = threadIdx.x; k < P.n_smem; k += blockDim.x) s_times[k] = P.times[k];
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 p = pts[i];
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return;             // (:292-294)
    const double ts = double(p.w) + P.start_time;                                // point.time + lidar_start_time
    // std::map::upper_bound: first sample strictly later than ts
    uint32_t lo = 0, hi = P.n_samples;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        const double tm = mid < P.n_smem ? s_times[mid] : P.times[mid];
        if (tm > ts) hi = mid; else lo = mid + 1;
    }
    uint32_t after = lo;
    if (after == P.n_samples) { after = P.n_samples - 1; atomicAdd(P.past_end, 1u); }   // end() upstream (UB): last interval
    if ((after < P.n_smem ? s_times[after] : P.times[after]) < 0.0001) after = 0;       // (:258-260)
    double qc[4], pc[3];
    const double* A = P.poses + 7 * size_t(after);
    if (after == 0) {
        qc[0] = A[3]; qc[1] = A[4]; qc[2] = A[5]; qc[3] = A[6];
        pc[0] = A[0]; pc[1] = A[1]; pc[2] = A[2];
    } else {
        const double* B = A - 7;
        const double tb = (after - 1) < P.n_smem ? s_times[after - 1] : P.times[after - 1];
        const double ta = after < P.n_smem ? s_times[after] : P.times[after];
        const double ratio = (ts - tb) / (ta - tb);
        slerp_xyzw(B + 3, ratio, A + 3, qc);
#pragma unroll
        for (int k = 0; k < 3; ++k) pc[k] = (1 - ratio) * B[k] + ratio * A[k];
    }
    normalize4(qc);
    // T_oc = T_w_original^-1 * T_w_current
    double q[4], t[3];
    qmul(P.q0_conj, qc, q);
    if (P.imu_only) { t[0] = t[1] = t[2] = 0.0; }
    else {
        const double d[3] = {pc[0] - P.p0[0], pc[1] - P.p0[1], pc[2] - P.p0[2]};
        qrot(P.q0_conj, d, t);
    }
    if (P.imu_only) {
        // T_l_i * T_oc * T_i_l
        double q1[4], t1[3], r[3];
        qrot(q, P.t_il, r);                                  // T_oc * T_i_l
        t1[0] = r[0] + t[0]; t1[1] = r[1] + t[1]; t1[2] = r[2] + t[2];
        qmul(q, P.q_il, q1);
        qrot(P.q_li, t1, r);                                 // T_l_i * (...)
        t[0] = r[0] + P.t_li[0]; t[1] = r[1] + P.t_li[1]; t[2] = r[2] + P.t_li[2];
        qmul(P.q_li, q1, q);
    }
    normalize4(q);
    const double v[3] = {double(p.x), double(p.y), double(p.z)};
    double o[3];
    qrot(q, v, o);
    p.x = float(o[0] + t[0]); p.y = float(o[1] + t[1]); p.z = float(o[2] + t[2]);
    pts[i] = p;
}

void launch_deskew(float4* pts, uint32_t n, const DeskewParams& P, cudaStream_t st) {
    if (n) k_deskew<<<(n + 255) / 256, 256, P.n_smem * sizeof(double), st>>>(pts, n, P);
}

// Candidate j is point i = 1 + j * skip (the loop of :507); flag = the keep predicate of :515-518 with its literal
// precedence, a || b || (c && range), in plain IEEE float (no contraction).
__global__ void __launch_bounds__(256) k_uniform_flags(const float4* __restrict__ pts, uint32_t n_cand, uint32_t skip, float block_range2, int int_abs,
                                                       uint32_t* __restrict__ flags) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_cand) return;
    const size_t i = 1 + size_t(j) * skip;
    const float4 p = pts[i], q = pts[i - 1];
    const float dx = __fsub_rn(p.x, q.x), dy = __fsub_rn(p.y, q.y), dz = __fsub_rn(p.z, q.z);
    double ax, ay, az;
    if (int_abs) {
        // int(NaN / inf / |d| >= 2^31) is undefined upstream: such a difference counts as "no difference" (the oracle does the same)
        ax = (isfinite(dx) && fabsf(dx) < 2147483648.0f) ? double(abs(int(dx))) : 0.0;
        ay = (isfinite(dy) && fabsf(dy) < 2147483648.0f) ? double(abs(int(dy))) : 0.0;
        az = (isfinite(dz) && fabsf(dz) < 2147483648.0f) ? double(abs(int(dz))) : 0.0;
    }
    else { ax = double(fabsf(dx)); ay = double(fabsf(dy)); az = double(fabsf(dz)); }
    const float r2 = __fadd_rn(__fadd_rn(__fmul_rn(p.x, p.x), __fmul_rn(p.y, p.y)), __fmul_rn(p.z, p.z));
    flags[j] = (ax > 1e-7 || ay > 1e-7 || (az > 1e-7 && r2 > block_range2)) ? 1u : 0u;
}

__global__ void __launch_bounds__(256) k_uniform_scatter(const float4* __restrict__ pts, uint32_t n_cand, uint32_t skip, const uint32_t* __restrict__ flags,
                                                         const uint32_t* __restrict__ rank, float4* __restrict__ out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_cand || !flags[j]) return;
    out[rank[j]] = pts[1 + size_t(j) * skip];                   // {x, y, z, intensity = time}
}

// d_scan -> d_scan_sorted (compacted, input order).  Scratch: d_svals (flags), d_svals_out (ranks), d_sort_tmp.
int scan_extract_uniform(Ctx* c, uint32_t n, uint32_t skip, float block_range, int int_abs, uint32_t* n_out) {
    cudaStream_t st = c->stream;
    *n_out = 0;
    if (n < 2) return SO_OK;
    const uint32_t n_cand = (n - 2) / skip + 1;                 // i = 1, 1+skip, ... < n
    const uint32_t grid = (n_cand + 255) / 256;
    k_uniform_flags<<<grid, 256, 0, st>>>(c->d_scan, n_cand, skip, block_range * block_range, int_abs, c->d_svals);
    size_t tmp = c->d_sort_tmp.cap();
    SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->d_sort_tmp, tmp, c->d_svals.get(), c->d_svals_out.get(), int(n_cand), st));
    uint32_t last_flag = 0, last_rank = 0;
    SO_CUDA_TRY(cudaMemcpyAsync(&last_flag, c->d_svals + n_cand - 1, 4, cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaMemcpyAsync(&last_rank, c->d_svals_out + n_cand - 1, 4, cudaMemcpyDeviceToHost, st));
    c->prefiltered_n = SIZE_MAX;
    k_uniform_scatter<<<grid, 256, 0, st>>>(c->d_scan, n_cand, skip, c->d_svals, c->d_svals_out, c->d_scan_sorted);
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    *n_out = last_rank + last_flag;
    c->launches += 3;
    SO_CUDA_TRY(cudaGetLastError());
    return SO_OK;
}

}  // namespace so

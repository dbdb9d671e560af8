// so_undistort.cu -- within-scan motion compensation, sm_90a: the warp of every point by its scan's motion D over dt, shared by modes
// APPROXIMATED and OPTIMIZED (und_point, so_undistort.cuh; tests/undistort_numpy.py restates its bits).  With alpha_i =
// double(tau_i) / dt (0 for a non-finite tau_i):
//   q_i     = slerp(identity, q_D, alpha_i)     (Eigen's QuaternionBase::slerp; identity when rotation == 0)
//   u_i     = float3(qrot(q_i, p_i) + alpha_i * t_D)
// The two modes differ only in where D comes from (the sources FromPose and FromMotion below):
//   APPROXIMATED  the reference's UndistortionMode::APPROXIMATED (LidarSlam.h:65-82; its branch of ComputePointInitAndFinalPose,
//                 LidarSlam.cpp:382-400, is empty upstream), a constant body-velocity model: D = T_prev^-1 * T_cur with T_cur the
//                 scan's current estimate, q_D = normalise(conj(q_prev) * q_cur), t_D = qrot(conj(q_prev), t_cur - t_prev)
//   OPTIMIZED     D is the motion block so_motion.cu estimates, rotation always on
// Three forms, each templated on the source:
//   k_warp_scan    the head of every ICP iteration: one thread per active point of the ordered scans, writes d_scan_sorted (w kept)
//   k_warp_edges   the same for the edge cloud (so_register_*_edges): d_escan -> und.d_ewarp, same index
//   k_warp_cloud   a contiguous cloud: the map and keyframe insert after a compensated registration, so_undistort_points
#include <cmath>
#include <vector>

#include "so_undistort.cuh"

namespace so {

// A source answers for one scan: skip() -- its points are left as they are; setup(x, sh) -- sh of D on the CTA's thread 0, x being
// the pose the points are warped at; params() -- und_point's dt and rotation.  The forms are templated on it rather than branching on
// the mode, so that each mode's kernels keep their own register allocation.

// APPROXIMATED: D = T_prev^-1 * T(x) from the scan's UndistortParams (und_setup); a scan with on == 0 is skipped
struct FromPose {
    UndistortParams P;
    __device__ explicit FromPose(const UndistortParams& p) : P(p) {}
    __device__ bool skip() const { return !P.on; }
    __device__ void setup(const double x[7], double sh[9]) const { und_setup(P, x, sh); }
    __device__ UndistortParams params() const { return P; }
};

// OPTIMIZED: D and dt of a MotionState or MotionD (motion_setup), whatever the pose; held by address, so each is read only where used
struct FromMotion {
    const double* D;
    const double* dt;
    template <class M> __device__ explicit FromMotion(const M& m) : D(m.D), dt(&m.dt) {}
    __device__ bool skip() const { return false; }
    __device__ void setup(const double*, double sh[9]) const { motion_setup(D, sh); }
    __device__ UndistortParams params() const {
        UndistortParams P{};
        P.dt = *dt; P.on = 1; P.rotation = 1;
        return P;
    }
};

// One thread per active point, CTAs laid out per scan like the other per-point kernels; exits at once for scans that are not in
// PH_CORR or that the source skips.  The raw point and its time are gathered from the upload buffers by the original index that scan
// ordering left in w (no ordered raw copy, so the ordering kernels stay as they are): ~52 B per point -- the ordered slot (16 B read
// for w), the raw point and its time (20 B, gathered), the store (16 B).
template <class Src, class Rec>
__global__ void __launch_bounds__(kThreads) k_warp_scan(BatchView bv, float4* __restrict__ sorted, const float4* __restrict__ raw,
                                                        const float* __restrict__ times, const Rec* __restrict__ rec) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    const Src src(rec[s]);
    if (src.skip()) return;
    const uint32_t n = uint32_t(st->n_points);
    if (blockIdx.x * kThreads >= n) return;
    __shared__ double sh[9];
    if (threadIdx.x == 0) src.setup(st->x, sh);
    __syncthreads();
    const UndistortParams P = src.params();
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const size_t base = size_t(bv.offset[s]), gi = base + i;
    const float w = sorted[gi].w;
    const size_t src_i = base + __float_as_uint(w);                      // original index (k_scan_gather / k_prepare_small)
    float4 o = und_point(P, sh, __ldg(&raw[src_i]), __ldg(&times[src_i]));
    o.w = w;
    sorted[gi] = o;
}

// The edge cloud: one thread per edge point; the edge cloud is not reordered, so raw point, time and output share the index.
// k_edge_fit / k_edge_evaluate then read `out` as their sensor-frame cloud.
template <class Src, class Rec>
__global__ void __launch_bounds__(kThreads) k_warp_edges(BatchView bv, const uint32_t* __restrict__ eoffset, float4* __restrict__ out,
                                                         const float4* __restrict__ raw, const float* __restrict__ times,
                                                         const Rec* __restrict__ rec) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    const Src src(rec[s]);
    if (src.skip()) return;
    const uint32_t n = uint32_t(st->n_edge);
    if (blockIdx.x * kThreads >= n) return;
    __shared__ double sh[9];
    if (threadIdx.x == 0) src.setup(st->x, sh);
    __syncthreads();
    const UndistortParams P = src.params();
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const size_t gi = size_t(eoffset[s]) + i;
    out[gi] = und_point(P, sh, __ldg(&raw[gi]), __ldg(&times[gi]));
}

struct UndPose { double v[7]; };
template <class Src, class Rec>
__global__ void __launch_bounds__(256) k_warp_cloud(float4* __restrict__ pts, const float* __restrict__ times, uint32_t n, Rec r, UndPose x) {
    const Src src(r);
    __shared__ double sh[9];
    if (threadIdx.x == 0) src.setup(x.v, sh);
    __syncthreads();
    const UndistortParams P = src.params();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pts[i] = und_point(P, sh, pts[i], times[i]);
}

template <class Src, class Rec>
static uint32_t launch_warp_from(const Ctx* c, const BatchView& bv, const uint32_t* eoffset, const Rec* rec, uint32_t grid_x, uint32_t grid_e,
                                 uint32_t n_scans, cudaStream_t st) {
    k_warp_scan<Src><<<dim3(grid_x, n_scans), kThreads, 0, st>>>(bv, c->d_scan_sorted, c->d_scan, c->und.d_time, rec);
    if (!grid_e) return 1;
    k_warp_edges<Src><<<dim3(grid_e, n_scans), kThreads, 0, st>>>(bv, eoffset, c->und.d_ewarp, c->d_escan, c->und.d_etime, rec);
    return 2;
}

uint32_t launch_warp(const Ctx* c, UndistortionMode mode, const BatchView& bv, const uint32_t* eoffset, uint32_t first, uint32_t grid_x,
                     uint32_t grid_e, uint32_t n_scans, cudaStream_t st) {
    if (mode == UndistortionMode::OPTIMIZED) return launch_warp_from<FromMotion>(c, bv, eoffset, c->mot.d_st + first, grid_x, grid_e, n_scans, st);
    return launch_warp_from<FromPose>(c, bv, eoffset, c->und.d_par + first, grid_x, grid_e, n_scans, st);
}

int warp_cloud(Ctx* c, float4* pts, const float* times, uint32_t n, const CloudWarp& w, const double pose[7]) {
    if (w.mode == UndistortionMode::NONE || !n) return SO_OK;
    UndPose x;
    for (int k = 0; k < 7; ++k) x.v[k] = pose[k];
    const uint32_t grid = (n + 255) / 256;
    timed_launch_begin(c);
    if (w.mode == UndistortionMode::OPTIMIZED) k_warp_cloud<FromMotion><<<grid, 256, 0, c->stream>>>(pts, times, n, w.motion, x);
    else k_warp_cloud<FromPose><<<grid, 256, 0, c->stream>>>(pts, times, n, w.par, x);
    timed_launch_end(c, 7, 1);
    SO_CUDA_TRY(cudaGetLastError());
    return SO_OK;
}


// ------------------------------------------------------------------------------------------------------------------ host side
bool finite_pose(const double p[7]) {
    for (int k = 0; k < 7; ++k) if (!std::isfinite(p[k])) return false;
    return p[3] * p[3] + p[4] * p[4] + p[5] * p[5] + p[6] * p[6] > 0.0;
}

int check_undistort(const so_undistort* u) {
    if (!u) return fail(SO_ERR_ARG, "bad args");
    if (u->mode == 2) return fail(SO_ERR_ARG, "so_undistort.mode 2 (OPTIMIZED) estimates a second pose: use so_register_optimized");
    if (u->mode != 0 && u->mode != 1) return fail(SO_ERR_ARG, "so_undistort.mode must be 0 (NONE) or 1 (APPROXIMATED)");
    if (u->mode == 0) return SO_OK;
    if (u->rotation != 0 && u->rotation != 1) return fail(SO_ERR_ARG, "so_undistort.rotation must be 0 or 1");
    if (!(std::isfinite(u->dt) && u->dt > 0.0)) return fail(SO_ERR_ARG, "so_undistort.dt must be finite and > 0");
    if (!finite_pose(u->prev_pose)) return fail(SO_ERR_ARG, "so_undistort.prev_pose must be finite with a non-zero quaternion");
    return SO_OK;
}

UndistortParams make_params(const so_undistort& u) {
    UndistortParams P{};
    P.on = u.mode == 1 ? 1 : 0;
    if (!P.on) return P;
    P.q_prev_conj[0] = -u.prev_pose[3]; P.q_prev_conj[1] = -u.prev_pose[4]; P.q_prev_conj[2] = -u.prev_pose[5]; P.q_prev_conj[3] = u.prev_pose[6];
    for (int a = 0; a < 3; ++a) P.t_prev[a] = u.prev_pose[a];
    P.dt = u.dt;
    P.rotation = u.rotation;
    return P;
}

// The float at byte time_offset of every record -> dst (device)
int upload_times(Ctx* c, const void* src, size_t n, size_t stride, size_t toff, float* dst) {
    if (n == 0) return SO_OK;
    std::vector<float> h(n);
    const unsigned char* p = static_cast<const unsigned char*>(src) + toff;
    for (size_t i = 0; i < n; ++i, p += stride) std::memcpy(&h[i], p, 4);
    SO_CUDA_TRY(cudaMemcpyAsync(dst, h.data(), n * sizeof(float), cudaMemcpyHostToDevice, c->stream));   // pageable: staged before return
    count_h2d(c, n * sizeof(float));
    return SO_OK;
}

int undistort_reserve(Ctx* c, size_t n_points) {
    int rc = c->und.d_par.reserve(c->max_batch);
    if (!rc) rc = c->und.d_time.reserve(std::max<size_t>(n_points, 1));
    return rc;
}

// Sized to the edge capacity on first use and never regrown, so that a captured schedule's pointer to d_ewarp stays valid
int undistort_edge_reserve(Ctx* c) {
    int rc = c->und.d_etime.reserve(std::max<size_t>(c->edge_cap, 1));
    if (!rc) rc = c->und.d_ewarp.reserve(std::max<size_t>(c->edge_cap, 1));
    return rc;
}

}  // namespace so

using namespace so;

extern "C" {

int so_undistort_points(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, size_t toff, const double pose[7],
                        const so_undistort* u, float* out_xyzi) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose || (n && (!xyzi || !out_xyzi)) || stride < 12 || toff + 4 > stride || !finite_pose(pose)) return fail(SO_ERR_ARG, "bad args");
    int rc = check_undistort(u);
    if (rc) return rc;
    if (n > c->scan_cap) return fail(SO_ERR_CAPACITY, "cloud larger than the context's scan capacity");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    if (n == 0) return SO_OK;
    rc = c->und.d_hook.reserve(n);
    if (!rc) rc = c->und.d_hook_time.reserve(n);
    if (!rc) rc = upload_cloud(c, xyzi, n, stride, ioff, c->und.d_hook);
    if (!rc) rc = upload_times(c, xyzi, n, stride, toff, c->und.d_hook_time);
    if (rc) return rc;
    CloudWarp w;
    if (u->mode == 1) { w.mode = UndistortionMode::APPROXIMATED; w.par = make_params(*u); }
    rc = warp_cloud(c, c->und.d_hook, c->und.d_hook_time, uint32_t(n), w, pose);
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemcpyAsync(out_xyzi, c->und.d_hook, n * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    count_d2h(c, n * sizeof(float4));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SO_OK;
}

}  // extern "C"

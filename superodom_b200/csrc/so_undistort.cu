// so_undistort.cu -- within-scan motion compensation inside the registration: the reference's UndistortionMode::APPROXIMATED
// (LidarSlam.h:65-82; its branch of ComputePointInitAndFinalPose, LidarSlam.cpp:382-400, is empty upstream), sm_90a.
//
// A constant body-velocity model.  At the start of every ICP iteration, with T_cur the scan's current estimate:
//   D       = T_prev^-1 * T_cur                 q_D = normalise(conj(q_prev) * q_cur), t_D = qrot(conj(q_prev), t_cur - t_prev)
//   alpha_i = double(tau_i) / dt                (a non-finite tau_i gives 0)
//   q_i     = slerp(identity, q_D, alpha_i)     (Eigen's QuaternionBase::slerp; identity when rotation == 0)
//   pInit_i = float3(qrot(q_i, p_i) + alpha_i * t_D)
// and the iteration runs on pInit in place of p (und_point, so_undistort.cuh; tests/undistort_numpy.py restates its bits).
//   k_undistort        the ICP form: one thread per active point of the ordered scans, writes d_scan_sorted (w kept)
//   k_undistort_edges  the ICP form for the edge cloud (so_register_undistort_edges): d_escan -> und.d_ewarp, same index
//   k_undistort_cloud  a contiguous cloud at a given pose: the map insert after an undistorted registration, so_undistort_points
#include <cmath>
#include <vector>

#include "so_undistort.cuh"

namespace so {

// One thread per active point, CTAs laid out per scan like the other per-point kernels; exits at once for scans that are not in
// PH_CORR or not undistorted.  The raw point and its time are gathered from the upload buffers by the original index that scan
// ordering left in w (no ordered raw copy, so the ordering kernels stay as they are): ~52 B per point -- the ordered slot
// (16 B read for w), the raw point and its time (20 B, gathered), the store (16 B).
__global__ void __launch_bounds__(kThreads) k_undistort(BatchView bv, float4* __restrict__ sorted, const float4* __restrict__ raw,
                                                        const float* __restrict__ times, const UndistortParams* __restrict__ par) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    const UndistortParams P = par[s];
    if (!P.on) return;
    const uint32_t n = uint32_t(st->n_points);
    if (blockIdx.x * kThreads >= n) return;
    __shared__ double sh[9];
    if (threadIdx.x == 0) und_setup(P, st->x, sh);
    __syncthreads();
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const size_t base = size_t(bv.offset[s]), gi = base + i;
    const float w = sorted[gi].w;
    const size_t src = base + __float_as_uint(w);                        // original index (k_scan_gather / k_prepare_small)
    float4 o = und_point(P, sh, __ldg(&raw[src]), __ldg(&times[src]));
    o.w = w;
    sorted[gi] = o;
}

void launch_undistort(const BatchView& bv, float4* sorted, const float4* raw, const float* times, const UndistortParams* par,
                      uint32_t grid_x, uint32_t n_scans, cudaStream_t st) {
    k_undistort<<<dim3(grid_x, n_scans), kThreads, 0, st>>>(bv, sorted, raw, times, par);
}

// The same warp for the edge cloud (so_register_undistort_edges): one thread per edge point; the edge cloud is not reordered, so
// raw point, time and output share the index.  k_edge_fit / k_edge_evaluate then read `out` as their sensor-frame cloud.
__global__ void __launch_bounds__(kThreads) k_undistort_edges(BatchView bv, const uint32_t* __restrict__ eoffset, float4* __restrict__ out,
                                                              const float4* __restrict__ raw, const float* __restrict__ times,
                                                              const UndistortParams* __restrict__ par) {
    const int s = blockIdx.y;
    const IcpState* st = bv.st + s;
    if (st->phase != PH_CORR) return;
    const UndistortParams P = par[s];
    if (!P.on) return;
    const uint32_t n = uint32_t(st->n_edge);
    if (blockIdx.x * kThreads >= n) return;
    __shared__ double sh[9];
    if (threadIdx.x == 0) und_setup(P, st->x, sh);
    __syncthreads();
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const size_t gi = size_t(eoffset[s]) + i;
    out[gi] = und_point(P, sh, __ldg(&raw[gi]), __ldg(&times[gi]));
}

void launch_undistort_edges(const BatchView& bv, const uint32_t* eoffset, float4* out, const float4* raw, const float* times,
                            const UndistortParams* par, uint32_t grid_e, uint32_t n_scans, cudaStream_t st) {
    k_undistort_edges<<<dim3(grid_e, n_scans), kThreads, 0, st>>>(bv, eoffset, out, raw, times, par);
}

struct UndPose { double v[7]; };
__global__ void __launch_bounds__(256) k_undistort_cloud(float4* __restrict__ pts, const float* __restrict__ times, uint32_t n,
                                                         UndistortParams P, UndPose x) {
    __shared__ double sh[9];
    if (threadIdx.x == 0) und_setup(P, x.v, sh);
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pts[i] = und_point(P, sh, pts[i], times[i]);
}

static void launch_undistort_cloud(Ctx* c, float4* pts, const float* times, uint32_t n, const UndistortParams& P, const double pose[7]) {
    UndPose x;
    for (int k = 0; k < 7; ++k) x.v[k] = pose[k];
    if (!n) return;
    timed_launch_begin(c);
    k_undistort_cloud<<<(n + 255) / 256, 256, 0, c->stream>>>(pts, times, n, P, x);
    timed_launch_end(c, 7);                                               // counts the launch
}

int undistort_tail(Ctx* c, float4* dst, const RegisteredScan& r, const double pose[7]) {
    launch_undistort_cloud(c, dst, c->und.d_time, r.n, r.par, pose);
    SO_CUDA_TRY(cudaGetLastError());
    return SO_OK;
}

int undistort_edge_tail(Ctx* c, float4* dst, const RegisteredScan& r, const double pose[7]) {
    launch_undistort_cloud(c, dst, c->und.d_etime, r.n_edge, r.par, pose);
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
    if (u->mode == 1) launch_undistort_cloud(c, c->und.d_hook, c->und.d_hook_time, uint32_t(n), make_params(*u), pose);
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaMemcpyAsync(out_xyzi, c->und.d_hook, n * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    count_d2h(c, n * sizeof(float4));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SO_OK;
}

}  // extern "C"

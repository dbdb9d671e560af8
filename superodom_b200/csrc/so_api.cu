// so_api.cu -- the C ABI (include/superodom_b200.h): context, uploads, the CUDA-graph ICP schedule, results.  Global localization
// (so_localize_*) is in so_global.cu.
// Host code above the kernels stays C++ (the reference's host language); no torch types anywhere.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "so_ctx.cuh"
#include "so_chunks.h"
#include "so_knn.cuh"

namespace so {

static thread_local std::string g_err;
void set_error(const std::string& s) { g_err = s; }

int fail(int code, const std::string& msg) { set_error(msg); return code; }

// ---------------------------------------------------------------------------------------------- host pose helpers
// tf2 Matrix3x3(q).getRPY of the quaternion {x, y, z, w}
void tf2_get_rpy(const double q[4], double* roll_out, double* pitch_out, double* yaw_out) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double d = x * x + y * y + z * z + w * w, s = 2.0 / d;
    const double xs = x * s, ys = y * s, zs = z * s, wx = w * xs, wy = w * ys, wz = w * zs;
    const double xx = x * xs, xy = x * ys, xz = x * zs, yy = y * ys, yz = y * zs, zz = z * zs;
    const double m00 = 1.0 - (yy + zz), m01 = xy - wz, m02 = xz + wy, m10 = xy + wz, m20 = xz - wy, m21 = yz + wx, m22 = 1.0 - (xx + yy);
    double roll, pitch, yaw;
    if (std::fabs(m20) >= 1) {
        yaw = 0;
        if (m20 < 0) { pitch = M_PI / 2.0; roll = std::atan2(m01, m02); }
        else { pitch = -M_PI / 2.0; roll = std::atan2(-m01, -m02); }
    } else {
        pitch = -std::asin(m20);
        roll = std::atan2(m21 / std::cos(pitch), m22 / std::cos(pitch));
        yaw = std::atan2(m10 / std::cos(pitch), m00 / std::cos(pitch));
    }
    *roll_out = roll; *pitch_out = pitch; *yaw_out = yaw;
}

// tf2 Matrix3x3(q).getRPY + Quaternion::setRPY round trip: LidarSLAM::MannualYawCorrection (LidarSlam.cpp:891-913)
static void manual_yaw_correction(const double last[7], double T[7], double yaw_ratio) {
    double tn, rn;
    rel_motion(last, T, &tn, &rn);
    const float translation_norm = float(tn);
    double roll, pitch, yaw;
    tf2_get_rpy(T + 3, &roll, &pitch, &yaw);
    const double cyaw = yaw + double(translation_norm) * yaw_ratio * M_PI / 180;
    const double hy = cyaw * 0.5, hp = pitch * 0.5, hr = roll * 0.5;
    const double cy = std::cos(hy), sy = std::sin(hy), cp = std::cos(hp), sp = std::sin(hp), cr = std::cos(hr), sr = std::sin(hr);
    double q[4] = {sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy};
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int i = 0; i < 4; ++i) T[3 + i] = q[i] / n;
}

static inline int block_coord_h(double v, int origin) { int c = int(v / kBlock); if (v < 0) c--; return c + origin; }

// LocalMap::get5x5LocalMapFeatureSize (LocalMap.h:291-318) on the host mirror of the block counts
static int counts_5x5(const Ctx* c, const MapStore& ms, const int32_t ijk[3]) {
    (void)c;
    int n = 0;
    for (int i = ijk[0] - 2; i <= ijk[0] + 2; ++i)
        for (int j = ijk[1] - 2; j <= ijk[1] + 2; ++j)
            for (int k = ijk[2] - 1; k <= ijk[2] + 1; ++k)
                if (i >= 0 && i < kW && j >= 0 && j < kH && k >= 0 && k < kD) n += ms.h_block_count[i + kW * j + kW * kH * k];
    return n;
}

int ensure_maps(Ctx* c) {
    if (c->surf.dirty) { int rc = map_rebuild(c, c->surf); if (rc) return rc; }
    if (c->edge.dirty) { int rc = map_rebuild(c, c->edge); if (rc) return rc; }
    return SO_OK;
}

void shift_origin(const int32_t o[3], const double t[3], int32_t out[3], int32_t cc_out[3]) {
    const int dims[3] = {kW, kH, kD};
    for (int a = 0; a < 3; ++a) {                           // LocalMap::shiftMap (LocalMap.h:169-287)
        int cc = block_coord_h(t[a] + kHalfBlock, o[a]), shift = 0;
        while (cc < 3) { cc++; shift++; }
        while (cc >= dims[a] - 3) { cc--; shift--; }
        out[a] = o[a] + shift;
        if (cc_out) cc_out[a] = cc;
    }
}

int move_window(Ctx* c, const int32_t o[3]) {
    if (o[0] != c->origin[0] || o[1] != c->origin[1] || o[2] != c->origin[2]) {
        for (int a = 0; a < 3; ++a) c->origin[a] = o[a];
        c->surf.dirty = true; c->edge.dirty = true;
    }
    return ensure_maps(c);
}

// ---------------------------------------------------------------------------------------------- allocation
static int ctx_alloc(Ctx* c) {
    SO_CUDA_TRY(cudaSetDevice(c->device));
    SO_CUDA_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    int rc = c->ev0.create();
    if (!rc) rc = c->ev1.create();
    if (!rc) rc = c->evp0.create();
    if (!rc) rc = c->evp1.create();
    if (rc) return rc;
    SO_CUDA_TRY(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    SO_CUDA_TRY(cudaStreamCreateWithFlags(&c->aux_stream, cudaStreamNonBlocking));
    rc = c->ev_fork.create(cudaEventDisableTiming);
    if (!rc) rc = c->ev_join.create(cudaEventDisableTiming);
    for (Event& e : c->ev_copy) if (!rc) rc = e.create(cudaEventDisableTiming);
    if (!rc) rc = map_alloc(c);
    if (rc) return rc;
    c->max_batch = c->cfg.max_batch;
    c->scan_cap = size_t(c->cfg.max_scan_points) * c->max_batch;
    c->grid_x_cap = (c->cfg.max_scan_points + kThreads - 1) / kThreads;
    rc = c->d_scan.reserve(c->scan_cap);
    if (!rc) rc = c->d_dec.reserve(kPrepareSmallCap);
    if (!rc) rc = c->ev_dec.create(cudaEventDisableTiming);
    if (!rc) rc = c->d_scan_sorted.reserve(c->scan_cap);
    if (!rc) rc = c->d_skeys.reserve(c->scan_cap);
    if (!rc) rc = c->d_skeys_out.reserve(c->scan_cap);
    if (!rc) rc = c->d_svals.reserve(c->scan_cap);
    if (!rc) rc = c->d_svals_out.reserve(c->scan_cap);
    if (!rc) rc = c->d_nn_pos.reserve(c->scan_cap * 5);
    if (!rc) rc = c->d_nn_d5.reserve(c->scan_cap);
    if (!rc) rc = c->d_nn_pre.reserve(c->scan_cap);
    if (!rc) rc = scan_sort_alloc(c);
    if (!rc) rc = c->d_offset.reserve(c->max_batch);
    if (!rc) rc = c->d_state.reserve(c->max_batch);
    if (!rc) rc = c->h_state.reserve(c->max_batch);
    if (!rc) rc = c->h_offset.reserve(2 * size_t(c->max_batch));       // [0, max_batch): scan offsets; then the edge clouds' offsets
    if (rc) return rc;
    c->nn.pos = c->d_nn_pos; c->nn.d5 = c->d_nn_d5; c->nn.pre = c->d_nn_pre; c->nn.cap = c->scan_cap;
    c->h_eoffset = c->h_offset + c->max_batch;
    c->edge_cap = c->cfg.max_scan_points;
    c->edge_grid_cap = uint32_t((c->edge_cap + kThreads - 1) / kThreads);
    rc = c->d_partials.reserve(size_t(c->max_batch) * (c->grid_x_cap + c->edge_grid_cap) * kAcc);
    if (!rc) rc = c->d_escan.reserve(c->edge_cap);
    if (!rc) rc = c->d_eoffset.reserve(c->max_batch);
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemset(c->d_eoffset, 0, c->max_batch * sizeof(uint32_t)));
    rc = c->d_ebuf_a.reserve(c->edge_cap);
    if (!rc) rc = c->d_ebuf_b.reserve(c->edge_cap);
    if (!rc) rc = c->d_ebuf_flags.reserve(c->edge_cap);
    if (!rc) rc = c->d_ebuf_nn.reserve(c->edge_cap * 10);
    if (!rc) rc = c->d_ebuf_selmask.reserve(c->edge_cap);
    if (rc) return rc;
    c->ebuf.a = c->d_ebuf_a; c->ebuf.b = c->d_ebuf_b; c->ebuf.flags = c->d_ebuf_flags; c->ebuf.nn = c->d_ebuf_nn; c->ebuf.selmask = c->d_ebuf_selmask;
    c->ebuf.scan = c->d_escan; c->ebuf.offset = c->d_eoffset;
    rc = c->d_counters.reserve(c->max_batch);
    if (!rc) rc = c->d_hist.reserve(size_t(c->max_batch) * kHistStride);
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemset(c->d_counters, 0, c->max_batch * sizeof(uint32_t)));
    SO_CUDA_TRY(cudaMemset(c->d_hist, 0, c->max_batch * kHistStride * sizeof(int32_t)));
    const size_t slots = corr_tile_cap(c->scan_cap, c->max_batch) * kCorrTile;
    rc = c->d_corr_x.reserve(slots * 4);
    if (!rc) rc = c->d_corr_w.reserve(slots);
    if (!rc) rc = c->d_corr_p.reserve(slots * 3);
    if (!rc) rc = c->d_corr_flags.reserve(c->scan_cap);
    if (!rc) rc = c->d_corr_nn.reserve(size_t(c->cfg.max_scan_points) * 5);
    if (!rc) rc = c->d_corr_nn_d2.reserve(size_t(c->cfg.max_scan_points) * 5);
    if (rc) return rc;
    c->corr.x = c->d_corr_x; c->corr.w = c->d_corr_w; c->corr.p = c->d_corr_p; c->corr.flags = c->d_corr_flags; c->corr.nn = c->d_corr_nn; c->corr.nn_d2 = c->d_corr_nn_d2;
    return SO_OK;
}

// The buffers and events free themselves with the context; the streams and graph execs are freed here
static void ctx_free(Ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    for (auto& g : c->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    if (c->aux_stream) cudaStreamDestroy(c->aux_stream);
    if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

static int ensure_stage(Ctx* c, size_t n) {
    if (n <= c->h_stage.cap()) return SO_OK;
    if (c->h_stage) cudaDeviceSynchronize();           // no copy out of the old buffer may still be in flight
    return c->h_stage.reserve(n);
}

// Copy a strided host cloud into device float4 {x,y,z,intensity}.  Packed float4 input goes straight through.
int upload_cloud(Ctx* c, const void* src, size_t n, size_t stride, size_t ioff, float4* dst) {
    if (n == 0) return SO_OK;
    if (stride == 16 && ioff == 12) {
        SO_CUDA_TRY(cudaMemcpyAsync(dst, src, n * sizeof(float4), cudaMemcpyHostToDevice, c->stream));
        c->bytes_h2d += n * sizeof(float4);
        return SO_OK;
    }
    int rc = ensure_stage(c, n);
    if (rc) return rc;
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));     // staging buffer reuse
    float4* h = c->h_stage;
    const unsigned char* p = static_cast<const unsigned char*>(src);
    for (size_t i = 0; i < n; ++i, p += stride) {
        float xyz[3], it = 0.f;
        std::memcpy(xyz, p, 12);
        if (ioff + 4 <= stride) std::memcpy(&it, p + ioff, 4);
        h[i] = make_float4(xyz[0], xyz[1], xyz[2], it);
    }
    SO_CUDA_TRY(cudaMemcpyAsync(dst, h, n * sizeof(float4), cudaMemcpyHostToDevice, c->stream));
    c->bytes_h2d += n * sizeof(float4);
    return SO_OK;
}

// shouldProcessPoint (LidarSlam.cpp:353-359) on the host: the same three IEEE operations as so_icp.cu's should_process (no FMA)
static inline bool should_process_h(uint32_t i, double rate) {
    const double x = double(i) * rate;
    const double rem = x - double(int64_t(x));            // x >= 0 and < 2^32: truncation == floor
    return !(rem + 0.001 > rate);
}

// Indices shouldProcessPoint keeps of an n-point scan capped at max_features (ascending).  A function of (n, max_features) only,
// so the list of the last call is kept.
static const std::vector<uint32_t>& decimation_list(Ctx* c, uint32_t n, int32_t max_features) {
    if (c->dec_n == n && c->dec_mf == max_features && !c->dec_idx.empty()) return c->dec_idx;
    const double rate = 1.0 * max_features / double(n);       // calculateSamplingRate (LidarSlam.cpp:346-351)
    c->dec_idx.clear();
    for (uint32_t i = 0; i < n; ++i) if (should_process_h(i, rate)) c->dec_idx.push_back(i);
    c->dec_n = n; c->dec_mf = max_features;
    return c->dec_idx;
}

// The pending whole-cloud upload of a decimated so_register (Ctx::defer), on the COPY stream: it only has to land before the scan
// is inserted, so it runs beside the registration instead of in front of it.  No-op when nothing is pending.
static int run_deferred_upload(Ctx* c) {
    if (!c->defer.src) return SO_OK;
    const void* src = c->defer.src;
    c->defer.src = nullptr;
    const size_t n = c->defer.n;
    if (c->defer.stride == 16 && c->defer.ioff == 12) {
        SO_CUDA_TRY(cudaMemcpyAsync(c->d_scan, src, n * sizeof(float4), cudaMemcpyHostToDevice, c->copy_stream));
    } else {
        float4* h = c->h_stage + c->defer.stage_off;
        const unsigned char* p = static_cast<const unsigned char*>(src);
        for (size_t i = 0; i < n; ++i, p += c->defer.stride) h[i] = read_point(p, c->defer.stride, c->defer.ioff);
        SO_CUDA_TRY(cudaMemcpyAsync(c->d_scan, h, n * sizeof(float4), cudaMemcpyHostToDevice, c->copy_stream));
    }
    c->bytes_h2d += n * sizeof(float4);
    SO_CUDA_TRY(cudaEventRecord(c->ev_dec, c->copy_stream));
    return SO_OK;
}

// ---------------------------------------------------------------------------------------------- ICP schedule
static BatchView batch_view(const Ctx* c, const float4* scan, uint32_t first = 0) {
    BatchView bv;
    bv.scan = scan; bv.offset = c->d_offset + first; bv.st = c->d_state + first;
    bv.partial_stride = c->grid_x_cap + c->edge_grid_cap; bv.edge_partial_offset = c->grid_x_cap;
    bv.partials = c->d_partials + size_t(first) * bv.partial_stride * kAcc; bv.hist = c->d_hist + size_t(first) * kHistStride;
    const double a = double(std::sqrt(3 * c->surf.res));     // float sqrt of a float product (LidarSlam.cpp:271)
    bv.tukey_a2 = a * a;
    const double al = double(std::sqrt(3 * c->edge.res));     // TukeyLoss(std::sqrt(3*lineRes_)) (LidarSlam.cpp:263)
    bv.tukey_a2_line = al * al;
    bv.counters = nullptr;
    return bv;
}

void count_h2d(Ctx* c, size_t b) { c->bytes_h2d += b; }
void count_d2h(Ctx* c, size_t b) { c->bytes_d2h += b; }

void timed_launch_begin(Ctx* c) { if (c->profiling) cudaEventRecord(c->evp0, c->stream); }
void timed_launch_end(Ctx* c, int cls, uint32_t n) {
    c->launches += n;
    if (!c->profiling) return;
    cudaEventRecord(c->evp1, c->stream);
    cudaEventSynchronize(c->evp1);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, c->evp0, c->evp1);
    c->prof[cls].ms += ms; c->prof[cls].launches++;
}

// With a valid neighbour graph the searches of a call queue the queries it does not answer (k_knn_scan<true>): the queue and the
// per-scan, per-iteration queue lengths of the call's n_scans scans, zeroed.
static int graph_queue_begin(Ctx* c, size_t n_scans) {
    if (!knn_graph_valid(c)) return SO_OK;
    int rc = c->d_nn_queue.reserve(c->scan_cap);
    if (!rc) rc = c->d_nn_qcount.reserve(size_t(c->max_batch) * SO_MAX_ICP_ITERS);
    if (rc) return rc;
    c->nn.queue = c->d_nn_queue; c->nn.qcount = c->d_nn_qcount;
    SO_CUDA_TRY(cudaMemsetAsync(c->nn.qcount, 0, n_scans * SO_MAX_ICP_ITERS * sizeof(uint32_t), c->stream));
    return SO_OK;
}

// A contiguous run of scans of the batch that is uploaded, ordered and registered together.
// grid_in: CTAs covering the longest scan as uploaded (scan ordering); small: every scan's survivors fit k_prepare_small.
// grid_x, fused, coop: set by plan_chunk
struct Chunk {
    uint32_t first, count, pt_first, pt_count, grid_x = 0, grid_e = 0, grid_in = 0; bool small = false; uint32_t max_kept = 0;
    bool fused = false, coop = false;
};

// The choices the ICP kernels of a chunk make, made once for the registration and the stage calls.  max_pts: the points of the
// chunk's longest scan the ICP kernels cover; own_step: the solves keep a step kernel of their own (mode OPTIMIZED, the
// degeneracy-aware step, the stage calls).
//   grid_x  CTAs covering max_pts, rounded up to a bucket of 16 CTAs so that scans of slightly different sizes (live SLAM: every
//           scan differs) share one captured graph; the kernels guard i < n_points and k_lm_step sums only the partial rows
//           n_points implies
//   fused   one or two scans in flight are launch-latency bound: the optimiser step is folded into the evaluation kernels
//           (k_evaluate_lm, which launch_first_eval / launch_evaluate take when the chunk has no edge cloud)
//   coop    the latency-bound search: a warp per query (k_knn_scan_coop)
static void plan_chunk(const Ctx* c, Chunk& ch, uint32_t max_pts, bool own_step) {
    const uint32_t g = (max_pts + kThreads - 1) / kThreads;
    ch.grid_x = g ? std::min<uint32_t>(c->grid_x_cap, (g + 15u) & ~15u) : 0;
    ch.fused = ch.count <= 2 && !c->profiling && !c->no_fused_lm && !own_step;
    ch.coop = ch.count <= 2 && ch.grid_x <= kCoopMaxGrid && !c->no_coop_knn;
}

// The BatchView of the chunk's scans in `scan`, with the chunk's choices
static BatchView chunk_view(const Ctx* c, const float4* scan, const Chunk& ch) {
    BatchView bv = batch_view(c, scan, ch.first);
    if (ch.fused) bv.counters = c->d_counters + ch.first;
    bv.coop_knn = ch.coop;
    return bv;
}

// Once per registration: order every scan by map cell at its prior pose (k_scan_keys -> radix sort -> k_scan_gather, or the one-CTA
// k_prepare_small for small registrations).  compact: drop the points the decimation skips here, once, instead of in every kernel.
// The dropped bit is only carried when a scan of the chunk is capped: without one it is zero in every key and k_scan_finish changes
// nothing, and leaving it out keeps 128-scan chunks of the 1 M-point map at 25 + 7 = 32 bits -- 32-bit keys, 4 radix passes over
// 8-byte pairs instead of 5 over 12-byte ones -- for the same permutation.
static int prepare_scans(Ctx* c, const float4* d_scan_in, const Chunk& ch, cudaStream_t st, bool compact) {
    c->prefiltered_n = SIZE_MAX;                                   // d_scan_sorted is about to be overwritten
    const MapView mv = map_view(c, c->surf);
    const BatchView bv = batch_view(c, d_scan_in, ch.first);
    timed_launch_begin(c);
    // key layout: [scan inside the chunk | dropped (compact only) | cell]; 32-bit keys whenever everything fits
    const uint64_t n_cells = scan_key_space(c->surf.n_slots, mv.nb);       // cell-order keys (so_knn.cuh)
    int cell_bits = 1, scan_bits = 0;
    while (cell_bits < 32 && (uint64_t(1) << cell_bits) <= n_cells) ++cell_bits;       // cells 0..n_cells-1 < mask = 2^cell_bits - 1
    if (compact && ch.small && !c->no_small_prepare) {
        timed_launch_end(c, 3, launch_prepare_small(mv, bv, c->d_scan_sorted, ch.count, cell_bits, ch.max_kept, st));
        SO_CUDA_TRY(cudaGetLastError());
        return SO_OK;
    }
    while ((1u << scan_bits) < ch.count) ++scan_bits;
    if (compact && !c->force_drop_bit) {
        bool capped = false;
        for (uint32_t s = ch.first; s < ch.first + ch.count; ++s) capped |= c->h_state[s].sampling_rate >= 0.0;     // init_state: -1 = no cap
        compact = capped;
    }
    const int extra = compact ? 1 : 0;
    const bool key32 = !c->force_key64 && cell_bits < 32 && cell_bits + extra + scan_bits <= 32;
    if (!key32) cell_bits = 32;
    uint32_t n = launch_scan_keys(mv, bv, c->d_skeys, c->d_svals, ch.grid_in, ch.count, cell_bits, key32, compact, st);
    int rc = scan_sort(c, ch.pt_first, ch.pt_count, int(ch.count), cell_bits + extra, key32, st);
    if (rc) return rc;
    n += launch_scan_gather(d_scan_in, c->d_svals_out, c->d_skeys_out, ch.pt_first, c->d_offset + ch.first, ch.pt_count,
                            c->d_scan_sorted + ch.pt_first, cell_bits + extra, key32, st);
    if (compact) n += launch_scan_finish(bv, c->d_skeys_out, ch.pt_first, ch.pt_first, cell_bits, key32, ch.count, st);
    timed_launch_end(c, 3, n);
    SO_CUDA_TRY(cudaGetLastError());
    return SO_OK;
}

// One solve phase of an ICP iteration for the chunk's scans (first: its first scan): PH_CORR opens a solve, PH_EVAL is one lm
// evaluation.  OPTIMIZED: the two-block motion solve; otherwise the six-column one, stepped by k_lm_step_deg when dg is given.
// me / eb: the edge map and the chunk's line buffers, read when grid_e > 0.  Returns the kernels it enqueued.
static uint32_t launch_solve(const Ctx* c, UndistortionMode mode, int phase, const BatchView& bv, const CorrBuf& cb, uint32_t first, uint32_t grid_x,
                             uint32_t n_scans, cudaStream_t st, const MapView* me, const EdgeBuf* eb, uint32_t grid_e, DegenState* dg) {
    if (mode == UndistortionMode::OPTIMIZED) {
        const MotionEdges med = grid_e ? MotionEdges{*me, *eb, c->d_escan, c->und.d_etime, c->mot.d_epartials, grid_e} : MotionEdges{};
        return launch_motion_solve(phase, bv, cb, c->d_scan, c->und.d_time, c->mot.d_st, first, c->mot.d_partials + size_t(first) * c->mot.stride * kMotionAcc,
                                   c->mot.stride, grid_x, n_scans, st, grid_e ? &med : nullptr);
    }
    if (phase == PH_CORR) return launch_first_eval(bv, cb, grid_x, n_scans, st, me, eb, grid_e, dg);
    return launch_evaluate(bv, cb, grid_x, n_scans, st, eb, grid_e, dg);
}

// One ICP iteration: [head, search, k_fit, first solve, lm solves].  Every kernel exits at once when its scan is not in the
// matching phase, so a fixed schedule follows whatever path the device-side state machine takes.
//   head         modes APPROXIMATED and OPTIMIZED: k_warp_scan (the scans warped by D, from the current pose or the motion block) +
//                k_warp_edges when the chunk has an edge cloud; NONE: none
//   search       k_knn_scan (k_knn_scan_coop for a coop chunk; k_knn_scan<true> + k_knn_round2 with the neighbour graph), or
//                k_knn_inject with injected neighbours
//   first solve  k_evaluate<PH_CORR> (+ k_edge_fit) + k_lm_step; OPTIMIZED: k_motion_eval<PH_CORR> (+ k_edge_fit + k_motion_eval_edge)
//                + k_motion_step
//   lm solves    k_evaluate<PH_EVAL> (+ k_edge_evaluate) + k_lm_step; OPTIMIZED: k_motion_eval<PH_EVAL> (+ k_motion_eval_edge) + k_motion_step
// Preferred form: a CUDA-graph WHILE node around ONE iteration (k_loop_cond ends the loop when every scan of the chunk is done);
// fallback: the schedule unrolled `iters` times.  Profiling or injected neighbours: launched one step at a time instead, each step
// only when a scan of the chunk is in its phase.  dg: the chunk's DegenState array of a degeneracy-aware registration
// (k_lm_step_deg steps its solves), else nullptr.
// Counts the kernels it launched, except in the loop form, whose passes only the final states tell: *body_launches is then the
// kernels one pass of the WHILE body launches, else 0.
static int run_schedule(Ctx* c, const Chunk& ch, int iters, int lm, UndistortionMode mode, const uint32_t* d_inject, int inject_iters,
                        cudaStream_t run_stream, DegenState* dg, uint32_t* body_launches) {
    const MapView mv = search_view(c);
    NnBuf nn = c->nn;                                     // queue lengths: indexed by the scan's position inside the chunk
    if (nn.qcount) nn.qcount += size_t(ch.first) * SO_MAX_ICP_ITERS;
    const BatchView bv = chunk_view(c, c->d_scan_sorted, ch);
    CorrBuf cb = c->corr;
    cb.nn = nullptr; cb.nn_d2 = nullptr; cb.first = ch.first;
    const uint32_t grid_x = ch.grid_x, n_scans = ch.count, grid_e = ch.grid_e;
    const MapView me = map_view(c, c->edge);
    EdgeBuf eb = c->ebuf;
    eb.offset = c->d_eoffset + ch.first;                  // like bv.offset: indexed by the scan's position inside the chunk
    eb.nn = nullptr; eb.selmask = nullptr;
    *body_launches = 0;
    const bool optimized = mode == UndistortionMode::OPTIMIZED;
    const bool warp_edges = mode != UndistortionMode::NONE && grid_e;     // the line branch runs on the warped edge cloud
    if (warp_edges) eb.scan = c->und.d_ewarp;
    // The iteration's steps in order, on c->stream: step(cls, phase, launch) with the step's profile class, the phase of the scans
    // it serves, and launch() enqueueing it and returning its kernels.  Returns the sum of what step returned.
    auto iteration = [&](auto&& step) -> uint32_t {
        cudaStream_t s = c->stream;
        uint32_t n = 0;
        if (mode != UndistortionMode::NONE) n += step(7, PH_CORR, [&] { return launch_warp(c, mode, bv, eb.offset, ch.first, grid_x, grid_e, n_scans, s); });
        n += step(0, PH_CORR, [&] {
            return d_inject ? launch_inject(mv, c->surf.d_xyzi, c->surf.n, bv, c->nn, d_inject, inject_iters, grid_x, n_scans, s)
                            : launch_match(mv, bv, cb, nn, grid_x, n_scans, s, 1);
        });
        n += step(5, PH_CORR, [&] { return launch_match(mv, bv, cb, nn, grid_x, n_scans, s, 2); });
        n += step(optimized ? 8 : 4, PH_CORR, [&] { return launch_solve(c, mode, PH_CORR, bv, cb, ch.first, grid_x, n_scans, s, &me, &eb, grid_e, dg); });
        for (int k = 0; k < lm; ++k)
            n += step(optimized ? 8 : 1, PH_EVAL, [&] { return launch_solve(c, mode, PH_EVAL, bv, cb, ch.first, grid_x, n_scans, s, &me, &eb, grid_e, dg); });
        return n;
    };
    auto enqueue = [](int, int, auto&& launch) { return launch(); };
    if (c->profiling || d_inject) {
        // profiling mode: one launch at a time, timed with events, and only launches that have work (the host peeks
        // at the phases) so that the per-class average is the duration of a kernel that actually ran
        std::vector<IcpState> peek(n_scans);
        auto any_in = [&](int ph) -> bool {
            cudaMemcpyAsync(peek.data(), c->d_state + ch.first, n_scans * sizeof(IcpState), cudaMemcpyDeviceToHost, c->stream);
            cudaStreamSynchronize(c->stream);
            for (uint32_t s = 0; s < n_scans; ++s) if (peek[s].phase == ph) return true;
            return false;
        };
        auto timed = [&](int cls, int ph, auto&& launch) -> uint32_t {
            if (!any_in(ph)) return 0;
            timed_launch_begin(c);
            const uint32_t n = launch();
            timed_launch_end(c, cls, n);
            return n;
        };
        for (int it = 0; it < iters; ++it) iteration(timed);
        SO_CUDA_TRY(cudaGetLastError());
        return SO_OK;
    }
    Ctx::GraphKey key;
    std::memset(&key, 0, sizeof(key));                      // padding bytes take part in the memcmp below
    key.first = ch.first; key.count = n_scans; key.grid_x = grid_x; key.grid_e = grid_e; key.iters = iters; key.lm = lm;
    key.ptrs[0] = mv.pts; key.ptrs[1] = mv.cell_start; key.ptrs[2] = mv.block_slot; key.ptrs[3] = mv.block_count;
    key.ptrs[4] = me.pts; key.ptrs[5] = me.cell_start; key.ptrs[6] = me.block_slot; key.ptrs[7] = me.block_count;
    for (int a = 0; a < 3; ++a) key.origin[a] = mv.origin[a];
    key.nb[0] = mv.nb; key.nb[1] = me.nb; key.res[0] = mv.plane_res; key.res[1] = me.plane_res;
    if (mode != UndistortionMode::NONE) { key.mode = mode; key.und_time = c->und.d_time; }
    if (warp_edges) key.und_edge = c->und.d_ewarp;
    key.degen = dg;
    key.graph[0] = mv.graph; key.graph[1] = mv.graph_radius; key.graph[2] = mv.graph_stats; key.graph[3] = nn.queue; key.graph[4] = nn.qcount;
    Ctx::GraphSlot* slot = nullptr;
    for (auto& g : c->graphs)
        if (g.exec && std::memcmp(&g.key, &key, sizeof(key)) == 0) slot = &g;
    if (!slot) {
        slot = &c->graphs[0];
        for (auto& g : c->graphs) { if (!g.exec) { slot = &g; break; } if (g.used < slot->used) slot = &g; }
        if (slot->exec) { cudaGraphExecDestroy(slot->exec); slot->exec = nullptr; }
        slot->is_loop = false;
        if (!c->no_cond_graph) {
            cudaGraph_t g = nullptr;
            cudaGraphConditionalHandle handle;
            bool ok = cudaGraphCreate(&g, 0) == cudaSuccess &&
                      cudaGraphConditionalHandleCreate(&handle, g, 1, cudaGraphCondAssignDefault) == cudaSuccess;
            cudaGraphNodeParams p = {cudaGraphNodeTypeConditional};
            cudaGraphNode_t node;
            if (ok) {
                p.conditional.handle = handle; p.conditional.type = cudaGraphCondTypeWhile; p.conditional.size = 1;
                ok = cudaGraphAddNode(&node, g, nullptr, 0, &p) == cudaSuccess;
            }
            if (ok) {
                cudaGraph_t body = p.conditional.phGraph_out[0];
                ok = cudaStreamBeginCaptureToGraph(c->stream, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
                if (ok) {
                    slot->launches = iteration(enqueue);
                    slot->launches += launch_loop_cond(bv, n_scans, handle, c->stream);
                    cudaGraph_t dummy = nullptr;
                    ok = cudaStreamEndCapture(c->stream, &dummy) == cudaSuccess;
                }
            }
            if (ok) ok = cudaGraphInstantiate(&slot->exec, g, 0) == cudaSuccess;
            if (g) cudaGraphDestroy(g);
            if (ok) slot->is_loop = true;
            else { cudaGetLastError(); slot->exec = nullptr; c->no_cond_graph = true; }      // fall back to the unrolled schedule
        }
        if (!slot->exec) {
            cudaGraph_t g = nullptr;
            SO_CUDA_TRY(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
            slot->launches = 0;
            for (int it = 0; it < iters; ++it) slot->launches += iteration(enqueue);
            SO_CUDA_TRY(cudaStreamEndCapture(c->stream, &g));
            cudaError_t e = cudaGraphInstantiate(&slot->exec, g, 0);
            cudaGraphDestroy(g);
            if (e != cudaSuccess) { slot->exec = nullptr; return fail(SO_ERR_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e)); }
        }
        slot->key = key;
    }
    slot->used = ++c->graph_clock;
    SO_CUDA_TRY(cudaGraphLaunch(slot->exec, run_stream));
    if (slot->is_loop) *body_launches = slot->launches;
    else c->launches += slot->launches;
    return SO_OK;
}

static void init_state(IcpState& s, const double pose[7], uint32_t n, const so_icp_opts& o, uint32_t n_edge = 0) {
    std::memset(&s, 0, sizeof(s));
    std::memcpy(s.x0, pose, 7 * sizeof(double));
    std::memcpy(s.x, pose, 7 * sizeof(double));
    std::memcpy(s.cand, pose, 7 * sizeof(double));
    s.n_points = int32_t(n);
    s.n_input = int32_t(n);
    s.n_edge = int32_t(n_edge);
    s.max_icp_iters = o.max_icp_iters;
    s.lm_max_iterations = o.lm_max_iterations;
    // calculateSamplingRate (LidarSlam.cpp:346-351)
    s.sampling_rate = (o.max_surface_features > 0 && n > uint32_t(o.max_surface_features)) ? 1.0 * o.max_surface_features / double(n) : -1.0;
    s.use_prior = o.use_pose_prior ? 1 : 0;
    s.prior_vcf = o.visual_confidence_factor;
    for (int a = 0; a < 3; ++a) s.prior_unc[a] = o.prior_uncertainty[a];
    s.phase = PH_CORR;
}

static void fill_result(const Ctx* c, const IcpState& s, const double pose_in[7], const so_icp_opts& o, so_icp_result* r) {
    r->n_iterations = s.n_iterations;
    for (int i = 0; i < SO_MAX_ICP_ITERS; ++i) {
        r->iter_n_surf[i] = s.iter_n_surf[i]; r->iter_n_edge[i] = s.iter_n_edge[i]; r->iter_dtrans[i] = s.iter_dtrans[i]; r->iter_drot[i] = s.iter_drot[i];
        r->iter_lm_steps[i] = s.iter_lm_steps[i]; r->iter_lm_successful[i] = s.iter_lm_successful[i];
        r->iter_lm_termination[i] = s.iter_lm_termination[i]; r->iter_cost[i] = s.iter_cost[i];
    }
    std::memcpy(r->hist_obs, s.hist_obs, sizeof(r->hist_obs));
    std::memcpy(r->hist_reject_plane, s.hist_rej, sizeof(r->hist_reject_plane));
    std::memcpy(r->hist_reject_line, s.hist_rej_line, sizeof(r->hist_reject_line));
    std::memcpy(r->cov, s.cov, sizeof(r->cov));
    r->pos_err = s.pos_err; r->pos_inv_cond = s.pos_inv_cond; r->ori_err_deg = s.ori_err_deg; r->ori_inv_cond = s.ori_inv_cond;
    for (int i = 0; i < 3; ++i) { r->pos_dir[i] = s.pos_dir[i]; r->ori_dir[i] = s.ori_dir[i]; }
    if (s.status) r->status = s.status;
    r->knn_searched = 0; r->knn_verified = 0;             // reserved
    r->prediction_source = s.use_prior ? 1 : 0;
    double T[7];
    std::memcpy(T, s.x, sizeof(T));
    std::memcpy(r->pose_opt, T, sizeof(T));
    // performPostOptimizationProcessing (LidarSlam.cpp:155-171): last_T_w_lidar == T_w_initial_guess == prior (:53-57)
    manual_yaw_correction(pose_in, T, double(o.yaw_ratio));
    std::memcpy(r->pose, T, sizeof(T));
    rel_motion(pose_in, T, &r->total_translation, &r->total_rotation);           // updateOptimizationStats (:198-210)
    r->translation_from_last = r->total_translation; r->rotation_from_last = r->total_rotation;
    (void)c;
}

int icp_opts_check(const so_icp_opts& o) {
    if (o.max_icp_iters <= 0 || o.max_icp_iters > SO_MAX_ICP_ITERS) return fail(SO_ERR_ARG, "max_icp_iters must be in [1,32]");
    if (o.lm_max_iterations > 16) return fail(SO_ERR_ARG, "lm_max_iterations must be <= 16");
    return SO_OK;
}

// The registration of q's scans once they are on the device: at q.scans for Source::DEVICE, else at d_scan, where Source::HOST_PACKED
// scans are uploaded here chunk by chunk on the copy stream.  Mode APPROXIMATED / OPTIMIZED: the scans' times, parameters or motion
// blocks are on the device too.
static int register_core(Ctx* c, const RegisterRequest& q) {
    const float4* const d_scan = q.src == RegisterRequest::Source::DEVICE ? static_cast<const float4*>(q.scans) : c->d_scan;
    const void* const host_src = q.src == RegisterRequest::Source::HOST_PACKED ? q.scans : nullptr;
    const uint32_t* const n_points = q.n_points;
    const uint32_t* const n_edge = q.n_edge;
    const size_t n_scans = q.n_scans;
    const double* const poses = q.poses;
    so_icp_result* const results = q.results;
    double* const sink = q.sink_rows ? c->d_pose_sink : nullptr;
    so_icp_opts o = *q.opts;
    if (o.lm_max_iterations <= 0) o.lm_max_iterations = 4;
    { int rc = icp_opts_check(o); if (rc) return rc; }
    { int rc = ensure_maps(c); if (rc) return rc; }
    uint32_t max_n = 0, off = 0, eoff = 0;
    bool any = false, any_edge = false;
    for (size_t s = 0; s < n_scans; ++s) {
        so_icp_result* r = results + s;
        std::memset(r, 0, sizeof(*r));
        const double* pose = poses + 7 * s;
        std::memcpy(r->pose, pose, 7 * sizeof(double));
        std::memcpy(r->pose_opt, pose, 7 * sizeof(double));
        r->scan_surf_num = int32_t(n_points[s]);
        // prepareOptimizationState (LidarSlam.cpp:361-369)
        int32_t ijk[3];
        if (q.allow_shift && !o.skip_map_checks) { int rc = so_map_shift(reinterpret_cast<so_ctx*>(c), pose, ijk); if (rc < 0) return rc; }
        else for (int a = 0; a < 3; ++a) ijk[a] = block_coord_h(pose[a] + kHalfBlock, c->origin[a]);
        for (int a = 0; a < 3; ++a) r->pos_in_localmap[a] = ijk[a];
        r->map_surf_5x5 = counts_5x5(c, c->surf, ijk);
        r->map_edge_5x5 = counts_5x5(c, c->edge, ijk);
        init_state(c->h_state[s], pose, n_points[s], o, n_edge ? n_edge[s] : 0);
        c->h_offset[s] = off;
        off += n_points[s];
        c->h_eoffset[s] = eoff;                                    // edge clouds: packed back to back in d_escan like the scans in d_scan
        if (n_edge) { eoff += n_edge[s]; any_edge |= n_edge[s] != 0; r->scan_edge_num = int32_t(n_edge[s]); }
        if (!o.skip_map_checks && !(r->map_surf_5x5 > 50)) {       // hasEnoughFeatures (:379-381): pose stays the prior
            r->status = SO_STATUS_NOT_ENOUGH_FEATURES;
            c->h_state[s].phase = PH_DONE; c->h_state[s].status = r->status;
        } else if (n_points[s] == 0) {
            r->status = SO_STATUS_NO_CORRESPONDENCES;
            c->h_state[s].phase = PH_DONE; c->h_state[s].status = r->status;
        } else { any = true; max_n = std::max(max_n, n_points[s]); }
    }
    if (sink && c->sink_cursor + n_scans > c->sink_cap) return fail(SO_ERR_CAPACITY, "pose sink full (so_set_pose_sink)");
    if (!any && sink) {                                         // nothing to register: the rows are the priors
        SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, n_scans * sizeof(IcpState), cudaMemcpyHostToDevice, c->stream));
        c->launches += launch_pack_poses(c->d_state, uint32_t(n_scans), sink + c->sink_cursor * 8, c->stream);
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    if (any) {
        SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, n_scans * sizeof(IcpState), cudaMemcpyHostToDevice, c->stream));
        SO_CUDA_TRY(cudaMemcpyAsync(c->d_offset, c->h_offset, n_scans * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
        if (any_edge || c->eoffset_dirty) {                        // the all-zero table of the edge-less case is already there
            SO_CUDA_TRY(cudaMemcpyAsync(c->d_eoffset, c->h_eoffset, n_scans * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
            c->eoffset_dirty = any_edge;
        }
        count_h2d(c, n_scans * (sizeof(IcpState) + sizeof(uint32_t)));
        {                                                           // the neighbour graph, when this call's searches pay for it
            size_t queries = 0;
            for (size_t s = 0; s < n_scans; ++s)
                if (c->h_state[s].phase == PH_CORR)
                    queries += c->h_state[s].sampling_rate < 0.0 ? n_points[s] : std::min<uint32_t>(n_points[s], uint32_t(o.max_surface_features) + 1);
            int rc = knn_graph_prepare(c, queries);
            if (!rc) rc = graph_queue_begin(c, n_scans);
            if (rc) return rc;
        }
        // Chunk the batch.  Even chunks run on `stream`, odd ones on aux_stream, so that one chunk's serial stretches (the
        // one-CTA optimiser steps, kernel tails, the loop condition) sit under the other's wide kernels; with host input
        // the H2D of chunk k+1 (copy stream) also overlaps the kernels of chunk k.
        // Device-resident scans: two chunks (one per stream).  Chunks stay >= 8 scans: below that the wide kernels stop filling the GPU.
        // (the rule -- growing chunks for host input -- lives in so_chunks.h, where a CPU test can reach it)
        const std::vector<uint32_t> bounds = chunk_bounds(n_scans, host_src != nullptr, c->profiling, c->chunk_override);
        const size_t n_chunks = bounds.size() - 1;
        std::vector<Chunk> chunks;
        for (size_t k = 0; k < n_chunks; ++k) {
            const uint32_t f = bounds[k], e = bounds[k + 1];
            if (e == f) continue;
            Chunk ch{f, e - f, c->h_offset[f], (e < n_scans ? c->h_offset[e] : off) - c->h_offset[f]};
            uint32_t mx = 0, mx_in = 0;
            for (uint32_t s = f; s < e; ++s) if (c->h_state[s].phase == PH_CORR) {
                mx_in = std::max(mx_in, n_points[s]);
                // shouldProcessPoint keeps at most max_surface_features + 1 points of a decimated scan (one per wrap of i * rate)
                const uint32_t kept = c->h_state[s].sampling_rate < 0.0 ? n_points[s] : std::min<uint32_t>(n_points[s], uint32_t(o.max_surface_features) + 1);
                mx = std::max(mx, kept);
            }
            ch.grid_in = (mx_in + kThreads - 1) / kThreads;
            ch.small = mx <= kPrepareSmallCap && mx_in > 0;
            ch.max_kept = mx;
            plan_chunk(c, ch, mx, q.mode == UndistortionMode::OPTIMIZED || q.degen);
            if (n_edge) for (uint32_t s = f; s < e; ++s) if (c->h_state[s].phase == PH_CORR) ch.grid_e = std::max(ch.grid_e, (n_edge[s] + kThreads - 1) / kThreads);
            chunks.push_back(ch);
        }
        SO_CUDA_TRY(cudaEventRecord(c->ev0, c->stream));
        const bool two_streams = chunks.size() > 1 && !c->single_stream;
        if (two_streams) {
            SO_CUDA_TRY(cudaEventRecord(c->ev_fork, c->stream));                    // aux starts after the state upload and all earlier work
            SO_CUDA_TRY(cudaStreamWaitEvent(c->aux_stream, c->ev_fork, 0));
        }
        if (host_src) {
            SO_CUDA_TRY(cudaEventRecord(c->ev_copy[16], c->stream));                // copies must not overtake earlier work on d_scan
            SO_CUDA_TRY(cudaStreamWaitEvent(c->copy_stream, c->ev_copy[16], 0));
            for (size_t k = 0; k < chunks.size(); ++k) {
                const Chunk& ch = chunks[k];
                if (ch.pt_count)
                    SO_CUDA_TRY(cudaMemcpyAsync(c->d_scan + ch.pt_first, static_cast<const float4*>(host_src) + ch.pt_first,
                                                size_t(ch.pt_count) * sizeof(float4), cudaMemcpyHostToDevice, c->copy_stream));
                count_h2d(c, size_t(ch.pt_count) * sizeof(float4));
                SO_CUDA_TRY(cudaEventRecord(c->ev_copy[k], c->copy_stream));
            }
        }
        std::vector<uint32_t> body_launches(chunks.size(), 0);       // a later chunk's capture may evict this chunk's graph
        for (size_t k = 0; k < chunks.size(); ++k) {
            const Chunk& ch = chunks[k];
            cudaStream_t st = (two_streams && (k & 1)) ? c->aux_stream : c->stream;
            if (host_src) SO_CUDA_TRY(cudaStreamWaitEvent(st, c->ev_copy[k], 0));
            if (ch.grid_x == 0) continue;
            int rc = prepare_scans(c, d_scan, ch, st, true);
            if (!rc) rc = run_schedule(c, ch, o.max_icp_iters, o.lm_max_iterations, q.mode, q.inject ? c->d_inject.get() : nullptr, q.inject_iters, st,
                                       q.degen ? c->deg.d_st + ch.first : nullptr, &body_launches[k]);
            if (rc) {                                       // leave no work behind on the side streams before reporting the error
                cudaStreamSynchronize(c->aux_stream);
                cudaStreamSynchronize(c->copy_stream);
                return rc;
            }
        }
        if (two_streams) {
            SO_CUDA_TRY(cudaEventRecord(c->ev_join, c->aux_stream));
            SO_CUDA_TRY(cudaStreamWaitEvent(c->stream, c->ev_join, 0));
        }
        SO_CUDA_TRY(cudaEventRecord(c->ev1, c->stream));
        { int rc = run_deferred_upload(c); if (rc) return rc; }      // host-side staging of the whole cloud while the registration runs
        if (sink) c->launches += launch_pack_poses(c->d_state, uint32_t(n_scans), sink + c->sink_cursor * 8, c->stream);
        SO_CUDA_TRY(cudaMemcpyAsync(c->h_state, c->d_state, n_scans * sizeof(IcpState), cudaMemcpyDeviceToHost, c->stream));
        count_d2h(c, n_scans * sizeof(IcpState));
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
        float ms = 0.f;
        cudaEventElapsedTime(&ms, c->ev0, c->ev1);
        for (size_t k = 0; k < chunks.size(); ++k) {                // the loop form: the WHILE body ran once per iteration of the longest registration
            int max_it = 0;
            for (uint32_t s = chunks[k].first; s < chunks[k].first + chunks[k].count; ++s) max_it = std::max(max_it, int(c->h_state[s].n_iterations));
            c->launches += uint64_t(max_it) * body_launches[k];
        }
        for (size_t s = 0; s < n_scans; ++s) {
            if (results[s].status == SO_STATUS_NOT_ENOUGH_FEATURES || n_points[s] == 0) continue;
            fill_result(c, c->h_state[s], poses + 7 * s, o, results + s);
            results[s].time_ms = double(ms);
        }
    }
    if (sink) c->sink_cursor += n_scans;
    return SO_OK;
}

// A capped so_register scan (the shipped configurations cap a 28 800-point scan at 2 000 features): the registration reads only the
// points shouldProcessPoint keeps, so only those go up in front of it, into d_dec (32 KB instead of 460 KB).  The whole cloud -- needed
// by so_map_add_registered_scan, not by the registration -- is staged and copied on the copy stream while the registration runs.
static int upload_kept(Ctx* c, const RegisterRequest& q, size_t n_edge, uint32_t* kept_out) {
    const uint32_t n = q.n_points[0];
    const std::vector<uint32_t>& keep = decimation_list(c, n, q.opts->max_surface_features);
    const uint32_t kept = uint32_t(keep.size());
    if (kept == 0 || kept > kPrepareSmallCap) return fail(SO_ERR_ARG, "decimation list out of range");
    const bool packed = q.stride == 16 && q.ioff == 12;
    if (n_edge && !packed) SO_CUDA_TRY(cudaStreamSynchronize(c->stream));     // a strided edge cloud has to have left the staging buffer
    SO_CUDA_TRY(cudaEventSynchronize(c->ev_dec));                              // so has the previous call's deferred copy
    int rc = ensure_stage(c, size_t(kPrepareSmallCap) + (packed ? 0 : n));
    if (rc) return rc;
    float4* h = c->h_stage;
    const unsigned char* p = static_cast<const unsigned char*>(q.scans);
    for (uint32_t j = 0; j < kept; ++j) h[j] = read_point(p + size_t(keep[j]) * q.stride, q.stride, q.ioff);
    SO_CUDA_TRY(cudaEventRecord(c->ev_copy[16], c->stream));                  // the whole-cloud copy must not overtake earlier readers of d_scan
    SO_CUDA_TRY(cudaStreamWaitEvent(c->copy_stream, c->ev_copy[16], 0));
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_dec, h, size_t(kept) * sizeof(float4), cudaMemcpyHostToDevice, c->stream));
    c->bytes_h2d += size_t(kept) * sizeof(float4);
    c->defer.src = q.scans; c->defer.n = n; c->defer.stride = q.stride; c->defer.ioff = q.ioff; c->defer.stage_off = kPrepareSmallCap;
    *kept_out = kept;
    return SO_OK;
}

int register_scans(Ctx* c, const RegisterRequest& q) {
    using Source = RegisterRequest::Source;
    SO_CUDA_TRY(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    size_t total = 0, total_e = 0;
    for (size_t s = 0; s < q.n_scans; ++s) { total += q.n_points[s]; if (q.n_edge) total_e += q.n_edge[s]; }
    const bool host = q.src == Source::HOST || q.src == Source::HOST_PACKED;
    const bool with_times = q.mode != UndistortionMode::NONE;
    if (q.src != Source::DEVICE) c->reg.valid = false;                         // d_scan is overwritten; valid again below if insertable
    int rc = SO_OK;
    if (q.mode == UndistortionMode::APPROXIMATED) rc = undistort_reserve(c, total);
    if (q.mode == UndistortionMode::OPTIMIZED) rc = motion_reserve(c, total);
    if (!rc && q.degen) rc = c->deg.d_st.reserve(c->max_batch);
    if (!rc && q.inject) {
        const size_t words = size_t(q.inject_iters) * total * 5;
        rc = c->d_inject.reserve(words);
        if (!rc) SO_CUDA_TRY(cudaMemcpyAsync(c->d_inject, q.inject, words * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    }
    const bool edge_times = q.mode != UndistortionMode::NONE && q.edge && total_e;    // so_register_undistort_edges / _optimized_edges
    if (!rc && edge_times) rc = undistort_edge_reserve(c);
    if (!rc && edge_times && q.mode == UndistortionMode::OPTIMIZED) rc = motion_edge_reserve(c);
    if (!rc && q.edge) rc = upload_cloud(c, q.edge, total_e, q.stride, q.ioff, c->d_escan);   // first: it may use the staging buffer
    if (!rc && edge_times) rc = upload_times(c, q.edge, total_e, q.stride, q.toff, c->und.d_etime);
    if (rc) return rc;
    RegisterRequest core = q;                      // what register_core registers: a capped so_register scan, its kept points
    const so_icp_opts& o = *q.opts;
    so_icp_opts o_kept = o;
    uint32_t kept = 0;
    const bool decimated = q.src == Source::HOST && q.insertable && q.mode == UndistortionMode::NONE && !c->no_dec_upload &&
                           o.max_surface_features > 0 && total > size_t(o.max_surface_features) && uint32_t(o.max_surface_features) + 1 <= kPrepareSmallCap;
    if (decimated) {
        rc = upload_kept(c, q, total_e, &kept);
        o_kept.max_surface_features = 0;                                         // the decimation has been applied
        core.src = Source::DEVICE; core.scans = c->d_dec; core.n_points = &kept; core.opts = &o_kept;
    } else if (q.src == Source::HOST) {
        rc = upload_cloud(c, q.scans, total, q.stride, q.ioff, c->d_scan);
    } else if (q.src == Source::PREFILTERED) {
        c->prefiltered_n = SIZE_MAX;
        if (total) SO_CUDA_TRY(cudaMemcpyAsync(c->d_scan, c->d_scan_sorted, total * sizeof(float4), cudaMemcpyDeviceToDevice, c->stream));
        // the filtered cloud's w (the VoxelGrid average of the time the extraction stored in intensity) is the time
        if (total && with_times)
            SO_CUDA_TRY(cudaMemcpy2DAsync(c->und.d_time, sizeof(float), reinterpret_cast<const char*>(c->d_scan_sorted.get()) + 12, sizeof(float4),
                                          sizeof(float), total, cudaMemcpyDeviceToDevice, c->stream));
    }
    if (!rc && host && with_times) rc = upload_times(c, q.scans, total, q.stride, q.toff, c->und.d_time);
    if (!rc && q.mode == UndistortionMode::APPROXIMATED) {
        SO_CUDA_TRY(cudaMemcpyAsync(c->und.d_par, q.und, q.n_scans * sizeof(UndistortParams), cudaMemcpyHostToDevice, c->stream));
        count_h2d(c, q.n_scans * sizeof(UndistortParams));
    }
    if (!rc && q.mode == UndistortionMode::OPTIMIZED) {
        SO_CUDA_TRY(cudaMemcpyAsync(c->mot.d_st, q.motion, q.n_scans * sizeof(MotionState), cudaMemcpyHostToDevice, c->stream));
        count_h2d(c, q.n_scans * sizeof(MotionState));
    }
    if (!rc && q.degen) {
        SO_CUDA_TRY(cudaMemcpyAsync(c->deg.d_st, q.degen, q.n_scans * sizeof(DegenState), cudaMemcpyHostToDevice, c->stream));
        count_h2d(c, q.n_scans * sizeof(DegenState));
    }
    if (rc) return rc;
    rc = register_core(c, core);
    if (decimated) {
        const int rc2 = run_deferred_upload(c);                                  // not yet run when nothing was launched (soft statuses) or on errors
        SO_CUDA_TRY(cudaStreamWaitEvent(c->stream, c->ev_dec, 0));               // later work on the context stream (the insert) sees the whole cloud
        if (!rc) rc = rc2;
        if (!rc) q.results[0].scan_surf_num = int32_t(total);
    }
    if (!rc && q.mode == UndistortionMode::OPTIMIZED) {
        SO_CUDA_TRY(cudaMemcpyAsync(q.motion, c->mot.d_st, q.n_scans * sizeof(MotionState), cudaMemcpyDeviceToHost, c->stream));
        count_d2h(c, q.n_scans * sizeof(MotionState));
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    if (!rc && q.degen) {
        SO_CUDA_TRY(cudaMemcpyAsync(q.degen, c->deg.d_st, q.n_scans * sizeof(DegenState), cudaMemcpyDeviceToHost, c->stream));
        count_d2h(c, q.n_scans * sizeof(DegenState));
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    if (rc) return rc;
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    for (size_t s = 0; s < q.n_scans; ++s) {
        q.results[s].time_total_ms = ms;
        if (q.motion_results) fill_motion(q.results[s], q.motion[s], q.motion_results + s);
    }
    if (q.insertable) {
        c->reg = RegisteredScan{};
        c->reg.n = uint32_t(total); c->reg.warp.mode = q.mode;
        if (q.edge) c->reg.n_edge = uint32_t(total_e);
        if (q.mode == UndistortionMode::APPROXIMATED) c->reg.warp.par = q.und[0];
        if (q.mode == UndistortionMode::OPTIMIZED) {
            std::memcpy(c->reg.warp.motion.D, q.motion[0].D, sizeof(c->reg.warp.motion.D)); c->reg.warp.motion.dt = q.motion[0].dt;
        }
    }
    return SO_OK;
}

// ---------------------------------------------------------------------------------------------- the so_register* family
// A single scan as the live loop registers it: the map may shift to the prior, the scan stays for so_map_add_registered_scan
static RegisterRequest single_scan(const uint32_t* n, const double* pose, const so_icp_opts* opts, so_icp_result* out) {
    RegisterRequest q;
    q.n_points = n; q.poses = pose; q.opts = opts; q.results = out; q.allow_shift = true; q.insertable = true;
    return q;
}
static int status_of(int rc, const so_icp_result& r) { return rc ? rc : r.status; }
static int check_batch(const Ctx* c, const uint32_t* n_points, size_t n_scans) {
    if (n_scans == 0 || n_scans > c->max_batch) return fail(SO_ERR_CAPACITY, "n_scans exceeds so_config.max_batch");
    for (size_t s = 0; s < n_scans; ++s) if (n_points[s] > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "scan too large");
    return SO_OK;
}
// A batch of host clouds: packed float4 ones go up chunk by chunk beside the kernels, strided ones whole first
static RegisterRequest batch_request(const void* surf, const uint32_t* n_points, size_t n_scans, size_t stride, size_t ioff, const double* poses,
                                     const so_icp_opts* opts, so_icp_result* results) {
    RegisterRequest q;
    q.src = stride == 16 && ioff == 12 ? RegisterRequest::Source::HOST_PACKED : RegisterRequest::Source::HOST;
    q.scans = surf; q.stride = stride; q.ioff = ioff; q.n_points = n_points; q.n_scans = n_scans; q.poses = poses; q.opts = opts; q.results = results;
    return q;
}

// dst[0..n) = the registered scan (Ctx::reg), still in d_scan, compensated for its motion as it was registered; with edges, its edge
// cloud, still in d_escan (left by so_register, so_register_undistort_edges and so_register_optimized_edges).  The map inserts place it
// at a store's tail, so_keyframe_add_registered at the keyframe pools' tails.
int put_registered_scan(Ctx* c, bool edges, float4* dst, const double pose[7]) {
    const RegisteredScan& r = c->reg;
    SO_CUDA_TRY(cudaMemcpyAsync(dst, edges ? c->d_escan : c->d_scan, size_t(edges ? r.n_edge : r.n) * sizeof(float4),
                                cudaMemcpyDeviceToDevice, c->stream));
    return warp_cloud(c, dst, edges ? c->und.d_etime : c->und.d_time, edges ? r.n_edge : r.n, r.warp, pose);   // OPTIMIZED: u(D_opt), whatever the pose
}

// so_degeneracy values of the degeneracy-aware entry points (so_register_degeneracy*, so_loop_verify_degeneracy, so_solve)
int check_degeneracy(const so_degeneracy* d, size_t n) {
    for (size_t s = 0; s < n; ++s) {
        if (!(d[s].pos_threshold >= 0.0 && d[s].pos_threshold < 1.0) || !(d[s].ori_threshold >= 0.0 && d[s].ori_threshold < 1.0))
            return fail(SO_ERR_ARG, "degeneracy thresholds must be in [0, 1)");
        if (d[s].constrain != 0 && d[s].constrain != 1) return fail(SO_ERR_ARG, "so_degeneracy.constrain must be 0 or 1");
    }
    return SO_OK;
}

}  // namespace so

// =================================================================================================== C ABI
using namespace so;
using Source = RegisterRequest::Source;

extern "C" {

const char* so_last_error(void) { return g_err.c_str(); }

int so_device_available(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return 0; }
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, 0) != cudaSuccess) { cudaGetLastError(); return 0; }
    return p.major == 9 ? 1 : 0;
}

so_ctx* so_create(const so_config* cfg_in) {
    so_config cfg{};
    if (cfg_in) cfg = *cfg_in;
    if (cfg.max_map_points == 0) cfg.max_map_points = 4u << 20;
    if (cfg.max_scan_points == 0) cfg.max_scan_points = 262144;
    if (cfg.max_batch == 0) cfg.max_batch = 1;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); set_error("no CUDA device: this library has no CPU fallback"); return nullptr; }
    if (cfg.device < 0 || cfg.device >= n) { set_error("bad device ordinal"); return nullptr; }
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, cfg.device);
    if (p.major != 9) { set_error("device is not compute capability 9.x (kernels are built for sm_90a only)"); return nullptr; }
    Ctx* c = new Ctx();
    c->device = cfg.device;
    c->cfg = cfg;
    if (cfg.plane_res > 0) c->surf.res = cfg.plane_res;
    if (cfg.line_res > 0) c->edge.res = cfg.line_res;
    if (std::getenv("SO_NO_COND_GRAPH")) c->no_cond_graph = true;
    if (std::getenv("SO_SINGLE_STREAM")) c->single_stream = true;
    if (std::getenv("SO_NO_FUSED_LM")) c->no_fused_lm = true;
    if (std::getenv("SO_NO_SMALL_PREPARE")) c->no_small_prepare = true;
    if (std::getenv("SO_NO_COOP_KNN")) c->no_coop_knn = true;
    if (std::getenv("SO_FORCE_KEY64")) c->force_key64 = true;
    if (std::getenv("SO_FORCE_DROP_BIT")) c->force_drop_bit = true;
    if (std::getenv("SO_NO_DEC_UPLOAD")) c->no_dec_upload = true;
    if (const char* e = std::getenv("SO_KNN_GRAPH")) c->knn_graph_mode = std::strcmp(e, "on") == 0 ? 1 : (std::strcmp(e, "off") == 0 ? -1 : 0);
    if (const char* e = std::getenv("SO_CHUNKS")) c->chunk_override = std::max(0, std::min(16, std::atoi(e)));      // profiling aid: ncu cannot see inside conditional-node bodies
    if (ctx_alloc(c) != SO_OK) { ctx_free(c); return nullptr; }
    return reinterpret_cast<so_ctx*>(c);
}

void so_destroy(so_ctx* ctx) { ctx_free(reinterpret_cast<Ctx*>(ctx)); }

int so_set_stream(so_ctx* ctx, void* cuda_stream) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (auto& g : c->graphs) if (g.exec) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; }
    if (cuda_stream) {
        if (c->own_stream) cudaStreamDestroy(c->stream);
        c->stream = static_cast<cudaStream_t>(cuda_stream); c->own_stream = false;
    } else if (!c->own_stream) {
        SO_CUDA_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)); c->own_stream = true;
    }
    return SO_OK;
}

// ---- map -------------------------------------------------------------------------------------------------------
int so_map_set_resolution(so_ctx* ctx, float line_res, float plane_res) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !(plane_res > 0)) return fail(SO_ERR_ARG, "bad args");
    if (line_res > 0 && line_res != c->edge.res) {
        const int nb_old = c->edge.nb;
        c->edge.res = line_res;
        if (map_cells_per_block(line_res) != nb_old) c->edge.dirty = true;
    }
    if (plane_res != c->surf.res) {
        const int nb_old = c->surf.nb;
        c->surf.res = plane_res;
        if (map_cells_per_block(plane_res) != nb_old) c->surf.dirty = true;
    }
    return SO_OK;
}

int so_map_set_origin(so_ctx* ctx, const double t[3], int32_t out_origin[3]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !t) return fail(SO_ERR_ARG, "bad args");
    for (int a = 0; a < 3; ++a) {                           // LocalMap::setOrigin (LocalMap.h:146-164)
        int cc = int((t[a] + kHalfBlock) / kBlock);
        if (t[a] + kHalfBlock < 0) cc--;
        c->origin[a] = -cc;
        if (out_origin) out_origin[a] = c->origin[a];
    }
    c->surf.dirty = true; c->edge.dirty = true;
    return SO_OK;
}

int so_map_get_origin(so_ctx* ctx, int32_t out[3]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !out) return fail(SO_ERR_ARG, "bad args");
    for (int a = 0; a < 3; ++a) out[a] = c->origin[a];
    return SO_OK;
}

int so_map_shift(so_ctx* ctx, const double t[3], int32_t out_ijk[3]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !t || !out_ijk) return fail(SO_ERR_ARG, "bad args");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    int32_t o[3], cc[3];
    shift_origin(c->origin, t, o, cc);
    { int rc = move_window(c, o); if (rc) return rc; }
    for (int a = 0; a < 3; ++a) out_ijk[a] = cc[a];
    return SO_OK;
}

static int store_set_points(Ctx* c, MapStore& ms, const void* xyzi, size_t n, size_t stride, size_t ioff) {
    if (!c || (!xyzi && n) || stride < 12) return fail(SO_ERR_ARG, "bad args");
    if (n > c->cfg.max_map_points + ms.arc.d_pool.cap()) return fail(SO_ERR_CAPACITY, "map larger than so_config.max_map_points (plus the block archive)");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    if (ms.arc.d_pool) {                                          // window and archive replaced together; the checks come before any change
        std::vector<float4> pts(n);
        const unsigned char* p = static_cast<const unsigned char*>(xyzi);
        for (size_t i = 0; i < n; ++i) pts[i] = read_point(p + i * stride, stride, ioff);
        int rc = archive_load(c, ms, pts.data(), n);
        return rc ? rc : map_rebuild(c, ms);
    }
    int rc = upload_cloud(c, xyzi, n, stride, ioff, ms.d_xyzi);
    if (rc) return rc;
    ms.n = uint32_t(n);
    return map_rebuild(c, ms);
}
// xyzi == nullptr with n != 0: the registered scan or its edge cloud (put_registered_scan)
static int store_add(Ctx* c, MapStore& ms, const void* xyzi, size_t n, size_t stride, size_t ioff, const double* pose) {
    if (!c || stride < 12) return fail(SO_ERR_ARG, "bad args");
    if (size_t(ms.n) + n > c->cfg.max_map_points) return fail(SO_ERR_CAPACITY, "map + new points exceed so_config.max_map_points");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    if (n == 0) return SO_OK;
    int rc = SO_OK;
    if (ms.dirty) { rc = map_rebuild(c, ms); if (rc) return rc; }           // pending origin / resolution change first: it may compact the cloud
    // ... or, with the block archive on, grow it by the blocks it restores: the new points must still fit behind it
    if (size_t(ms.n) + n > c->cfg.max_map_points) return fail(SO_ERR_CAPACITY, "map + new points exceed so_config.max_map_points");
    rc = xyzi ? upload_cloud(c, xyzi, n, stride, ioff, ms.d_xyzi + ms.n) : put_registered_scan(c, &ms == &c->edge, ms.d_xyzi + ms.n, pose);
    if (rc) return rc;
    if (pose) { rc = map_transform_tail(c, ms, uint32_t(n), pose); if (rc) return rc; }
    timed_launch_begin(c);
    rc = map_add_points(c, ms, uint32_t(n));
    timed_launch_end(c, 3, 1);
    return rc;
}

int so_map_set_points(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    return c ? store_set_points(c, c->surf, xyzi, n, stride, ioff) : fail(SO_ERR_ARG, "null ctx");
}
int so_map_set_edge_points(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    return c ? store_set_points(c, c->edge, xyzi, n, stride, ioff) : fail(SO_ERR_ARG, "null ctx");
}
int so_map_add_surf(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!xyzi && n) return fail(SO_ERR_ARG, "bad args");
    return c ? store_add(c, c->surf, xyzi, n, stride, ioff, nullptr) : fail(SO_ERR_ARG, "null ctx");
}
int so_map_add_edge(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!xyzi && n) return fail(SO_ERR_ARG, "bad args");
    return c ? store_add(c, c->edge, xyzi, n, stride, ioff, nullptr) : fail(SO_ERR_ARG, "null ctx");
}
int so_map_add_scan(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, const double pose[7]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!pose || (!xyzi && n)) return fail(SO_ERR_ARG, "bad args");
    return c ? store_add(c, c->surf, xyzi, n, stride, ioff, pose) : fail(SO_ERR_ARG, "null ctx");
}
int so_map_add_registered_scan(so_ctx* ctx, const double pose[7]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose) return fail(SO_ERR_ARG, "bad args");
    if (!c->reg.valid) return fail(SO_ERR_ARG, "so_map_add_registered_scan needs a preceding single-scan so_register* (and nothing that reuses the scan buffers in between)");
    if (c->reg.n == 0) return SO_OK;
    return store_add(c, c->surf, nullptr, c->reg.n, 16, 12, pose);
}
int so_map_add_registered_edges(so_ctx* ctx, const double pose[7]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose) return fail(SO_ERR_ARG, "bad args");
    if (!c->reg.valid || !c->reg.edge_valid)
        return fail(SO_ERR_ARG, "so_map_add_registered_edges needs a preceding single-scan so_register* (and nothing that reuses the scan or edge buffers in between)");
    if (c->reg.n_edge == 0) return SO_OK;
    return store_add(c, c->edge, nullptr, c->reg.n_edge, 16, 12, pose);
}
int so_map_add_scan_edge(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, const double pose[7]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!pose || (!xyzi && n)) return fail(SO_ERR_ARG, "bad args");
    return c ? store_add(c, c->edge, xyzi, n, stride, ioff, pose) : fail(SO_ERR_ARG, "null ctx");
}

void so_free_space_defaults(so_free_space* opts) { if (opts) free_space_defaults(opts); }

int so_map_clear_free_space(so_ctx* ctx, int stores, const void* xyzi, size_t n, size_t stride, size_t ioff, const double pose[7],
                            const so_free_space* opts, so_free_space_result* result) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || (!xyzi && n) || stride < 12) return fail(SO_ERR_ARG, "bad args");
    { int rc = free_space_check(opts, stores, pose); if (rc) return rc; }
    if (n > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "so_map_clear_free_space: cloud larger than so_config.max_scan_points");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    int rc = free_space_prepare(c, stores);
    if (!rc) rc = free_space_reserve_points(c, n);
    if (!rc) rc = upload_cloud(c, xyzi, n, stride, ioff, c->fs.d_pts);
    return rc ? rc : free_space_clear(c, stores, c->fs.d_pts, uint32_t(n), pose, *opts, result);
}

// The image comes from the surf store's tail, where put_registered_scan leaves the scan as so_map_add_registered_scan would insert it
// (before the transform to the world frame); d_scan, the times and the record are only read
int so_map_clear_free_space_registered(so_ctx* ctx, int stores, const double pose[7], const so_free_space* opts, so_free_space_result* result) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    { int rc = free_space_check(opts, stores, pose); if (rc) return rc; }
    if (!c->reg.valid) return fail(SO_ERR_ARG, "so_map_clear_free_space_registered needs a preceding single-scan so_register* (and nothing that reuses the scan buffers in between)");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    if (c->reg.n == 0) {
        if (result) { *result = so_free_space_result{}; result->n_after[0] = c->surf.n; result->n_after[1] = c->edge.n; }
        return SO_OK;
    }
    int rc = free_space_prepare(c, stores | 1);
    if (rc) return rc;
    MapStore& ms = c->surf;
    if (size_t(ms.n) + c->reg.n > c->cfg.max_map_points) return fail(SO_ERR_CAPACITY, "map + registered scan exceed so_config.max_map_points");
    rc = put_registered_scan(c, false, ms.d_xyzi + ms.n, pose);
    return rc ? rc : free_space_clear(c, stores, ms.d_xyzi + ms.n, c->reg.n, pose, *opts, result);
}

int so_map_counts_5x5(so_ctx* ctx, const int32_t ijk[3], int32_t* n_edge, int32_t* n_surf) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !ijk) return fail(SO_ERR_ARG, "bad args");
    { int rc = ensure_maps(c); if (rc) return rc; }
    if (n_edge) *n_edge = counts_5x5(c, c->edge, ijk);
    if (n_surf) *n_surf = counts_5x5(c, c->surf, ijk);
    return SO_OK;
}

size_t so_map_size(so_ctx* ctx) { Ctx* c = reinterpret_cast<Ctx*>(ctx); return c ? size_t(c->surf.n) + size_t(c->edge.n) : 0; }

int so_map_archive(so_ctx* ctx, size_t cap_points) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    return archive_set_cap(c, cap_points);
}

int so_map_archive_info(so_ctx* ctx, int store, size_t* n_points, size_t* n_blocks, size_t* cap_points) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || (store != 0 && store != 1)) return fail(SO_ERR_ARG, "bad args");
    const BlockArchive& a = (store ? c->edge : c->surf).arc;
    if (n_points) *n_points = a.live;
    if (n_blocks) *n_blocks = a.dir.size();
    if (cap_points) *cap_points = a.d_pool.cap();
    return SO_OK;
}

int so_map_download_all(so_ctx* ctx, int store, float* out, size_t cap, size_t* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !n_out || (store != 0 && store != 1)) return fail(SO_ERR_ARG, "bad args");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    { int rc = ensure_maps(c); if (rc) return rc; }
    return archive_download_all(c, store ? c->edge : c->surf, out, cap, n_out);
}

int so_map_download(so_ctx* ctx, int mode, const int32_t ijk[3], float* out, size_t cap, size_t* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !n_out) return fail(SO_ERR_ARG, "bad args");
    if (mode == 1 && !ijk) return fail(SO_ERR_ARG, "mode 1 needs ijk");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    { int rc = ensure_maps(c); if (rc) return rc; }
    // LocalMap::getAllLocalMap / get5x5LocalMap (LocalMap.h:647-687): cubes in index order, each cube's edge cloud then its surf cloud
    std::vector<float4> he(c->edge.n), hs(c->surf.n);
    if (c->edge.n) SO_CUDA_TRY(cudaMemcpy(he.data(), c->edge.d_xyzi, size_t(c->edge.n) * sizeof(float4), cudaMemcpyDeviceToHost));
    if (c->surf.n) SO_CUDA_TRY(cudaMemcpy(hs.data(), c->surf.d_xyzi, size_t(c->surf.n) * sizeof(float4), cudaMemcpyDeviceToHost));
    struct Ref { int32_t lin; uint8_t kind; uint32_t idx; };
    std::vector<Ref> refs;
    refs.reserve(he.size() + hs.size());
    auto push = [&](const std::vector<float4>& h, uint8_t kind) {
        for (uint32_t i = 0; i < h.size(); ++i) {
            int g[3]; const float q[3] = {h[i].x, h[i].y, h[i].z};
            for (int a = 0; a < 3; ++a) g[a] = block_coord_h(double(q[a]) + kHalfBlock, c->origin[a]);
            if (mode == 1 && (std::abs(g[0] - ijk[0]) > 2 || std::abs(g[1] - ijk[1]) > 2 || std::abs(g[2] - ijk[2]) > 1)) continue;
            refs.push_back(Ref{g[0] + kW * g[1] + kW * kH * g[2], kind, i});
        }
    };
    push(he, 0); push(hs, 1);
    if (mode == 1) {    // get5x5LocalMap loops i (x) outermost, then j, then k: order by (i, j, k), not by the linear cube index
        std::stable_sort(refs.begin(), refs.end(), [](const Ref& a, const Ref& b) {
            const int ai = a.lin % kW, aj = (a.lin / kW) % kH, ak = a.lin / (kW * kH), bi = b.lin % kW, bj = (b.lin / kW) % kH, bk = b.lin / (kW * kH);
            if (ai != bi) return ai < bi; if (aj != bj) return aj < bj; if (ak != bk) return ak < bk; return a.kind < b.kind; });
    } else {
        std::stable_sort(refs.begin(), refs.end(), [](const Ref& a, const Ref& b) { return a.lin != b.lin ? a.lin < b.lin : a.kind < b.kind; });
    }
    size_t k = 0;
    for (const Ref& r : refs) {
        if (out && k < cap) std::memcpy(out + 4 * k, r.kind ? &hs[r.idx] : &he[r.idx], sizeof(float4));
        ++k;
    }
    *n_out = k;
    return SO_OK;
}

// ---- scan pre-filter ---------------------------------------------------------------------------------------------
int so_scan_prefilter(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, int auto_voxel_size, float* line_res,
                      float* plane_res, float* out_xyzi, size_t cap, size_t* n_out, double* average_distance) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || (!xyzi && n) || stride < 12 || !line_res || !plane_res || !n_out || (!out_xyzi && cap)) return fail(SO_ERR_ARG, "bad args");
    if (n > c->scan_cap) return fail(SO_ERR_CAPACITY, "cloud larger than the scan buffers");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    *n_out = 0;
    if (auto_voxel_size && n) {
        // laserMapping::adjustVoxelSize (laserMapping.cpp:603-636): float accumulators in cloud order, exactly as written there
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        int far_points = 0;
        const unsigned char* p = static_cast<const unsigned char*>(xyzi);
        for (size_t i = 0; i < n; ++i, p += stride) {
            float v[3];
            std::memcpy(v, p, 12);
            a0 += std::fabs(v[0]); a1 += std::fabs(v[1]); a2 += std::fabs(v[2]);
            if (v[0] * v[0] + v[1] * v[1] + v[2] * v[2] > 9) far_points++;
        }
        (void)far_points;                                          // increase_blind_radius is computed and never used upstream
        const float sz = float(n);
        a0 /= sz; a1 /= sz; a2 /= sz;
        const double avg = double(a0 * a1 * a2);                   // float product stored into a float64 field
        if (average_distance) *average_distance = avg;
        if (avg < 25) { *line_res = 0.1f; *plane_res = 0.2f; }
        else if (avg > 65) { *line_res = 0.4f; *plane_res = 0.8f; }
    }
    int rc = so_map_set_resolution(ctx, *line_res, *plane_res);   // slam.localMap.lineRes_/planeRes_ = config_ (:648-649)
    if (rc) return rc;
    c->reg.valid = false;
    rc = upload_cloud(c, xyzi, n, stride, ioff, c->d_scan);
    if (rc) return rc;
    uint32_t m = 0;
    timed_launch_begin(c);
    rc = scan_voxel_filter(c, uint32_t(n), *plane_res, &m);
    timed_launch_end(c, 3, 1);
    if (rc) return rc;
    *n_out = m;
    c->prefiltered_n = m;                                          // so_register_prefiltered: the filtered cloud stays in d_scan_sorted
    const size_t ncopy = std::min<size_t>(m, cap);
    if (ncopy) {
        SO_CUDA_TRY(cudaMemcpyAsync(out_xyzi, c->d_scan_sorted, ncopy * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
        count_d2h(c, ncopy * sizeof(float4));
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    return SO_OK;
}

// ---- scan preparation: deskew + uniform extraction (featureExtraction.cpp:222-314,504-525) ----------------------
namespace {
struct HPose { double q[4]; double p[3]; };      // xyzw
HPose hpose_from7(const double* v) { return HPose{{v[3], v[4], v[5], v[6]}, {v[0], v[1], v[2]}}; }
void hnormalize(double q[4]) {
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int k = 0; k < 4; ++k) q[k] /= n;
}
// Eigen::QuaternionBase::slerp
void hslerp(const double a[4], double t, const double b[4], double o[4]) {
    const double one = 1.0 - std::numeric_limits<double>::epsilon();
    const double d = a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3];
    const double ad = std::fabs(d);
    double s0, s1;
    if (ad >= one) { s0 = 1.0 - t; s1 = t; }
    else {
        const double th = std::acos(ad), st = std::sin(th);
        s0 = std::sin((1.0 - t) * th) / st;
        s1 = std::sin(t * th) / st;
    }
    if (d < 0) s1 = -s1;
    for (int k = 0; k < 4; ++k) o[k] = s0 * a[k] + s1 * b[k];
}
// the sign Eigen's matrix -> quaternion conversion produces (w > 0 when the trace is positive, else the dominant axis > 0)
void hcanonical_sign(double q[4]) {
    const double tr = 4.0 * q[3] * q[3] - 1.0;        // trace of R(q) for a unit q
    bool flip;
    if (tr > 0) flip = q[3] < 0;
    else {
        int i = 0;
        if (std::fabs(q[1]) > std::fabs(q[0])) i = 1;
        if (std::fabs(q[2]) > std::fabs(q[i])) i = 2;
        flip = q[i] < 0;
    }
    if (flip) for (int k = 0; k < 4; ++k) q[k] = -q[k];
}
}  // namespace

int so_scan_deskew(so_ctx* ctx, void* points, size_t n, size_t stride, size_t time_offset, double lidar_start_time, const double* sample_times,
                   const double* sample_poses, size_t n_samples, int imu_only, const double T_i_l[7], double start_pose_out[7], size_t* n_past_end) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || (!points && n) || stride < 12 || time_offset + 4 > stride || !sample_times || !sample_poses || n_samples == 0 || (imu_only && !T_i_l))
        return fail(SO_ERR_ARG, "bad args");
    if (n > c->scan_cap) return fail(SO_ERR_CAPACITY, "cloud larger than the scan buffers");
    if (n_samples * 8 > c->scan_cap) return fail(SO_ERR_CAPACITY, "more pose samples than the scratch holds (max_scan_points / 8)");
    for (size_t k = 1; k < n_samples; ++k)
        if (!(sample_times[k] > sample_times[k - 1])) return fail(SO_ERR_ARG, "sample_times must be strictly ascending (std::map keys)");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    // getInterpolatedPoseAtTime(lidar_start_time) on the host (:279): same rule as the kernel
    size_t after = size_t(std::upper_bound(sample_times, sample_times + n_samples, lidar_start_time) - sample_times);
    if (after == n_samples) after = n_samples - 1;
    if (sample_times[after] < 0.0001) after = 0;
    HPose start;
    if (after == 0) start = hpose_from7(sample_poses);
    else {
        const HPose a = hpose_from7(sample_poses + 7 * (after - 1)), b = hpose_from7(sample_poses + 7 * after);
        const double ratio = (lidar_start_time - sample_times[after - 1]) / (sample_times[after] - sample_times[after - 1]);
        hslerp(a.q, ratio, b.q, start.q);
        for (int k = 0; k < 3; ++k) start.p[k] = (1 - ratio) * a.p[k] + ratio * b.p[k];
    }
    if (imu_only) start.p[0] = start.p[1] = start.p[2] = 0.0;          // Imu::Ptr samples carry no translation (:232-236)
    hnormalize(start.q);
    DeskewParams P{};
    P.start_time = lidar_start_time;
    P.n_samples = uint32_t(n_samples);
    P.n_smem = uint32_t(std::min<size_t>(n_samples, 2048));
    P.imu_only = imu_only ? 1 : 0;
    P.q0_conj[0] = -start.q[0]; P.q0_conj[1] = -start.q[1]; P.q0_conj[2] = -start.q[2]; P.q0_conj[3] = start.q[3];
    for (int k = 0; k < 3; ++k) P.p0[k] = start.p[k];
    double out7[7] = {start.p[0], start.p[1], start.p[2], start.q[0], start.q[1], start.q[2], start.q[3]};
    if (imu_only) {
        HPose il = hpose_from7(T_i_l);
        hnormalize(il.q);
        for (int k = 0; k < 4; ++k) P.q_il[k] = il.q[k];
        for (int k = 0; k < 3; ++k) P.t_il[k] = il.p[k];
        P.q_li[0] = -il.q[0]; P.q_li[1] = -il.q[1]; P.q_li[2] = -il.q[2]; P.q_li[3] = il.q[3];
        double r[3];
        qrot(P.q_li, il.p, r);                                           // Twist::inverse (Twist.h:172-179)
        P.t_li[0] = -r[0]; P.t_li[1] = -r[1]; P.t_li[2] = -r[2];
        // T_w_original_sensor = T_w_original * T_i_l (:283-286)
        double q[4];
        qmul(start.q, il.q, q);
        hnormalize(q);
        hcanonical_sign(q);
        qrot(start.q, il.p, r);
        out7[0] = r[0] + start.p[0]; out7[1] = r[1] + start.p[1]; out7[2] = r[2] + start.p[2];
        out7[3] = q[0]; out7[4] = q[1]; out7[5] = q[2]; out7[6] = q[3];
    }
    if (start_pose_out) std::memcpy(start_pose_out, out7, sizeof(out7));
    if (n_past_end) *n_past_end = 0;
    if (n == 0) return SO_OK;
    c->reg.valid = false;
    int rc = upload_cloud(c, points, n, stride, time_offset, c->d_scan);          // float4 {x, y, z, time}
    if (rc) return rc;
    // pose samples into device scratch (the scan-sort key buffer): [times n][poses 7n]; IMU samples lose their translation here
    std::vector<double> hs(n_samples * 8);
    for (size_t k = 0; k < n_samples; ++k) {
        hs[k] = sample_times[k];
        for (int j = 0; j < 7; ++j) hs[n_samples + 7 * k + j] = (imu_only && j < 3) ? 0.0 : sample_poses[7 * k + j];
    }
    double* d_samples = reinterpret_cast<double*>(c->d_skeys.get());
    SO_CUDA_TRY(cudaMemcpyAsync(d_samples, hs.data(), hs.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    count_h2d(c, hs.size() * sizeof(double));
    SO_CUDA_TRY(cudaMemsetAsync(c->d_svals, 0, 4, c->stream));
    P.times = d_samples; P.poses = d_samples + n_samples; P.past_end = c->d_svals;
    timed_launch_begin(c);
    launch_deskew(c->d_scan, uint32_t(n), P, c->stream);
    c->launches++;
    timed_launch_end(c, 3, 1);
    rc = ensure_stage(c, n);
    if (rc) return rc;
    uint32_t past = 0;
    SO_CUDA_TRY(cudaMemcpyAsync(c->h_stage, c->d_scan, n * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(&past, c->d_svals, 4, cudaMemcpyDeviceToHost, c->stream));
    count_d2h(c, n * sizeof(float4) + 4);
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));                                 // also covers hs going out of scope
    const float4* h = c->h_stage;
    unsigned char* dst = static_cast<unsigned char*>(points);
    for (size_t i = 0; i < n; ++i, dst += stride) std::memcpy(dst, &h[i], 12);     // x, y, z only; every other field untouched
    if (n_past_end) *n_past_end = past;
    return SO_OK;
}

int so_scan_extract_uniform(so_ctx* ctx, const void* points, size_t n, size_t stride, size_t time_offset, int skip_num, float block_range,
                            int int_abs, float* out_xyzi, size_t cap, size_t* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || (!points && n) || stride < 12 || time_offset + 4 > stride || !n_out || (!out_xyzi && cap)) return fail(SO_ERR_ARG, "bad args");
    if (skip_num <= 0) return fail(SO_ERR_ARG, "skip_num must be positive (the reference loop would not terminate)");
    if (n > c->scan_cap) return fail(SO_ERR_CAPACITY, "cloud larger than the scan buffers");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    *n_out = 0;
    c->reg.valid = false;
    int rc = upload_cloud(c, points, n, stride, time_offset, c->d_scan);
    if (rc) return rc;
    uint32_t m = 0;
    timed_launch_begin(c);
    rc = scan_extract_uniform(c, uint32_t(n), uint32_t(skip_num), block_range, int_abs, &m);
    timed_launch_end(c, 3, 1);
    if (rc) return rc;
    *n_out = m;
    const size_t ncopy = std::min<size_t>(m, cap);
    if (ncopy) {
        SO_CUDA_TRY(cudaMemcpyAsync(out_xyzi, c->d_scan_sorted, ncopy * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
        count_d2h(c, ncopy * sizeof(float4));
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    return SO_OK;
}

// ---- registration: the so_register* family.  Each entry point checks its own arguments, in its own order and with its own messages,
// describes the call and hands it to register_scans.  Single-scan calls return the registration's status, batches SO_OK.
int so_register(so_ctx* ctx, const void* surf, size_t n_surf, const void* edge, size_t n_edge, size_t stride, size_t ioff,
                const double pose_in[7], const so_icp_opts* opts, so_icp_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose_in || !opts || !out || (!surf && n_surf) || (!edge && n_edge) || stride < 12) return fail(SO_ERR_ARG, "bad args");
    if (n_edge > c->edge_cap) return fail(SO_ERR_CAPACITY, "edge cloud larger than so_config.max_scan_points");
    if (n_surf > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "scan larger than so_config.max_scan_points");
    const uint32_t n = uint32_t(n_surf), ne = uint32_t(n_edge);
    RegisterRequest q = single_scan(&n, pose_in, opts, out);
    q.scans = surf; q.stride = stride; q.ioff = ioff;
    q.edge = edge; q.n_edge = &ne;                                       // edge branch input (empty upstream: featureExtraction.cpp:429-436)
    return status_of(register_scans(c, q), *out);
}

int so_register_prefiltered(so_ctx* ctx, const double pose_in[7], const so_icp_opts* opts, so_icp_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose_in || !opts || !out) return fail(SO_ERR_ARG, "bad args");
    if (c->prefiltered_n == SIZE_MAX) return fail(SO_ERR_ARG, "so_register_prefiltered needs a preceding so_scan_prefilter (and nothing that reuses the scan buffers in between)");
    const uint32_t n = uint32_t(c->prefiltered_n);
    RegisterRequest q = single_scan(&n, pose_in, opts, out);
    q.src = Source::PREFILTERED;
    return status_of(register_scans(c, q), *out);
}

int so_register_injected(so_ctx* ctx, const void* surf, size_t n_surf, size_t stride, size_t ioff, const double pose_in[7], const so_icp_opts* opts,
                         const uint32_t* nn_ids, int32_t n_trace_iters, so_icp_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose_in || !opts || !out || !surf || !nn_ids || n_surf == 0 || n_trace_iters <= 0 || stride < 12) return fail(SO_ERR_ARG, "bad args");
    if (n_surf > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "scan larger than so_config.max_scan_points");
    const uint32_t n = uint32_t(n_surf);
    RegisterRequest q = single_scan(&n, pose_in, opts, out);
    q.scans = surf; q.stride = stride; q.ioff = ioff; q.inject = nn_ids; q.inject_iters = n_trace_iters;
    q.insertable = false;                                                // a test hook: its scan is not the live loop's
    return status_of(register_scans(c, q), *out);
}

int so_register_batch(so_ctx* ctx, const void* surf, const uint32_t* n_points, size_t n_scans, size_t stride, size_t ioff,
                      const double* poses_in, const so_icp_opts* opts, so_icp_result* results) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !surf || !n_points || !poses_in || !opts || !results || stride < 12) return fail(SO_ERR_ARG, "bad args");
    int rc = check_batch(c, n_points, n_scans);
    return rc ? rc : register_scans(c, batch_request(surf, n_points, n_scans, stride, ioff, poses_in, opts, results));
}

int so_register_batch_edges(so_ctx* ctx, const void* surf, const uint32_t* n_points, const void* edge, const uint32_t* n_edge, size_t n_scans,
                            size_t stride, size_t ioff, const double* poses_in, const so_icp_opts* opts, so_icp_result* results) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !surf || !n_points || !n_edge || !poses_in || !opts || !results || stride < 12) return fail(SO_ERR_ARG, "bad args");
    int rc = check_batch(c, n_points, n_scans);
    if (rc) return rc;
    size_t total_e = 0;
    for (size_t s = 0; s < n_scans; ++s) total_e += n_edge[s];
    if (total_e > c->edge_cap) return fail(SO_ERR_CAPACITY, "edge clouds of the batch exceed so_config.max_scan_points points in total");
    if (total_e && !edge) return fail(SO_ERR_ARG, "bad args");
    RegisterRequest q = batch_request(surf, n_points, n_scans, stride, ioff, poses_in, opts, results);
    q.src = Source::HOST;                                                // uploaded whole, packed or not
    q.edge = edge; q.n_edge = n_edge;
    return register_scans(c, q);
}

int so_register_batch_device(so_ctx* ctx, const void* d_scans, const uint32_t* n_points, size_t n_scans, const double* poses_in,
                             const so_icp_opts* opts, so_icp_result* results) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !d_scans || !n_points || !poses_in || !opts || !results) return fail(SO_ERR_ARG, "bad args");
    int rc = check_batch(c, n_points, n_scans);
    if (rc) return rc;
    RegisterRequest q = batch_request(d_scans, n_points, n_scans, 16, 12, poses_in, opts, results);
    q.src = Source::DEVICE;
    return register_scans(c, q);
}

// Keyframes of src registered against dst's map as so_register_batch_device registers device scans: mode NONE (a keyframe is already
// compensated), dst's registered-scan record untouched.  degen: NULL, or one DegenState per keyframe (so_register_keyframes_degeneracy)
static int register_keyframes(Ctx* c, Ctx* s, const int32_t* ids, size_t n, const double* priors7, const so_icp_opts* opts,
                              so_icp_result* results, DegenState* degen) {
    SO_CUDA_TRY(cudaSetDevice(c->device));
    const float4* scans = nullptr;
    std::vector<uint32_t> n_points;
    int rc = keyframe_scans(c, s, ids, n, &scans, &n_points);
    if (!rc) rc = check_batch(c, n_points.data(), n);
    if (rc) return rc;
    RegisterRequest q = batch_request(scans, n_points.data(), n, 16, 12, priors7, opts, results);
    q.src = Source::DEVICE;
    q.degen = degen;
    return register_scans(c, q);
}

int so_register_keyframes(so_ctx* dst_ctx, so_ctx* src_ctx, const int32_t* ids, size_t n, const double* priors7, const so_icp_opts* opts,
                          so_icp_result* results) {
    Ctx* c = reinterpret_cast<Ctx*>(dst_ctx);
    Ctx* s = reinterpret_cast<Ctx*>(src_ctx);
    if (!c || !s || !ids || !priors7 || !opts || !results) return fail(SO_ERR_ARG, "bad args");
    if (c->device != s->device) return fail(SO_ERR_ARG, "so_register_keyframes: the two contexts are on different devices");
    return register_keyframes(c, s, ids, n, priors7, opts, results, nullptr);
}

// ---- degeneracy-aware registration: so_register's schedule with k_lm_step_deg stepping the solves (DESIGN.md section 3)
static DegenState degen_state(const so_degeneracy& d) {
    DegenState s{};
    s.pos_thr2 = d.pos_threshold * d.pos_threshold;
    s.ori_thr2 = d.ori_threshold * d.ori_threshold;
    s.constrain = d.constrain;
    s.m = 6;
    return s;
}
static void fill_degeneracy(const DegenState& s, so_degeneracy_result* out) {
    std::memcpy(out->iter_n_flag_pos, s.iter_n_flag_pos, sizeof(out->iter_n_flag_pos));
    std::memcpy(out->iter_n_flag_ori, s.iter_n_flag_ori, sizeof(out->iter_n_flag_ori));
    std::memcpy(out->pos_info, s.pos_info, sizeof(out->pos_info)); std::memcpy(out->pos_axes, s.pos_axes, sizeof(out->pos_axes));
    std::memcpy(out->ori_info, s.ori_info, sizeof(out->ori_info)); std::memcpy(out->ori_axes, s.ori_axes, sizeof(out->ori_axes));
    out->flags_pos = s.flags_pos; out->flags_ori = s.flags_ori;
}

int so_register_degeneracy(so_ctx* ctx, const void* surf, size_t n_surf, const void* edge, size_t n_edge, size_t stride, size_t ioff,
                           const double pose_in[7], const so_degeneracy* d, const so_icp_opts* opts, so_degeneracy_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose_in || !d || !opts || !out || (!surf && n_surf) || (!edge && n_edge) || stride < 12) return fail(SO_ERR_ARG, "bad args");
    int rc = check_degeneracy(d, 1);
    if (rc) return rc;
    if (n_edge > c->edge_cap) return fail(SO_ERR_CAPACITY, "edge cloud larger than so_config.max_scan_points");
    if (n_surf > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "scan larger than so_config.max_scan_points");
    const uint32_t n = uint32_t(n_surf), ne = uint32_t(n_edge);
    DegenState S = degen_state(*d);
    RegisterRequest q = single_scan(&n, pose_in, opts, &out->icp);
    q.scans = surf; q.stride = stride; q.ioff = ioff;
    q.edge = edge; q.n_edge = &ne;
    q.degen = &S;
    rc = register_scans(c, q);
    if (rc) return rc;
    fill_degeneracy(S, out);
    return out->icp.status;
}

int so_register_batch_degeneracy(so_ctx* ctx, const void* surf, const uint32_t* n_points, const void* edge, const uint32_t* n_edge, size_t n_scans,
                                 size_t stride, size_t ioff, const double* poses_in, const so_degeneracy* d, const so_icp_opts* opts,
                                 so_degeneracy_result* results) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !surf || !n_points || !poses_in || !d || !opts || !results || stride < 12) return fail(SO_ERR_ARG, "bad args");
    int rc = check_batch(c, n_points, n_scans);
    if (!rc) rc = check_degeneracy(d, n_scans);
    if (rc) return rc;
    size_t total_e = 0;
    if (n_edge) for (size_t s = 0; s < n_scans; ++s) total_e += n_edge[s];
    if (total_e > c->edge_cap) return fail(SO_ERR_CAPACITY, "edge clouds of the batch exceed so_config.max_scan_points points in total");
    if (total_e && !edge) return fail(SO_ERR_ARG, "bad args");
    std::vector<so_icp_result> icp(n_scans);
    std::vector<DegenState> S(n_scans);
    for (size_t s = 0; s < n_scans; ++s) S[s] = degen_state(d[s]);
    RegisterRequest q = batch_request(surf, n_points, n_scans, stride, ioff, poses_in, opts, icp.data());
    if (n_edge) { q.src = Source::HOST; q.edge = edge; q.n_edge = n_edge; }      // as so_register_batch_edges
    q.degen = S.data();
    rc = register_scans(c, q);
    if (rc) return rc;
    for (size_t s = 0; s < n_scans; ++s) { results[s].icp = icp[s]; fill_degeneracy(S[s], results + s); }
    return SO_OK;
}

// so_register_keyframes with the degeneracy-aware step, as so_register_batch_degeneracy adds it to so_register_batch
int so_register_keyframes_degeneracy(so_ctx* dst_ctx, so_ctx* src_ctx, const int32_t* ids, size_t n, const double* priors7,
                                     const so_degeneracy* d, const so_icp_opts* opts, so_degeneracy_result* results) {
    Ctx* c = reinterpret_cast<Ctx*>(dst_ctx);
    Ctx* s = reinterpret_cast<Ctx*>(src_ctx);
    if (!c || !s || !ids || !priors7 || !d || !opts || !results) return fail(SO_ERR_ARG, "bad args");
    if (c->device != s->device) return fail(SO_ERR_ARG, "so_register_keyframes_degeneracy: the two contexts are on different devices");
    int rc = check_degeneracy(d, n);
    if (rc) return rc;
    std::vector<so_icp_result> icp(std::max<size_t>(n, 1));
    std::vector<DegenState> S(std::max<size_t>(n, 1));
    for (size_t k = 0; k < n; ++k) S[k] = degen_state(d[k]);
    rc = register_keyframes(c, s, ids, n, priors7, opts, icp.data(), S.data());
    if (rc) return rc;
    for (size_t k = 0; k < n; ++k) { results[k].icp = icp[k]; fill_degeneracy(S[k], results + k); }
    return SO_OK;
}

// so_register_undistort (edge == nullptr, n_edge == 0) and so_register_undistort_edges: both clouds share the layout and the time offset
static int register_undistort(so_ctx* ctx, const void* surf, size_t n_surf, const void* edge, size_t n_edge, size_t stride, size_t ioff,
                              size_t toff, const double pose_in[7], const so_undistort* u, const so_icp_opts* opts, so_icp_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose_in || !opts || !out || (!surf && n_surf) || (!edge && n_edge) || stride < 12 || toff + 4 > stride) return fail(SO_ERR_ARG, "bad args");
    if (n_edge > c->edge_cap) return fail(SO_ERR_CAPACITY, "edge cloud larger than so_config.max_scan_points");
    int rc = check_undistort(u);
    if (rc) return rc;
    if (u->mode == 0) return so_register(ctx, surf, n_surf, n_edge ? edge : nullptr, n_edge, stride, ioff, pose_in, opts, out);
    if (n_surf > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "scan larger than so_config.max_scan_points");
    const uint32_t n = uint32_t(n_surf), ne = uint32_t(n_edge);
    const UndistortParams P = make_params(*u);
    RegisterRequest q = single_scan(&n, pose_in, opts, out);
    q.scans = surf; q.stride = stride; q.ioff = ioff; q.toff = toff; q.mode = UndistortionMode::APPROXIMATED; q.und = &P;
    if (ne) { q.edge = edge; q.n_edge = &ne; }
    return status_of(register_scans(c, q), *out);
}

int so_register_undistort(so_ctx* ctx, const void* surf, size_t n_surf, size_t stride, size_t ioff, size_t toff, const double pose_in[7],
                          const so_undistort* u, const so_icp_opts* opts, so_icp_result* out) {
    return register_undistort(ctx, surf, n_surf, nullptr, 0, stride, ioff, toff, pose_in, u, opts, out);
}

int so_register_undistort_edges(so_ctx* ctx, const void* surf, size_t n_surf, const void* edge, size_t n_edge, size_t stride, size_t ioff,
                                size_t toff, const double pose_in[7], const so_undistort* u, const so_icp_opts* opts, so_icp_result* out) {
    return register_undistort(ctx, surf, n_surf, edge, n_edge, stride, ioff, toff, pose_in, u, opts, out);
}

int so_register_prefiltered_undistort(so_ctx* ctx, const double pose_in[7], const so_undistort* u, const so_icp_opts* opts, so_icp_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose_in || !opts || !out) return fail(SO_ERR_ARG, "bad args");
    int rc = check_undistort(u);
    if (rc) return rc;
    if (u->mode == 0) return so_register_prefiltered(ctx, pose_in, opts, out);
    if (c->prefiltered_n == SIZE_MAX) return fail(SO_ERR_ARG, "so_register_prefiltered_undistort needs a preceding so_scan_prefilter (and nothing that reuses the scan buffers in between)");
    const uint32_t n = uint32_t(c->prefiltered_n);
    const UndistortParams P = make_params(*u);
    RegisterRequest q = single_scan(&n, pose_in, opts, out);
    q.src = Source::PREFILTERED; q.mode = UndistortionMode::APPROXIMATED; q.und = &P;
    return status_of(register_scans(c, q), *out);
}

int so_register_batch_undistort(so_ctx* ctx, const void* surf, const uint32_t* n_points, size_t n_scans, size_t stride, size_t ioff, size_t toff,
                                const double* poses_in, const so_undistort* u, const so_icp_opts* opts, so_icp_result* results) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !surf || !n_points || !poses_in || !u || !opts || !results || stride < 12 || toff + 4 > stride) return fail(SO_ERR_ARG, "bad args");
    int rc = check_batch(c, n_points, n_scans);
    if (rc) return rc;
    std::vector<UndistortParams> P(n_scans);
    bool any = false;
    for (size_t s = 0; s < n_scans; ++s) {
        if ((rc = check_undistort(u + s))) return rc;
        P[s] = make_params(u[s]);
        any |= P[s].on != 0;
    }
    RegisterRequest q = batch_request(surf, n_points, n_scans, stride, ioff, poses_in, opts, results);
    q.toff = toff; q.und = P.data();
    q.mode = any ? UndistortionMode::APPROXIMATED : UndistortionMode::NONE;   // mode 0 scans in an APPROXIMATED batch: the warp skips them
    return register_scans(c, q);
}

// so_register_optimized (edge == nullptr, n_edge == 0) and so_register_optimized_edges: both clouds share the layout and the time offset
static int register_optimized(so_ctx* ctx, const void* surf, size_t n_surf, const void* edge, size_t n_edge, size_t stride, size_t ioff,
                              size_t toff, const double pose_in[7], const so_motion* m, const so_icp_opts* opts, so_motion_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose_in || !opts || !out || (!surf && n_surf) || (!edge && n_edge) || stride < 12 || toff + 4 > stride) return fail(SO_ERR_ARG, "bad args");
    if (n_edge > c->edge_cap) return fail(SO_ERR_CAPACITY, "edge cloud larger than so_config.max_scan_points");
    int rc = check_motion(m, opts);
    if (rc) return rc;
    if (n_surf > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "scan larger than so_config.max_scan_points");
    const uint32_t n = uint32_t(n_surf), ne = uint32_t(n_edge);
    MotionState M = make_state(*m);
    so_icp_result icp;
    RegisterRequest q = single_scan(&n, pose_in, opts, &icp);
    q.scans = surf; q.stride = stride; q.ioff = ioff; q.toff = toff;
    q.mode = UndistortionMode::OPTIMIZED; q.motion = &M; q.motion_results = out;
    if (ne) { q.edge = edge; q.n_edge = &ne; }
    return status_of(register_scans(c, q), icp);
}

int so_register_optimized(so_ctx* ctx, const void* surf, size_t n_surf, size_t stride, size_t ioff, size_t toff, const double pose_in[7],
                          const so_motion* m, const so_icp_opts* opts, so_motion_result* out) {
    return register_optimized(ctx, surf, n_surf, nullptr, 0, stride, ioff, toff, pose_in, m, opts, out);
}

int so_register_optimized_edges(so_ctx* ctx, const void* surf, size_t n_surf, const void* edge, size_t n_edge, size_t stride, size_t ioff,
                                size_t toff, const double pose_in[7], const so_motion* m, const so_icp_opts* opts, so_motion_result* out) {
    return register_optimized(ctx, surf, n_surf, edge, n_edge, stride, ioff, toff, pose_in, m, opts, out);
}

int so_register_prefiltered_optimized(so_ctx* ctx, const double pose_in[7], const so_motion* m, const so_icp_opts* opts, so_motion_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose_in || !opts || !out) return fail(SO_ERR_ARG, "bad args");
    int rc = check_motion(m, opts);
    if (rc) return rc;
    if (c->prefiltered_n == SIZE_MAX) return fail(SO_ERR_ARG, "so_register_prefiltered_optimized needs a preceding so_scan_prefilter (and nothing that reuses the scan buffers in between)");
    const uint32_t n = uint32_t(c->prefiltered_n);
    MotionState M = make_state(*m);
    so_icp_result icp;
    RegisterRequest q = single_scan(&n, pose_in, opts, &icp);
    q.src = Source::PREFILTERED; q.mode = UndistortionMode::OPTIMIZED; q.motion = &M; q.motion_results = out;
    return status_of(register_scans(c, q), icp);
}

int so_register_batch_optimized(so_ctx* ctx, const void* surf, const uint32_t* n_points, size_t n_scans, size_t stride, size_t ioff, size_t toff,
                                const double* poses_in, const so_motion* m, const so_icp_opts* opts, so_motion_result* results) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !surf || !n_points || !poses_in || !m || !opts || !results || stride < 12 || toff + 4 > stride) return fail(SO_ERR_ARG, "bad args");
    int rc = check_batch(c, n_points, n_scans);
    if (rc) return rc;
    std::vector<MotionState> M(n_scans);
    for (size_t s = 0; s < n_scans; ++s) {
        if ((rc = check_motion(m + s, opts))) return rc;
        M[s] = make_state(m[s]);
    }
    std::vector<so_icp_result> icp(n_scans);
    RegisterRequest q = batch_request(surf, n_points, n_scans, stride, ioff, poses_in, opts, icp.data());
    q.toff = toff; q.mode = UndistortionMode::OPTIMIZED; q.motion = M.data(); q.motion_results = results;
    return register_scans(c, q);
}

int so_set_pose_sink(so_ctx* ctx, void* d_rows, size_t cap_rows, size_t first_row) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || (d_rows && first_row > cap_rows)) return fail(SO_ERR_ARG, "bad args");
    // no synchronisation: rows are written by kernels on the context stream, so work already enqueued there keeps its order
    c->d_pose_sink = static_cast<double*>(d_rows); c->sink_cap = d_rows ? cap_rows : 0; c->sink_cursor = d_rows ? first_row : 0;
    return SO_OK;
}

// ---- stage-level entry points ------------------------------------------------------------------------------------
// so_correspond / so_correspond_seeded: pose_prev == nullptr -> the search and fit of iteration 0 at `pose`; otherwise the scan is
// ordered at pose_prev, iteration 0 runs there unreported, and iteration 1 runs at `pose` on the neighbour records it left.
static int correspond_stage(Ctx* c, const void* surf, size_t n, size_t stride, size_t ioff, const double pose[7], const double* pose_prev,
                            int32_t max_surface_features, so_corr* corr, int32_t hist_obs[9], int32_t hist_rej[7]) {
    if (n > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "scan larger than so_config.max_scan_points");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    { int rc0 = ensure_maps(c); if (rc0) return rc0; }
    c->reg.valid = false;
    int rc = upload_cloud(c, surf, n, stride, ioff, c->d_scan);
    if (rc) return rc;
    so_icp_opts o{}; o.max_icp_iters = -1; o.lm_max_iterations = 4; o.max_surface_features = max_surface_features;
    init_state(c->h_state[0], pose_prev ? pose_prev : pose, uint32_t(n), o);
    c->h_offset[0] = 0;
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, sizeof(IcpState), cudaMemcpyHostToDevice, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_offset, c->h_offset, sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    Chunk ch{0, 1, 0, uint32_t(n)};
    ch.grid_in = (uint32_t(n) + kThreads - 1) / kThreads;
    plan_chunk(c, ch, uint32_t(n), true);                               // as a single small registration would search
    rc = prepare_scans(c, c->d_scan, ch, c->stream, false);              // stage API reports every point: decimation stays inside the kernels
    if (rc) return rc;
    rc = knn_graph_prepare(c, 0);                                       // a stage call builds the neighbour graph only when it is forced on
    if (!rc) rc = graph_queue_begin(c, 1);
    if (rc) return rc;
    const MapView mv = search_view(c);
    const BatchView bv = chunk_view(c, c->d_scan_sorted, ch);
    auto correspond = [&] {
        timed_launch_begin(c);
        const uint32_t k = launch_match(mv, bv, c->corr, c->nn, ch.grid_x, 1, c->stream);
        timed_launch_end(c, 0, k + launch_first_eval(bv, c->corr, ch.grid_x, 1, c->stream));
    };
    correspond();
    SO_CUDA_TRY(cudaGetLastError());
    if (pose_prev) {
        // iteration 1 at `pose`: same scan order, the neighbour records (pre, d5, pos) of iteration 0 are what seed_bound reads
        init_state(c->h_state[0], pose, uint32_t(n), o);
        c->h_state[0].icp_iter = 1;
        SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, sizeof(IcpState), cudaMemcpyHostToDevice, c->stream));
        correspond();
        SO_CUDA_TRY(cudaGetLastError());
    }
    std::vector<double> x(n * 3), w(n); std::vector<uchar4> fl(n); std::vector<uint32_t> nn(n * 5); std::vector<float> d2(n * 5);
    std::vector<float4> sorted(n);
    SO_CUDA_TRY(cudaMemcpyAsync(x.data(), c->corr.x, n * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));     // scan 0 at offset 0: slot j
    SO_CUDA_TRY(cudaMemcpyAsync(w.data(), c->corr.w, n * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(fl.data(), c->corr.flags, n * sizeof(uchar4), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(nn.data(), c->corr.nn, n * 5 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(d2.data(), c->corr.nn_d2, n * 5 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(sorted.data(), c->d_scan_sorted, n * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(c->h_state, c->d_state, sizeof(IcpState), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (size_t j = 0; j < n; ++j) {          // kernels work in cell order; report in the caller's order
        uint32_t orig;
        std::memcpy(&orig, &sorted[j].w, 4);
        so_corr& r = corr[orig];
        std::memset(&r, 0, sizeof(r));
        // plane_of_solution's steps as IEEE operations (every one correctly rounded, so the same bits); rejected points report 0
        if (fl[j].x == SO_MATCH_SUCCESS) {
            const double* xj = &x[j * 3];
            const double nn = std::sqrt(std::fma(xj[2], xj[2], std::fma(xj[0], xj[0], xj[1] * xj[1])));
            r.d = 1.0 / nn;
            for (int k = 0; k < 3; ++k) r.n[k] = xj[k] / nn;
        }
        r.w = w[j];
        for (int k = 0; k < 5; ++k) { r.nn[k] = nn[j * 5 + k]; r.nn_d2[k] = d2[j * 5 + k]; }
        r.status = fl[j].x; r.obs[0] = fl[j].y; r.obs[1] = fl[j].z; r.obs[2] = fl[j].w;
    }
    if (hist_obs) std::memcpy(hist_obs, c->h_state[0].hist_obs, 9 * sizeof(int32_t));
    if (hist_rej) std::memcpy(hist_rej, c->h_state[0].hist_rej, 7 * sizeof(int32_t));
    return SO_OK;
}

int so_correspond(so_ctx* ctx, const void* surf, size_t n, size_t stride, size_t ioff, const double pose[7], int32_t max_surface_features,
                  so_corr* corr, int32_t hist_obs[9], int32_t hist_rej[7]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !surf || !pose || !corr || n == 0 || stride < 12) return fail(SO_ERR_ARG, "bad args");
    return correspond_stage(c, surf, n, stride, ioff, pose, nullptr, max_surface_features, corr, hist_obs, hist_rej);
}

int so_ordered_scans(so_ctx* ctx, float* out, size_t n) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || (!out && n)) return fail(SO_ERR_ARG, "bad args");
    if (n > c->scan_cap) return fail(SO_ERR_CAPACITY, "more points than the scan buffer holds");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    SO_CUDA_TRY(cudaStreamSynchronize(c->aux_stream));
    SO_CUDA_TRY(cudaMemcpyAsync(out, c->d_scan_sorted, n * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SO_OK;
}

int so_correspond_seeded(so_ctx* ctx, const void* surf, size_t n, size_t stride, size_t ioff, const double pose[7], int32_t max_surface_features,
                         so_corr* corr, int32_t hist_obs[9], int32_t hist_rej[7], const double pose_prev[7]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !surf || !pose || !corr || n == 0 || stride < 12 || !pose_prev) return fail(SO_ERR_ARG, "bad args");
    return correspond_stage(c, surf, n, stride, ioff, pose, pose_prev, max_surface_features, corr, hist_obs, hist_rej);
}

int so_correspond_edge(so_ctx* ctx, const void* edge, size_t n, size_t stride, size_t ioff, const double pose[7], so_edge_corr* corr,
                       int32_t hist_rej_line[7]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !edge || !pose || !corr || n == 0 || stride < 12) return fail(SO_ERR_ARG, "bad args");
    if (n > c->edge_cap) return fail(SO_ERR_CAPACITY, "edge cloud larger than so_config.max_scan_points");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    { int rc0 = ensure_maps(c); if (rc0) return rc0; }
    c->reg.edge_valid = false;                                           // d_escan is overwritten below
    int rc = upload_cloud(c, edge, n, stride, ioff, c->d_escan);
    if (rc) return rc;
    so_icp_opts o{}; o.max_icp_iters = -1; o.lm_max_iterations = 4;
    init_state(c->h_state[0], pose, 0, o, uint32_t(n));
    c->h_offset[0] = 0;
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, sizeof(IcpState), cudaMemcpyHostToDevice, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_offset, c->h_offset, sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    const uint32_t grid_e = (uint32_t(n) + kThreads - 1) / kThreads;
    const MapView me = map_view(c, c->edge);
    const BatchView bv = batch_view(c, c->d_scan_sorted);
    timed_launch_begin(c);
    const uint32_t k = launch_first_eval(bv, c->corr, 0, 1, c->stream, &me, &c->ebuf, grid_e);     // 0 plane CTAs: only the edge kernel + k_lm_step have work
    timed_launch_end(c, 4, k);
    SO_CUDA_TRY(cudaGetLastError());
    std::vector<double4> a(n), b(n); std::vector<uchar4> fl(n); std::vector<uint32_t> nn(n * 10), sel(n);
    SO_CUDA_TRY(cudaMemcpyAsync(a.data(), c->ebuf.a, n * sizeof(double4), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(b.data(), c->ebuf.b, n * sizeof(double4), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(fl.data(), c->ebuf.flags, n * sizeof(uchar4), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(nn.data(), c->ebuf.nn, n * 10 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(sel.data(), c->ebuf.selmask, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(c->h_state, c->d_state, sizeof(IcpState), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (size_t i = 0; i < n; ++i) {
        so_edge_corr& r = corr[i];
        std::memset(&r, 0, sizeof(r));
        r.a[0] = a[i].x; r.a[1] = a[i].y; r.a[2] = a[i].z; r.w = a[i].w; r.b[0] = b[i].x; r.b[1] = b[i].y; r.b[2] = b[i].z;
        for (int k = 0; k < 10; ++k) r.nn[k] = nn[i * 10 + k];
        r.selected_mask = sel[i]; r.status = fl[i].x; r.n_selected = fl[i].y;
    }
    if (hist_rej_line) std::memcpy(hist_rej_line, c->h_state[0].hist_rej_line, 7 * sizeof(int32_t));
    return SO_OK;
}

int so_evaluate(so_ctx* ctx, const double pose[7], double H[36], double g[6], double* cost) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose) return fail(SO_ERR_ARG, "bad args");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    IcpState& s = c->h_state[0];
    const uint32_t n = uint32_t(s.n_points);
    const uint32_t grid_e = (uint32_t(s.n_edge) + kThreads - 1) / kThreads;
    if (n == 0 && grid_e == 0) return fail(SO_ERR_ARG, "so_evaluate needs a preceding so_correspond / so_correspond_edge");
    std::memcpy(s.cand, pose, 7 * sizeof(double));
    s.phase = PH_EVAL; s.max_icp_iters = -1;
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, sizeof(IcpState), cudaMemcpyHostToDevice, c->stream));
    const uint32_t grid_x = (n + kThreads - 1) / kThreads;
    const BatchView bv = batch_view(c, c->d_scan_sorted);
    timed_launch_begin(c);
    timed_launch_end(c, 1, launch_evaluate(bv, c->corr, grid_x, 1, c->stream, &c->ebuf, grid_e));
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaMemcpyAsync(c->h_state, c->d_state, sizeof(IcpState), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (H) for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) H[i * 6 + j] = s.H[i <= j ? tri(i, j) : tri(j, i)];
    if (g) for (int i = 0; i < 6; ++i) g[i] = s.g[i];
    if (cost) *cost = s.cost;
    return SO_OK;
}

int so_covariance(so_ctx* ctx, const double* H, int32_t n, so_icp_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !H || !out || (n != 6 && n != 12)) return fail(SO_ERR_ARG, "bad args");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    IcpState& s = c->h_state[0];                              // the state of a preceding so_correspond* is replaced
    std::memset(&s, 0, sizeof(s));
    timed_launch_begin(c);
    uint32_t k = 0;
    if (n == 6) {
        for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) s.H[tri(i, j)] = H[i * 6 + j];
        SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, sizeof(IcpState), cudaMemcpyHostToDevice, c->stream));
        k = launch_covariance(c->d_state, c->stream);
    } else {
        { int rc = c->mot.d_st.reserve(std::max<size_t>(c->max_batch, 1)); if (rc) return rc; }
        MotionState M{};
        for (int i = 0; i < 12; ++i) for (int j = i; j < 12; ++j) M.H[i * 12 - (i * (i - 1)) / 2 + (j - i)] = H[i * 12 + j];
        SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, sizeof(IcpState), cudaMemcpyHostToDevice, c->stream));
        SO_CUDA_TRY(cudaMemcpyAsync(c->mot.d_st, &M, sizeof(MotionState), cudaMemcpyHostToDevice, c->stream));
        k = launch_covariance12(c->d_state, c->mot.d_st, c->stream);
    }
    timed_launch_end(c, 1, k);
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaMemcpyAsync(c->h_state, c->d_state, sizeof(IcpState), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    std::memset(out, 0, sizeof(*out));
    std::memcpy(out->cov, s.cov, sizeof(out->cov));
    out->pos_err = s.pos_err; out->pos_inv_cond = s.pos_inv_cond; out->ori_err_deg = s.ori_err_deg; out->ori_inv_cond = s.ori_inv_cond;
    for (int i = 0; i < 3; ++i) { out->pos_dir[i] = s.pos_dir[i]; out->ori_dir[i] = s.ori_dir[i]; }
    return SO_OK;
}

int so_degeneracy_analysis(so_ctx* ctx, const double* H, const so_degeneracy* d, so_degeneracy_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !H || !d || !out) return fail(SO_ERR_ARG, "bad args");
    { int rc = check_degeneracy(d, 1); if (rc) return rc; }
    SO_CUDA_TRY(cudaSetDevice(c->device));
    { int rc = c->deg.d_st.reserve(std::max<size_t>(c->max_batch, 1)); if (rc) return rc; }
    IcpState& s = c->h_state[0];                              // the state of a preceding so_correspond* is replaced
    std::memset(&s, 0, sizeof(s));
    for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) s.H[tri(i, j)] = H[i * 6 + j];
    DegenState S = degen_state(*d);
    timed_launch_begin(c);
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, sizeof(IcpState), cudaMemcpyHostToDevice, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(c->deg.d_st, &S, sizeof(DegenState), cudaMemcpyHostToDevice, c->stream));
    timed_launch_end(c, 1, launch_degeneracy_analysis(c->d_state, c->deg.d_st, c->stream));
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaMemcpyAsync(&S, c->deg.d_st, sizeof(DegenState), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    std::memset(out, 0, sizeof(*out));
    fill_degeneracy(S, out);
    return SO_OK;
}

// so_solve / so_solve_optimized, once the caller has checked its arguments and initialised h_state[0..n_problems): the buffers k_fit
// fills (scan point with its index in w, {n, d}, weight, flags, the accepted-row histogram) are written from the caller's rows; then the
// first evaluation and lm evaluations run as one ICP iteration of a registration launches them.  ms (mode OPTIMIZED): the problems'
// motion blocks, updated in place; the rows' raw points also go to d_scan and their times to und.d_time, where k_motion_eval reads them.
// dg: the degeneracy-aware solve's states (so_solve), updated in place.
static int solve_stage(Ctx* c, const so_solve_row* rows, const float* times, size_t n_problems, int lm, MotionState* ms, DegenState* dg,
                       so_solve_result* out) {
    size_t total = 0;
    uint32_t max_n = 0;
    for (size_t b = 0; b < n_problems; ++b) { total += uint32_t(c->h_state[b].n_points); max_n = std::max(max_n, uint32_t(c->h_state[b].n_points)); }
    SO_CUDA_TRY(cudaSetDevice(c->device));
    if (dg) { int rc = c->deg.d_st.reserve(c->max_batch); if (rc) return rc; }
    if (ms) { int rc = motion_reserve(c, total); if (rc) return rc; }
    c->prefiltered_n = SIZE_MAX;                                  // d_scan_sorted is overwritten
    if (ms) c->reg.valid = false;                                 // so are d_scan and the times
    std::vector<float4> raw(ms ? total : 0), sp(total);
    // the record in its ND form ({n, d} per slot): slots of scan b from corr_first(b, offset) on; the gaps between scans are not read
    const size_t slots = corr_first(uint32_t(n_problems), uint32_t(total));
    std::vector<double> nd(slots * 4), w(slots);
    std::vector<float> pr(slots * 3);
    std::vector<int32_t> hist(n_problems * kHistStride, 0);
    uint32_t off = 0;
    for (size_t b = 0; b < n_problems; ++b) {
        const uint32_t n = uint32_t(c->h_state[b].n_points);
        c->h_offset[b] = off;
        const size_t r0 = corr_first(uint32_t(b), off);
        for (uint32_t i = 0; i < n; ++i) {
            const so_solve_row& r = rows[off + i];
            float4 p = make_float4(r.p[0], r.p[1], r.p[2], 0.f);
            if (ms) raw[off + i] = p;
            std::memcpy(&p.w, &i, 4);                             // the point's index inside its scan, as k_scan_gather writes it
            sp[off + i] = p;
            for (int k = 0; k < 3; ++k) { nd[(r0 + i) * 4 + k] = r.n[k]; pr[(r0 + i) * 3 + k] = r.p[k]; }
            nd[(r0 + i) * 4 + 3] = r.d;
            w[r0 + i] = r.w;
        }
        hist[b * kHistStride + 9] = int32_t(n);                   // hist_rej[SUCCESS]: every row is accepted
        off += n;
    }
    cudaStream_t st = c->stream;
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_state, c->h_state, n_problems * sizeof(IcpState), cudaMemcpyHostToDevice, st));
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_offset, c->h_offset, n_problems * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    SO_CUDA_TRY(cudaMemcpyAsync(c->d_hist, hist.data(), hist.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (total) {
        SO_CUDA_TRY(cudaMemcpyAsync(c->d_scan_sorted, sp.data(), total * sizeof(float4), cudaMemcpyHostToDevice, st));
        SO_CUDA_TRY(cudaMemcpyAsync(c->corr.x, nd.data(), slots * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
        SO_CUDA_TRY(cudaMemcpyAsync(c->corr.w, w.data(), slots * sizeof(double), cudaMemcpyHostToDevice, st));
        SO_CUDA_TRY(cudaMemcpyAsync(c->corr.p, pr.data(), slots * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
        SO_CUDA_TRY(cudaMemsetAsync(c->corr.flags, 0, total * sizeof(uchar4), st));
        if (ms) {
            SO_CUDA_TRY(cudaMemcpyAsync(c->d_scan, raw.data(), total * sizeof(float4), cudaMemcpyHostToDevice, st));
            SO_CUDA_TRY(cudaMemcpyAsync(c->und.d_time, times, total * sizeof(float), cudaMemcpyHostToDevice, st));
        }
    }
    if (dg) SO_CUDA_TRY(cudaMemcpyAsync(c->deg.d_st, dg, n_problems * sizeof(DegenState), cudaMemcpyHostToDevice, st));
    if (ms) SO_CUDA_TRY(cudaMemcpyAsync(c->mot.d_st, ms, n_problems * sizeof(MotionState), cudaMemcpyHostToDevice, st));
    Chunk ch{0, uint32_t(n_problems), 0, uint32_t(total)};
    plan_chunk(c, ch, max_n, ms || dg);
    const BatchView bv = chunk_view(c, c->d_scan_sorted, ch);
    const UndistortionMode mode = ms ? UndistortionMode::OPTIMIZED : UndistortionMode::NONE;
    CorrBuf cb = c->corr;
    cb.nn = nullptr; cb.nn_d2 = nullptr; cb.given = true;
    DegenState* const ddg = dg ? c->deg.d_st.get() : nullptr;
    auto solve = [&](int phase) { return launch_solve(c, mode, phase, bv, cb, 0, ch.grid_x, ch.count, st, nullptr, nullptr, 0, ddg); };
    timed_launch_begin(c);
    timed_launch_end(c, ms ? 8 : 4, solve(PH_CORR));
    SO_CUDA_TRY(cudaGetLastError());
    std::vector<double> cost0(n_problems);                        // the cost IterationZero evaluated (the state's cost moves with the steps)
    SO_CUDA_TRY(cudaMemcpyAsync(c->h_state, c->d_state, n_problems * sizeof(IcpState), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    for (size_t b = 0; b < n_problems; ++b) cost0[b] = c->h_state[b].cost;
    for (int k = 0; k < lm; ++k) {
        timed_launch_begin(c); timed_launch_end(c, ms ? 8 : 1, solve(PH_EVAL));
    }
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaMemcpyAsync(c->h_state, c->d_state, n_problems * sizeof(IcpState), cudaMemcpyDeviceToHost, st));
    if (dg) SO_CUDA_TRY(cudaMemcpyAsync(dg, c->deg.d_st, n_problems * sizeof(DegenState), cudaMemcpyDeviceToHost, st));
    if (ms) SO_CUDA_TRY(cudaMemcpyAsync(ms, c->mot.d_st, n_problems * sizeof(MotionState), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    for (size_t b = 0; b < n_problems; ++b) {
        const IcpState& s = c->h_state[b];
        so_solve_result& r = out[b];
        std::memset(&r, 0, sizeof(r));
        std::memcpy(r.pose, s.x, sizeof(r.pose));
        r.initial_cost = cost0[b]; r.final_cost = s.cost;
        r.lm_iterations = s.lm_iter; r.successful = s.num_successful; r.unsuccessful = s.num_unsuccessful; r.termination = s.termination;
        r.radius = s.radius; r.decrease_factor = s.decrease_factor; r.gmax = s.gmax;
        if (dg) { r.n_flag_pos = dg[b].iter_n_flag_pos[0]; r.n_flag_ori = dg[b].iter_n_flag_ori[0]; }
        r.status = s.status;
    }
    return SO_OK;
}

int so_solve(so_ctx* ctx, const so_solve_row* rows, const so_solve_problem* pr, size_t n_problems, const so_degeneracy* d, so_solve_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pr || !out || n_problems == 0) return fail(SO_ERR_ARG, "bad args");
    if (n_problems > size_t(c->max_batch)) return fail(SO_ERR_CAPACITY, "more problems than so_config.max_batch");
    if (d) { int rc = check_degeneracy(d, n_problems); if (rc) return rc; }
    size_t total = 0;
    int lm = 0;
    for (size_t b = 0; b < n_problems; ++b) {
        if (pr[b].n_rows > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "problem larger than so_config.max_scan_points");
        if (pr[b].lm_max_iterations > 16) return fail(SO_ERR_ARG, "lm_max_iterations must be <= 16");
        total += pr[b].n_rows;
        lm = std::max(lm, pr[b].lm_max_iterations <= 0 ? 4 : pr[b].lm_max_iterations);
    }
    if (total && !rows) return fail(SO_ERR_ARG, "bad args");
    std::vector<DegenState> dg(d ? n_problems : 0);
    for (size_t b = 0; b < n_problems; ++b) {
        so_icp_opts o{};
        o.max_icp_iters = 1; o.lm_max_iterations = pr[b].lm_max_iterations <= 0 ? 4 : pr[b].lm_max_iterations;
        o.use_pose_prior = pr[b].use_pose_prior; o.visual_confidence_factor = pr[b].visual_confidence_factor;
        for (int a = 0; a < 3; ++a) o.prior_uncertainty[a] = pr[b].prior_uncertainty[a];
        init_state(c->h_state[b], pr[b].pose, pr[b].n_rows, o);
        std::memcpy(c->h_state[b].x0, pr[b].x0, sizeof(c->h_state[b].x0));      // the prior's measurement, apart from the start
        if (d) dg[b] = degen_state(d[b]);
    }
    return solve_stage(c, rows, nullptr, n_problems, lm, nullptr, d ? dg.data() : nullptr, out);
}

// The two-block solve of so_register_optimized: each problem's motion block from its so_motion, with D and Dc at the start motion
int so_solve_optimized(so_ctx* ctx, const so_solve_row* rows, const float* times, const so_solve_optimized_problem* pr, size_t n_problems,
                       so_solve_optimized_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pr || !out || n_problems == 0) return fail(SO_ERR_ARG, "bad args");
    if (n_problems > size_t(c->max_batch)) return fail(SO_ERR_CAPACITY, "more problems than so_config.max_batch");
    size_t total = 0;
    int lm = 0;
    std::vector<MotionState> ms(n_problems);
    for (size_t b = 0; b < n_problems; ++b) {
        if (pr[b].n_rows > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "problem larger than so_config.max_scan_points");
        so_icp_opts o{};
        o.max_icp_iters = 1; o.lm_max_iterations = pr[b].lm_max_iterations <= 0 ? 4 : pr[b].lm_max_iterations;
        { int rc = check_motion(&pr[b].m, &o); if (rc) return rc; }
        if (!finite_pose(pr[b].pose) || !finite_pose(pr[b].motion)) return fail(SO_ERR_ARG, "pose and motion must be finite with a non-zero quaternion");
        total += pr[b].n_rows;
        lm = std::max(lm, o.lm_max_iterations);
        init_state(c->h_state[b], pr[b].pose, pr[b].n_rows, o);
        ms[b] = make_state(pr[b].m);
        const double* D = pr[b].motion;
        const double n = std::sqrt(D[3] * D[3] + D[4] * D[4] + D[5] * D[5] + D[6] * D[6]);      // normalised as make_state normalises D0
        for (int k = 0; k < 7; ++k) ms[b].D[k] = ms[b].Dc[k] = k < 3 ? D[k] : D[k] / n;
    }
    if (total && (!rows || !times)) return fail(SO_ERR_ARG, "bad args");
    std::vector<so_solve_result> res(n_problems);
    const int rc = solve_stage(c, rows, times, n_problems, lm, ms.data(), nullptr, res.data());
    if (rc) return rc;
    for (size_t b = 0; b < n_problems; ++b) {
        so_solve_optimized_result& r = out[b];
        std::memset(&r, 0, sizeof(r));
        r.solve = res[b];
        std::memcpy(r.motion, ms[b].D, sizeof(r.motion));
        std::memcpy(r.cov, c->h_state[b].cov, sizeof(r.cov));
    }
    return SO_OK;
}

// ---- k-NN --------------------------------------------------------------------------------------------------------
int so_knn_device(so_ctx* ctx, const void* d_q, size_t nq, int k, float max_d2, uint32_t* d_idx, float* d_d2) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !d_q || !d_idx || !d_d2 || k < 1 || k > 8) return fail(SO_ERR_ARG, "bad args");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    { int rc0 = ensure_maps(c); if (rc0) return rc0; }
    if (nq == 0) return SO_OK;
    // Large query sets are first ordered by map cell (cell key -> radix sort); threads then take queries in that order and
    // write their answers at the caller's positions.  Small sets skip the ordering.
    const uint32_t* order = nullptr;
    const MapView mv = map_view(c, c->surf);
    timed_launch_begin(c);
    if (nq >= 32768 && nq < (size_t(1) << 31)) {
        int rc = query_sort_reserve(c, nq);
        if (rc) return rc;
        launch_query_keys(mv, static_cast<const float4*>(d_q), nq, c->d_qkeys, c->d_qvals, c->stream);
        rc = query_sort(c, nq);
        if (rc) return rc;
        order = c->d_qvals_out;
        c->launches++;
    }
    if (launch_knn(mv, static_cast<const float4*>(d_q), order, nq, k, max_d2, d_idx, d_d2, c->stream)) return fail(SO_ERR_ARG, "bad k");
    timed_launch_end(c, 2, 1);
    SO_CUDA_TRY(cudaGetLastError());
    return SO_OK;
}

int so_knn(so_ctx* ctx, const float* q_xyz, size_t nq, size_t stride, int k, float max_d2, uint32_t* idx, float* d2) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !q_xyz || !idx || !d2 || k < 1 || k > 8 || stride < 12) return fail(SO_ERR_ARG, "bad args");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    int rc = c->d_q.reserve(nq);
    if (!rc) rc = c->d_knn_idx.reserve(nq * 8);
    if (!rc) rc = c->d_knn_d2.reserve(nq * 8);
    if (rc) return rc;
    rc = upload_cloud(c, q_xyz, nq, stride, stride /* no intensity */, c->d_q);
    if (rc) return rc;
    rc = so_knn_device(ctx, c->d_q, nq, k, max_d2, c->d_knn_idx, c->d_knn_d2);
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemcpyAsync(idx, c->d_knn_idx, nq * k * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(d2, c->d_knn_d2, nq * k * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SO_OK;
}

// ---- instrumentation -----------------------------------------------------------------------------------------------
uint64_t so_kernel_launches(so_ctx* ctx, int reset) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return 0;
    const uint64_t v = c->launches;
    if (reset) c->launches = 0;
    return v;
}

int so_sampling_indices(uint32_t n, int32_t max_surface_features, uint32_t* out, size_t cap, size_t* n_out) {
    if (!n_out || (!out && cap)) return fail(SO_ERR_ARG, "bad args");
    const double rate = (max_surface_features > 0 && n > uint32_t(max_surface_features)) ? 1.0 * max_surface_features / double(n) : -1.0;
    size_t k = 0;
    for (uint32_t i = 0; i < n; ++i) {
        if (rate >= 0.0 && !should_process_h(i, rate)) continue;
        if (k < cap) out[k] = i;
        ++k;
    }
    *n_out = k;
    return SO_OK;
}

int so_bytes_copied(so_ctx* ctx, uint64_t* h2d, uint64_t* d2h, int reset) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    if (h2d) *h2d = c->bytes_h2d;
    if (d2h) *d2h = c->bytes_d2h;
    if (reset) { c->bytes_h2d = 0; c->bytes_d2h = 0; }
    return SO_OK;
}

int so_build_flags(void) { return 0; }

int so_profile_enable(so_ctx* ctx, int on) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    c->profiling = on != 0;
    return SO_OK;
}

int so_profile_get(so_ctx* ctx, int cls, double* ms, uint64_t* launches, int reset) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || cls < 0 || cls > 8) return fail(SO_ERR_ARG, "bad args");
    if (ms) *ms = c->prof[cls].ms;
    if (launches) *launches = c->prof[cls].launches;
    if (reset) c->prof[cls] = ProfileSlot{};
    return SO_OK;
}

int so_knn_graph(so_ctx* ctx, uint32_t* point_id, uint32_t* nbr_id, float* radius, size_t cap_points, uint32_t* k, size_t* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !n_out) return fail(SO_ERR_ARG, "null argument");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    if (k) *k = uint32_t(kGraphK);
    { int rc = ensure_maps(c); if (rc) return rc; }
    MapStore& ms = c->surf;
    *n_out = ms.n;
    if (ms.n == 0) return SO_OK;
    if (!knn_graph_valid(c)) {
        const int mode = c->knn_graph_mode;
        c->knn_graph_mode = 1;
        const int rc = knn_graph_prepare(c, 0);
        c->knn_graph_mode = mode;
        if (rc) return rc;
    }
    if (!point_id || !nbr_id || !radius) return SO_OK;
    if (cap_points < ms.n) return fail(SO_ERR_CAPACITY, "so_knn_graph: cap_points below the store's points");
    std::vector<float4> sorted(ms.n);
    std::vector<uint32_t> pos(size_t(ms.n) * kGraphK);
    SO_CUDA_TRY(cudaMemcpyAsync(sorted.data(), ms.d_sorted, sorted.size() * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(pos.data(), ms.d_graph, pos.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaMemcpyAsync(radius, ms.d_graph_radius, size_t(ms.n) * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (size_t t = 0; t < ms.n; ++t) {
        std::memcpy(&point_id[t], &sorted[t].w, 4);
        for (int j = 0; j < kGraphK; ++j) {
            const uint32_t p = pos[t * kGraphK + j];
            uint32_t id = 0xFFFFFFFFu;
            if (p != 0xFFFFFFFFu) std::memcpy(&id, &sorted[p].w, 4);
            nbr_id[t * kGraphK + j] = id;
        }
    }
    return SO_OK;
}

int so_knn_graph_stats(so_ctx* ctx, int on, uint64_t* counts) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    const size_t bytes = 2 * SO_MAX_ICP_ITERS * sizeof(uint32_t);
    if (counts) {
        uint32_t h[2 * SO_MAX_ICP_ITERS] = {};
        if (c->d_graph_stats) {
            SO_CUDA_TRY(cudaMemcpyAsync(h, c->d_graph_stats, bytes, cudaMemcpyDeviceToHost, c->stream));
            SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
        }
        for (int i = 0; i < 2 * SO_MAX_ICP_ITERS; ++i) counts[i] = h[i];
    }
    if (on) {
        int rc = c->d_graph_stats.reserve(2 * SO_MAX_ICP_ITERS);
        if (rc) return rc;
        SO_CUDA_TRY(cudaMemsetAsync(c->d_graph_stats, 0, bytes, c->stream));
    }
    if (!on && c->d_graph_stats) {
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
        c->d_graph_stats.reset();
    }
    return SO_OK;
}

}  // extern "C"

// so_ctx.cuh -- the context behind the C ABI: owns every device buffer, the stream, CUDA graphs and host mirrors.
#pragma once
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "so_icp.cuh"

namespace so {

#define SO_CUDA_TRY(expr)                                                                         \
    do {                                                                                          \
        cudaError_t e__ = (expr);                                                                 \
        if (e__ != cudaSuccess) {                                                                 \
            so::set_error(std::string(#expr) + ": " + cudaGetErrorString(e__));                   \
            return SO_ERR_CUDA;                                                                   \
        }                                                                                         \
    } while (0)

void set_error(const std::string& s);

// Grow-only device buffer: when n elements (bytes for void) exceed cap, free the old buffer and allocate n; the contents are not
// kept.  A failed allocation leaves cap at 0, so the next call retries.
template <class T>
int grow_buffer(T*& p, size_t& cap, size_t n) {
    if (n <= cap) return SO_OK;
    cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t bytes = n;
    if constexpr (!std::is_void_v<T>) bytes *= sizeof(T);
    SO_CUDA_TRY(cudaMalloc(&p, bytes));
    cap = n;
    return SO_OK;
}

struct ProfileSlot { double ms = 0.0; uint64_t launches = 0; };
constexpr int kMotionAcc = 91;                     // 78 (upper triangle of the 12x12 H) + 12 (g) + 1 (cost)

// Within-scan motion compensation of a registration (the reference's UndistortionMode, LidarSlam.h:65-82): NONE, APPROXIMATED
// (so_undistort.cu: k_undistort heads every ICP iteration), OPTIMIZED (so_motion.cu: the motion is a second parameter block).
enum class UndistortionMode : int32_t { NONE = 0, APPROXIMATED = 1, OPTIMIZED = 2 };

// Within-scan motion compensation of one scan (so_undistort, mode APPROXIMATED): everything k_undistort needs besides the
// current pose.  Kept out of IcpState so that the other kernels do not change.
struct UndistortParams {
    double q_prev_conj[4];                         // conj(q_prev), xyzw
    double t_prev[3];
    double dt;                                     // seconds from prev_pose to the pose being estimated, > 0
    int32_t on;                                    // 0: the scan registers exactly as so_register
    int32_t rotation;                              // 1: slerp the rotation too; 0: translation only
};

// Per-scan motion block of mode OPTIMIZED (so_motion.cu), next to the scan's IcpState
struct MotionState {
    double D0[7];              // motion prior (quaternion normalised)
    double info[6];            // its information diagonal per accepted correspondence
    double dt;                 // seconds the motion spans, > 0
    double D[7], Dc[7];        // accepted / candidate motion
    double H[78], g[12];       // at (x, D): upper triangle of the 12x12, gradient; prior rows included
    double cost;               // so_evaluate_optimized: the plane rows' cost
    double scale[12], diag[12], sqrt_info[6];
    int32_t stage;             // so_evaluate_optimized: the first evaluation reports H, g, cost and ends the registration
    int32_t pad;
};
static_assert(sizeof(MotionState) % 8 == 0, "copied as 8-byte words");

// The scan so_map_add_registered_scan inserts: d_scan[0..n) in upload order and, unless mode NONE, its times in und.d_time[0..n)
struct RegisteredScan {
    bool valid = true;                             // false: a call has overwritten d_scan or the times since that scan registered
    uint32_t n = 0;                                // 0: no scan registered yet, nothing to insert
    UndistortionMode mode = UndistortionMode::NONE;
    UndistortParams par{};                         // APPROXIMATED: the parameters it registered with
    double D[7] = {0, 0, 0, 0, 0, 0, 1}, dt = 0;   // OPTIMIZED: the estimated motion D_opt and the time it spans
};

// One registration call (register_scans, so_api.cu): where the scans come from, what they are, how they register, where the
// results go.  Serves every so_register* entry point, so_evaluate_optimized and the candidate refinement of so_localize_global*.
struct RegisterRequest {
    enum class Source {
        HOST,                                      // host cloud(s) in the stride / ioff layout, uploaded whole first
        HOST_PACKED,                               // host batch of packed float4, uploaded chunk by chunk beside the kernels
        DEVICE,                                    // packed float4 scans in device memory (d_scan and its record untouched)
        PREFILTERED,                               // the cloud so_scan_prefilter left in d_scan_sorted; its w is the time
    };
    Source src = Source::HOST;
    const void* scans = nullptr;                   // HOST*: the host cloud; DEVICE: the device scans
    size_t stride = 16, ioff = 12, toff = 12;      // host layout: bytes per point, offsets of the intensity and of the time
    const uint32_t* n_points = nullptr;            // [n_scans], scans back to back
    size_t n_scans = 1;
    const void* edge = nullptr;                    // optional host edge clouds (host layout), n_edge[s] points each, back to back
    const uint32_t* n_edge = nullptr;
    const double* poses = nullptr;                 // [n_scans][7] priors
    const so_icp_opts* opts = nullptr;
    UndistortionMode mode = UndistortionMode::NONE;
    const UndistortParams* und = nullptr;          // APPROXIMATED: [n_scans]
    MotionState* motion = nullptr;                 // OPTIMIZED: [n_scans], uploaded first and read back after the registration
    const uint32_t* inject = nullptr;              // host neighbour ids [inject_iters][n][5] in place of the search
    int inject_iters = 0;
    bool allow_shift = false;                      // the map may shift to the priors (single-scan registration)
    bool sink_rows = true;                         // an attached pose sink gets a row per scan
    bool insertable = false;                       // the scan stays for so_map_add_registered_scan
    so_icp_result* results = nullptr;              // [n_scans]
    so_motion_result* motion_results = nullptr;    // OPTIMIZED, optional: [n_scans] results with the motion
};

// One per-block cloud family of the LocalMap (surf or edge): points in id order, the sorted hash grid, block tables.
struct MapStore {
    float res = 0.4f;                              // planeRes_ (surf) / lineRes_ (edge): voxel leaf and gate / search radius
    uint32_t n = 0;                                // points held (on-grid)
    float4* d_xyzi = nullptr;                      // [max_map] id order, w = intensity
    float4* d_sorted = nullptr;                    // [max_map] sorted by (slot, cell), w = bitcast(id)
    int32_t* d_block_slot = nullptr;               // [4851]
    int32_t* d_block_count = nullptr;              // [4851]
    uint32_t* d_cell_start = nullptr;              // [cell_cap]
    size_t cell_cap = 0;
    std::vector<int32_t> h_block_count, h_block_slot;   // host mirrors
    int n_slots = 0;
    int nb = 64;                                   // cells per block axis
    bool dirty = true;                             // the index is not built for the current cloud, origin and resolution
};

struct Ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = true;
    so_config cfg{};

    // ---- maps: raw (id order) + sorted hash grid; one store for surf points, one for edge points -------------------
    int32_t origin[3] = {kW / 2, kH / 2, kD / 2};  // LocalMap() ctor (LocalMap.h:141-144)
    MapStore surf, edge;                           // psurf_pc_ / pedge_pc_ of every MapBlock
    // scratch shared by both stores (builds are sequential on the context stream)
    uint64_t* d_keys = nullptr;                    // [max_map] sort keys (in)
    uint64_t* d_keys_out = nullptr;                // [max_map]
    uint32_t* d_vals = nullptr;                    // [max_map] ids (in)
    uint32_t* d_vals_out = nullptr;                // [max_map]
    void* d_cub_tmp = nullptr;
    size_t cub_tmp_bytes = 0;
    struct MapScratch* d_map_scratch = nullptr;    // device-side bookkeeping of a store change or a scan pre-filter (so_map.cu)
    struct InsertInfo* h_map_info = nullptr;       // pinned read-back target of its InsertInfo

    // ---- scans / correspondences / optimiser state -------------------------------------------------------------
    uint32_t max_batch = 1;
    size_t scan_cap = 0;                           // points over the whole batch
    size_t prefiltered_n = SIZE_MAX;               // points so_scan_prefilter left in d_scan_sorted (SIZE_MAX: none / overwritten since)
    RegisteredScan reg;                            // what d_scan (and und.d_time) hold for so_map_add_registered_scan
    float4* d_scan = nullptr;                      // upload target for host scans (original order)
    float4* d_scan_sorted = nullptr;               // cell-ordered copy the kernels read; w = original index
    uint64_t* d_skeys = nullptr; uint64_t* d_skeys_out = nullptr;   // scan sort keys (scan id << 32 | cell)
    uint32_t* d_svals = nullptr; uint32_t* d_svals_out = nullptr;
    void* d_sort_tmp = nullptr; size_t sort_tmp_bytes = 0;
    void* d_sort_tmp2 = nullptr;                   // second radix-sort scratch: scan ordering of the chunks that run on aux_stream
    NnBuf nn{};
    uint32_t* d_offset = nullptr;
    IcpState* d_state = nullptr;
    IcpState* h_state = nullptr;                   // pinned
    uint32_t* h_offset = nullptr;                  // pinned
    uint32_t* h_eoffset = nullptr;                 // second half of the same allocation
    bool eoffset_dirty = false;                    // d_eoffset holds non-zero entries from the last batch
    double* d_partials = nullptr;
    uint32_t* d_counters = nullptr;
    int32_t* d_hist = nullptr;
    CorrBuf corr{};
    // edge / line branch (single-scan so_register only)
    size_t edge_cap = 0; uint32_t edge_grid_cap = 0;
    float4* d_escan = nullptr; uint32_t* d_eoffset = nullptr; EdgeBuf ebuf{};
    uint32_t grid_x_cap = 0;
    double* d_pose_sink = nullptr; size_t sink_cap = 0, sink_cursor = 0;   // so_set_pose_sink: device rows the batch calls append to
    uint32_t* d_inject = nullptr; size_t inject_cap = 0;   // so_register_injected: caller-supplied neighbour ids [iters][n][5]
    void* h_stage = nullptr;                       // pinned staging for strided host clouds
    size_t h_stage_bytes = 0;
    // so_register of a DECIMATED scan (max_surface_features < n): only the points shouldProcessPoint keeps go up before the
    // registration is launched; the whole cloud (what so_map_add_registered_scan inserts) follows on the copy stream while it runs
    float4* d_dec = nullptr;                       // [kPrepareSmallCap] the kept points, index order, w = intensity
    std::vector<uint32_t> dec_idx;                 // kept indices for (dec_n, dec_mf): the list depends on nothing else
    uint32_t dec_n = 0; int32_t dec_mf = 0;
    cudaEvent_t ev_dec = nullptr;                  // the deferred upload of the whole cloud has landed in d_scan
    struct { const void* src = nullptr; size_t n = 0, stride = 0, ioff = 0, stage_off = 0; } defer;      // pending whole-cloud upload (src == nullptr: none)
    bool no_dec_upload = false;                    // SO_NO_DEC_UPLOAD: A/B aid, always upload the whole cloud first

    // ---- k-NN scratch -------------------------------------------------------------------------------------------
    float4* d_q = nullptr; uint32_t* d_knn_idx = nullptr; float* d_knn_d2 = nullptr;
    size_t q_cap = 0, knn_idx_cap = 0, knn_d2_cap = 0;
    uint32_t* d_qkeys = nullptr; uint32_t* d_qkeys_out = nullptr; uint32_t* d_qvals = nullptr; uint32_t* d_qvals_out = nullptr;   // cell ordering of so_knn* queries
    size_t qkeys_cap = 0, qkeys_out_cap = 0, qvals_cap = 0, qvals_out_cap = 0;
    void* d_qsort_tmp = nullptr; size_t qsort_tmp_bytes = 0;

    // ---- CUDA graph cache for the ICP schedule (one entry per batch chunk shape) ------------------------------------
    // Everything a captured schedule bakes into its kernel arguments: the chunk shape and both MapViews (pointers, origin, grid,
    // resolutions).  Keyed on these VALUES, not on a "map changed" counter, so that a map insert that leaves the index arrays
    // where they are (the usual live-SLAM case) keeps hitting the cache.
    struct GraphKey {
        uint32_t first, count, grid_x, grid_e; int32_t iters, lm;
        const void* ptrs[8]; int32_t origin[3]; int32_t nb[2]; float res[2];
        UndistortionMode mode; const void* und_time;   // the head of every iteration (NONE / nullptr: none)
    };
    struct GraphSlot {
        cudaGraphExec_t exec = nullptr;
        GraphKey key{}; bool is_loop = false; uint64_t used = 0;
    };
    GraphSlot graphs[20];
    uint64_t graph_clock = 0;
    bool force_key64 = false;                      // SO_FORCE_KEY64: test aid, take the 64-bit scan-order key path even when 32 bits suffice
    bool no_coop_knn = false;                      // SO_NO_COOP_KNN: A/B aid, always one query per thread
    bool no_small_prepare = false;                 // SO_NO_SMALL_PREPARE: A/B aid, always the device-wide scan ordering
    bool no_fused_lm = false;                      // SO_NO_FUSED_LM: A/B aid, always the two-kernel evaluation + optimiser step
    bool single_stream = false;                    // SO_SINGLE_STREAM: tuning aid, all chunks on `stream`
    int chunk_override = 0;                        // SO_CHUNKS: tuning aid, upload/compute chunks per host batch (0 = built-in rule)
    bool no_cond_graph = false;                    // conditional nodes unavailable (or SO_NO_COND_GRAPH): unrolled schedule
    cudaStream_t aux_stream = nullptr;             // odd chunks of a batch run here, concurrently with the even ones on `stream`:
                                                   // one chunk's serial optimiser steps and kernel tails hide under the other's wide kernels
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    cudaStream_t copy_stream = nullptr;            // H2D of batch chunks overlaps the previous chunk's kernels
    cudaEvent_t ev_copy[17] = {};           // [0..15]: per upload chunk; [16]: guard

    // ---- global localization (so_localize_global): allocated on first use, grown on demand --------------------------
    struct Reloc {
        uint32_t* d_bits[2] = {nullptr, nullptr}; size_t bit_words[2] = {0, 0};     // occupancy bitmap, ping-pong for the dilation passes
        uint64_t* d_keys = nullptr; uint64_t* d_keys_out = nullptr; size_t key_cap = 0, key_out_cap = 0;
        void* d_tmp = nullptr; size_t tmp_bytes = 0;                        // radix-sort scratch
        float4* d_pts = nullptr;                                           // [kRelocMaxPoints] score points
        double* d_q = nullptr; size_t q_cap = 0;                           // one quaternion per yaw
        cudaEvent_t ev[5] = {};                                            // stage boundaries
    } reloc;
    // ---- branch-and-bound search (so_localize_global_bnb): allocated on first use, grown on demand ---------------------
    struct Bnb {
        uint32_t* d_pyr = nullptr; size_t pyr_words = 0;                   // every level of the clipped pyramid, back to back
        uint32_t* d_scratch = nullptr; size_t scratch_words = 0;           // raster / dilation ping-pong partner of level 0
        int4* d_off = nullptr; size_t off_cap = 0;                         // [nyaw][nz][n_pts] voxel offsets of the score points
        uint64_t* d_nodes = nullptr;                                       // level buffers: [kBnbRoot] root chunk + [4C] per finer level
        uint64_t* d_unsorted = nullptr;                                    // [kBnbRoot] scored nodes before the sort
        uint64_t* d_merge[2] = {nullptr, nullptr};                         // [kBnbMerge] running top-P + new leaves, sorted copy
        void* d_tmp = nullptr; size_t tmp_bytes = 0;                       // radix-sort scratch
        struct BnbCtl* d_ctl = nullptr; struct BnbCtl* h_ctl = nullptr;    // K*, level counts and statistics (pinned mirror)
        uint32_t* d_bounds = nullptr;                                      // [6] map bounding box (ordered float bits)
        cudaEvent_t ev[4] = {};                                            // build start, build end / search start, search end, spare
    } bnb;
    // ---- within-scan motion compensation (so_register_undistort*): allocated on first use, grown on demand ------------
    struct Und {
        UndistortParams* d_par = nullptr; size_t par_cap = 0;              // [max_batch] per-scan parameters of the registration
        float* d_time = nullptr; size_t time_cap = 0;                      // per-point times of the scans in d_scan (upload order)
        float4* d_hook = nullptr; size_t hook_cap = 0;                     // so_undistort_points: the cloud and its times
        float* d_hook_time = nullptr; size_t hook_time_cap = 0;
    } und;
    // ---- within-scan motion estimated by the registration (so_register_optimized*): allocated on first use ------------------
    struct Mot {
        MotionState* d_st = nullptr; size_t st_cap = 0;                    // [max_batch] per-scan motion blocks
        double* d_partials = nullptr; size_t partials_cap = 0;             // [max_batch][stride][kMotionAcc] per-CTA sums
        uint32_t stride = 0;                                               // CTAs per scan the partials are laid out for
    } mot;
    // ---- edge extraction (so_scan_extract_edges): allocated on first use, grown on demand; never touches the scan buffers ----
    struct Feat {
        unsigned char* d_raw = nullptr; size_t raw_cap = 0;                // the caller's records as given
        size_t cap = 0;                                                    // points every per-point buffer below holds
        uint64_t* d_keys[2] = {nullptr, nullptr};                          // sort keys in / out: (ring, time), then (ring, sector, curvature)
        uint32_t* d_vals[2] = {nullptr, nullptr};
        float4* d_pts = nullptr;                                           // valid points in (ring, time, index) order, w = time
        uint8_t* d_excl = nullptr; uint8_t* d_reach = nullptr;             // excluded marks; neighbour-mark reach of each candidate
        uint32_t* d_sel = nullptr; uint32_t* d_rank = nullptr;             // accepted flags and their exclusive scan
        float4* d_out = nullptr; float4* d_vout = nullptr;                 // edge cloud; after the voxel filter
        void* d_tmp = nullptr; size_t tmp_bytes = 0;                       // radix-sort / scan scratch
        uint32_t* d_ring = nullptr;                                        // [65536] first position, [65536] end, [65536] ring list, [4] control
    } feat;

    // ---- instrumentation ----------------------------------------------------------------------------------------
    uint64_t launches = 0;
    uint64_t bytes_h2d = 0, bytes_d2h = 0;         // host<->device bytes moved by registration / k-NN calls
    bool profiling = false;
    ProfileSlot prof[9];
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evp0 = nullptr, evp1 = nullptr;
};

// so_api.cu
int fail(int code, const std::string& msg);                 // set_error(msg), return code
void tf2_get_rpy(const double q[4], double* roll, double* pitch, double* yaw);
int ensure_maps(Ctx* c);                                    // rebuild dirty map stores
int upload_cloud(Ctx* c, const void* src, size_t n, size_t stride, size_t ioff, float4* dst);
void count_h2d(Ctx* c, size_t b);
void count_d2h(Ctx* c, size_t b);
void timed_launch_begin(Ctx* c);
void timed_launch_end(Ctx* c, int cls);                     // counts one launch; profile class cls when profiling
int icp_opts_check(const so_icp_opts& o);                   // max_icp_iters and lm_max_iterations in the supported range
// Serves one request: puts the scans, their times and the mode's parameters on the device, registers, reads the motion back, fills
// results (time_total_ms included) and keeps the record of the scan left in d_scan.  The caller has checked the arguments.
int register_scans(Ctx* c, const RegisterRequest& q);
inline float4 read_point(const unsigned char* p, size_t stride, size_t ioff) {     // one point of a strided host cloud
    float xyz[3], it = 0.f;
    std::memcpy(xyz, p, 12);
    if (ioff + 4 <= stride) std::memcpy(&it, p + ioff, 4);
    return make_float4(xyz[0], xyz[1], xyz[2], it);
}
// so_global.cu
void global_free(Ctx* c);                                   // the search buffers and events of Ctx::reloc / Ctx::bnb
// so_undistort.cu
void undistort_free(Ctx* c);                                // the buffers of Ctx::und
int undistort_reserve(Ctx* c, size_t n_points);             // Ctx::und's parameters (max_batch) and times (n_points)
int check_undistort(const so_undistort* u);                 // argument errors of one so_undistort
UndistortParams make_params(const so_undistort& u);
bool finite_pose(const double p[7]);                        // finite, with a non-zero quaternion
int upload_times(Ctx* c, const void* src, size_t n, size_t stride, size_t toff, float* dst);   // the float at toff of every record -> dst
// k_undistort: pInit of every active point of the chunk's scans (bv.st / bv.offset / par already offset to the chunk), from the
// raw points in upload order (raw, times: indexed offset + original index) into the ordered copy `sorted`, w kept
void launch_undistort(const BatchView& bv, float4* sorted, const float4* raw, const float* times, const UndistortParams* par,
                      uint32_t grid_x, uint32_t n_scans, cudaStream_t st);
// ms tail = the registered scan r (APPROXIMATED): pInit at pose, in place
int undistort_tail(Ctx* c, MapStore& ms, const RegisteredScan& r, const double pose[7]);
// so_motion.cu
void motion_free(Ctx* c);                                   // the buffers of Ctx::mot
int motion_reserve(Ctx* c, size_t n_points);                // Ctx::mot's blocks and partials (max_batch), Ctx::und's times (n_points)
int check_motion(const so_motion* m, const so_icp_opts* o); // argument errors of one so_motion and the options it registers with
MotionState make_state(const so_motion& m);
void fill_motion(const so_icp_result& icp, const MotionState& M, so_motion_result* out);   // out = icp + motion, pose_end = T * D
int motion_tail(Ctx* c, MapStore& ms, const RegisteredScan& r);   // ms tail = the registered scan r (OPTIMIZED): u(r.D), in place
// One ICP iteration's kernels of mode OPTIMIZED for the chunk's scans (bv.st / bv.offset / partials already offset to the chunk, ms
// the whole array and `first` the chunk's first scan): the warp u(D) into `sorted`, and one evaluation + trust-region step (phase
// PH_CORR: the first of a solve)
void launch_motion_warp(const BatchView& bv, float4* sorted, const float4* raw, const float* times, const MotionState* ms, uint32_t first,
                        uint32_t grid_x, uint32_t n_scans, cudaStream_t st);
void launch_motion_solve(int phase, const BatchView& bv, const CorrBuf& cb, const float4* raw, const float* times, MotionState* ms, uint32_t first,
                         double* partials, uint32_t stride, uint32_t grid_x, uint32_t n_scans, cudaStream_t st);
// so_covariance: cov12_warp on ms->H into st's covariance and error fields (device memory)
void launch_covariance12(IcpState* st, const MotionState* ms, cudaStream_t stream);
// so_map.cu
int map_alloc(Ctx* c);
void map_free(Ctx* c);
int map_add_points(Ctx* c, MapStore& ms, uint32_t n_new);   // ms.d_xyzi[n .. n+n_new) holds the new points: voxel-filter touched blocks, index
int map_transform_tail(Ctx* c, MapStore& ms, uint32_t n_new, const double pose[7]);   // sensor-frame tail points -> world frame
int scan_voxel_filter(Ctx* c, uint32_t n, float leaf, uint32_t* n_out);   // d_scan -> d_scan_sorted (VoxelGrid on a scan)
// The same filter on any packed cloud in[0..n) -> out, with the caller's sort buffers (keys: 2n words of head scratch after the sort)
struct VoxelBufs { uint64_t* keys; uint64_t* keys_out; uint32_t* vals; uint32_t* vals_out; void* tmp; size_t tmp_bytes; };
int cloud_voxel_filter(Ctx* c, const float4* in, uint32_t n, float leaf, const VoxelBufs& b, float4* out, uint32_t* n_out);
// so_features.cu
void features_free(Ctx* c);                                 // the buffers of Ctx::feat
// so_scan.cu
struct DeskewParams {
    double start_time;                     // lidar_start_time
    const double* times;                   // n_samples ascending sample stamps (device)
    const double* poses;                   // n_samples x {tx,ty,tz,qx,qy,qz,qw} (device; translation zeroed for IMU samples)
    uint32_t n_samples, n_smem;            // n_smem: stamps cached in shared memory
    int imu_only;
    double q0_conj[4], p0[3];              // T_w_original: conjugate of its (normalised) rotation, its position
    double q_il[4], t_il[3], q_li[4], t_li[3];   // T_i_l and its inverse (parameter.cpp:192-193)
    uint32_t* past_end;                    // points later than the last sample
};
void launch_deskew(float4* pts, uint32_t n, const DeskewParams& P, cudaStream_t st);
int scan_extract_uniform(Ctx* c, uint32_t n, uint32_t skip, float block_range, int int_abs, uint32_t* n_out);   // d_scan -> d_scan_sorted   // d_scan -> d_scan_sorted (VoxelGrid on a scan)
int map_rebuild(Ctx* c, MapStore& ms);    // (re)bin, drop off-grid points, index; the store stays dirty when it fails
MapView map_view(const Ctx* c, const MapStore& ms);
int map_cells_per_block(float plane_res);
int scan_sort_alloc(Ctx* c);             // temp storage for the per-registration scan sort
int query_sort(Ctx* c, size_t n);         // d_qkeys/d_qvals -> *_out (allocates on growth)
int query_sort_reserve(Ctx* c, size_t n);
int scan_sort(Ctx* c, size_t first, size_t n, int n_scans, int cell_bits, bool key32, cudaStream_t st);   // d_skeys/d_svals[first..first+n) -> *_out
// so_reloc.cu (global localization search)
struct RelocGrid {
    int32_t nx, ny, nz, nyaw;              // hypotheses per axis: 2I+1, 2J+1, 2K+1, yaw steps
    int32_t e;                             // ceil(max_range / res): the scan's reach in voxels
    int32_t bx, by, bz, wpr;               // bitmap voxels per axis (nx + 2e, ...), 32-bit words per x row
    double lo[3];                          // world position of bitmap voxel (0, 0, 0): t_c - (I + e, J + e, K + e) * res
    double res;
};
constexpr int kRelocMaxPoints = 4097;      // score_points <= 4096; shouldProcessPoint keeps at most one more
constexpr int kRelocThreads = 256, kRelocRows = 8;   // k_reloc_score: CTA size, y shifts per CTA
uint32_t* launch_reloc_dilate(const RelocGrid& g, int d, uint32_t* a, uint32_t* b, cudaStream_t st);   // 3 passes; returns the result buffer
int launch_reloc_score(const float4* spts, int n_pts, const double* d_q, const RelocGrid& g, const uint32_t* bits, uint64_t* keys, cudaStream_t st);
size_t reloc_sort_bytes(size_t n);
int reloc_sort(void* tmp, size_t tmp_bytes, const uint64_t* in, uint64_t* out, size_t n, cudaStream_t st);

// so_reloc.cu (branch-and-bound search over an occupancy pyramid)
constexpr int kBnbLevels = 32;             // levels 0..31 (nx <= 2^25 + 1 needs at most 26)
constexpr int kBnbBatch = 1 << 14;         // C: nodes expanded per step, so a finer level buffer holds at most 4C
constexpr int kBnbRoot = 1 << 16;          // root nodes scored per chunk, and the root size the Lmax rule aims for
constexpr int kBnbMaxKeys = 64 * 64;       // P <= 64 k with k <= 64
constexpr int kBnbMerge = kBnbMaxKeys + 4 * kBnbBatch;
constexpr uint64_t kBnbNone = ~0ull;       // a discarded node: sorts after every valid key (bit 48 set, sorted bits 0..48)
// The clipped pyramid.  Level L stores B_L(x, y, z) = OR_{a,b in [0,2^L)} B(x+a, y+b, z) for box voxels x in [x0 - (2^L-1), x0 + wx),
// y in [y0 - (2^L-1), y0 + wy), z in [z0, z0 + wz), where [x0, x0+wx) x [y0, y0+wy) x [z0, z0+wz) is the window W of the search box
// that the surf map's voxel bounding box, grown by the dilation, covers.  B is 0 outside W, so so is B_L outside its array.
struct BnbPyramid {
    int32_t x0, y0, z0, wx, wy, wz;
    int32_t lmax;
    int32_t wpr[kBnbLevels];               // 32-bit words per row of each level
    uint64_t off[kBnbLevels];              // first word of each level in Ctx::Bnb::d_pyr
};
struct BnbCtl {                            // device control block, read back after every step
    uint64_t kstar;                        // P-th smallest leaf key found so far (kBnbNone while fewer than P are known)
    uint64_t cnt[kBnbLevels];              // per level: end of the nodes still admitted by K*
    unsigned long long scored[kBnbLevels], discarded[kBnbLevels];
};
void launch_map_bounds(const float4* pts, uint32_t n, uint32_t* d_bounds, cudaStream_t st);   // d_bounds: min xyz, max xyz (ordered bits)
// Raster of the surf store into the window W of p (the whole box: x0 = y0 = z0 = 0, wx/wy/wz = bx/by/bz, wpr[0] = g.wpr)
void launch_bnb_raster(const float4* pts, uint32_t n, const RelocGrid& g, const BnbPyramid& p, uint32_t* bits, cudaStream_t st);
void launch_bnb_levels(const BnbPyramid& p, uint32_t* pyr, cudaStream_t st);                  // levels 1..lmax from level 0
void launch_bnb_offsets(const float4* spts, int n_pts, const double* d_q, const RelocGrid& g, const BnbPyramid& p, int4* off,
                        cudaStream_t st);
// Bound of level-`level` nodes: parents == nullptr scores nodes first .. first+n-1 of the level in (m, k, tile y, tile x) order;
// otherwise node c is child (c & 3) of parents[c >> 2] (key order).  out[c] = the node key, or kBnbNone when it is clipped away,
// its parent is above K* or its own key is above K*.
void launch_bnb_score(const RelocGrid& g, const BnbPyramid& p, const uint32_t* pyr, const int4* off, int n_pts, int level,
                      const uint64_t* parents, uint64_t first, uint32_t n, BnbCtl* ctl, uint64_t* out, cudaStream_t st);
// cnt[l] for l in 1..lmax: the end of the keys <= K* among nodes[l][head[l], cnt_in[l]) (sorted); the rest are counted as discarded
struct BnbTrim { uint64_t head[kBnbLevels], cnt[kBnbLevels], base[kBnbLevels]; int32_t lmax; };
void launch_bnb_trim(const BnbTrim& t, const uint64_t* nodes, BnbCtl* ctl, cudaStream_t st);
size_t bnb_sort_bytes(size_t n);
int bnb_sort(void* tmp, size_t tmp_bytes, const uint64_t* in, uint64_t* out, size_t n, cudaStream_t st);

}  // namespace so

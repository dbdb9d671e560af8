// so_ctx.cuh -- the context behind the C ABI: owns every device buffer, the stream, CUDA graphs and host mirrors.
#pragma once
#include <cstring>
#include <map>
#include <string>
#include <utility>
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

// Owner of one device (Pinned = false: cudaMalloc) or pinned host (true: cudaMallocHost) allocation of T; freed by its destructor and
// by move-assignment.  Grow-only: reserve(n) does nothing when n <= cap(), else frees the old allocation first (the contents are not
// kept, so peak memory does not grow) and allocates n elements.  A failed allocation leaves the buffer empty, so the next call retries.
// Converts to T* (and has ->), so kernel arguments, copies and pointer arithmetic take the buffer as they took the pointer.
template <class T, bool Pinned>
class Buffer {
public:
    Buffer() = default;
    Buffer(const Buffer&) = delete;
    Buffer& operator=(const Buffer&) = delete;
    Buffer(Buffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), cap_(std::exchange(o.cap_, 0)) {}
    Buffer& operator=(Buffer&& o) noexcept {
        if (this != &o) { reset(); p_ = std::exchange(o.p_, nullptr); cap_ = std::exchange(o.cap_, 0); }
        return *this;
    }
    ~Buffer() { reset(); }
    int reserve(size_t n) {                        // the only member that needs T complete
        if (n <= cap_) return SO_OK;
        reset();
        void* p = nullptr;
        if constexpr (Pinned) SO_CUDA_TRY(cudaMallocHost(&p, n * sizeof(T)));
        else SO_CUDA_TRY(cudaMalloc(&p, n * sizeof(T)));
        p_ = static_cast<T*>(p);
        cap_ = n;
        return SO_OK;
    }
    void reset() {
        if (p_) { if constexpr (Pinned) cudaFreeHost(p_); else cudaFree(p_); }
        p_ = nullptr;
        cap_ = 0;
    }
    T* get() const { return p_; }
    size_t cap() const { return cap_; }
    operator T*() const { return p_; }
    T* operator->() const { return p_; }
private:
    T* p_ = nullptr;
    size_t cap_ = 0;
};
template <class T> using DeviceBuffer = Buffer<T, false>;
template <class T> using PinnedBuffer = Buffer<T, true>;

// Owner of one CUDA event: create(flags) makes it (replacing any it held), the destructor destroys it
class Event {
public:
    Event() = default;
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    ~Event() { if (e_) cudaEventDestroy(e_); }
    int create(unsigned flags = cudaEventDefault) {
        if (e_) cudaEventDestroy(e_);
        e_ = nullptr;
        SO_CUDA_TRY(cudaEventCreateWithFlags(&e_, flags));
        return SO_OK;
    }
    operator cudaEvent_t() const { return e_; }
private:
    cudaEvent_t e_ = nullptr;
};

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

// The scan so_map_add_registered_scan inserts: d_scan[0..n) in upload order and, unless mode NONE, its times in und.d_time[0..n);
// the edge cloud so_map_add_registered_edges inserts: d_escan[0..n_edge) and, unless mode NONE, its times in und.d_etime
struct RegisteredScan {
    bool valid = true;                             // false: a call has overwritten d_scan or the times since that scan registered
    bool edge_valid = true;                        // false: so_correspond_edge has overwritten d_escan since
    uint32_t n = 0;                                // 0: no scan registered yet, nothing to insert
    uint32_t n_edge = 0;                           // 0: the registration had no edge cloud, nothing to insert
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
    DegenState* degen = nullptr;                   // degeneracy-aware registration (mode NONE): [n_scans], uploaded first and read back
    const uint32_t* inject = nullptr;              // host neighbour ids [inject_iters][n][5] in place of the search
    int inject_iters = 0;
    bool allow_shift = false;                      // the map may shift to the priors (single-scan registration)
    bool sink_rows = true;                         // an attached pose sink gets a row per scan
    bool insertable = false;                       // the scan stays for so_map_add_registered_scan
    so_icp_result* results = nullptr;              // [n_scans]
    so_motion_result* motion_results = nullptr;    // OPTIMIZED, optional: [n_scans] results with the motion
};

// Block archive of one store (so_map_archive; so_archive.h): the clouds of blocks the window dropped, each kept as one segment of a
// point pool in its in-block order, found through a directory sorted by world key.  d_pool.cap() == 0: off, nothing allocated.
struct GatherSeg { uint64_t src, dst; uint32_t n, pad; };      // one block cloud copied src[0..n) -> dst[0..n) (k_seg_gather)
struct BlockArchive {
    struct Seg { uint64_t off; uint32_t n; };
    DeviceBuffer<float4> d_pool;                   // [cap()]: segments in [0, used), holes where blocks were restored
    size_t used = 0, live = 0;                     // pool tail; points in live segments
    std::map<uint64_t, Seg> dir;                   // world key -> segment, key order (host: every origin change goes through the host)
    DeviceBuffer<GatherSeg> d_segs;                // segment lists of the gathers
};

// Keyframe store (so_keyframes.cu; so_keyframe_reserve): registered scans kept on the device with their poses, for a loop-closing back
// end.  Per store (0 surf, 1 edge) one float4 pool holds the keyframes back to back in id order, each as put_registered_scan places
// it (sensor frame, motion-compensated as registered).  cap_frames == 0: off, nothing allocated.
struct KeyframeStore {
    size_t cap_points = 0, cap_frames = 0;         // points per pool, keyframes
    DeviceBuffer<float4> d_pool[2];                // [cap_points] each
    std::vector<uint64_t> off[2];                  // [frames + 1] first point of every keyframe, then the pool's tail
    std::vector<double> poses;                     // [frames][7]
    size_t frames() const { return poses.size() / 7; }
    // Scan Context descriptors (so_loop.cu), by keyframe id: [cap_frames][rings][sectors] images and [cap_frames][sectors] column
    // norms for the options in desc_opts (rings == 0: no table, else one of cap_frames keyframes); desc_ok[id] = 1 while id's
    // descriptor is valid for them and its pose
    DeviceBuffer<float> d_desc;
    DeviceBuffer<double> d_desc_norm;
    so_loop_opts desc_opts{};
    std::vector<uint8_t> desc_ok;
};
// One selected keyframe of so_map_from_keyframes: pool[src .. src + n) becomes union[start .. start + n), transformed by pose
struct KfSeg { uint64_t src; uint32_t start, n; double pose[7]; };
// Scratch of so_map_from_keyframes and so_register_keyframes (so_keyframes.cu), grown on demand: the union of the selected keyframes
// in the world frame, its sort, and the filtered cloud of each store until both have passed their capacity checks
struct KeyframeScratch {
    DeviceBuffer<KfSeg> d_segs;
    DeviceBuffer<float4> d_raw;
    DeviceBuffer<uint64_t> d_keys, d_keys_out;
    DeviceBuffer<uint32_t> d_vals, d_vals_out;
    DeviceBuffer<float4> d_out[2];
    DeviceBuffer<uint32_t> d_blk;                          // block of every filtered point, then the block runs
    DeviceBuffer<unsigned char> d_tmp;
    DeviceBuffer<int32_t> d_ctl;                           // [8] world-block bounds and run count
    PinnedBuffer<int32_t> h_ctl;                           // its mirror
    // loop detection (so_loop.cu): keyframes to describe, the queries, one chunk's pair table and every query's top k
    DeviceBuffer<struct DescSeg> d_dsegs;
    DeviceBuffer<struct LoopQuery> d_queries;
    DeviceBuffer<struct LoopPair> d_pairs, d_top;
    Event ev_loop[4];                                      // describe start / end, search start / end
};

// One per-block cloud family of the LocalMap (surf or edge): points in id order, the sorted hash grid, block tables.
struct MapStore {
    float res = 0.4f;                              // planeRes_ (surf) / lineRes_ (edge): voxel leaf and gate / search radius
    uint32_t n = 0;                                // points held (on-grid)
    DeviceBuffer<float4> d_xyzi;                   // [max_map] id order, w = intensity
    DeviceBuffer<float4> d_sorted;                 // [max_map] sorted by (slot, cell), w = bitcast(id)
    DeviceBuffer<int32_t> d_block_slot;            // [4851]
    DeviceBuffer<int32_t> d_block_count;           // [4851]
    DeviceBuffer<uint32_t> d_cell_start;
    std::vector<int32_t> h_block_count, h_block_slot;   // host mirrors
    int n_slots = 0;
    int nb = 64;                                   // cells per block axis
    bool dirty = true;                             // the index is not built for the current cloud, origin and resolution
    uint64_t index_gen = 0;                        // bumped by every index build: a neighbour graph is valid for one index only
    // neighbour graph of the sorted cloud (surf store; knn_graph_prepare): kGraphK positions per point, AoS, and the radius below
    // which a row is complete.  Valid while graph_gen == index_gen and the store is clean.
    DeviceBuffer<uint32_t> d_graph;                         // [points][kGraphK]
    DeviceBuffer<float> d_graph_radius;
    uint64_t graph_gen = ~uint64_t(0);
    BlockArchive arc;
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
    DeviceBuffer<uint64_t> d_keys;                 // [max_map] sort keys (in)
    DeviceBuffer<uint64_t> d_keys_out;             // [max_map]
    DeviceBuffer<uint32_t> d_vals;                 // [max_map] ids (in)
    DeviceBuffer<uint32_t> d_vals_out;             // [max_map]
    DeviceBuffer<unsigned char> d_cub_tmp;
    DeviceBuffer<struct MapScratch> d_map_scratch; // device-side bookkeeping of a store change or a scan pre-filter (so_map.cu)
    PinnedBuffer<struct InsertInfo> h_map_info;    // read-back target of its InsertInfo

    // ---- scans / correspondences / optimiser state -------------------------------------------------------------
    uint32_t max_batch = 1;
    size_t scan_cap = 0;                           // points over the whole batch
    size_t prefiltered_n = SIZE_MAX;               // points so_scan_prefilter left in d_scan_sorted (SIZE_MAX: none / overwritten since)
    RegisteredScan reg;                            // what d_scan (and und.d_time) hold for so_map_add_registered_scan
    DeviceBuffer<float4> d_scan;                   // upload target for host scans (original order)
    DeviceBuffer<float4> d_scan_sorted;            // cell-ordered copy the kernels read; w = original index
    DeviceBuffer<uint64_t> d_skeys, d_skeys_out;   // scan sort keys (scan id << 32 | cell)
    DeviceBuffer<uint32_t> d_svals, d_svals_out;
    DeviceBuffer<unsigned char> d_sort_tmp;
    DeviceBuffer<unsigned char> d_sort_tmp2;       // second radix-sort scratch: scan ordering of the chunks that run on aux_stream
    NnBuf nn{};                                    // views of the five buffers below
    DeviceBuffer<uint32_t> d_nn_pos;
    DeviceBuffer<float> d_nn_d5;
    DeviceBuffer<unsigned char> d_nn_pre;
    DeviceBuffer<uint32_t> d_nn_queue, d_nn_qcount;   // allocated with the first neighbour graph a search uses
    DeviceBuffer<uint32_t> d_offset;
    DeviceBuffer<IcpState> d_state;
    PinnedBuffer<IcpState> h_state;
    PinnedBuffer<uint32_t> h_offset;
    uint32_t* h_eoffset = nullptr;                 // second half of h_offset
    bool eoffset_dirty = false;                    // d_eoffset holds non-zero entries from the last batch
    DeviceBuffer<double> d_partials;
    DeviceBuffer<uint32_t> d_counters;
    DeviceBuffer<int32_t> d_hist;
    CorrBuf corr{};                                // views of the five buffers below
    DeviceBuffer<double4> d_corr_nd;
    DeviceBuffer<double> d_corr_w;
    DeviceBuffer<uchar4> d_corr_flags;
    DeviceBuffer<uint32_t> d_corr_nn;
    DeviceBuffer<float> d_corr_nn_d2;
    // edge / line branch (single-scan so_register only)
    size_t edge_cap = 0; uint32_t edge_grid_cap = 0;
    DeviceBuffer<float4> d_escan;
    DeviceBuffer<uint32_t> d_eoffset;
    EdgeBuf ebuf{};                                // views of d_escan, d_eoffset and the five buffers below
    DeviceBuffer<double4> d_ebuf_a, d_ebuf_b;
    DeviceBuffer<uchar4> d_ebuf_flags;
    DeviceBuffer<uint32_t> d_ebuf_nn, d_ebuf_selmask;
    uint32_t grid_x_cap = 0;
    double* d_pose_sink = nullptr; size_t sink_cap = 0, sink_cursor = 0;   // so_set_pose_sink: device rows the batch calls append to
    DeviceBuffer<uint32_t> d_inject;               // so_register_injected: caller-supplied neighbour ids [iters][n][5]
    PinnedBuffer<float4> h_stage;                  // staging for strided host clouds
    // so_register of a DECIMATED scan (max_surface_features < n): only the points shouldProcessPoint keeps go up before the
    // registration is launched; the whole cloud (what so_map_add_registered_scan inserts) follows on the copy stream while it runs
    DeviceBuffer<float4> d_dec;                    // [kPrepareSmallCap] the kept points, index order, w = intensity
    std::vector<uint32_t> dec_idx;                 // kept indices for (dec_n, dec_mf): the list depends on nothing else
    uint32_t dec_n = 0; int32_t dec_mf = 0;
    Event ev_dec;                                  // the deferred upload of the whole cloud has landed in d_scan
    struct { const void* src = nullptr; size_t n = 0, stride = 0, ioff = 0, stage_off = 0; } defer;      // pending whole-cloud upload (src == nullptr: none)
    bool no_dec_upload = false;                    // SO_NO_DEC_UPLOAD: A/B aid, always upload the whole cloud first
    int knn_graph_mode = 0;                        // SO_KNN_GRAPH: test / A/B aid; 0 = built by the rule, 1 (on) = built for every search call,
                                                   // -1 (off) = never used
    DeviceBuffer<uint32_t> d_graph_stats;          // so_knn_graph_stats: [SO_MAX_ICP_ITERS][2] counters while on, else empty

    // ---- k-NN scratch -------------------------------------------------------------------------------------------
    DeviceBuffer<float4> d_q;
    DeviceBuffer<uint32_t> d_knn_idx;
    DeviceBuffer<float> d_knn_d2;
    DeviceBuffer<uint32_t> d_qkeys, d_qkeys_out, d_qvals, d_qvals_out;   // cell ordering of so_knn* queries
    DeviceBuffer<unsigned char> d_qsort_tmp;

    // ---- CUDA graph cache for the ICP schedule (one entry per batch chunk shape) ------------------------------------
    // Everything a captured schedule bakes into its kernel arguments: the chunk shape and both MapViews (pointers, origin, grid,
    // resolutions).  Keyed on these VALUES, not on a "map changed" counter, so that a map insert that leaves the index arrays
    // where they are (the usual live-SLAM case) keeps hitting the cache.
    struct GraphKey {
        uint32_t first, count, grid_x, grid_e; int32_t iters, lm;
        const void* ptrs[8]; int32_t origin[3]; int32_t nb[2]; float res[2];
        UndistortionMode mode; const void* und_time;   // the head of every iteration (NONE / nullptr: none)
        const void* und_edge;                          // APPROXIMATED with an edge cloud: the warped edge cloud the line branch reads
        const void* degen;                             // degeneracy-aware registration: the DegenState array (nullptr: off)
        const void* graph[5];                          // MapView::graph, graph_radius, graph_stats of the surf view (nullptr: none), NnBuf::queue, qcount
    };
    struct GraphSlot {
        cudaGraphExec_t exec = nullptr;
        GraphKey key{}; bool is_loop = false; uint64_t used = 0;
    };
    GraphSlot graphs[20];
    uint64_t graph_clock = 0;
    bool force_key64 = false;                      // SO_FORCE_KEY64: test aid, take the 64-bit scan-order key path even when 32 bits suffice
    bool force_drop_bit = false;                   // SO_FORCE_DROP_BIT: test aid, carry the scan-order key's dropped bit even when no scan of the chunk is capped
    bool no_coop_knn = false;                      // SO_NO_COOP_KNN: A/B aid, always one query per thread
    bool no_small_prepare = false;                 // SO_NO_SMALL_PREPARE: A/B aid, always the device-wide scan ordering
    bool no_fused_lm = false;                      // SO_NO_FUSED_LM: A/B aid, always the two-kernel evaluation + optimiser step
    bool single_stream = false;                    // SO_SINGLE_STREAM: tuning aid, all chunks on `stream`
    int chunk_override = 0;                        // SO_CHUNKS: tuning aid, upload/compute chunks per host batch (0 = built-in rule)
    bool no_cond_graph = false;                    // conditional nodes unavailable (or SO_NO_COND_GRAPH): unrolled schedule
    cudaStream_t aux_stream = nullptr;             // odd chunks of a batch run here, concurrently with the even ones on `stream`:
                                                   // one chunk's serial optimiser steps and kernel tails hide under the other's wide kernels
    Event ev_fork, ev_join;
    cudaStream_t copy_stream = nullptr;            // H2D of batch chunks overlaps the previous chunk's kernels
    Event ev_copy[17];                             // [0..15]: per upload chunk; [16]: guard

    // ---- global localization (so_localize_global*): allocated on first use, grown on demand ---------------------------
    struct Bnb {
        DeviceBuffer<float4> d_pts;                                        // [kRelocMaxPoints] score points
        DeviceBuffer<double> d_q;                                          // one quaternion per yaw
        DeviceBuffer<uint32_t> d_pyr;                                      // every level of the clipped pyramid, back to back
        DeviceBuffer<uint32_t> d_scratch;                                  // raster / dilation ping-pong partner of level 0
        DeviceBuffer<int4> d_off;                                          // [nyaw][n_pts] voxel offsets of the score points
        DeviceBuffer<uint64_t> d_nodes;                                    // level buffers: [kBnbRoot] root chunk + [4C] per finer level
        DeviceBuffer<uint64_t> d_unsorted;                                 // [kBnbRoot] scored nodes before the sort
        DeviceBuffer<uint64_t> d_merge[2];                                 // [kBnbMerge] running top-P + new leaves, sorted copy
        DeviceBuffer<unsigned char> d_tmp;                                 // radix-sort scratch
        DeviceBuffer<struct BnbCtl> d_ctl;                                 // K*, level counts and statistics
        PinnedBuffer<struct BnbCtl> h_ctl;                                 // their mirror
        DeviceBuffer<uint32_t> d_bounds;                                   // [6] map bounding box (ordered float bits)
        Event ev[4];                                                       // build start, build end / search start, search end, spare
    } bnb;
    // ---- within-scan motion compensation (so_register_undistort*): allocated on first use, grown on demand ------------
    struct Und {
        DeviceBuffer<UndistortParams> d_par;                               // [max_batch] per-scan parameters of the registration
        DeviceBuffer<float> d_time;                                        // per-point times of the scans in d_scan (upload order)
        DeviceBuffer<float4> d_hook;                                       // so_undistort_points: the cloud and its times
        DeviceBuffer<float> d_hook_time;
        DeviceBuffer<float> d_etime;                                       // [edge_cap] times of the edge cloud in d_escan
        DeviceBuffer<float4> d_ewarp;                                      // [edge_cap] its pInit at the current pose (EdgeBuf::scan)
    } und;
    // ---- within-scan motion estimated by the registration (so_register_optimized*): allocated on first use ------------------
    struct Mot {
        DeviceBuffer<MotionState> d_st;                                    // [max_batch] per-scan motion blocks
        DeviceBuffer<double> d_partials;                                   // [max_batch][stride][kMotionAcc] per-CTA sums
        uint32_t stride = 0;                                               // CTAs per scan the partials are laid out for
        DeviceBuffer<double> d_epartials;                                  // the edge clouds' per-CTA sums (so_register_optimized_edges)
    } mot;
    // ---- degeneracy-aware registration (so_register_degeneracy*, so_degeneracy_analysis): allocated on first use --------------
    struct Deg {
        DeviceBuffer<DegenState> d_st;                                     // [max_batch] per-scan analysis and solve columns
    } deg;
    // ---- edge extraction (so_scan_extract_edges): allocated on first use, grown on demand; never touches the scan buffers ----
    struct Feat {
        DeviceBuffer<unsigned char> d_raw;                                 // the caller's records as given
        // the per-point buffers, each of d_pts.cap() points
        DeviceBuffer<uint64_t> d_keys[2];                                  // sort keys in / out: (ring, time), then (ring, sector, curvature)
        DeviceBuffer<uint32_t> d_vals[2];
        DeviceBuffer<float4> d_pts;                                        // valid points in (ring, time, index) order, w = time
        DeviceBuffer<uint8_t> d_excl, d_reach;                             // excluded marks; neighbour-mark reach of each candidate
        DeviceBuffer<uint32_t> d_sel, d_rank;                              // accepted flags and their exclusive scan
        DeviceBuffer<float4> d_out, d_vout;                                // edge cloud; after the voxel filter
        DeviceBuffer<unsigned char> d_tmp;                                 // radix-sort / scan scratch
        DeviceBuffer<uint32_t> d_ring;                                     // [65536] first position, [65536] end, [65536] ring list, [4] control
    } feat;

    // ---- free-space clearing (so_map_clear_free_space*, so_free.cu): allocated on first use, grown on demand ---------------------
    struct FreeSpace {
        DeviceBuffer<uint32_t> d_img;                                      // range image: float bits of the minimum range per pixel
        DeviceBuffer<float4> d_pts;                                        // the host form's cloud
        DeviceBuffer<uint8_t> d_keep;                                      // [2][max_map_points] keep flags of the surf and edge windows
        DeviceBuffer<struct FreeCounters> d_cnt;                           // counters of one call
        PinnedBuffer<struct FreeCounters> h_cnt;                           // their mirror
        // so_map_clear_free_space_keyframes: one tile's images in d_img, and for every selected keyframe its pool segment and pose
        DeviceBuffer<struct KfImgSeg> d_kseg;
        DeviceBuffer<struct FreePose> d_kpose;
        DeviceBuffer<uint32_t> d_ccount, d_coff, d_clist;                  // per window block: candidate keyframes, offsets, the lists
        DeviceBuffer<unsigned char> d_tmp;                                 // scan scratch
        DeviceBuffer<struct FreeKfCounters> d_kcnt;                        // counters of one call
        PinnedBuffer<struct FreeKfCounters> h_kcnt;                        // their mirror
        Event ev[2];                                                       // start / end of the call's device work
    } fs;

    // ---- keyframes (so_keyframe_*, so_map_from_keyframes, so_register_keyframes): allocated on first use ---------------------------
    KeyframeStore kf;
    KeyframeScratch kfs;

    // ---- loop verification (so_loop_verify, so_verify.cu), on the scratch context: allocated on first use, grown on demand -----------
    struct Verify {
        DeviceBuffer<float4> d_q;                                          // the query's surf points at the aligned pose
        DeviceBuffer<uint32_t> d_img;                                      // the query's range image, then the submap keyframes' images
        DeviceBuffer<struct KfImgSeg> d_kseg;                              // the submap keyframes' pool segments
        DeviceBuffer<struct FreePose> d_kpose;                             // and their poses
        DeviceBuffer<double> d_partials;                                   // per-CTA sums of d^2 over the inliers
        DeviceBuffer<struct VerifyCounters> d_cnt;                         // counters of one candidate
        PinnedBuffer<struct VerifyCounters> h_cnt;                         // their mirror
        Event ev[2];                                                       // start / end of one candidate's device work
    } ver;

    // ---- pose graph (so_pose_graph_solve, so_pose_graph.cu): allocated on first use, grown on demand ------------------------------
    // Two linearisation sets: [cur] at the iterate, [1 - cur] at the candidate of the last trial (an accepted step swaps them)
    struct Pg {
        DeviceBuffer<so_pose_edge> d_edges;                                // [m]
        DeviceBuffer<int32_t> d_inc;                                       // [n + 1] offsets, then [2m] incident edge ids, ascending per node
        DeviceBuffer<uint8_t> d_const;                                     // [n] 1: the node is held constant
        DeviceBuffer<double> d_x[2];                                       // [n][7]
        DeviceBuffer<struct PgEdgeBlk> d_blk[2];                           // [m] per-edge Jacobian products
        DeviceBuffer<double> d_ecost[2], d_w[2];                           // [m] 1/2 rho and rho' per edge
        DeviceBuffer<double> d_H[2], d_C[2], d_g[2];                       // [n][36] node blocks, [n][36] chain blocks (k, k+1), [n][6]
        DeviceBuffer<double> d_scale, d_diag, d_dd;                        // [6n] Jacobi scaling, LM diagonal, diag / radius
        DeviceBuffer<double> d_vec;                                        // [6][6n] PCG vectors b, y, r, z, p, q
        DeviceBuffer<double> d_crD, d_crL, d_crU, d_crB;                   // cyclic-reduction levels: [T][36] x 3, [T][6]
        DeviceBuffer<double> d_red;                                        // [2][max_blocks] CTA partials of the trial's grid reductions
        int max_blocks = 0;                                                // co-resident CTAs of k_pg_trial on the context's device
        DeviceBuffer<struct PgCtl> d_ctl;
        PinnedBuffer<struct PgCtl> h_ctl;
        Event ev[2];
    } pg;

    // ---- instrumentation ----------------------------------------------------------------------------------------
    uint64_t launches = 0;
    uint64_t bytes_h2d = 0, bytes_d2h = 0;         // host<->device bytes moved by registration / k-NN calls
    bool profiling = false;
    ProfileSlot prof[9];
    Event ev0, ev1, evp0, evp1;
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
// so_undistort.cu
int undistort_reserve(Ctx* c, size_t n_points);             // Ctx::und's parameters (max_batch) and times (n_points)
int undistort_edge_reserve(Ctx* c);                         // Ctx::und's edge times and warped edge cloud (edge_cap, fixed once allocated)
int check_undistort(const so_undistort* u);                 // argument errors of one so_undistort
UndistortParams make_params(const so_undistort& u);
bool finite_pose(const double p[7]);                        // finite, with a non-zero quaternion
int upload_times(Ctx* c, const void* src, size_t n, size_t stride, size_t toff, float* dst);   // the float at toff of every record -> dst
// k_undistort: pInit of every active point of the chunk's scans (bv.st / bv.offset / par already offset to the chunk), from the
// raw points in upload order (raw, times: indexed offset + original index) into the ordered copy `sorted`, w kept
void launch_undistort(const BatchView& bv, float4* sorted, const float4* raw, const float* times, const UndistortParams* par,
                      uint32_t grid_x, uint32_t n_scans, cudaStream_t st);
// k_undistort_edges: pInit of every edge point of the chunk's scans (eoffset already offset to the chunk), from the raw edge cloud
// and its times (indexed eoffset + i) into `out` at the same index, w kept
void launch_undistort_edges(const BatchView& bv, const uint32_t* eoffset, float4* out, const float4* raw, const float* times,
                            const UndistortParams* par, uint32_t grid_e, uint32_t n_scans, cudaStream_t st);
// dst[0..r.n) = the registered scan r (APPROXIMATED): pInit at pose, in place
int undistort_tail(Ctx* c, float4* dst, const RegisteredScan& r, const double pose[7]);
// dst[0..r.n_edge) = the registered edge cloud r (APPROXIMATED): pInit at pose, in place
int undistort_edge_tail(Ctx* c, float4* dst, const RegisteredScan& r, const double pose[7]);
// so_motion.cu
int motion_reserve(Ctx* c, size_t n_points);                // Ctx::mot's blocks and partials (max_batch), Ctx::und's times (n_points)
int check_motion(const so_motion* m, const so_icp_opts* o); // argument errors of one so_motion and the options it registers with
MotionState make_state(const so_motion& m);
void fill_motion(const so_icp_result& icp, const MotionState& M, so_motion_result* out);   // out = icp + motion, pose_end = T * D
int motion_tail(Ctx* c, float4* dst, const RegisteredScan& r);   // dst[0..r.n) = the registered scan r (OPTIMIZED): u(r.D), in place
int motion_edge_tail(Ctx* c, float4* dst, const RegisteredScan& r);   // dst[0..r.n_edge) = its edge cloud: u(r.D) with the edge times, in place
int motion_edge_reserve(Ctx* c);                             // Ctx::mot's edge partials
// The edge cloud of an OPTIMIZED chunk: the edge map, the line buffers (eb.scan: where the warp puts float(u(D)) of the edge points,
// eb.offset: the chunk's edge offsets), the raw edge points and their times, the edge partials and the CTAs covering the largest cloud
struct MotionEdges { MapView map; EdgeBuf eb; const float4* raw; const float* times; double* partials; uint32_t grid_e; };
// One ICP iteration's kernels of mode OPTIMIZED for the chunk's scans (bv.st / bv.offset / partials already offset to the chunk, ms
// the whole array and `first` the chunk's first scan): the warp u(D) into `sorted`, and one evaluation + trust-region step (phase
// PH_CORR: the first of a solve)
// me (optional): the chunk's edge clouds -- the warp also writes float(u(D)) of the edge points, the solve adds k_edge_fit (PH_CORR)
// and the line rows (k_motion_eval_edge) to the sums k_motion_step reduces
void launch_motion_warp(const BatchView& bv, float4* sorted, const float4* raw, const float* times, const MotionState* ms, uint32_t first,
                        uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const MotionEdges* me = nullptr);
void launch_motion_solve(int phase, const BatchView& bv, const CorrBuf& cb, const float4* raw, const float* times, MotionState* ms, uint32_t first,
                         double* partials, uint32_t stride, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const MotionEdges* me = nullptr);
// so_covariance: cov12_warp on ms->H into st's covariance and error fields (device memory)
void launch_covariance12(IcpState* st, const MotionState* ms, cudaStream_t stream);
// so_map.cu
int map_alloc(Ctx* c);
int map_add_points(Ctx* c, MapStore& ms, uint32_t n_new);   // ms.d_xyzi[n .. n+n_new) holds the new points: voxel-filter touched blocks, index
int map_transform_tail(Ctx* c, MapStore& ms, uint32_t n_new, const double pose[7]);   // sensor-frame tail points -> world frame
int scan_voxel_filter(Ctx* c, uint32_t n, float leaf, uint32_t* n_out);   // d_scan -> d_scan_sorted (VoxelGrid on a scan)
// The same filter on any packed cloud in[0..n) -> out, with the caller's sort buffers (keys: 2n words of head scratch after the sort)
struct VoxelBufs { uint64_t* keys; uint64_t* keys_out; uint32_t* vals; uint32_t* vals_out; void* tmp; size_t tmp_bytes; };
int cloud_voxel_filter(Ctx* c, const float4* in, uint32_t n, float leaf, const VoxelBufs& b, float4* out, uint32_t* n_out);
// Removal of the points whose keep flag is 0 from the built store ms (stable), then its index: n_keep points are left
int map_compact(Ctx* c, MapStore& ms, const uint8_t* keep, uint32_t n_keep, uint32_t* d_num_selected);
// so_free.cu (free-space clearing)
void free_space_defaults(so_free_space* o);
int free_space_check(const so_free_space* o, int stores, const double pose[7]);   // SO_ERR_ARG cases of so_map_clear_free_space*
int free_space_prepare(Ctx* c, int stores);                 // rebuild the selected stores that are dirty
int free_space_reserve_points(Ctx* c, size_t n);            // Ctx::fs.d_pts for a host cloud of n points
// The range image of d_pts[0..n_pts) (sensor frame at pose), then every selected store carved against it; the stores are built
int free_space_clear(Ctx* c, int stores, const float4* d_pts, uint32_t n_pts, const double pose[7], const so_free_space& o,
                     so_free_space_result* out);
// The surf clouds of src's keyframes ids[0..n_ids) (n_ids > 0; ids and poses checked) imaged at poses7 and every selected store of c
// carved against all of them: what so_map_clear_free_space of each keyframe in turn leaves; the stores are built
int free_space_clear_keyframes(Ctx* c, Ctx* src, const int32_t* ids, size_t n_ids, const double* poses7, int stores, const so_free_space& o,
                               so_free_space_keyframes_result* out);
// so_api.cu: dst[0..n) = the registered scan (edges: its edge cloud) as the map inserts place it before the world transform
int put_registered_scan(Ctx* c, bool edges, float4* dst, const double pose[7]);
// so_keyframes.cu
// The surf clouds of src's keyframes ids[0..n) back to back on the device as registration input for dst, with their sizes: src's pool
// in place when the ids are consecutive, else a gather into dst's scratch.  SO_ERR_ARG for an id src does not hold.
int keyframe_scans(Ctx* dst, Ctx* src, const int32_t* ids, size_t n, const float4** scans, std::vector<uint32_t>* n_points);
// so_loop.cu: the descriptor table at cap_frames keyframes (valid descriptors kept) into *desc / *norm, not yet the store's; left
// empty when there is no table.  Moved into the store after its pools
int loop_table_alloc(const KeyframeStore& s, size_t cap_frames, DeviceBuffer<float>* desc, DeviceBuffer<double>* norm);
// so_map.cu: pts[0..n) at pose, in place, by k_transform_points (utils::TransformPoint: qrot in double, float store)
void launch_transform(float4* pts, uint32_t n, const double pose[7], cudaStream_t st);
// so_map.cu, so_map_from_keyframes in two steps so that two stores change together or not at all.  keyframe_map_filter: the map of the
// union that segs[0..n_segs) (host, total points) cut from `pool`, filtered for store ms (0 surf, 1 edge) under c's origin and leaf into
// the scratch c->kfs.d_out[store]; SO_ERR_CAPACITY when it does not fit ms, nothing changed either way.  keyframe_map_commit: ms
// replaced by that map and its index built.
struct KfBuild {
    uint32_t n_win = 0, n_win_blocks = 0;          // window points and blocks
    size_t n_arc = 0;                              // points of off-window blocks (archive on)
    std::vector<GatherSeg> win;                    // filtered cloud -> window, block by block
    std::vector<std::pair<uint64_t, GatherSeg>> arc;   // world key, filtered cloud -> archive pool
};
int keyframe_map_filter(Ctx* c, MapStore& ms, int store, const KfSeg* segs, uint32_t n_segs, uint32_t total, const float4* pool, KfBuild* b);
int keyframe_map_commit(Ctx* c, MapStore& ms, int store, const KfBuild& b);
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
// Block archive (so_map.cu): off-window points go to the archive and archived blocks the window reaches come back inside map_rebuild
int archive_set_cap(Ctx* c, size_t cap);                  // both stores: on / resize (contents kept) / 0: off and freed; all or nothing
// so_map_set_points with the archive on: pts[0..n) (finite, host) -> window part in d_xyzi, the rest in the archive; no rebuild
int archive_load(Ctx* c, MapStore& ms, const float4* pts, size_t n);
int archive_download_all(Ctx* c, MapStore& ms, float* out, size_t cap, size_t* n_out);   // window + archive by world key
// The live segments of ms's archive as {pool offset, -, points} in ms.arc.d_segs (host directory walk, no point copied): *n_segs of
// them, the largest holding *max_n points
int archive_segments(Ctx* c, MapStore& ms, uint32_t* n_segs, uint32_t* max_n);
// LocalMap::shiftMap's rule: the origin so_map_shift(t) leaves when called at origin o, and t's block under it (cc, may be NULL)
void shift_origin(const int32_t o[3], const double t[3], int32_t out[3], int32_t cc[3]);
int move_window(Ctx* c, const int32_t o[3]);                // origin = o (both stores dirty when it changes), then ensure_maps
MapView map_view(const Ctx* c, const MapStore& ms);
// Neighbour graph of the surf store (so_knn.cuh): built for the current index when a search call of `queries` queries pays for it
// (queries >= kGraphQueriesPerPoint x the store's points) or the graph is forced on, and none is valid
int knn_graph_prepare(Ctx* c, size_t queries);
bool knn_graph_valid(const Ctx* c);
MapView search_view(const Ctx* c);      // map_view of the surf store with its graph when one is valid and the graph is not off
int map_cells_per_block(float plane_res);
int scan_sort_alloc(Ctx* c);             // temp storage for the per-registration scan sort
int query_sort(Ctx* c, size_t n);         // d_qkeys/d_qvals -> *_out (allocates on growth)
int query_sort_reserve(Ctx* c, size_t n);
int scan_sort(Ctx* c, size_t first, size_t n, int n_scans, int cell_bits, bool key32, cudaStream_t st);   // d_skeys/d_svals[first..first+n) -> *_out
// so_reloc.cu (global localization: branch-and-bound search over an occupancy pyramid)
struct RelocGrid {
    int32_t nx, ny, nz, nyaw;              // hypotheses per axis: 2I+1, 2J+1, 2K+1, yaw steps
    int32_t e;                             // ceil(max_range / res): the scan's reach in voxels
    int32_t bx, by, bz, wpr;               // bitmap voxels per axis (nx + 2e, ...), 32-bit words per x row
    double lo[3];                          // world position of bitmap voxel (0, 0, 0): t_c - (I + e, J + e, K + e) * res
    double res;
};
constexpr int kRelocMaxPoints = 4097;      // score_points <= 4096; shouldProcessPoint keeps at most one more
uint32_t* launch_reloc_dilate(const RelocGrid& g, int d, uint32_t* a, uint32_t* b, cudaStream_t st);   // 3 passes; returns the result buffer
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
// Raster of the surf store into level 0 of p's window W
void launch_bnb_raster(const float4* pts, uint32_t n, const RelocGrid& g, const BnbPyramid& p, uint32_t* bits, cudaStream_t st);
// The same two over the live segments of an archive pool (segs[s].src: first point, .n: points; max_n: the largest .n), read in place
void launch_seg_bounds(const float4* pool, const GatherSeg* segs, uint32_t n_segs, uint32_t max_n, uint32_t* d_bounds, cudaStream_t st);
void launch_seg_raster(const float4* pool, const GatherSeg* segs, uint32_t n_segs, uint32_t max_n, const RelocGrid& g, const BnbPyramid& p,
                       uint32_t* bits, cudaStream_t st);
void launch_bnb_levels(const BnbPyramid& p, uint32_t* pyr, cudaStream_t st);                  // levels 1..lmax from level 0
// off[m][p]: box voxel {x, y} of score point p at yaw m and shift (0, 0, 0), and its z relative to W's first plane
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

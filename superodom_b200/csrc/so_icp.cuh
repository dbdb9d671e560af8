// so_icp.cuh -- kernel-side views and host launchers shared by so_icp.cu / so_api.cu.
#pragma once
#include "so_internal.cuh"

namespace so {

struct CorrBuf {
    double4* nd;        // {n.x,n.y,n.z,d}; all zero for rejected points
    double* w;          // residualCoefficient (0 for rejected)
    uchar4* flags;      // {status, obs0, obs1, obs2}
    uint32_t* nn;       // optional [5 per point] neighbour ids (stage tests); may be null
    float* nn_d2;       // optional [5 per point]
};

constexpr int kHistStride = 24;

// edge / line branch buffers (single-scan registration only; batches carry no edge clouds)
struct EdgeBuf {
    const float4* scan;       // edge points, sensor frame
    const uint32_t* offset;   // [n_scans] first edge point of each scan
    double4* a;               // {point_a, residualCoefficient}; w == 0 for rejected points
    double4* b;               // {point_b, 0}
    uchar4* flags;            // {status, n_selected, 0, 0}
    uint32_t* nn;             // optional [10 per point] neighbour ids (stage tests)
    uint32_t* selmask;        // optional: bit j set = j-th neighbour kept by the best-line selection
};

struct BatchView {
    const float4* scan;       // all scans back to back
    const uint32_t* offset;   // [n_scans] first point of each scan
    IcpState* st;             // [n_scans]
    double* partials;         // [n_scans][partial_stride][kAcc] per-CTA sums of the last per-point kernel
    uint32_t partial_stride;  // CTAs per scan the partials buffer is laid out for
    int32_t* hist;            // [n_scans][kHistStride] histogram accumulators (self-resetting): 9 obs + 7 plane + 7 line rejection causes
    uint32_t edge_partial_offset;   // first partial slot of the edge kernels
    double tukey_a2_line;     // a^2 for edges, a = double(sqrtf(3*lineRes_))  (LidarSlam.cpp:263)
    double tukey_a2;          // a^2, a = double(sqrtf(3*planeRes_))  (LidarSlam.cpp:271)
    uint32_t* counters;       // [n_scans] CTA tickets of k_evaluate_lm; nullptr = two-kernel form (k_evaluate + k_lm_step)
    bool coop_knn = false;    // small registration: one warp per query (k_knn_scan_coop)
};

// neighbour hand-off between k_knn_scan and k_fit: positions only.  k_fit gathers the five points from the sorted map, which
// (16 B per map point, 16 MB at the bench shape) fits in L2; handing over the points would send 160 B per query through HBM.
struct NnBuf {
    uint32_t* pos;       // [5][cap] positions of the 5 neighbours in the sorted map (0xFFFFFFFF = none); k_fit's input, seeds the next iteration
    float* d5;           // [cap] exact 5th-neighbour d2 of the last search (decides whether its neighbours seed the next one)
    unsigned char* pre;  // [cap] SO_MATCH_SKIPPED / NOT_ENOUGH_NEIGHBORS / NEIGHBORS_TOO_FAR / SUCCESS (= has 5 neighbours)
    size_t cap;
};

constexpr uint32_t kCoopMaxGrid = 32;     // k_knn_scan_coop serves scans of up to 32 x 256 queries (a decimated live scan is ~2 000)
constexpr int kEvalPts = 16;              // points per thread in k_evaluate (large scans); part of the partial-sum layout, so of the result bits
// Points per thread of the evaluation kernels as a function of the scan's own size (never of the batch it is in, so that a scan's
// partial sums -- and with them its result, bit for bit -- do not depend on its neighbours): small scans spread over more CTAs,
// because ONE CTA looping over 16 points per thread was most of a latency-bound optimiser step.
__host__ __device__ inline int eval_pts(uint32_t n) { return n <= 4096u ? 1 : (n <= 65536u ? 4 : kEvalPts); }
__host__ __device__ inline uint32_t eval_ctas(uint32_t n) { const uint32_t per = uint32_t(eval_pts(n)) * 256u; return (n + per - 1) / per; }
// CTAs that cover every scan of up to n_max points (a smaller scan with fewer points per thread may need more CTAs than the largest)
__host__ inline uint32_t eval_grid(uint32_t n_max) {
    if (n_max <= 4096u) return (n_max + 255u) / 256u;
    if (n_max <= 65536u) { const uint32_t g = (n_max + 1023u) / 1024u; return g > 16u ? g : 16u; }
    const uint32_t per = uint32_t(kEvalPts) * 256u, g = (n_max + per - 1u) / per;
    return g > 64u ? g : 64u;
}
// k_fit launch shape, re-measured on an H100 80GB HBM3 (700 W limit; scripts/ab_knn.py, 64 cfg2 scans = 8.4 M points per launch,
// two alternating rounds, ms per launch): 2 points x 256 threads x 4 CTAs/SM 0.554-0.560; 1 point per thread 0.544-0.545;
// 128 threads x 8 CTAs/SM 0.552-0.554; neighbours re-read and re-converted per pass instead of kept in shared memory 0.594-0.609.
// The defaults are kept: the other shapes are within 3 % and were not carried through the full suite.  These times are with the
// neighbour points handed over through HBM; with positions handed over (NnBuf) the default shape takes 0.487-0.489 ms.
// k_fit only matches / fits; the first evaluation of the solve is a k_evaluate<PH_CORR> launch, so k_fit carries no
// normal-equation accumulators (64 registers, 4 CTAs per SM).
constexpr int kFitPts = 2;               // points per thread in k_fit
constexpr int kFitThreads = 256;
constexpr int kFitMinBlocks = 4;

void launch_scan_keys(const MapView& m, const BatchView& bv, uint64_t* keys, uint32_t* vals, uint32_t grid_x, uint32_t n_scans, int cell_bits, bool key32,
                      bool compact, cudaStream_t st);
void launch_scan_finish(const BatchView& bv, const uint64_t* sorted_keys, size_t first, uint32_t pt_first, int cell_bits, bool key32, uint32_t n_scans, cudaStream_t st);
constexpr uint32_t kPrepareSmallCap = 4096;    // survivors k_prepare_small can order (one CTA per scan)
void launch_prepare_small(const MapView& m, const BatchView& bv, float4* out, uint32_t n_scans, int key_bits, uint32_t max_kept, cudaStream_t st);
void launch_scan_gather(const float4* in, const uint32_t* vals, const uint64_t* keys, size_t first, const uint32_t* offset, size_t total, float4* out,
                        int cell_bits, bool key32, cudaStream_t st);
// part: 0 = the whole stage; 1 = k_knn_scan alone, 2 = k_fit alone (profiling)
void launch_match(const MapView& m, const BatchView& bv, const CorrBuf& cb, const NnBuf& nb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, int part = 0);
void launch_inject(const MapView& m, const float4* by_id, uint32_t n_map, const BatchView& bv, const NnBuf& nb, const uint32_t* ids, int n_trace_iters,
                   uint32_t grid_x, uint32_t n_scans, cudaStream_t st);
void launch_first_eval(const BatchView& bv, const CorrBuf& cb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const MapView* medge = nullptr,
                       const EdgeBuf* eb = nullptr, uint32_t grid_e = 0);
void launch_correspond(const MapView& m, const BatchView& bv, const CorrBuf& cb, const NnBuf& nb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st,
                       const MapView* medge = nullptr, const EdgeBuf* eb = nullptr, uint32_t grid_e = 0);
void launch_evaluate(const BatchView& bv, const CorrBuf& cb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const EdgeBuf* eb = nullptr, uint32_t grid_e = 0);
void launch_loop_cond(const BatchView& bv, uint32_t n_scans, cudaGraphConditionalHandle handle, cudaStream_t st);
void launch_pack_poses(const IcpState* st, uint32_t n_scans, double* rows, cudaStream_t stream);
// so_covariance: covariance_and_errors_warp on st->H (one scan's state, device memory)
void launch_covariance(IcpState* st, cudaStream_t stream);
void launch_query_keys(const MapView& m, const float4* q, size_t nq, uint32_t* keys, uint32_t* vals, cudaStream_t st);
int launch_knn(const MapView& m, const float4* q, const uint32_t* order, size_t nq, int k, float max_d2, uint32_t* idx, float* d2, cudaStream_t st);

}  // namespace so

// so_icp.cuh -- kernel-side views and host launchers shared by so_icp.cu / so_api.cu.
#pragma once
#include "so_corr_tiles.h"
#include "so_internal.cuh"

namespace so {

// The solve's correspondence record: what every evaluation pass reads per point.  Its three arrays are indexed by record slot
// (corr_first(first + s, offset[s]) + i for point i of scan s of the chunk, so_corr_tiles.h); flags, nn and nn_d2 by the point's
// position in the scan buffer.  A fitted plane is kept as the QR solution x it comes from (24 B, plane_of_solution gives n and d),
// not as {n, d} (32 B): the evaluation streams 44 B per point instead of 56.  Given rows (so_solve*) have no QR solution, so their
// record holds {n.x, n.y, n.z, d} (the ND form of the evaluation kernels); x holds 4 doubles per slot so that both forms fit.
struct CorrBuf {
    double* x;          // [3 per slot] QR solution x (ND form: [4 per slot] {n, d}); 0 for rejected points
    double* w;          // [slot] residualCoefficient (0 for rejected)
    float* p;           // [3 per slot] the scan point, as the scan buffer holds it
    uchar4* flags;      // {status, obs0, obs1, obs2}
    uint32_t* nn;       // optional [5 per point] neighbour ids (stage tests); may be null
    float* nn_d2;       // optional [5 per point]
    uint32_t first = 0; // the chunk's first scan inside the batch
    bool given = false; // the record holds {n, d} (so_solve*): the launchers take the ND form of the evaluation kernels
};

// The plane of a fit from its unnormalised QR solution x (A x = -1 over the neighbours): negative_OA_dot_norm = 1 / norm.norm();
// norm.normalize() (LidarSlam.cpp:812-816).  k_fit gates on what this returns and every reader of the record decodes x with it, so
// the rounding of each step is spelt out: |x|^2 as the compiler contracted the expression x0 x0 + x1 x1 + x2 x2 where the fit used
// to compute it (x1 x1 rounded, then two FMAs), IEEE square root and reciprocal, and x / |x| as the division (div_rcp from the
// reciprocal, which gives the same bits, where it is valid).
__device__ __forceinline__ void plane_of_solution(double x0, double x1, double x2, double n[3], double& d) {
    const double nn = __dsqrt_rn(__fma_rn(x2, x2, __fma_rn(x0, x0, __dmul_rn(x1, x1))));
    d = __drcp_rn(nn);
    n[0] = div_rcp_ok(x0, nn) ? div_rcp(x0, nn, d) : __ddiv_rn(x0, nn);
    n[1] = div_rcp_ok(x1, nn) ? div_rcp(x1, nn, d) : __ddiv_rn(x1, nn);
    n[2] = div_rcp_ok(x2, nn) ? div_rcp(x2, nn, d) : __ddiv_rn(x2, nn);
}

// Slots per record entry of the two forms: the QR solution, or {n, d} (given rows)
template <bool ND> constexpr int kCorrX = ND ? 4 : 3;

// n and d of the record entry at rec (kCorrX<ND> doubles)
template <bool ND>
__device__ __forceinline__ void corr_plane(const double* rec, double n[3], double& d) {
    if (ND) { n[0] = rec[0]; n[1] = rec[1]; n[2] = rec[2]; d = rec[3]; }
    else plane_of_solution(rec[0], rec[1], rec[2], n, d);
}

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
    // with the neighbour graph (MapView::graph): the queries it did not answer, handed from k_knn_scan to k_knn_round2
    uint32_t* queue;     // [cap] point indices, scan s's from offset[s] on; their round-1 bound waits in d5
    uint32_t* qcount;    // [scans][SO_MAX_ICP_ITERS] queue lengths, zeroed before every registration call
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

// The launchers of the registration's kernels return the number of kernels they enqueued (Ctx::launches counts from that).
uint32_t launch_scan_keys(const MapView& m, const BatchView& bv, uint64_t* keys, uint32_t* vals, uint32_t grid_x, uint32_t n_scans, int cell_bits, bool key32,
                          bool compact, cudaStream_t st);
uint32_t launch_scan_finish(const BatchView& bv, const uint64_t* sorted_keys, size_t first, uint32_t pt_first, int cell_bits, bool key32, uint32_t n_scans, cudaStream_t st);
constexpr uint32_t kPrepareSmallCap = 4096;    // survivors k_prepare_small can order (one CTA per scan)
uint32_t launch_prepare_small(const MapView& m, const BatchView& bv, float4* out, uint32_t n_scans, int key_bits, uint32_t max_kept, cudaStream_t st);
uint32_t launch_scan_gather(const float4* in, const uint32_t* vals, const uint64_t* keys, size_t first, const uint32_t* offset, size_t total, float4* out,
                            int cell_bits, bool key32, cudaStream_t st);
// part: 0 = the whole stage; 1 = the search alone, 2 = k_fit alone
uint32_t launch_match(const MapView& m, const BatchView& bv, const CorrBuf& cb, const NnBuf& nb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, int part = 0);
uint32_t launch_inject(const MapView& m, const float4* by_id, uint32_t n_map, const BatchView& bv, const NnBuf& nb, const uint32_t* ids, int n_trace_iters,
                       uint32_t grid_x, uint32_t n_scans, cudaStream_t st);
// dg: the chunk's DegenState array of a degeneracy-aware registration (k_lm_step_deg in place of k_lm_step, no fused form)
uint32_t launch_first_eval(const BatchView& bv, const CorrBuf& cb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const MapView* medge = nullptr,
                           const EdgeBuf* eb = nullptr, uint32_t grid_e = 0, DegenState* dg = nullptr);
// k_edge_fit alone (mode OPTIMIZED: the line correspondences and histogram; its 6-column sums are not read there)
uint32_t launch_edge_fit(const MapView& medge, const BatchView& bv, const EdgeBuf& eb, uint32_t grid_e, uint32_t n_scans, cudaStream_t st);
uint32_t launch_evaluate(const BatchView& bv, const CorrBuf& cb, uint32_t grid_x, uint32_t n_scans, cudaStream_t st, const EdgeBuf* eb = nullptr,
                         uint32_t grid_e = 0, DegenState* dg = nullptr);
uint32_t launch_loop_cond(const BatchView& bv, uint32_t n_scans, cudaGraphConditionalHandle handle, cudaStream_t st);
uint32_t launch_pack_poses(const IcpState* st, uint32_t n_scans, double* rows, cudaStream_t stream);
// so_covariance: covariance_and_errors_warp on st->H (one scan's state, device memory)
uint32_t launch_covariance(IcpState* st, cudaStream_t stream);
// so_degeneracy_analysis: the analysis a degeneracy-aware solve begins with, on st->H, into *dg (device memory, thresholds set)
uint32_t launch_degeneracy_analysis(const IcpState* st, DegenState* dg, cudaStream_t stream);
void launch_query_keys(const MapView& m, const float4* q, size_t nq, uint32_t* keys, uint32_t* vals, cudaStream_t st);
int launch_knn(const MapView& m, const float4* q, const uint32_t* order, size_t nq, int k, float max_d2, uint32_t* idx, float* d2, cudaStream_t st);

}  // namespace so

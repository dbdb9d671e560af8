// so_map.cu -- device-resident LocalMap: block binning + sorted spatial hash grid (SURVEY 2.3: K1).
//
// Replaces the per-block nanoflann::Octree build (flann/octree.h:355-400,536-738, called from LocalMap.h:580,638):
// points are keyed by (block slot, cell inside the block), radix-sorted, and a dense per-slot cell-start table is
// built by histogram + exclusive scan.  Cells have edge cs = 50/nb >= sqrt(3*planeRes): every neighbour that can
// pass the NEIGHBORS_TOO_FAR gate lies in the 27 cells around the query's cell, and because nb divides the 50 m
// block exactly, "same block" (LocalMap.h:488-507) is "same slot".
//
// Every change to a store goes through one pipeline: an optional filter stage (voxel filter of the touched blocks, drop of
// off-grid points; filter_stage) and one index stage (block counts, slots, cell table; count_blocks + index_cells).
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <set>

#include <cub/cub.cuh>

#include "so_archive.h"
#include "so_ctx.cuh"
#include "so_knn.cuh"

namespace so {

// Cells per 50 m block axis: cell edge cs = 50/nb is about half the search radius sqrt(3*planeRes) (so the pruned
// walk over (2R+1)^2 rows visits few points beyond the true k-NN ball), capped at 192 (28 MB cell table per block).
int map_cells_per_block(float plane_res) {
    const float bound = 3 * plane_res;                               // float product, as LidarSlam.cpp:526
    const double r = std::sqrt(double(bound)) * (1.0 + 1e-4);
    int nb = int(2.0 * kBlock / r);
    if (nb < 1) nb = 1;
    if (nb > 192) nb = 192;
    return nb;
}

static int map_rings(float plane_res, int nb) {
    const float bound = 3 * plane_res;
    const double r = std::sqrt(double(bound)) * (1.0 + 1e-4);
    const double cs = kBlock / double(nb);
    int R = int(std::ceil(r / cs));
    return R < 1 ? 1 : R;
}

// Device-side bookkeeping of a store change or a scan pre-filter: everything the host would otherwise read back between launches.
struct InsertInfo {
    uint32_t begin, end;        // sorted filter keys: [0, begin) kept in order, [begin, end) voxel-filtered, [end, total) dropped
    uint32_t n_out;             // points of the filtered cloud (the cloud the index stage indexes)
    uint32_t n_slots;           // non-empty blocks of that cloud
    uint32_t n_kept;            // its points on the grid
    uint32_t error;             // 1: more slots than the cell table was sized for
    uint32_t fallback;          // cloud voxel filter: PCL's voxel index would overflow, the output is the input
    uint32_t pad;
};
struct MapScratch {
    InsertInfo info;
    uint32_t bounds[6];                                              // cloud voxel filter: float_order min, ~max per axis (atomicMin)
    uint8_t touched[kNumBlocks];                                     // blocks the new points of an insert reach
    uint32_t runs;                                                   // eviction: blocks (and the dropped run) of the off-window points
};

constexpr size_t kMaxCells = size_t(1) << 31;      // cell indices are 32-bit in the kernels and the scan length is an int

__device__ __forceinline__ int block_coord(double v, int origin) {   // LocalMap.h:594-605
    int c = int(v / kBlock);
    if (v < 0) c--;
    return c + origin;
}

// Linear grid block of a point under `origin`, or -1 when the block is off the 21 x 21 x 11 grid or the point is not finite
__device__ __forceinline__ int grid_block(const float4 p, int3 origin) {
    const int gx = block_coord(double(p.x) + kHalfBlock, origin.x), gy = block_coord(double(p.y) + kHalfBlock, origin.y),
              gz = block_coord(double(p.z) + kHalfBlock, origin.z);
    if (gx >= 0 && gx < kW && gy >= 0 && gy < kH && gz >= 0 && gz < kD && isfinite(p.x) && isfinite(p.y) && isfinite(p.z))
        return gx + kW * gy + kW * kH * gz;
    return -1;
}

static int store_alloc(Ctx* c, MapStore& ms) {
    const size_t M = c->cfg.max_map_points;
    int rc = ms.d_xyzi.reserve(M);
    if (!rc) rc = ms.d_sorted.reserve(M);
    if (!rc) rc = ms.d_block_slot.reserve(kNumBlocks);
    if (!rc) rc = ms.d_block_count.reserve(kNumBlocks);
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemset(ms.d_block_slot, 0xFF, kNumBlocks * sizeof(int32_t)));
    SO_CUDA_TRY(cudaMemset(ms.d_block_count, 0, kNumBlocks * sizeof(int32_t)));
    ms.h_block_count.assign(kNumBlocks, 0);
    ms.h_block_slot.assign(kNumBlocks, -1);
    return SO_OK;
}

int map_alloc(Ctx* c) {
    const size_t M = c->cfg.max_map_points;
    int rc = store_alloc(c, c->surf);
    if (rc) return rc;
    rc = store_alloc(c, c->edge);
    if (rc) return rc;
    rc = c->d_keys.reserve(M);
    if (!rc) rc = c->d_keys_out.reserve(M);
    if (!rc) rc = c->d_vals.reserve(M);
    if (!rc) rc = c->d_vals_out.reserve(M);
    if (rc) return rc;
    // cub temp: the 64-bit filter sort (the 32-bit cell sort needs less) and the scan of its voxel heads at full capacity;
    // reserve_cells grows it for the scan of the cell table
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, c->d_keys.get(), c->d_keys_out.get(), c->d_vals.get(), c->d_vals_out.get(), int(M), 0, 64);
    cub::DeviceScan::ExclusiveSum(nullptr, b, (uint32_t*)nullptr, (uint32_t*)nullptr, int(M));
    rc = c->d_cub_tmp.reserve(std::max(a, b) + 256);
    if (!rc) rc = c->d_map_scratch.reserve(1);
    if (!rc) rc = c->h_map_info.reserve(1);
    return rc;
}

MapView map_view(const Ctx* c, const MapStore& ms) {
    MapView m;
    m.pts = ms.d_sorted; m.block_slot = ms.d_block_slot; m.block_count = ms.d_block_count; m.cell_start = ms.d_cell_start;
    m.origin[0] = c->origin[0]; m.origin[1] = c->origin[1]; m.origin[2] = c->origin[2];
    m.nb = ms.nb; m.inv_cs = double(ms.nb) / kBlock; m.cs = float(kBlock / double(ms.nb));
    m.bound_d2 = 3 * ms.res;        // float product (LidarSlam.cpp:526)
    m.inv_bound_d2 = 1.0 / double(m.bound_d2);
    m.plane_res = ms.res;
    m.R = map_rings(ms.res, ms.nb);
    m.graph = nullptr; m.graph_radius = nullptr; m.graph_stats = nullptr;
    return m;
}

// ------------------------------------------------------------------------------------------------------------------
// Neighbour graph of the sorted cloud (so_knn.cuh): row t = the kGraphK nearest in-block points of point t, from the exact in-block
// search for kGraphK + 1 neighbours with t itself dropped, and the radius below which the row is complete.  A point the search does
// not return (more than kGraphK duplicates with smaller ids) or whose block lookup disagrees with its place in the index gets radius 0.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kGraphThreads = 64;
__global__ void __launch_bounds__(kGraphThreads) k_knn_graph(MapView m, uint32_t n, uint32_t* __restrict__ graph, float* __restrict__ radius) {
    __shared__ uint32_t s_buf[kBufCap * kGraphThreads];
    const uint32_t t = blockIdx.x * kGraphThreads + threadIdx.x;
    if (t >= n) return;                                          // no CTA-wide synchronisation below
    const float4 p = m.pts[t];
    QueryCell qc;
    locate(m, p.x, p.y, p.z, qc);
    uint32_t* row = graph + size_t(t) * kGraphK;
    int j = 0;
    float r = 0.f;
    if (qc.slot >= 0) {
        const uint32_t cells = uint32_t(m.nb) * uint32_t(m.nb) * uint32_t(m.nb);
        const uint32_t lo = m.cell_start[uint32_t(qc.slot) * cells], hi = m.cell_start[uint32_t(qc.slot) * cells + cells];
        if (t >= lo && t < hi) {
            TopK<kGraphK + 1> tk;
            tk.init(FLT_MAX);
            knn_search<kGraphK + 1>(BlockGrid(m, qc.slot), m, qc, p.x, p.y, p.z, 0.f, s_buf, tk);
            bool self = false;
            float last = 0.f;
#pragma unroll
            for (int i = 0; i < kGraphK + 1; ++i) {
                // a block of at most kGraphK points also hands back the far-away dummies its walks pad spans with (for_span): entries
                // whose position does not hold the point they name
                const bool real = tk.id[i] != 0xFFFFFFFFu && tk.pos[i] >= lo && tk.pos[i] < hi && __float_as_uint(m.pts[tk.pos[i]].w) == tk.id[i] &&
                                  exact_d2(m.pts[tk.pos[i]], p.x, p.y, p.z) == tk.d2[i];
                const bool me = real && tk.pos[i] == t;
                self |= me;
                if (real && !me && j < kGraphK) { row[j++] = tk.pos[i]; last = tk.d2[i]; }
            }
            if (self) r = (hi - lo - 1u <= uint32_t(kGraphK)) ? INFINITY : kGraphRadiusScale * sqrtf(last);
        }
    }
    for (; j < kGraphK; ++j) row[j] = 0xFFFFFFFFu;
    radius[t] = r;
}

bool knn_graph_valid(const Ctx* c) {
    const MapStore& ms = c->surf;
    return c->knn_graph_mode >= 0 && !ms.dirty && ms.n > 0 && ms.graph_gen == ms.index_gen && ms.d_graph;
}

int knn_graph_prepare(Ctx* c, size_t queries) {
    MapStore& ms = c->surf;
    if (ms.dirty || knn_graph_valid(c) || !graph_build_due(c->knn_graph_mode, queries, ms.n)) return SO_OK;
    int rc = ms.d_graph.reserve(size_t(ms.n) * kGraphK);
    if (!rc) rc = ms.d_graph_radius.reserve(ms.n);
    if (rc) return rc;
    k_knn_graph<<<(ms.n + kGraphThreads - 1) / kGraphThreads, kGraphThreads, 0, c->stream>>>(map_view(c, ms), ms.n, ms.d_graph, ms.d_graph_radius);
    c->launches++;
    SO_CUDA_TRY(cudaGetLastError());
    ms.graph_gen = ms.index_gen;
    return SO_OK;
}

MapView search_view(const Ctx* c) {
    MapView m = map_view(c, c->surf);
    if (knn_graph_valid(c)) {
        m.graph = reinterpret_cast<const uint4*>(c->surf.d_graph.get());
        m.graph_radius = c->surf.d_graph_radius;
        m.graph_stats = c->d_graph_stats;
    }
    return m;
}

int scan_sort_alloc(Ctx* c) {
    size_t need = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, need, c->d_skeys.get(), c->d_skeys_out.get(), c->d_svals.get(), c->d_svals_out.get(), int(c->scan_cap), 0, 64);
    int rc = c->d_sort_tmp.reserve(need + 256);
    if (!rc) rc = c->d_sort_tmp2.reserve(need + 256);
    return rc;
}

int query_sort_reserve(Ctx* c, size_t n) {
    int rc = c->d_qkeys.reserve(n);
    if (!rc) rc = c->d_qkeys_out.reserve(n);
    if (!rc) rc = c->d_qvals.reserve(n);
    if (!rc) rc = c->d_qvals_out.reserve(n);
    if (rc) return rc;
    size_t need = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, need, c->d_qkeys.get(), c->d_qkeys_out.get(), c->d_qvals.get(), c->d_qvals_out.get(), int(n), 0, 32);
    return c->d_qsort_tmp.reserve(need + 256);
}

int query_sort(Ctx* c, size_t n) {
    size_t tmp = c->d_qsort_tmp.cap();
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_qsort_tmp, tmp, c->d_qkeys.get(), c->d_qkeys_out.get(), c->d_qvals.get(), c->d_qvals_out.get(), int(n), 0, 32, c->stream));
    c->launches += 5;
    return SO_OK;
}

int scan_sort(Ctx* c, size_t first, size_t n, int n_scans, int cell_bits, bool key32, cudaStream_t st) {
    int bits = cell_bits;
    while ((1 << (bits - cell_bits)) < n_scans) ++bits;
    size_t tmp = c->d_sort_tmp.cap();
    void* scratch = st == c->aux_stream ? c->d_sort_tmp2 : c->d_sort_tmp;
    if (key32)
        SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(scratch, tmp, reinterpret_cast<uint32_t*>(c->d_skeys.get()) + first, reinterpret_cast<uint32_t*>(c->d_skeys_out.get()) + first,
                                                    c->d_svals + first, c->d_svals_out + first, int(n), 0, bits, st));
    else
        SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(scratch, tmp, c->d_skeys.get() + first, c->d_skeys_out.get() + first,
                                                    c->d_svals + first, c->d_svals_out + first, int(n), 0, bits, st));
    c->launches += 5;
    return SO_OK;
}

struct Pose7 { double v[7]; };
// utils::TransformPoint (superodom_utils.h:116-127): double math, float store; w kept
__device__ __forceinline__ float4 pose_point(const double* pose, float4 p) {
    const double v[3] = {double(p.x), double(p.y), double(p.z)};
    double o[3];
    qrot(pose + 3, v, o);
    p.x = float(o[0] + pose[0]); p.y = float(o[1] + pose[1]); p.z = float(o[2] + pose[2]);
    return p;
}

__global__ void k_transform_points(float4* __restrict__ pts, uint32_t n, Pose7 pose) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pts[i] = pose_point(pose.v, pts[i]);
}

void launch_transform(float4* pts, uint32_t n, const double pose[7], cudaStream_t st) {
    if (!n) return;
    Pose7 P;
    for (int k = 0; k < 7; ++k) P.v[k] = pose[k];                            // by value in the launch: no staging copy, no wait
    k_transform_points<<<(n + 255) / 256, 256, 0, st>>>(pts, n, P);
}

int map_transform_tail(Ctx* c, MapStore& ms, uint32_t n_new, const double pose[7]) {
    launch_transform(ms.d_xyzi + ms.n, n_new, pose, c->stream);
    c->launches++;
    return SO_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Voxel reduction shared by the map's filter stage and the scan pre-filter: pcl::VoxelGrid semantics (voxel =
// floor(coord * (1.0f/leaf)) in float32, centroid of all four fields accumulated in float32 and divided by float(count), output
// ordered by voxel index).  PCL leaves the in-voxel accumulation order unspecified (std::sort on the voxel index); here it is
// ascending cloud order, the order the stable radix sort preserves.  Sorted keys below t_voxel are copied through in order, keys
// in [t_voxel, t_drop) are averaged voxel by voxel, keys from t_drop on are dropped.
// ------------------------------------------------------------------------------------------------------------------
// boundaries of the three key classes in the sorted keys, by binary search (one thread)
__global__ void k_voxel_bounds(const uint64_t* __restrict__ keys, uint32_t total, uint64_t t_voxel, uint64_t t_drop, InsertInfo* __restrict__ info) {
    if (threadIdx.x || blockIdx.x) return;
    uint32_t lo = 0, hi = total;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (keys[mid] >= t_voxel) hi = mid; else lo = mid + 1; }      // first filtered key
    info->begin = lo;
    hi = total;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (keys[mid] >= t_drop) hi = mid; else lo = mid + 1; }       // first dropped key
    info->end = lo;
}

__global__ void k_voxel_heads(const uint64_t* __restrict__ keys, uint32_t total, const InsertInfo* __restrict__ info, uint32_t* __restrict__ head) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    head[i] = (i >= info->begin && i < info->end && (i == info->begin || keys[i] != keys[i - 1])) ? 1u : 0u;
}

// rank[] = exclusive scan of head[] over [0, total): rank[i] counts the voxels before sorted position i
__global__ void k_voxel_centroid(const float4* __restrict__ raw, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                 const uint32_t* __restrict__ head, const uint32_t* __restrict__ rank, uint32_t total, InsertInfo* __restrict__ info,
                                 float4* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const uint32_t begin = info->begin, end = info->end;
    if (i == total - 1) info->n_out = begin + rank[i] + head[i];      // voxels in total
    if (i < begin) { out[i] = raw[vals[i]]; return; }                   // kept points: copied through in order
    if (i >= end || !head[i]) return;
    const uint64_t key = keys[i];
    float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
    uint32_t cnt = 0;
    for (uint32_t j = i; j < end && keys[j] == key; ++j) {             // pcl::CentroidPoint: float accumulators, cloud order
        const float4 p = raw[vals[j]];
        ax = __fadd_rn(ax, p.x); ay = __fadd_rn(ay, p.y); az = __fadd_rn(az, p.z); aw = __fadd_rn(aw, p.w);
        ++cnt;
    }
    const float nf = float(cnt);
    out[begin + rank[i]] = make_float4(__fdiv_rn(ax, nf), __fdiv_rn(ay, nf), __fdiv_rn(az, nf), __fdiv_rn(aw, nf));
}

// raw[0..total) sorted by keys / vals -> out[0..info->n_out); head: scratch of 2 * total words (heads, then ranks)
static int voxel_reduce(Ctx* c, const float4* raw, const uint64_t* keys, const uint32_t* vals, uint32_t total, uint64_t t_voxel, uint64_t t_drop,
                        uint32_t* head, void* tmp, size_t tmp_bytes, float4* out) {
    cudaStream_t st = c->stream;
    InsertInfo* d_info = &c->d_map_scratch->info;
    const uint32_t grid = (total + 255) / 256;
    uint32_t* rank = head + total;
    k_voxel_bounds<<<1, 32, 0, st>>>(keys, total, t_voxel, t_drop, d_info);
    k_voxel_heads<<<grid, 256, 0, st>>>(keys, total, d_info, head);
    SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, head, rank, int(total), st));
    k_voxel_centroid<<<grid, 256, 0, st>>>(raw, keys, vals, head, rank, total, d_info, out);
    c->launches += 5;
    return SO_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Filter stage: LocalMap::addSurfPointCloud (LocalMap.h:591-645).  New world-frame points are appended, every block they
// touch is re-filtered as a whole by a voxel-centroid filter of leaf planeRes_ (output ordered by voxel index (k, j, i)),
// untouched blocks keep their clouds, points off the grid (what LocalMap::shiftMap does to blocks rolled off it,
// LocalMap.h:169-287) are dropped.  The in-voxel accumulation order is old points, then new points in input order.
// ------------------------------------------------------------------------------------------------------------------
__global__ void k_mark_touched_new(const float4* __restrict__ pts, uint32_t n_new, int3 origin, uint8_t* __restrict__ touched) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_new) return;
    const int b = grid_block(pts[i], origin);
    if (b >= 0) touched[b] = 1;
}

// Voxel of p inside world block w (grid block g = w + origin) as [vk][vj][vi], vb bits each.  PCL orders a block's output by the voxel
// index relative to the block cloud's bounding box; subtracting any per-block constant keeps that order, so the index is taken relative
// to the block's minimum corner (minus a 2-voxel guard for the float rounding of x * inv_leaf at the faces).
__device__ __forceinline__ uint64_t block_voxel(const float4 p, int wx, int wy, int wz, float inv_leaf, int vb) {
    const double il = double(inv_leaf);
    const int64_t bx = int64_t(floor((double(wx) * kBlock - kHalfBlock) * il)) - 2;
    const int64_t by = int64_t(floor((double(wy) * kBlock - kHalfBlock) * il)) - 2;
    const int64_t bz = int64_t(floor((double(wz) * kBlock - kHalfBlock) * il)) - 2;
    const int64_t vmax = (int64_t(1) << vb) - 1;
    auto local = [vmax](int64_t v) { return uint64_t(v < 0 ? 0 : (v > vmax ? vmax : v)); };
    const uint64_t vi = local(int64_t(floorf(__fmul_rn(p.x, inv_leaf))) - bx);      // pcl::VoxelGrid: floor(coord * inverse_leaf_size) in float
    const uint64_t vj = local(int64_t(floorf(__fmul_rn(p.y, inv_leaf))) - by);
    const uint64_t vk = local(int64_t(floorf(__fmul_rn(p.z, inv_leaf))) - bz);
    return (vk << (2 * vb)) | (vj << vb) | vi;
}

// bits of a block-local voxel index: 50 m / leaf + 5 values
static int voxel_bits(float inv_leaf) {
    int vb = 1;
    while (vb < 16 && double(1 << vb) < kBlock * double(inv_leaf) + 5.0) ++vb;
    return vb;
}

// insert key of every point (old cloud followed by the new points), the block recomputed from the coordinates:
// [class: 0 untouched block, 1 touched, 2 dropped][block 13 bits][vk][vj][vi], vb bits per block-local voxel index (50 m / leaf + 5
// values: 8 bits at leaf 0.2) -- 39 key bits = 5 radix passes instead of the 8 of a full 64-bit key.
__global__ void k_insert_keys(const float4* __restrict__ raw, uint32_t n, float inv_leaf, int3 origin, const uint8_t* __restrict__ touched,
                              int vb, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = raw[i];
    const int b = grid_block(p, origin);
    const int cls_shift = 13 + 3 * vb;
    uint64_t key = uint64_t(2) << cls_shift;                              // off-grid / non-finite: dropped
    if (b >= 0) {
        if (!touched[b]) key = 0;                                         // untouched block: kept in place (stable sort)
        else {
            const int gx = b % kW, gy = (b / kW) % kH, gz = b / (kW * kH);
            key = (uint64_t(1) << cls_shift) | (uint64_t(b) << (3 * vb)) | block_voxel(p, gx - origin.x, gy - origin.y, gz - origin.z, inv_leaf, vb);
        }
    }
    keys[i] = key;
    vals[i] = i;
}

// d_xyzi[0..ms.n + n_new) (the store's cloud, then n_new new points) -> the filtered cloud in d_xyzi[0..info->n_out); the two cloud
// buffers swap roles (no device-to-device copy of the map).  n_new == 0: nothing is touched, only the off-grid points are dropped
// (the sort then runs over the two class bits alone).
static int filter_stage(Ctx* c, MapStore& ms, uint32_t n_new) {
    cudaStream_t st = c->stream;
    const uint32_t total = ms.n + n_new;
    const int3 origin = make_int3(c->origin[0], c->origin[1], c->origin[2]);
    uint8_t* d_touched = c->d_map_scratch->touched;
    SO_CUDA_TRY(cudaMemsetAsync(d_touched, 0, kNumBlocks, st));
    if (n_new) k_mark_touched_new<<<(n_new + 255) / 256, 256, 0, st>>>(ms.d_xyzi + ms.n, n_new, origin, d_touched);
    const float inv_leaf = 1.0f / ms.res;                               // Eigen::Array4f::Ones() / leaf_size_
    const int vb = voxel_bits(inv_leaf);
    const int cls_shift = 13 + 3 * vb;
    k_insert_keys<<<(total + 255) / 256, 256, 0, st>>>(ms.d_xyzi, total, inv_leaf, origin, d_touched, vb, c->d_keys, c->d_vals);
    size_t tmp = c->d_cub_tmp.cap();
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_cub_tmp, tmp, c->d_keys.get(), c->d_keys_out.get(), c->d_vals.get(), c->d_vals_out.get(), int(total),
                                                n_new ? 0 : cls_shift, cls_shift + 2, st));
    c->launches += 8;
    const int rc = voxel_reduce(c, ms.d_xyzi, c->d_keys_out, c->d_vals_out, total, uint64_t(1) << cls_shift, uint64_t(2) << cls_shift,
                                reinterpret_cast<uint32_t*>(c->d_keys.get()), c->d_cub_tmp, c->d_cub_tmp.cap(), ms.d_sorted);   // keys_in is free after the sort
    std::swap(ms.d_xyzi, ms.d_sorted);                                  // d_xyzi: the new cloud in id order; d_sorted: free for the new index
    return rc;
}

// ------------------------------------------------------------------------------------------------------------------
// Index stage: the search index of d_xyzi[0..info->n_out) (every point on the grid): block counts, slots in block order, cell
// keys through locate() -- the searches bin a point with the same code -- a 32-bit sort, the gather and the cell table.
// ------------------------------------------------------------------------------------------------------------------
// One atomic per (warp, block) instead of one per point: the cloud is ordered block by block, so a warp almost always holds a
// single block (1.1 M same-address atomics took 660 us; aggregated they take a few).  Off-grid points are counted nowhere.
__global__ void k_block_count(const float4* __restrict__ raw, const InsertInfo* __restrict__ info, int3 origin, int32_t* __restrict__ block_count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lin = i < info->n_out ? grid_block(raw[i], origin) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, lin);
    if (lin >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&block_count[lin], __popc(peers));
}

// slots of the non-empty blocks in block order, the points they hold, and the error flag of a slot count above slot_cap (one CTA)
__global__ void __launch_bounds__(1024) k_assign_slots(const int32_t* __restrict__ block_count, int32_t* __restrict__ block_slot, InsertInfo* __restrict__ info,
                                                       uint32_t slot_cap) {
    __shared__ uint32_t s_part[1024];
    __shared__ uint32_t s_kept;
    const int per = (kNumBlocks + 1023) / 1024;
    const int b0 = threadIdx.x * per;
    uint32_t mine = 0, kept = 0;
    for (int k = 0; k < per; ++k) { const int b = b0 + k; if (b < kNumBlocks && block_count[b] > 0) { ++mine; kept += uint32_t(block_count[b]); } }
    s_part[threadIdx.x] = mine;
    if (threadIdx.x == 0) s_kept = 0;
    __syncthreads();
    if (kept) atomicAdd(&s_kept, kept);
    for (int o = 1; o < 1024; o <<= 1) {                                // Hillis-Steele inclusive scan
        const uint32_t v = threadIdx.x >= o ? s_part[threadIdx.x - o] : 0;
        __syncthreads();
        s_part[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t slot = s_part[threadIdx.x] - mine;
    for (int k = 0; k < per; ++k) {
        const int b = b0 + k;
        if (b < kNumBlocks) block_slot[b] = block_count[b] > 0 ? int32_t(slot++) : -1;
    }
    if (threadIdx.x == 1023) { info->n_slots = s_part[1023]; info->n_kept = s_kept; info->error = s_part[1023] > slot_cap; }
}

// cell key + histogram; positions >= n_out (and every position after a slot overflow) get the largest key and sort behind every
// real point
__global__ void k_cell_keys(const float4* __restrict__ raw, uint32_t total, const InsertInfo* __restrict__ info, MapView m,
                            uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ cell_count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    vals[i] = i;
    if (i >= info->n_out || info->error) { keys[i] = 0xFFFFFFFFu; return; }
    const float4 p = raw[i];
    QueryCell qc;
    locate(m, p.x, p.y, p.z, qc);
    const uint32_t key = scan_order_key(m, qc);
    keys[i] = key;
    atomicAdd(&cell_count[key], 1u);
}

__global__ void k_gather(const float4* __restrict__ raw, const uint32_t* __restrict__ vals, uint32_t total, const InsertInfo* __restrict__ info,
                         float4* __restrict__ sorted) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total || i >= info->n_out) return;
    const uint32_t id = vals[i];
    const float4 p = raw[id];
    sorted[i] = make_float4(p.x, p.y, p.z, __uint_as_float(id));
}

// Cell table for `slots` slots, with up to `spare` slots of headroom where the limit allows, and the cub scratch to scan it.
// SO_ERR_CAPACITY, before anything grows, when `slots` alone reach the limit.
static int reserve_cells(Ctx* c, MapStore& ms, size_t slots, size_t spare) {
    const size_t cells_per_slot = size_t(ms.nb) * ms.nb * ms.nb;
    const size_t max_slots = (kMaxCells - 2) / cells_per_slot;         // slots * cells_per_slot + 1 < 2^31
    if (slots > max_slots) {
        set_error("map spans too many 50 m blocks for the dense cell table (n_slots * nb^3 >= 2^31)");
        return SO_ERR_CAPACITY;
    }
    if (slots * cells_per_slot + 1 <= ms.d_cell_start.cap()) return SO_OK;
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    int rc = ms.d_cell_start.reserve(std::min(slots + spare, max_slots) * cells_per_slot + 1);
    if (rc) return rc;
    size_t need = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, need, ms.d_cell_start.get(), ms.d_cell_start.get(), int(ms.d_cell_start.cap()));
    return c->d_cub_tmp.reserve(need + 256);
}

// block counts and slots of d_xyzi[0..info->n_out); more than slot_cap slots raise info->error
static int count_blocks(Ctx* c, MapStore& ms, uint32_t n_max, uint32_t slot_cap) {
    cudaStream_t st = c->stream;
    InsertInfo* d_info = &c->d_map_scratch->info;
    SO_CUDA_TRY(cudaMemsetAsync(ms.d_block_count, 0, kNumBlocks * sizeof(int32_t), st));
    k_block_count<<<(n_max + 255) / 256, 256, 0, st>>>(ms.d_xyzi, d_info, make_int3(c->origin[0], c->origin[1], c->origin[2]), ms.d_block_count);
    k_assign_slots<<<1, 1024, 0, st>>>(ms.d_block_count, ms.d_block_slot, d_info, slot_cap);
    c->launches += 3;
    return SO_OK;
}

// The cell table of slot_cap slots over the slots count_blocks assigned, then the one read-back of the sizes, the error flag and
// the host mirrors.  The store is clean (its index built) when no slot overflowed.
static int index_cells(Ctx* c, MapStore& ms, uint32_t n_max, uint32_t slot_cap) {
    cudaStream_t st = c->stream;
    InsertInfo* d_info = &c->d_map_scratch->info;
    InsertInfo* h_info = c->h_map_info;
    const uint32_t grid = (n_max + 255) / 256;
    const size_t cells_used = size_t(slot_cap) * ms.nb * ms.nb * ms.nb + 1;
    SO_CUDA_TRY(cudaMemsetAsync(ms.d_cell_start, 0, cells_used * sizeof(uint32_t), st));
    uint32_t* keys32 = reinterpret_cast<uint32_t*>(c->d_keys.get());
    uint32_t* keys32_out = reinterpret_cast<uint32_t*>(c->d_keys_out.get());
    k_cell_keys<<<grid, 256, 0, st>>>(ms.d_xyzi, n_max, d_info, map_view(c, ms), keys32, c->d_vals, ms.d_cell_start);
    size_t tmp = c->d_cub_tmp.cap();
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_cub_tmp, tmp, keys32, keys32_out, c->d_vals.get(), c->d_vals_out.get(), int(n_max), 0, 32, st));
    k_gather<<<grid, 256, 0, st>>>(ms.d_xyzi, c->d_vals_out, n_max, d_info, ms.d_sorted);
    tmp = c->d_cub_tmp.cap();
    SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->d_cub_tmp, tmp, ms.d_cell_start.get(), ms.d_cell_start.get(), int(cells_used), st));
    SO_CUDA_TRY(cudaMemcpyAsync(h_info, d_info, sizeof(InsertInfo), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaMemcpyAsync(ms.h_block_count.data(), ms.d_block_count, kNumBlocks * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaMemcpyAsync(ms.h_block_slot.data(), ms.d_block_slot, kNumBlocks * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    c->launches += 10;
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    ms.n = h_info->n_out;
    ms.n_slots = int(h_info->n_slots);
    ms.dirty = h_info->error != 0;
    ms.index_gen++;
    return SO_OK;
}

static int map_rebuild_archive(Ctx* c, MapStore& ms);
static int set_empty_index(Ctx* c, MapStore& ms);

// Removal of flagged points from a built store: the id-order cloud compacted stably (cub::DeviceSelect::Flagged keeps input order)
// into the other cloud buffer, the two swapped, then the index stage over the n_keep points left.  Removal empties slots but never
// opens one, so the cell table of the current slot count holds the new index.
int map_compact(Ctx* c, MapStore& ms, const uint8_t* keep, uint32_t n_keep, uint32_t* d_num_selected) {
    cudaStream_t st = c->stream;
    size_t need = 0;
    cub::DeviceSelect::Flagged(nullptr, need, ms.d_xyzi.get(), keep, ms.d_sorted.get(), d_num_selected, int(ms.n));
    int rc = c->d_cub_tmp.reserve(need + 256);
    if (rc) return rc;
    ms.dirty = true;
    size_t tmp = c->d_cub_tmp.cap();
    SO_CUDA_TRY(cub::DeviceSelect::Flagged(c->d_cub_tmp, tmp, ms.d_xyzi.get(), keep, ms.d_sorted.get(), d_num_selected, int(ms.n), st));
    c->launches += 2;
    std::swap(ms.d_xyzi, ms.d_sorted);                                  // d_xyzi: the kept cloud in id order; d_sorted: free for the index
    const uint32_t slots = uint32_t(ms.n_slots);
    ms.n = n_keep;
    if (n_keep == 0) return set_empty_index(c, ms);
    InsertInfo* h_info = c->h_map_info;
    *h_info = InsertInfo{};
    h_info->n_out = n_keep;
    SO_CUDA_TRY(cudaMemcpyAsync(&c->d_map_scratch->info, h_info, sizeof(InsertInfo), cudaMemcpyHostToDevice, st));
    rc = count_blocks(c, ms, n_keep, slots);
    return rc ? rc : index_cells(c, ms, n_keep, slots);
}

static int set_empty_index(Ctx* c, MapStore& ms) {
    cudaStream_t st = c->stream;
    SO_CUDA_TRY(cudaMemsetAsync(ms.d_block_count, 0, kNumBlocks * sizeof(int32_t), st));
    SO_CUDA_TRY(cudaMemsetAsync(ms.d_block_slot, 0xFF, kNumBlocks * sizeof(int32_t), st));
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    std::fill(ms.h_block_count.begin(), ms.h_block_count.end(), 0);
    std::fill(ms.h_block_slot.begin(), ms.h_block_slot.end(), -1);
    ms.n_slots = 0;
    ms.dirty = false;
    ms.index_gen++;
    return SO_OK;
}

// (Re)build the index of d_xyzi[0..n) under the current origin and resolution: count blocks and assign slots over the raw cloud,
// size the cell table, drop off-grid points (filter stage, nothing touched) when there are any, index.  With the block archive on,
// off-grid points move to the archive and archived blocks the grid covers come back instead (map_rebuild_archive).
int map_rebuild(Ctx* c, MapStore& ms) {
    cudaStream_t st = c->stream;
    ms.nb = map_cells_per_block(ms.res);
    ms.dirty = true;
    if (ms.arc.d_pool) return map_rebuild_archive(c, ms);
    if (ms.n == 0) return set_empty_index(c, ms);
    const uint32_t n = ms.n;
    InsertInfo* h_info = c->h_map_info;
    *h_info = InsertInfo{};
    h_info->n_out = n;
    SO_CUDA_TRY(cudaMemcpyAsync(&c->d_map_scratch->info, h_info, sizeof(InsertInfo), cudaMemcpyHostToDevice, st));
    int rc = count_blocks(c, ms, n, kNumBlocks);
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemcpyAsync(h_info, &c->d_map_scratch->info, sizeof(InsertInfo), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    const uint32_t n_slots = h_info->n_slots;
    rc = reserve_cells(c, ms, n_slots, n_slots / 4);
    if (rc) return rc;
    if (h_info->n_kept < n) { rc = filter_stage(c, ms, 0); if (rc) return rc; }
    return index_cells(c, ms, n, n_slots);
}

// LocalMap::addSurfPointCloud without a host round trip between its steps: the filter stage, then the index stage bounded to the
// current slots plus 4 new ones.  The host reads the sizes, block tables and the error flag back ONCE, at the end; when the new
// cloud opened more blocks, the table grows to the slot count read back and the index stage runs again (not the filter).
int map_add_points(Ctx* c, MapStore& ms, uint32_t n_new) {
    if (n_new == 0) return SO_OK;
    const uint32_t total = ms.n + n_new;                                // the caller rebuilt a dirty store BEFORE appending the new points
    ms.nb = map_cells_per_block(ms.res);
    const size_t cells_per_slot = size_t(ms.nb) * ms.nb * ms.nb;
    const uint32_t slot_cap = uint32_t(std::min<size_t>(size_t(ms.n_slots) + 4, (kMaxCells - 2) / cells_per_slot));
    int rc = reserve_cells(c, ms, slot_cap, 4);
    if (rc) return rc;
    ms.dirty = true;
    rc = filter_stage(c, ms, n_new);
    if (!rc) rc = count_blocks(c, ms, total, slot_cap);
    if (!rc) rc = index_cells(c, ms, total, slot_cap);
    if (rc || !ms.dirty) return rc;
    const uint32_t n_slots = uint32_t(ms.n_slots);                      // more new blocks than the table was sized for
    rc = reserve_cells(c, ms, n_slots, 4);
    if (!rc) rc = count_blocks(c, ms, total, n_slots);
    return rc ? rc : index_cells(c, ms, total, n_slots);
}

// ------------------------------------------------------------------------------------------------------------------
// Block archive (so_archive.h): with it on, the rebuild that applies an origin change moves every block the window drops to the
// archive, unchanged, and brings back every archived block the window now covers.  Per store: one float4 point pool holding one
// segment per block (its cloud in store order) and a host directory {world key -> segment} in key order.  Evicted segments are
// appended at the pool's tail; restored ones leave a hole, and the pool is compacted (stably, in pool order) only when an eviction
// does not fit behind the tail -- so a shift costs the blocks that move, not the size of the archive.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kEvictShift = 60;                   // eviction key: class above the 60-bit world key
static_assert(archive::kWinW == kW && archive::kWinH == kH && archive::kWinD == kD, "the archive's window is the block grid");
static_assert(3 * archive::kKeyBits <= kEvictShift, "world key fits below the class bits");

// Eviction key of every point of the store's cloud under the new origin: 0 in the window (kept in place by the stable sort);
// [1][world key] off the window (to the archive: grouped by block, cloud order inside each); [2] not finite or beyond the key
// range (dropped, as the filter stage drops them)
__global__ void k_evict_keys(const float4* __restrict__ raw, uint32_t n, int3 origin, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = raw[i];
    uint64_t key = 0;
    if (grid_block(p, origin) < 0) {
        const uint64_t w = archive::point_key(p.x, p.y, p.z);
        key = w == archive::kKeyNone ? uint64_t(2) << kEvictShift : (uint64_t(1) << kEvictShift) | w;
    }
    keys[i] = key;
    vals[i] = i;
}

// sorted positions [0, n_kept): the window's points, in order -> window; [n_kept, n_kept + n_evict): the evicted blocks -> pool tail
__global__ void k_evict_gather(const float4* __restrict__ raw, const uint32_t* __restrict__ vals, uint32_t n_kept, uint32_t n_evict,
                               float4* __restrict__ window, float4* __restrict__ pool_tail) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_kept) window[i] = raw[vals[i]];
    else if (i < n_kept + n_evict) pool_tail[i - n_kept] = raw[vals[i]];
}

// one CTA per block cloud: src[s.src .. +s.n) -> dst[s.dst .. +s.n)
__global__ void k_seg_gather(const float4* __restrict__ src, float4* __restrict__ dst, const GatherSeg* __restrict__ segs) {
    const GatherSeg s = segs[blockIdx.x];
    for (uint32_t j = threadIdx.x; j < s.n; j += blockDim.x) dst[s.dst + j] = src[s.src + j];
}

static int seg_gather(Ctx* c, BlockArchive& a, const std::vector<GatherSeg>& segs, const float4* src, float4* dst) {
    if (segs.empty()) return SO_OK;
    int rc = a.d_segs.reserve(segs.size());
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemcpyAsync(a.d_segs, segs.data(), segs.size() * sizeof(GatherSeg), cudaMemcpyHostToDevice, c->stream));
    k_seg_gather<<<unsigned(segs.size()), 256, 0, c->stream>>>(src, dst, a.d_segs);
    c->launches++;
    return SO_OK;
}

// Every live segment but those in `skip`, in pool order, packed from the front of dst.  The directory is not touched: the segments'
// new offsets go to *moved, for the caller to apply once everything it depends on has succeeded.  Returns the points packed.
using SegMoves = std::vector<std::pair<BlockArchive::Seg*, uint64_t>>;
static void apply_moves(const SegMoves& m) { for (const auto& x : m) x.first->off = x.second; }
static int repack(Ctx* c, BlockArchive& a, float4* dst, size_t* packed, SegMoves* moved, const std::set<const BlockArchive::Seg*>& skip = {}) {
    std::vector<BlockArchive::Seg*> order;
    order.reserve(a.dir.size());
    for (auto& kv : a.dir) if (!skip.count(&kv.second)) order.push_back(&kv.second);
    std::sort(order.begin(), order.end(), [](const BlockArchive::Seg* x, const BlockArchive::Seg* y) { return x->off < y->off; });
    std::vector<GatherSeg> segs;
    segs.reserve(order.size());
    uint64_t o = 0;
    for (const BlockArchive::Seg* s : order) { segs.push_back(GatherSeg{s->off, o, s->n, 0}); o += s->n; }
    int rc = seg_gather(c, a, segs, a.d_pool, dst);
    if (rc) return rc;
    moved->clear();
    for (size_t k = 0; k < order.size(); ++k) moved->emplace_back(order[k], segs[k].dst);
    *packed = size_t(o);
    return SO_OK;
}

// Both stores at once: every new pool is allocated before either store changes, so a failure leaves both as they were
int archive_set_cap(Ctx* c, size_t cap) {
    MapStore* stores[2] = {&c->surf, &c->edge};
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (cap == 0) {
        for (MapStore* ms : stores) ms->arc = BlockArchive{};
        return SO_OK;
    }
    for (MapStore* ms : stores)
        if (cap < ms->arc.live) { set_error("so_map_archive: capacity below the points the archive holds"); return SO_ERR_CAPACITY; }
    DeviceBuffer<float4> pool[2];
    for (int k = 0; k < 2; ++k) {
        if (cap == stores[k]->arc.d_pool.cap()) continue;
        if (pool[k].reserve(cap)) {
            cudaGetLastError();
            set_error("so_map_archive: cudaMalloc of the archive pool failed");
            return SO_ERR_CUDA;
        }
    }
    size_t packed[2] = {0, 0};
    SegMoves moved[2];
    int rc = SO_OK;
    for (int k = 0; k < 2 && !rc; ++k) if (pool[k]) rc = repack(c, stores[k]->arc, pool[k], &packed[k], &moved[k]);
    if (!rc && cudaStreamSynchronize(c->stream) != cudaSuccess) rc = SO_ERR_CUDA;
    if (rc) return rc;                                                   // both directories as they were
    for (int k = 0; k < 2; ++k) {
        if (!pool[k]) continue;
        BlockArchive& a = stores[k]->arc;
        apply_moves(moved[k]);
        a.d_pool = std::move(pool[k]);
        a.used = packed[k];
    }
    return SO_OK;
}

int archive_load(Ctx* c, MapStore& ms, const float4* pts, size_t n) {
    BlockArchive& a = ms.arc;
    std::vector<float4> win;
    std::vector<std::pair<uint64_t, uint32_t>> off;                  // (world key, index) of the points outside the window
    for (size_t i = 0; i < n; ++i) {
        const uint64_t key = archive::point_key(pts[i].x, pts[i].y, pts[i].z);
        if (key == archive::kKeyNone) continue;                         // not finite: dropped, as the rebuild drops it
        int w[3];
        archive::unpack_key(key, w);
        if (archive::in_window(w, c->origin)) win.push_back(pts[i]);
        else off.emplace_back(key, uint32_t(i));
    }
    if (win.size() > c->cfg.max_map_points) { set_error("map points inside the window exceed so_config.max_map_points"); return SO_ERR_CAPACITY; }
    if (off.size() > a.d_pool.cap()) { set_error("map points outside the window exceed the block archive (so_map_archive)"); return SO_ERR_CAPACITY; }
    std::stable_sort(off.begin(), off.end(), [](const auto& x, const auto& y) { return x.first < y.first; });
    std::vector<float4> arc(off.size());
    for (size_t i = 0; i < off.size(); ++i) arc[i] = pts[off[i].second];
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (!win.empty()) SO_CUDA_TRY(cudaMemcpy(ms.d_xyzi, win.data(), win.size() * sizeof(float4), cudaMemcpyHostToDevice));
    if (!arc.empty()) SO_CUDA_TRY(cudaMemcpy(a.d_pool, arc.data(), arc.size() * sizeof(float4), cudaMemcpyHostToDevice));
    a.dir.clear();
    for (size_t i = 0; i < off.size();) {
        size_t j = i;
        while (j < off.size() && off[j].first == off[i].first) ++j;
        a.dir[off[i].first] = BlockArchive::Seg{uint64_t(i), uint32_t(j - i)};
        i = j;
    }
    a.used = a.live = off.size();
    ms.n = uint32_t(win.size());
    ms.dirty = true;
    return SO_OK;
}

int archive_segments(Ctx* c, MapStore& ms, uint32_t* n_segs, uint32_t* max_n) {
    BlockArchive& a = ms.arc;
    std::vector<GatherSeg> segs;
    segs.reserve(a.dir.size());
    uint32_t m = 0;
    for (const auto& kv : a.dir) { segs.push_back(GatherSeg{kv.second.off, 0, kv.second.n, 0}); m = std::max(m, kv.second.n); }
    *n_segs = uint32_t(segs.size());
    *max_n = m;
    if (segs.empty()) return SO_OK;
    int rc = a.d_segs.reserve(segs.size());
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemcpyAsync(a.d_segs, segs.data(), segs.size() * sizeof(GatherSeg), cudaMemcpyHostToDevice, c->stream));
    return SO_OK;
}

int archive_download_all(Ctx* c, MapStore& ms, float* out, size_t cap, size_t* n_out) {
    const BlockArchive& a = ms.arc;
    std::vector<float4> win(ms.n), pool(a.used);
    if (ms.n) SO_CUDA_TRY(cudaMemcpy(win.data(), ms.d_xyzi, size_t(ms.n) * sizeof(float4), cudaMemcpyDeviceToHost));
    if (a.used) SO_CUDA_TRY(cudaMemcpy(pool.data(), a.d_pool, a.used * sizeof(float4), cudaMemcpyDeviceToHost));
    std::vector<std::pair<uint64_t, uint32_t>> wk(win.size());
    for (size_t i = 0; i < win.size(); ++i) wk[i] = {archive::point_key(win[i].x, win[i].y, win[i].z), uint32_t(i)};
    std::stable_sort(wk.begin(), wk.end(), [](const auto& x, const auto& y) { return x.first < y.first; });
    size_t k = 0, i = 0;
    auto put = [&](const float4& p) { if (out && k < cap) std::memcpy(out + 4 * k, &p, sizeof(float4)); ++k; };
    for (auto it = a.dir.begin(); it != a.dir.end() || i < wk.size();) {        // window and archive hold different blocks
        if (it == a.dir.end() || (i < wk.size() && wk[i].first < it->first)) { put(win[wk[i].second]); ++i; }
        else { for (uint32_t j = 0; j < it->second.n; ++j) put(pool[it->second.off + j]); ++it; }
    }
    *n_out = k;
    return SO_OK;
}

static int map_rebuild_archive(Ctx* c, MapStore& ms) {
    cudaStream_t st = c->stream;
    BlockArchive& a = ms.arc;
    InsertInfo* d_info = &c->d_map_scratch->info;
    InsertInfo* h_info = c->h_map_info;
    const int3 origin = make_int3(c->origin[0], c->origin[1], c->origin[2]);
    // blocks to restore: the directory's entries inside the window, one lookup per row of blocks
    std::vector<std::map<uint64_t, BlockArchive::Seg>::iterator> back;
    size_t n_back = 0;
    archive::window_rows(c->origin, [&](uint64_t lo, uint64_t hi) {
        for (auto it = a.dir.lower_bound(lo); it != a.dir.end() && it->first <= hi; ++it) { back.push_back(it); n_back += it->second.n; }
    });
    // points of the store that stay: block counts and slots of the cloud under the new origin (one read-back, as map_rebuild)
    const uint32_t n = ms.n;
    uint32_t n_kept = 0, n_slots = 0;
    if (n) {
        *h_info = InsertInfo{};
        h_info->n_out = n;
        SO_CUDA_TRY(cudaMemcpyAsync(d_info, h_info, sizeof(InsertInfo), cudaMemcpyHostToDevice, st));
        int rc = count_blocks(c, ms, n, kNumBlocks);
        if (rc) return rc;
        SO_CUDA_TRY(cudaMemcpyAsync(h_info, d_info, sizeof(InsertInfo), cudaMemcpyDeviceToHost, st));
        SO_CUDA_TRY(cudaGetLastError());
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        n_kept = h_info->n_kept; n_slots = h_info->n_slots;
    }
    // points that leave: sorted by (class, world key), stable, and the runs of that order (one per block, one for the dropped)
    std::vector<uint64_t> run_key;
    std::vector<uint32_t> run_n;
    size_t n_evict = 0;
    if (n_kept < n) {
        const uint32_t m = n - n_kept;
        uint32_t* d_runs = &c->d_map_scratch->runs;
        size_t need = 0;
        cub::DeviceRunLengthEncode::Encode(nullptr, need, c->d_keys_out.get(), c->d_keys.get(), c->d_vals.get(), d_runs, int(m));
        int rc = c->d_cub_tmp.reserve(need + 256);
        if (rc) return rc;
        k_evict_keys<<<(n + 255) / 256, 256, 0, st>>>(ms.d_xyzi, n, origin, c->d_keys, c->d_vals);
        size_t tmp = c->d_cub_tmp.cap();
        SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_cub_tmp, tmp, c->d_keys.get(), c->d_keys_out.get(), c->d_vals.get(), c->d_vals_out.get(), int(n), 0,
                                                    kEvictShift + 2, st));
        tmp = c->d_cub_tmp.cap();           // run keys and counts into the sort's inputs, free now
        SO_CUDA_TRY(cub::DeviceRunLengthEncode::Encode(c->d_cub_tmp, tmp, c->d_keys_out.get() + n_kept, c->d_keys.get(), c->d_vals.get(), d_runs, int(m), st));
        uint32_t runs = 0;
        SO_CUDA_TRY(cudaMemcpyAsync(&h_info->pad, d_runs, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        SO_CUDA_TRY(cudaGetLastError());
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        runs = h_info->pad;
        run_key.resize(runs); run_n.resize(runs);
        SO_CUDA_TRY(cudaMemcpyAsync(run_key.data(), c->d_keys, runs * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        SO_CUDA_TRY(cudaMemcpyAsync(run_n.data(), c->d_vals, runs * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        c->launches += 1 + 5 + 3;
        for (uint32_t r = 0; r < runs; ++r) if ((run_key[r] >> kEvictShift) == 1) n_evict += run_n[r];
    }
    // every check before the first change: the store stays as it was (and unbuilt) when one fails
    if (size_t(n_kept) + n_back > c->cfg.max_map_points) {
        set_error("restoring archived blocks would exceed so_config.max_map_points");
        return SO_ERR_CAPACITY;
    }
    if (a.live - n_back + n_evict > a.d_pool.cap()) { set_error("block archive full: grow it with so_map_archive"); return SO_ERR_CAPACITY; }
    n_slots += uint32_t(back.size());                                   // restored blocks are not in the window's cloud
    if (n_kept + n_back) { int rc = reserve_cells(c, ms, n_slots, n_slots / 4); if (rc) return rc; }
    const bool compact = a.used + n_evict > a.d_pool.cap();
    DeviceBuffer<float4> scratch;
    if (compact) { int rc = scratch.reserve(std::max<size_t>(a.live - n_back, 1)); if (rc) return rc; }
    // restore: the blocks' clouds behind the window's points, then out of the directory
    float4* dst = n_kept < n ? ms.d_sorted : ms.d_xyzi;
    std::vector<GatherSeg> segs;
    uint64_t at = n_kept;
    for (const auto& it : back) { segs.push_back(GatherSeg{it->second.off, at, it->second.n, 0}); at += it->second.n; }
    int rc = seg_gather(c, a, segs, a.d_pool, dst);
    size_t packed = 0;
    SegMoves moved;
    if (!rc && compact) {                                               // the other segments, stably, through the scratch
        std::set<const BlockArchive::Seg*> skip;
        for (const auto& it : back) skip.insert(&it->second);
        rc = repack(c, a, scratch, &packed, &moved, skip);
        if (!rc && packed && cudaMemcpyAsync(a.d_pool, scratch, packed * sizeof(float4), cudaMemcpyDeviceToDevice, st) != cudaSuccess) rc = SO_ERR_CUDA;
        if (!rc && cudaStreamSynchronize(st) != cudaSuccess) rc = SO_ERR_CUDA;
    }
    scratch.reset();
    if (rc) return rc;            // the directory and the store still describe what they held: nothing restored, nothing lost
    if (compact) { apply_moves(moved); a.used = packed; }
    for (const auto& it : back) a.dir.erase(it);
    a.live -= n_back;
    // evict: the window's points to the front of dst, the leaving blocks behind the pool's tail
    if (n_kept < n) {
        const uint32_t total = n_kept + uint32_t(n_evict);
        if (total) k_evict_gather<<<(total + 255) / 256, 256, 0, st>>>(ms.d_xyzi, c->d_vals_out, n_kept, uint32_t(n_evict), ms.d_sorted, a.d_pool + a.used);
        c->launches++;
        for (size_t r = 0; r < run_key.size(); ++r) {
            if ((run_key[r] >> kEvictShift) != 1) continue;
            a.dir[run_key[r] & ((uint64_t(1) << kEvictShift) - 1)] = BlockArchive::Seg{uint64_t(a.used), run_n[r]};
            a.used += run_n[r];
        }
        a.live += n_evict;
        std::swap(ms.d_xyzi, ms.d_sorted);
    }
    ms.n = n_kept + uint32_t(n_back);
    if (ms.n == 0) return set_empty_index(c, ms);
    *h_info = InsertInfo{};
    h_info->n_out = ms.n;
    SO_CUDA_TRY(cudaMemcpyAsync(d_info, h_info, sizeof(InsertInfo), cudaMemcpyHostToDevice, st));
    rc = count_blocks(c, ms, ms.n, n_slots);
    return rc ? rc : index_cells(c, ms, ms.n, n_slots);
}

// ------------------------------------------------------------------------------------------------------------------
// Scan pre-filter: the pcl::VoxelGrid(planeRes) that laserMapping::adjustVoxelSize applies to the sensor-frame surf
// cloud before Localization (laserMapping.cpp:639-645), and the corner filter of the edge extraction.  One grid for the
// whole cloud, indexed as VoxelGrid<PointT>::applyFilter (PCL 1.12, filters/impl/voxel_grid.hpp) indexes it: relative to
// the bounding box of the finite points, and the cloud returned verbatim when dx * dy * dz would overflow an int32.
// In: in[0..n); out: out[0..*n_out) ordered by PCL's voxel index.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kCloudKeyBits = 33;                     // uint32 voxel index, non-finite points at bit 32: five 8-bit radix passes

// Bounding box of the finite points (getMinMax3D of a cloud that is not dense): k_map_bounds' reduction with the non-finite points
// left out, the maximum stored as ~max (one atomicMin and one 0xFF fill serve both), and the warps of a CTA combined in shared
// memory first: a few CTAs, 6 atomics each, instead of 6 same-address atomics per warp of the cloud.
constexpr uint32_t kBoundsCtas = 256;
__global__ void __launch_bounds__(256) k_cloud_bounds(const float4* __restrict__ pts, uint32_t n, uint32_t* __restrict__ b) {
    __shared__ uint32_t s[8][6];
    uint32_t v6[6] = {~0u, ~0u, ~0u, ~0u, ~0u, ~0u};                   // min x, y, z; ~max x, y, z
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 p = pts[i];
        if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) continue;
        const uint32_t v[3] = {float_order(p.x), float_order(p.y), float_order(p.z)};
        for (int a = 0; a < 3; ++a) { v6[a] = min(v6[a], v[a]); v6[3 + a] = min(v6[3 + a], ~v[a]); }
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int a = 0; a < 6; ++a) v6[a] = __reduce_min_sync(0xffffffffu, v6[a]);
    if (lane == 0)
        for (int a = 0; a < 6; ++a) s[w][a] = v6[a];
    __syncthreads();
    if (threadIdx.x < 6) {
        uint32_t m = ~0u;
        for (int k = 0; k < 8; ++k) m = min(m, s[k][threadIdx.x]);
        atomicMin(b + threadIdx.x, m);
    }
}

// PCL's voxel index of every point: ijk = int(floor(p * inv) - float(min_b)) per axis, idx = ijk0 + ijk1 div0 + ijk2 div0 div1 in
// 32-bit arithmetic (PCL's int products, mod 2^32).  Non-finite points get bit 32 and sort last.  Every thread derives the grid
// from the bounds; thread 0 stores PCL's overflow test, dx dy dz > INT32_MAX with dx = int64((max - min) * inv) + 1, decided
// exactly in double (inside the contract dx dy < 2^44 is exact, and the rounding of the last product is monotone, so it cannot
// cross INT32_MAX); the float -> int conversions saturate outside the contract.
__global__ void k_voxel_keys_cloud(const float4* __restrict__ raw, uint32_t n, float inv_leaf, const uint32_t* __restrict__ bounds,
                                   uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ fallback) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float lo[3];
    uint32_t min_b[3], div[3];
    double cells = 1.0;
    for (int a = 0; a < 3; ++a) {
        lo[a] = float_unorder(bounds[a]);
        const float hi = float_unorder(~bounds[3 + a]);
        cells *= double(int64_t(__fmul_rn(__fsub_rn(hi, lo[a]), inv_leaf)) + 1);
        min_b[a] = uint32_t(int(floorf(__fmul_rn(lo[a], inv_leaf))));
        div[a] = uint32_t(int(floorf(__fmul_rn(hi, inv_leaf)))) - min_b[a] + 1u;
    }
    if (i == 0) *fallback = bounds[0] != ~0u && cells > 2147483647.0;        // no finite point: no fall-back, nothing out
    const float4 p = raw[i];
    uint64_t key = uint64_t(1) << 32;                                // non-finite points are skipped, as PCL does
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
        const float v[3] = {p.x, p.y, p.z};
        uint32_t ijk[3];
        for (int a = 0; a < 3; ++a) ijk[a] = uint32_t(int(__fsub_rn(floorf(__fmul_rn(v[a], inv_leaf)), float(int(min_b[a])))));
        key = ijk[0] + ijk[1] * div[0] + ijk[2] * (div[0] * div[1]);
    }
    keys[i] = key;
    vals[i] = i;
}

int cloud_voxel_filter(Ctx* c, const float4* in, uint32_t n, float leaf, const VoxelBufs& b, float4* out, uint32_t* n_out) {
    cudaStream_t st = c->stream;
    *n_out = 0;
    if (n == 0) return SO_OK;
    const uint32_t grid = (n + 255) / 256;
    const float inv_leaf = 1.0f / leaf;
    InsertInfo* d_info = &c->d_map_scratch->info;
    InsertInfo* h_info = c->h_map_info;
    uint32_t* d_bounds = c->d_map_scratch->bounds;
    SO_CUDA_TRY(cudaMemsetAsync(d_bounds, 0xFF, 6 * sizeof(uint32_t), st));
    k_cloud_bounds<<<std::min(grid, kBoundsCtas), 256, 0, st>>>(in, n, d_bounds);
    k_voxel_keys_cloud<<<grid, 256, 0, st>>>(in, n, inv_leaf, d_bounds, b.keys, b.vals, &d_info->fallback);
    size_t tmp = b.tmp_bytes;
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(b.tmp, tmp, b.keys, b.keys_out, b.vals, b.vals_out, int(n), 0, kCloudKeyBits, st));
    c->launches += 8;
    const int rc = voxel_reduce(c, in, b.keys_out, b.vals_out, n, 0, uint64_t(1) << 32,
                                reinterpret_cast<uint32_t*>(b.keys), b.tmp, b.tmp_bytes, out);   // keys_in is free after the sort
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemcpyAsync(h_info, d_info, sizeof(InsertInfo), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    if (h_info->fallback) {                                         // PCL: "Integer indices would overflow", output = input
        SO_CUDA_TRY(cudaMemcpyAsync(out, in, size_t(n) * sizeof(float4), cudaMemcpyDeviceToDevice, st));
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        *n_out = n;
        return SO_OK;
    }
    *n_out = h_info->n_out;
    return SO_OK;
}

int scan_voxel_filter(Ctx* c, uint32_t n, float leaf, uint32_t* n_out) {
    const VoxelBufs b{c->d_skeys, c->d_skeys_out, c->d_svals, c->d_svals_out, c->d_sort_tmp, c->d_sort_tmp.cap()};
    return cloud_voxel_filter(c, c->d_scan, n, leaf, b, c->d_scan_sorted, n_out);
}


// ------------------------------------------------------------------------------------------------------------------
// Map from keyframes (so_map_from_keyframes): ONE voxel filter over the union of the selected keyframes, each at its pose -- not a
// replay of inserts.  Every block of the union is filtered on its own at the store's leaf, as the insert filters a touched block, with
// the centroids summed in union order.  A thread per union point finds its keyframe in the segment table, transforms the point with
// k_transform_points' arithmetic (pose_point) and bins it by world block; the sort key is [drop][block][vk][vj][vi], with the block
// numbered in the box of the kept world blocks (z, y, x: world key order) and the voxel as the insert numbers it (block_voxel).  One
// stable sort then orders the union by world block, by voxel, and by union order inside a voxel; voxel_reduce averages it.
// Kept: the window's blocks, and with the archive on every block in the key range.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool kf_block(const float4 p, int3 origin, int archive, int w[3]) {
    if (!archive::world_axis(p.x, &w[0]) || !archive::world_axis(p.y, &w[1]) || !archive::world_axis(p.z, &w[2])) return false;
    if (archive) return true;
    const int gx = w[0] + origin.x, gy = w[1] + origin.y, gz = w[2] + origin.z;
    return gx >= 0 && gx < kW && gy >= 0 && gy < kH && gz >= 0 && gz < kD;
}

// union point i -> raw[i] in the world frame; ctl[0..3) = min, ctl[3..6) = max world block of the kept points (warp-reduced atomics)
__global__ void __launch_bounds__(256) k_kf_transform(const float4* __restrict__ pool, const KfSeg* __restrict__ segs, uint32_t n_segs,
                                                      uint32_t total, int3 origin, int archive, float4* __restrict__ raw, int32_t* __restrict__ ctl) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    int w[3] = {0, 0, 0};
    bool kept = false;
    if (i < total) {
        uint32_t lo = 0, hi = n_segs;                                  // the last segment starting at or before i: the one holding it
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (segs[mid].start <= i) lo = mid; else hi = mid; }
        const KfSeg& s = segs[lo];
        const float4 p = pose_point(s.pose, pool[s.src + (i - s.start)]);
        raw[i] = p;
        kept = kf_block(p, origin, archive, w);
    }
    for (int a = 0; a < 3; ++a) {                                      // every lane takes part: no early return above
        const int mn = __reduce_min_sync(0xffffffffu, kept ? w[a] : INT_MAX);
        const int mx = __reduce_max_sync(0xffffffffu, kept ? w[a] : INT_MIN);
        if ((threadIdx.x & 31) == 0 && mn <= mx) { atomicMin(ctl + a, mn); atomicMax(ctl + 3 + a, mx); }
    }
}

struct KfBox { int32_t lo[3]; uint32_t nx, ny; int32_t kb; };          // first block per axis, blocks along x and y; key bits below the drop bit

__global__ void k_kf_keys(const float4* __restrict__ raw, uint32_t total, int3 origin, int archive, KfBox box, float inv_leaf, int vb,
                          uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const float4 p = raw[i];
    int w[3];
    uint64_t key = uint64_t(1) << box.kb;                              // dropped
    if (kf_block(p, origin, archive, w)) {
        const uint64_t b = (uint64_t(w[2] - box.lo[2]) * box.ny + uint64_t(w[1] - box.lo[1])) * box.nx + uint64_t(w[0] - box.lo[0]);
        key = (b << (3 * vb)) | block_voxel(p, w[0], w[1], w[2], inv_leaf, vb);
    }
    keys[i] = key;
    vals[i] = i;
}

// blk[rank[i]] = the block of the voxel starting at sorted position i (voxel_reduce's heads and ranks)
__global__ void k_kf_voxel_blocks(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ head, const uint32_t* __restrict__ rank, uint32_t total,
                                  int shift, uint32_t* __restrict__ blk) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total && head[i]) blk[rank[i]] = uint32_t(keys[i] >> shift);
}

int keyframe_map_filter(Ctx* c, MapStore& ms, int store, const KfSeg* segs, uint32_t n_segs, uint32_t total, const float4* pool, KfBuild* b) {
    cudaStream_t st = c->stream;
    KeyframeScratch& k = c->kfs;
    *b = KfBuild{};
    if (total == 0) return SO_OK;
    const int archive_on = ms.arc.d_pool ? 1 : 0;
    const int3 origin = make_int3(c->origin[0], c->origin[1], c->origin[2]);
    int rc = k.d_segs.reserve(n_segs);
    if (!rc) rc = k.d_raw.reserve(total);
    if (!rc) rc = k.d_keys.reserve(total);
    if (!rc) rc = k.d_keys_out.reserve(total);
    if (!rc) rc = k.d_vals.reserve(total);
    if (!rc) rc = k.d_vals_out.reserve(total);
    if (!rc) rc = k.d_out[store].reserve(total);
    if (!rc) rc = k.d_blk.reserve(total);
    if (!rc) rc = k.d_ctl.reserve(8);
    if (!rc) rc = k.h_ctl.reserve(8);
    if (rc) return rc;
    {
        size_t a = 0, s2 = 0, r = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, a, k.d_keys.get(), k.d_keys_out.get(), k.d_vals.get(), k.d_vals_out.get(), int(total), 0, 64);
        cub::DeviceScan::ExclusiveSum(nullptr, s2, k.d_vals.get(), k.d_vals.get(), int(total));
        cub::DeviceRunLengthEncode::Encode(nullptr, r, k.d_blk.get(), k.d_vals.get(), k.d_vals_out.get(), k.d_ctl.get(), int(total));
        rc = k.d_tmp.reserve(std::max({a, s2, r}) + 256);
        if (rc) return rc;
    }
    // the box of the kept world blocks (one read-back)
    const int32_t init[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
    std::memcpy(k.h_ctl, init, sizeof(init));
    SO_CUDA_TRY(cudaMemcpyAsync(k.d_ctl, k.h_ctl, 6 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    SO_CUDA_TRY(cudaMemcpyAsync(k.d_segs, segs, n_segs * sizeof(KfSeg), cudaMemcpyHostToDevice, st));
    const uint32_t grid = (total + 255) / 256;
    k_kf_transform<<<grid, 256, 0, st>>>(pool, k.d_segs, n_segs, total, origin, archive_on, k.d_raw, k.d_ctl);
    SO_CUDA_TRY(cudaMemcpyAsync(k.h_ctl, k.d_ctl, 6 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    c->launches++;
    int32_t lo[3], hi[3];
    for (int a = 0; a < 3; ++a) { lo[a] = k.h_ctl[a]; hi[a] = k.h_ctl[3 + a]; }
    if (lo[0] > hi[0]) return SO_OK;                                   // no point is kept: the store becomes empty
    const float inv_leaf = 1.0f / ms.res;                              // Eigen::Array4f::Ones() / leaf_size_
    const int vb = voxel_bits(inv_leaf);
    const uint64_t nx = uint64_t(hi[0] - lo[0]) + 1, ny = uint64_t(hi[1] - lo[1]) + 1, nz = uint64_t(hi[2] - lo[2]) + 1;
    int bb = 0;
    while ((uint64_t(1) << bb) < nx * ny * nz) ++bb;
    if (bb > 32 || 3 * vb + bb > 63) {
        set_error("so_map_from_keyframes: the keyframes span too many 50 m blocks for the sort key at this leaf");
        return SO_ERR_CAPACITY;
    }
    const KfBox box{{lo[0], lo[1], lo[2]}, uint32_t(nx), uint32_t(ny), 3 * vb + bb};
    k_kf_keys<<<grid, 256, 0, st>>>(k.d_raw, total, origin, archive_on, box, inv_leaf, vb, k.d_keys, k.d_vals);
    size_t tmp = k.d_tmp.cap();
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(k.d_tmp, tmp, k.d_keys.get(), k.d_keys_out.get(), k.d_vals.get(), k.d_vals_out.get(), int(total), 0, box.kb + 1, st));
    c->launches += 6;
    uint32_t* head = reinterpret_cast<uint32_t*>(k.d_keys.get());           // keys_in is free after the sort: 2 * total words
    rc = voxel_reduce(c, k.d_raw, k.d_keys_out, k.d_vals_out, total, 0, uint64_t(1) << box.kb, head, k.d_tmp, k.d_tmp.cap(), k.d_out[store]);
    if (rc) return rc;
    k_kf_voxel_blocks<<<grid, 256, 0, st>>>(k.d_keys_out, head, head + total, total, 3 * vb, k.d_blk);
    InsertInfo* h_info = c->h_map_info;
    SO_CUDA_TRY(cudaMemcpyAsync(h_info, &c->d_map_scratch->info, sizeof(InsertInfo), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    const uint32_t n_out = h_info->n_out;
    // the runs of blocks in the filtered cloud: the block directory, the only thing the host reads
    uint32_t* run_blk = k.d_vals;                                      // free after the reduction
    uint32_t* run_n = k.d_vals_out;
    tmp = k.d_tmp.cap();
    SO_CUDA_TRY(cub::DeviceRunLengthEncode::Encode(k.d_tmp, tmp, k.d_blk.get(), run_blk, run_n, k.d_ctl.get() + 6, int(n_out), st));
    SO_CUDA_TRY(cudaMemcpyAsync(k.h_ctl + 6, k.d_ctl + 6, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    const uint32_t runs = uint32_t(k.h_ctl[6]);
    std::vector<uint32_t> hb(runs), hn(runs);
    SO_CUDA_TRY(cudaMemcpyAsync(hb.data(), run_blk, runs * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaMemcpyAsync(hn.data(), run_n, runs * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    c->launches += 3 + 5;
    uint64_t at = 0, n_win = 0;
    for (uint32_t r = 0; r < runs; ++r) {
        const int w[3] = {int(hb[r] % nx) + lo[0], int(hb[r] / nx % ny) + lo[1], int(hb[r] / (nx * ny)) + lo[2]};   // nx * ny may be 2^32
        if (archive::in_window(w, c->origin)) { b->win.push_back(GatherSeg{at, n_win, hn[r], 0}); n_win += hn[r]; }
        else { b->arc.emplace_back(archive::world_key(w[0], w[1], w[2]), GatherSeg{at, b->n_arc, hn[r], 0}); b->n_arc += hn[r]; }
        at += hn[r];
    }
    b->n_win = uint32_t(n_win);
    b->n_win_blocks = uint32_t(b->win.size());
    // every check before the first change
    if (n_win > c->cfg.max_map_points) { set_error("so_map_from_keyframes: the window's points exceed so_config.max_map_points"); return SO_ERR_CAPACITY; }
    if (b->n_arc > ms.arc.d_pool.cap()) { set_error("so_map_from_keyframes: the blocks outside the window exceed the block archive (so_map_archive)"); return SO_ERR_CAPACITY; }
    const size_t cells_per_slot = size_t(map_cells_per_block(ms.res));
    if (b->n_win_blocks > (kMaxCells - 2) / (cells_per_slot * cells_per_slot * cells_per_slot)) {
        set_error("map spans too many 50 m blocks for the dense cell table (n_slots * nb^3 >= 2^31)");
        return SO_ERR_CAPACITY;
    }
    return SO_OK;
}

int keyframe_map_commit(Ctx* c, MapStore& ms, int store, const KfBuild& b) {
    BlockArchive& a = ms.arc;
    const float4* out = c->kfs.d_out[store];
    int rc = seg_gather(c, a, b.win, out, ms.d_xyzi);
    if (rc) return rc;
    if (a.d_pool) {
        std::vector<GatherSeg> segs;
        segs.reserve(b.arc.size());
        for (const auto& kv : b.arc) segs.push_back(kv.second);
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));                 // the window's gather list has left the segment buffer
        rc = seg_gather(c, a, segs, out, a.d_pool);
        if (rc) return rc;
        a.dir.clear();
        for (const auto& kv : b.arc) a.dir[kv.first] = BlockArchive::Seg{kv.second.dst, kv.second.n};
        a.used = a.live = b.n_arc;
    }
    ms.n = b.n_win;
    return map_rebuild(c, ms);                                         // index stage; nothing is left to evict or restore
}

}  // namespace so

// so_map.cu -- device-resident LocalMap: block binning + sorted spatial hash grid (SURVEY 2.3: K1).
//
// Replaces the per-block nanoflann::Octree build (flann/octree.h:355-400,536-738, called from LocalMap.h:580,638):
// points are keyed by (block slot, cell inside the block), radix-sorted, and a dense per-slot cell-start table is
// built by histogram + exclusive scan.  Cells have edge cs = 50/nb >= sqrt(3*planeRes): every neighbour that can
// pass the NEIGHBORS_TOO_FAR gate lies in the 27 cells around the query's cell, and because nb divides the 50 m
// block exactly, "same block" (LocalMap.h:488-507) is "same slot".
#include <algorithm>
#include <cmath>

#include <cub/cub.cuh>

#include "so_ctx.cuh"

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

__device__ __forceinline__ int block_coord(double v, int origin) {   // LocalMap.h:594-605
    int c = int(v / kBlock);
    if (v < 0) c--;
    return c + origin;
}

__global__ void k_block_of(const float4* __restrict__ raw, uint32_t n, int3 origin, int32_t* __restrict__ block_of_point,
                           int32_t* __restrict__ block_count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = raw[i];
    const int gx = block_coord(double(p.x) + kHalfBlock, origin.x);
    const int gy = block_coord(double(p.y) + kHalfBlock, origin.y);
    const int gz = block_coord(double(p.z) + kHalfBlock, origin.z);
    int lin = -1;
    if (gx >= 0 && gx < kW && gy >= 0 && gy < kH && gz >= 0 && gz < kD && isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
        lin = gx + kW * gy + kW * kH * gz;
        atomicAdd(&block_count[lin], 1);
    }
    block_of_point[i] = lin;
}

__global__ void k_flags(const int32_t* __restrict__ block_of_point, uint32_t n, uint8_t* __restrict__ flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flags[i] = block_of_point[i] >= 0;
}

__global__ void k_keys(const float4* __restrict__ raw, uint32_t n, int3 origin, const int32_t* __restrict__ block_slot,
                       int nb, double inv_cs, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                       uint32_t* __restrict__ cell_count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = raw[i];
    const float q[3] = {p.x, p.y, p.z};
    const int o[3] = {origin.x, origin.y, origin.z};
    int g[3], c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double v = double(q[a]) + kHalfBlock;
        int b = int(v / kBlock);
        if (v < 0) b--;
        g[a] = b + o[a];
        int cc = int((v - kBlock * double(b)) * inv_cs);
        c[a] = cc < 0 ? 0 : (cc > nb - 1 ? nb - 1 : cc);
    }
    const int lin = g[0] + kW * g[1] + kW * kH * g[2];
    const uint64_t slot = uint64_t(block_slot[lin]);
    const uint64_t key = slot * uint64_t(nb) * uint64_t(nb) * uint64_t(nb) + uint64_t((c[2] * nb + c[1]) * nb + c[0]);
    keys[i] = key;
    vals[i] = i;
    atomicAdd(&cell_count[key], 1u);
}

__global__ void k_gather(const float4* __restrict__ raw, const uint32_t* __restrict__ vals, uint32_t n, float4* __restrict__ sorted) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t id = vals[i];
    const float4 p = raw[id];
    sorted[i] = make_float4(p.x, p.y, p.z, __uint_as_float(id));
}

static int store_alloc(Ctx* c, MapStore& ms) {
    const size_t M = c->cfg.max_map_points;
    SO_CUDA_TRY(cudaMalloc(&ms.d_xyzi, M * sizeof(float4)));
    SO_CUDA_TRY(cudaMalloc(&ms.d_sorted, M * sizeof(float4)));
    SO_CUDA_TRY(cudaMalloc(&ms.d_block_slot, kNumBlocks * sizeof(int32_t)));
    SO_CUDA_TRY(cudaMalloc(&ms.d_block_count, kNumBlocks * sizeof(int32_t)));
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
    SO_CUDA_TRY(cudaMalloc(&c->d_keys, M * sizeof(uint64_t)));
    SO_CUDA_TRY(cudaMalloc(&c->d_keys_out, M * sizeof(uint64_t)));
    SO_CUDA_TRY(cudaMalloc(&c->d_vals, M * sizeof(uint32_t)));
    SO_CUDA_TRY(cudaMalloc(&c->d_vals_out, M * sizeof(uint32_t)));
    SO_CUDA_TRY(cudaMalloc(&c->d_block_of_point, M * sizeof(int32_t)));
    // cub temp: the larger of sort / scan / select requirements at full capacity
    size_t a = 0, b = 0, d = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, c->d_keys, c->d_keys_out, c->d_vals, c->d_vals_out, int(M), 0, 64);
    cub::DeviceSelect::Flagged(nullptr, d, c->surf.d_xyzi, (uint8_t*)nullptr, c->surf.d_sorted, (uint32_t*)nullptr, int(M));
    const size_t max_cells = size_t(64) * 128 * 128 * 128 + 1;     // scan temp is tiny; size for a generous table
    cub::DeviceScan::ExclusiveSum(nullptr, b, (uint32_t*)nullptr, (uint32_t*)nullptr, int(std::min<size_t>(max_cells, size_t(1) << 30)));
    c->cub_tmp_bytes = std::max(a, std::max(b, d)) + 256;
    SO_CUDA_TRY(cudaMalloc(&c->d_cub_tmp, c->cub_tmp_bytes));
    SO_CUDA_TRY(cudaMalloc(&c->d_insert_info, 8192));
    SO_CUDA_TRY(cudaMallocHost(&c->h_insert_info, 256));
    return SO_OK;
}

void map_free(Ctx* c) {
    for (MapStore* ms : {&c->surf, &c->edge}) {
        cudaFree(ms->d_xyzi); cudaFree(ms->d_sorted); cudaFree(ms->d_block_slot); cudaFree(ms->d_block_count); cudaFree(ms->d_cell_start);
    }
    cudaFree(c->d_keys); cudaFree(c->d_keys_out); cudaFree(c->d_vals); cudaFree(c->d_vals_out); cudaFree(c->d_block_of_point); cudaFree(c->d_cub_tmp);
    cudaFree(c->d_insert_info);
    if (c->h_insert_info) cudaFreeHost(c->h_insert_info);
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
    return m;
}

// (Re)build the index from d_map_xyzi[0..map_n): bin to blocks under the current origin, drop off-grid points
// (what LocalMap::shiftMap does to blocks rolled off the grid, LocalMap.h:169-287), sort, build the cell table.
int map_rebuild(Ctx* c, MapStore& ms) {
    cudaStream_t st = c->stream;
    ms.nb = map_cells_per_block(ms.res);
    c->map_epoch++;
    ms.dirty = false;
    const int3 origin = make_int3(c->origin[0], c->origin[1], c->origin[2]);
    SO_CUDA_TRY(cudaMemsetAsync(ms.d_block_count, 0, kNumBlocks * sizeof(int32_t), st));
    std::fill(ms.h_block_count.begin(), ms.h_block_count.end(), 0);
    std::fill(ms.h_block_slot.begin(), ms.h_block_slot.end(), -1);
    ms.n_slots = 0;
    if (ms.n == 0) {
        SO_CUDA_TRY(cudaMemsetAsync(ms.d_block_slot, 0xFF, kNumBlocks * sizeof(int32_t), st));
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        return SO_OK;
    }
    const uint32_t n = ms.n;
    const uint32_t grid = (n + 255) / 256;
    k_block_of<<<grid, 256, 0, st>>>(ms.d_xyzi, n, origin, c->d_block_of_point, ms.d_block_count);
    c->launches++;
    SO_CUDA_TRY(cudaMemcpyAsync(ms.h_block_count.data(), ms.d_block_count, kNumBlocks * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    uint64_t kept = 0;
    for (int b = 0; b < kNumBlocks; ++b) if (ms.h_block_count[b] > 0) { ms.h_block_slot[b] = ms.n_slots++; kept += uint64_t(ms.h_block_count[b]); }
    SO_CUDA_TRY(cudaMemcpyAsync(ms.d_block_slot, ms.h_block_slot.data(), kNumBlocks * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (kept < n) {
        // compact away the points whose block rolled off the grid, preserving order (ids are ranks in this order)
        uint8_t* flags = reinterpret_cast<uint8_t*>(c->d_vals_out);
        uint32_t* d_num = reinterpret_cast<uint32_t*>(c->d_keys_out);
        k_flags<<<grid, 256, 0, st>>>(c->d_block_of_point, n, flags);
        size_t tmp = c->cub_tmp_bytes;
        SO_CUDA_TRY(cub::DeviceSelect::Flagged(c->d_cub_tmp, tmp, ms.d_xyzi, flags, ms.d_sorted, d_num, int(n), st));
        SO_CUDA_TRY(cudaMemcpyAsync(ms.d_xyzi, ms.d_sorted, kept * sizeof(float4), cudaMemcpyDeviceToDevice, st));
        c->launches += 3;
        ms.n = uint32_t(kept);
    }
    if (kept == 0) { SO_CUDA_TRY(cudaStreamSynchronize(st)); return SO_OK; }
    const uint32_t m = ms.n;
    const size_t cells = size_t(ms.n_slots) * ms.nb * ms.nb * ms.nb;
    if (cells + 1 >= (size_t(1) << 31)) {          // cell indices are 32-bit in the kernels and the scan length is an int
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        set_error("map spans too many 50 m blocks for the dense cell table (n_slots * nb^3 >= 2^31)");
        return SO_ERR_CAPACITY;
    }
    if (cells + 1 > ms.cell_cap) {
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        int rc = grow_buffer(ms.d_cell_start, ms.cell_cap, cells + 1 + cells / 4);
        if (rc) return rc;
        size_t need = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, need, ms.d_cell_start, ms.d_cell_start, int(ms.cell_cap));
        rc = grow_buffer(c->d_cub_tmp, c->cub_tmp_bytes, need + 256);
        if (rc) return rc;
    }
    SO_CUDA_TRY(cudaMemsetAsync(ms.d_cell_start, 0, (cells + 1) * sizeof(uint32_t), st));
    const uint32_t g2 = (m + 255) / 256;
    k_keys<<<g2, 256, 0, st>>>(ms.d_xyzi, m, origin, ms.d_block_slot, ms.nb, double(ms.nb) / kBlock, c->d_keys, c->d_vals, ms.d_cell_start);
    int bits = 1;
    while ((uint64_t(1) << bits) < uint64_t(cells)) ++bits;
    size_t tmp = c->cub_tmp_bytes;
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_cub_tmp, tmp, c->d_keys, c->d_keys_out, c->d_vals, c->d_vals_out, int(m), 0, bits, st));
    k_gather<<<g2, 256, 0, st>>>(ms.d_xyzi, c->d_vals_out, m, ms.d_sorted);
    tmp = c->cub_tmp_bytes;
    SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->d_cub_tmp, tmp, ms.d_cell_start, ms.d_cell_start, int(cells + 1), st));
    c->launches += 8;
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    return SO_OK;
}

int scan_sort_alloc(Ctx* c) {
    size_t need = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, need, c->d_skeys, c->d_skeys_out, c->d_svals, c->d_svals_out, int(c->scan_cap), 0, 64);
    c->sort_tmp_bytes = need + 256;
    SO_CUDA_TRY(cudaMalloc(&c->d_sort_tmp, c->sort_tmp_bytes));
    SO_CUDA_TRY(cudaMalloc(&c->d_sort_tmp2, c->sort_tmp_bytes));
    return SO_OK;
}

int query_sort_reserve(Ctx* c, size_t n) {
    int rc = grow_buffer(c->d_qkeys, c->qkeys_cap, n);
    if (!rc) rc = grow_buffer(c->d_qkeys_out, c->qkeys_out_cap, n);
    if (!rc) rc = grow_buffer(c->d_qvals, c->qvals_cap, n);
    if (!rc) rc = grow_buffer(c->d_qvals_out, c->qvals_out_cap, n);
    if (rc) return rc;
    size_t need = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, need, c->d_qkeys, c->d_qkeys_out, c->d_qvals, c->d_qvals_out, int(n), 0, 32);
    return grow_buffer(c->d_qsort_tmp, c->qsort_tmp_bytes, need + 256);
}

int query_sort(Ctx* c, size_t n) {
    size_t tmp = c->qsort_tmp_bytes;
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_qsort_tmp, tmp, c->d_qkeys, c->d_qkeys_out, c->d_qvals, c->d_qvals_out, int(n), 0, 32, c->stream));
    c->launches += 5;
    return SO_OK;
}

int scan_sort(Ctx* c, size_t first, size_t n, int n_scans, int cell_bits, bool key32, cudaStream_t st) {
    int bits = cell_bits;
    while ((1 << (bits - cell_bits)) < n_scans) ++bits;
    size_t tmp = c->sort_tmp_bytes;
    void* scratch = st == c->aux_stream ? c->d_sort_tmp2 : c->d_sort_tmp;
    if (key32)
        SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(scratch, tmp, reinterpret_cast<uint32_t*>(c->d_skeys) + first, reinterpret_cast<uint32_t*>(c->d_skeys_out) + first,
                                                    c->d_svals + first, c->d_svals_out + first, int(n), 0, bits, st));
    else
        SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(scratch, tmp, c->d_skeys + first, c->d_skeys_out + first,
                                                    c->d_svals + first, c->d_svals_out + first, int(n), 0, bits, st));
    c->launches += 5;
    return SO_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Map insert: LocalMap::addSurfPointCloud (LocalMap.h:591-645).  New world-frame points are appended, every block they
// touch is re-filtered as a whole by a voxel-centroid filter of leaf planeRes_ (pcl::VoxelGrid semantics: voxel =
// floor(coord * (1.0f/leaf)) in float32, centroid of all four fields accumulated in float32 and divided by
// float(count), output ordered by voxel index (k, j, i)), untouched blocks keep their clouds.  PCL leaves the in-voxel
// accumulation order unspecified (std::sort on the voxel index); here it is ascending cloud order (old points, then
// new points in input order), the order the stable radix sort preserves.
// ------------------------------------------------------------------------------------------------------------------
__global__ void k_mark_touched(const int32_t* __restrict__ block_of_point, uint32_t first_new, uint32_t n, uint8_t* __restrict__ touched) {
    const uint32_t i = first_new + blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && block_of_point[i] >= 0) touched[block_of_point[i]] = 1;
}

// Sort key of the insert: [63] touched flag | [48..60] grid block (13 bits: 0..4850) | 3 x 16 bits of BLOCK-LOCAL voxel index (k, j, i).
// PCL orders a block's output by the voxel index relative to the block cloud's bounding box; subtracting any per-block constant
// keeps that order, so the index is taken relative to the block's minimum corner (minus a 2-voxel guard for the float rounding of
// x * inv_leaf at the faces): 50 m / leaf + 4 values per axis -- 16 bits hold leaf >= 1 mm, wherever the block is in the world.
__global__ void k_voxel_keys(const float4* __restrict__ raw, const int32_t* __restrict__ block_of_point, const uint8_t* __restrict__ touched,
                             uint32_t n, float inv_leaf, int3 origin, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t b = block_of_point[i];
    uint64_t key;
    if (b < 0) key = ~uint64_t(0);                                  // off-grid: dropped
    else if (!touched[b]) key = 0;                                  // untouched block: keep, in place (stable sort)
    else {
        const float4 p = raw[i];
        const int gx = b % kW, gy = (b / kW) % kH, gz = b / (kW * kH);
        const double il = double(inv_leaf);
        const int64_t bx = int64_t(floor((double(gx - origin.x) * kBlock - kHalfBlock) * il)) - 2;
        const int64_t by = int64_t(floor((double(gy - origin.y) * kBlock - kHalfBlock) * il)) - 2;
        const int64_t bz = int64_t(floor((double(gz - origin.z) * kBlock - kHalfBlock) * il)) - 2;
        auto local = [](int64_t v) { return uint64_t(v < 0 ? 0 : (v > 65535 ? 65535 : v)); };
        const uint64_t vi = local(int64_t(floorf(__fmul_rn(p.x, inv_leaf))) - bx);      // pcl::VoxelGrid: floor(coord * inverse_leaf_size) in float
        const uint64_t vj = local(int64_t(floorf(__fmul_rn(p.y, inv_leaf))) - by);
        const uint64_t vk = local(int64_t(floorf(__fmul_rn(p.z, inv_leaf))) - bz);
        key = (uint64_t(1) << 63) | (uint64_t(b) << 48) | (vk << 32) | (vj << 16) | vi;
    }
    keys[i] = key;
    vals[i] = i;
}

__global__ void k_voxel_heads(const uint64_t* __restrict__ keys, uint32_t begin, uint32_t end, uint32_t* __restrict__ head) {
    const uint32_t i = begin + blockIdx.x * blockDim.x + threadIdx.x;
    if (i < end) head[i - begin] = (i == begin || keys[i] != keys[i - 1]) ? 1u : 0u;
}

__global__ void k_voxel_centroid(const float4* __restrict__ raw, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                 const uint32_t* __restrict__ rank, uint32_t begin, uint32_t end, float4* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < begin) { out[i] = raw[vals[i]]; return; }               // untouched blocks: copied through in order
    if (i >= end) return;
    if (!(i == begin || keys[i] != keys[i - 1])) return;             // not a voxel head
    const uint64_t key = keys[i];
    float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
    uint32_t cnt = 0;
    for (uint32_t j = i; j < end && keys[j] == key; ++j) {           // pcl::CentroidPoint: float accumulators, cloud order
        const float4 p = raw[vals[j]];
        ax = __fadd_rn(ax, p.x); ay = __fadd_rn(ay, p.y); az = __fadd_rn(az, p.z); aw = __fadd_rn(aw, p.w);
        ++cnt;
    }
    const float nf = float(cnt);
    out[begin + rank[i - begin]] = make_float4(__fdiv_rn(ax, nf), __fdiv_rn(ay, nf), __fdiv_rn(az, nf), __fdiv_rn(aw, nf));
}

struct Pose7 { double v[7]; };
__global__ void k_transform_points(float4* __restrict__ pts, uint32_t n, Pose7 pose) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 p = pts[i];
    const double v[3] = {double(p.x), double(p.y), double(p.z)};
    double o[3];
    qrot(pose.v + 3, v, o);                            // utils::TransformPoint (superodom_utils.h:116-127): double math, float store
    p.x = float(o[0] + pose.v[0]); p.y = float(o[1] + pose.v[1]); p.z = float(o[2] + pose.v[2]);
    pts[i] = p;
}

int map_transform_tail(Ctx* c, MapStore& ms, uint32_t n_new, const double pose[7]) {
    Pose7 P;
    for (int k = 0; k < 7; ++k) P.v[k] = pose[k];                            // by value in the launch: no staging copy, no wait
    k_transform_points<<<(n_new + 255) / 256, 256, 0, c->stream>>>(ms.d_xyzi + ms.n, n_new, P);
    c->launches++;
    return SO_OK;
}

static int map_add_points_sync(Ctx* c, MapStore& ms, uint32_t n_new) {
    cudaStream_t st = c->stream;
    const uint32_t total = ms.n + n_new;
    if (n_new == 0) return SO_OK;
    const int3 origin = make_int3(c->origin[0], c->origin[1], c->origin[2]);
    const uint32_t grid = (total + 255) / 256;
    uint8_t* d_touched = reinterpret_cast<uint8_t*>(c->d_vals_out);          // scratch: 4851 bytes
    SO_CUDA_TRY(cudaMemsetAsync(ms.d_block_count, 0, kNumBlocks * sizeof(int32_t), st));
    SO_CUDA_TRY(cudaMemsetAsync(d_touched, 0, kNumBlocks, st));
    k_block_of<<<grid, 256, 0, st>>>(ms.d_xyzi, total, origin, c->d_block_of_point, ms.d_block_count);
    k_mark_touched<<<(n_new + 255) / 256, 256, 0, st>>>(c->d_block_of_point, ms.n, total, d_touched);
    std::vector<uint8_t> h_touched(kNumBlocks);
    SO_CUDA_TRY(cudaMemcpyAsync(ms.h_block_count.data(), ms.d_block_count, kNumBlocks * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaMemcpyAsync(h_touched.data(), d_touched, kNumBlocks, cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    uint64_t n_untouched = 0, n_touched = 0;
    for (int b = 0; b < kNumBlocks; ++b) (h_touched[b] ? n_touched : n_untouched) += uint64_t(ms.h_block_count[b]);
    // keys need the touched flags: keep them in a scratch that the sort does not use
    uint8_t* d_touched2 = reinterpret_cast<uint8_t*>(c->d_cub_tmp);
    SO_CUDA_TRY(cudaMemcpyAsync(d_touched2, h_touched.data(), kNumBlocks, cudaMemcpyHostToDevice, st));
    const float inv_leaf = 1.0f / ms.res;                               // Eigen::Array4f::Ones() / leaf_size_
    k_voxel_keys<<<grid, 256, 0, st>>>(ms.d_xyzi, c->d_block_of_point, d_touched2, total, inv_leaf, origin, c->d_keys, c->d_vals);
    SO_CUDA_TRY(cudaStreamSynchronize(st));                                   // d_cub_tmp is reused by the sort next
    size_t tmp = c->cub_tmp_bytes;
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_cub_tmp, tmp, c->d_keys, c->d_keys_out, c->d_vals, c->d_vals_out, int(total), 0, 64, st));
    const uint32_t begin = uint32_t(n_untouched), end = uint32_t(n_untouched + n_touched);
    uint32_t n_vox = 0;
    uint32_t* d_head = reinterpret_cast<uint32_t*>(c->d_keys);               // keys_in is free after the sort
    if (n_touched) {
        k_voxel_heads<<<(uint32_t(n_touched) + 255) / 256, 256, 0, st>>>(c->d_keys_out, begin, end, d_head);
        uint32_t last_flag = 0, last_rank = 0;
        tmp = c->cub_tmp_bytes;
        uint32_t* d_rank = d_head + n_touched;                                // second half of the same scratch (8 B/pt available)
        SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->d_cub_tmp, tmp, d_head, d_rank, int(n_touched), st));
        SO_CUDA_TRY(cudaMemcpyAsync(&last_flag, d_head + n_touched - 1, 4, cudaMemcpyDeviceToHost, st));
        SO_CUDA_TRY(cudaMemcpyAsync(&last_rank, d_rank + n_touched - 1, 4, cudaMemcpyDeviceToHost, st));
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        n_vox = last_rank + last_flag;
        k_voxel_centroid<<<(end + 255) / 256, 256, 0, st>>>(ms.d_xyzi, c->d_keys_out, c->d_vals_out, d_rank, begin, end, ms.d_sorted);
    } else if (begin) {
        k_voxel_centroid<<<(begin + 255) / 256, 256, 0, st>>>(ms.d_xyzi, c->d_keys_out, c->d_vals_out, nullptr, begin, begin, ms.d_sorted);
    }
    ms.n = begin + n_vox;
    if (ms.n) SO_CUDA_TRY(cudaMemcpyAsync(ms.d_xyzi, ms.d_sorted, size_t(ms.n) * sizeof(float4), cudaMemcpyDeviceToDevice, st));
    c->launches += 12;
    SO_CUDA_TRY(cudaGetLastError());
    return map_rebuild(c, ms);
}

// Device-side bookkeeping of an insert: everything the host used to read back between launches.
struct InsertInfo {
    uint32_t begin, end;        // sorted insert keys: [0, begin) untouched blocks, [begin, end) touched blocks, [end, total) dropped
    uint32_t n_out;             // points of the new cloud
    uint32_t n_slots;           // non-empty blocks of the new cloud
    uint32_t error;             // 1: cell table capacity exceeded
    uint32_t pad[3];
};

__global__ void k_mark_touched_new(const float4* __restrict__ pts, uint32_t n_new, int3 origin, uint8_t* __restrict__ touched) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_new) return;
    const float4 p = pts[i];
    const int gx = block_coord(double(p.x) + kHalfBlock, origin.x), gy = block_coord(double(p.y) + kHalfBlock, origin.y),
              gz = block_coord(double(p.z) + kHalfBlock, origin.z);
    if (gx >= 0 && gx < kW && gy >= 0 && gy < kH && gz >= 0 && gz < kD && isfinite(p.x) && isfinite(p.y) && isfinite(p.z))
        touched[gx + kW * gy + kW * kH * gz] = 1;
}

// insert key of every point (old cloud followed by the new points), the block recomputed from the coordinates:
// [class: 0 untouched block, 1 touched, 2 dropped][block 13 bits][vk][vj][vi], vb bits per block-local voxel index (50 m / leaf + 5
// values: 8 bits at leaf 0.2) -- 39 key bits = 5 radix passes instead of the 8 of a full 64-bit key
__global__ void k_insert_keys(const float4* __restrict__ raw, uint32_t n, float inv_leaf, int3 origin, const uint8_t* __restrict__ touched,
                              int vb, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = raw[i];
    const int gx = block_coord(double(p.x) + kHalfBlock, origin.x), gy = block_coord(double(p.y) + kHalfBlock, origin.y),
              gz = block_coord(double(p.z) + kHalfBlock, origin.z);
    const int cls_shift = 13 + 3 * vb;
    uint64_t key = uint64_t(2) << cls_shift;                              // off-grid / non-finite: dropped
    if (gx >= 0 && gx < kW && gy >= 0 && gy < kH && gz >= 0 && gz < kD && isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
        const int b = gx + kW * gy + kW * kH * gz;
        if (!touched[b]) key = 0;                                         // untouched block: kept in place (stable sort)
        else {
            const double il = double(inv_leaf);
            const int64_t bx = int64_t(floor((double(gx - origin.x) * kBlock - kHalfBlock) * il)) - 2;
            const int64_t by = int64_t(floor((double(gy - origin.y) * kBlock - kHalfBlock) * il)) - 2;
            const int64_t bz = int64_t(floor((double(gz - origin.z) * kBlock - kHalfBlock) * il)) - 2;
            const int64_t vmax = (int64_t(1) << vb) - 1;
            auto local = [vmax](int64_t v) { return uint64_t(v < 0 ? 0 : (v > vmax ? vmax : v)); };
            const uint64_t vi = local(int64_t(floorf(__fmul_rn(p.x, inv_leaf))) - bx);      // pcl::VoxelGrid: floor(coord * inverse_leaf_size) in float
            const uint64_t vj = local(int64_t(floorf(__fmul_rn(p.y, inv_leaf))) - by);
            const uint64_t vk = local(int64_t(floorf(__fmul_rn(p.z, inv_leaf))) - bz);
            key = (uint64_t(1) << cls_shift) | (uint64_t(b) << (3 * vb)) | (vk << (2 * vb)) | (vj << vb) | vi;
        }
    }
    keys[i] = key;
    vals[i] = i;
}

// boundaries of the three key classes in the sorted keys, by binary search (one thread)
__global__ void k_insert_bounds(const uint64_t* __restrict__ keys, uint32_t total, int cls_shift, InsertInfo* __restrict__ info) {
    if (threadIdx.x || blockIdx.x) return;
    uint32_t lo = 0, hi = total;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((keys[mid] >> cls_shift) >= 1) hi = mid; else lo = mid + 1; }      // first touched key
    info->begin = lo;
    hi = total;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((keys[mid] >> cls_shift) >= 2) hi = mid; else lo = mid + 1; }      // first dropped key
    info->end = lo;
    info->error = 0;
}

__global__ void k_voxel_heads_dev(const uint64_t* __restrict__ keys, uint32_t total, const InsertInfo* __restrict__ info, uint32_t* __restrict__ head) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    head[i] = (i >= info->begin && i < info->end && (i == info->begin || keys[i] != keys[i - 1])) ? 1u : 0u;
}

// rank[] = exclusive scan of head[] over [0, total): rank[i] counts the voxels before sorted position i
__global__ void k_voxel_centroid_dev(const float4* __restrict__ raw, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                     const uint32_t* __restrict__ head, const uint32_t* __restrict__ rank, uint32_t total, InsertInfo* __restrict__ info,
                                     float4* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const uint32_t begin = info->begin, end = info->end;
    if (i == total - 1) info->n_out = begin + rank[i] + head[i];      // voxels in total
    if (i < begin) { out[i] = raw[vals[i]]; return; }                   // untouched blocks: copied through in order
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

// ---- index of a cloud whose size lives on the device (every point on-grid): block counts, slots, cell keys, cell table ------------
// One atomic per (warp, block) instead of one per point: the cloud is ordered block by block, so a warp almost always holds a
// single block (1.1 M same-address atomics took 660 us; aggregated they take a few).
__global__ void k_block_count_dev(const float4* __restrict__ raw, const InsertInfo* __restrict__ info, int3 origin, int32_t* __restrict__ block_count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    int lin = -1;
    if (i < info->n_out) {
        const float4 p = raw[i];
        const int gx = block_coord(double(p.x) + kHalfBlock, origin.x), gy = block_coord(double(p.y) + kHalfBlock, origin.y),
                  gz = block_coord(double(p.z) + kHalfBlock, origin.z);
        if (gx >= 0 && gx < kW && gy >= 0 && gy < kH && gz >= 0 && gz < kD) lin = gx + kW * gy + kW * kH * gz;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, lin);
    if (lin >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&block_count[lin], __popc(peers));
}

// slots of the non-empty blocks in block order (what the host loop of map_rebuild does), one CTA
__global__ void __launch_bounds__(1024) k_assign_slots(const int32_t* __restrict__ block_count, int32_t* __restrict__ block_slot, InsertInfo* __restrict__ info,
                                                       uint32_t slot_cap) {
    __shared__ uint32_t s_part[1024];
    const int per = (kNumBlocks + 1023) / 1024;
    const int b0 = threadIdx.x * per;
    uint32_t mine = 0;
    for (int k = 0; k < per; ++k) { const int b = b0 + k; if (b < kNumBlocks && block_count[b] > 0) ++mine; }
    s_part[threadIdx.x] = mine;
    __syncthreads();
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
    if (threadIdx.x == 1023) { info->n_slots = s_part[1023]; if (s_part[1023] > slot_cap) info->error = 1; }
}

// cell key + histogram; positions >= n_out get the largest key so that they sort behind every real point
__global__ void k_keys_dev(const float4* __restrict__ raw, uint32_t total, const InsertInfo* __restrict__ info, int3 origin, const int32_t* __restrict__ block_slot,
                           int nb, double inv_cs, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ cell_count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    vals[i] = i;
    if (i >= info->n_out || info->error) { keys[i] = 0xFFFFFFFFu; return; }
    const float4 p = raw[i];
    const float q[3] = {p.x, p.y, p.z};
    const int o[3] = {origin.x, origin.y, origin.z};
    int g[3], c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double v = double(q[a]) + kHalfBlock;
        int b = int(v / kBlock);
        if (v < 0) b--;
        g[a] = b + o[a];
        int cc = int((v - kBlock * double(b)) * inv_cs);
        c[a] = cc < 0 ? 0 : (cc > nb - 1 ? nb - 1 : cc);
    }
    const uint32_t slot = uint32_t(block_slot[g[0] + kW * g[1] + kW * kH * g[2]]);
    const uint32_t key = slot * uint32_t(nb) * uint32_t(nb) * uint32_t(nb) + uint32_t((c[2] * nb + c[1]) * nb + c[0]);
    keys[i] = key;
    atomicAdd(&cell_count[key], 1u);
}

__global__ void k_gather_dev(const float4* __restrict__ raw, const uint32_t* __restrict__ vals, uint32_t total, const InsertInfo* __restrict__ info,
                             float4* __restrict__ sorted) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total || i >= info->n_out) return;
    const uint32_t id = vals[i];
    const float4 p = raw[id];
    sorted[i] = make_float4(p.x, p.y, p.z, __uint_as_float(id));
}

// LocalMap::addSurfPointCloud without a host round trip between its steps: mark touched blocks, one stable sort by
// (touched, block, voxel), voxel heads + scan + centroids into the other cloud buffer, then the search index of the new cloud
// (block counts and slots on the device, cell keys + histogram, sort, gather, scan).  The host reads the sizes, block tables and
// the error flag back ONCE, at the end.  The two cloud buffers swap roles (no device-to-device copy of the map).
int map_add_points(Ctx* c, MapStore& ms, uint32_t n_new) {
    cudaStream_t st = c->stream;
    if (n_new == 0) return SO_OK;
    const uint32_t total = ms.n + n_new;                                // the caller rebuilt a dirty store BEFORE appending the new points
    const int3 origin = make_int3(c->origin[0], c->origin[1], c->origin[2]);
    const uint32_t grid = (total + 255) / 256;
    const int nb = map_cells_per_block(ms.res);
    const uint32_t cells_per_slot = uint32_t(nb) * uint32_t(nb) * uint32_t(nb);
    // cell table capacity for the slots this insert can need: the current ones plus every block a new point may open
    {
        const size_t want_slots = size_t(ms.n_slots) + 4;
        const size_t want = want_slots * cells_per_slot + 1;
        if (want > ms.cell_cap || ms.nb != nb) {
            size_t slots = want_slots + 4;
            while (slots > want_slots && slots * cells_per_slot + 1 >= (size_t(1) << 31)) --slots;
            if (slots * cells_per_slot + 1 >= (size_t(1) << 31)) return map_add_points_sync(c, ms, n_new);
            SO_CUDA_TRY(cudaStreamSynchronize(st));
            int rc = grow_buffer(ms.d_cell_start, ms.cell_cap, slots * cells_per_slot + 1);
            if (rc) return rc;
            size_t need = 0;
            cub::DeviceScan::ExclusiveSum(nullptr, need, ms.d_cell_start, ms.d_cell_start, int(ms.cell_cap));
            rc = grow_buffer(c->d_cub_tmp, c->cub_tmp_bytes, need + 256);
            if (rc) return rc;
        }
    }
    // this insert indexes at most the current slots + 4 new ones (more: error flag -> synchronous rebuild); table work is sized for that
    const uint32_t slot_cap = uint32_t(std::min<size_t>((ms.cell_cap - 1) / cells_per_slot, size_t(ms.n_slots) + 4));
    const size_t cells_used = size_t(slot_cap) * cells_per_slot + 1;
    ms.nb = nb;
    InsertInfo* d_info = reinterpret_cast<InsertInfo*>(c->d_insert_info);
    uint8_t* d_touched = reinterpret_cast<uint8_t*>(c->d_insert_info) + 64;         // 4851 bytes behind the info struct
    SO_CUDA_TRY(cudaMemsetAsync(d_touched, 0, kNumBlocks, st));
    k_mark_touched_new<<<(n_new + 255) / 256, 256, 0, st>>>(ms.d_xyzi + ms.n, n_new, origin, d_touched);
    const float inv_leaf = 1.0f / ms.res;                               // Eigen::Array4f::Ones() / leaf_size_
    int vb = 1;                                                         // bits of a block-local voxel index: 50 m / leaf + 5 values
    while (vb < 16 && double(1 << vb) < kBlock * double(inv_leaf) + 5.0) ++vb;
    const int cls_shift = 13 + 3 * vb;
    k_insert_keys<<<grid, 256, 0, st>>>(ms.d_xyzi, total, inv_leaf, origin, d_touched, vb, c->d_keys, c->d_vals);
    size_t tmp = c->cub_tmp_bytes;
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_cub_tmp, tmp, c->d_keys, c->d_keys_out, c->d_vals, c->d_vals_out, int(total), 0, cls_shift + 2, st));
    k_insert_bounds<<<1, 32, 0, st>>>(c->d_keys_out, total, cls_shift, d_info);
    uint32_t* d_head = reinterpret_cast<uint32_t*>(c->d_keys);          // keys_in is free after the sort: [heads total][ranks total]
    uint32_t* d_rank = d_head + total;
    k_voxel_heads_dev<<<grid, 256, 0, st>>>(c->d_keys_out, total, d_info, d_head);
    tmp = c->cub_tmp_bytes;
    SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->d_cub_tmp, tmp, d_head, d_rank, int(total), st));
    k_voxel_centroid_dev<<<grid, 256, 0, st>>>(ms.d_xyzi, c->d_keys_out, c->d_vals_out, d_head, d_rank, total, d_info, ms.d_sorted);
    std::swap(ms.d_xyzi, ms.d_sorted);                                  // d_xyzi: the new cloud in id order; d_sorted: free for the new index
    // ---- search index of the new cloud
    SO_CUDA_TRY(cudaMemsetAsync(ms.d_block_count, 0, kNumBlocks * sizeof(int32_t), st));
    k_block_count_dev<<<grid, 256, 0, st>>>(ms.d_xyzi, d_info, origin, ms.d_block_count);
    k_assign_slots<<<1, 1024, 0, st>>>(ms.d_block_count, ms.d_block_slot, d_info, slot_cap);
    SO_CUDA_TRY(cudaMemsetAsync(ms.d_cell_start, 0, cells_used * sizeof(uint32_t), st));
    uint32_t* keys32 = reinterpret_cast<uint32_t*>(c->d_keys);          // heads / ranks are dead now
    uint32_t* keys32_out = reinterpret_cast<uint32_t*>(c->d_keys_out);
    k_keys_dev<<<grid, 256, 0, st>>>(ms.d_xyzi, total, d_info, origin, ms.d_block_slot, nb, double(nb) / kBlock, keys32, c->d_vals, ms.d_cell_start);
    int bits = 1;
    while (bits < 32 && (uint64_t(1) << bits) < uint64_t(ms.cell_cap)) ++bits;
    tmp = c->cub_tmp_bytes;
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_cub_tmp, tmp, keys32, keys32_out, c->d_vals, c->d_vals_out, int(total), 0, 32, st));
    (void)bits;
    k_gather_dev<<<grid, 256, 0, st>>>(ms.d_xyzi, c->d_vals_out, total, d_info, ms.d_sorted);
    tmp = c->cub_tmp_bytes;
    SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->d_cub_tmp, tmp, ms.d_cell_start, ms.d_cell_start, int(cells_used), st));
    // ---- the one read-back
    InsertInfo* h_info = reinterpret_cast<InsertInfo*>(c->h_insert_info);
    SO_CUDA_TRY(cudaMemcpyAsync(h_info, d_info, sizeof(InsertInfo), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaMemcpyAsync(ms.h_block_count.data(), ms.d_block_count, kNumBlocks * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaMemcpyAsync(ms.h_block_slot.data(), ms.d_block_slot, kNumBlocks * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    c->launches += 26;
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    ms.n = h_info->n_out;
    ms.n_slots = int(h_info->n_slots);
    if (h_info->error) {                                                // more new blocks than the table was sized for: index again, synchronously
        ms.dirty = true;
        return map_rebuild(c, ms);
    }
    return SO_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Scan pre-filter: the pcl::VoxelGrid(planeRes) that laserMapping::adjustVoxelSize applies to the sensor-frame surf
// cloud before Localization (laserMapping.cpp:639-645).  Same voxel/centroid semantics as the map insert, one grid
// for the whole cloud.  In: d_scan[0..n); out: d_scan_sorted[0..*n_out) ordered by voxel index (k, j, i).
// ------------------------------------------------------------------------------------------------------------------
// VB bits per voxel index (offset 2^(VB-1)); the key of a skipped point has bit 3*VB set and sorts last.  VB = 13 covers +-4096
// voxels around the sensor (819 m at leaf 0.2) in 40 key bits = 5 radix passes; a point beyond that raises *overflow and the caller
// repeats the filter with VB = 17 (the layout every cloud fits).
template <int VB>
__global__ void k_voxel_keys_cloud(const float4* __restrict__ raw, uint32_t n, float inv_leaf, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                   uint32_t* __restrict__ overflow) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = raw[i];
    constexpr int64_t kOff = int64_t(1) << (VB - 1), kMask = (int64_t(1) << VB) - 1;
    uint64_t key = uint64_t(1) << (3 * VB);                          // non-finite points are skipped, as PCL does
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
        const int64_t vi = int64_t(floorf(__fmul_rn(p.x, inv_leaf))) + kOff;
        const int64_t vj = int64_t(floorf(__fmul_rn(p.y, inv_leaf))) + kOff;
        const int64_t vk = int64_t(floorf(__fmul_rn(p.z, inv_leaf))) + kOff;
        if (((vi | vj | vk) & ~kMask) != 0) *overflow = 1;           // outside the VB-bit range (negative values have high bits set)
        key = (uint64_t(vk & kMask) << (2 * VB)) | (uint64_t(vj & kMask) << VB) | uint64_t(vi & kMask);
    }
    keys[i] = key;
    vals[i] = i;
}

__global__ void k_count_valid(const uint64_t* __restrict__ keys, uint32_t n, uint64_t skipped_key, uint32_t* __restrict__ count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && keys[i] != skipped_key && (i + 1 == n || keys[i + 1] == skipped_key)) *count = i + 1;   // sorted: last valid key
}

int scan_voxel_filter(Ctx* c, uint32_t n, float leaf, uint32_t* n_out) {
    cudaStream_t st = c->stream;
    *n_out = 0;
    if (n == 0) return SO_OK;
    const uint32_t grid = (n + 255) / 256;
    const float inv_leaf = 1.0f / leaf;
    uint32_t* d_flag = reinterpret_cast<uint32_t*>(c->d_insert_info) + 2000;     // scratch word behind the insert bookkeeping
    uint32_t* d_cnt = reinterpret_cast<uint32_t*>(c->d_skeys);      // keys_in is free after the sort: [count][heads...][ranks...]
    uint32_t n_valid = 0;
    for (int wide = 0; wide < 2; ++wide) {
        const int vb = wide ? 17 : 13;
        SO_CUDA_TRY(cudaMemsetAsync(d_flag, 0, 4, st));
        if (wide) k_voxel_keys_cloud<17><<<grid, 256, 0, st>>>(c->d_scan, n, inv_leaf, c->d_skeys, c->d_svals, d_flag);
        else k_voxel_keys_cloud<13><<<grid, 256, 0, st>>>(c->d_scan, n, inv_leaf, c->d_skeys, c->d_svals, d_flag);
        size_t tmp = c->sort_tmp_bytes;
        SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->d_sort_tmp, tmp, c->d_skeys, c->d_skeys_out, c->d_svals, c->d_svals_out, int(n), 0, 3 * vb + 1, st));
        SO_CUDA_TRY(cudaMemsetAsync(d_cnt, 0, 4, st));
        k_count_valid<<<grid, 256, 0, st>>>(c->d_skeys_out, n, uint64_t(1) << (3 * vb), d_cnt);
        uint32_t h[2] = {0, 0};
        SO_CUDA_TRY(cudaMemcpyAsync(&h[0], d_cnt, 4, cudaMemcpyDeviceToHost, st));
        SO_CUDA_TRY(cudaMemcpyAsync(&h[1], d_flag, 4, cudaMemcpyDeviceToHost, st));
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        n_valid = h[0];
        if (!h[1]) break;                                           // every voxel index fitted the narrow key
    }
    if (n_valid == 0) return SO_OK;
    uint32_t* d_head = d_cnt + 4;
    uint32_t* d_rank = d_head + n_valid;
    k_voxel_heads<<<(n_valid + 255) / 256, 256, 0, st>>>(c->d_skeys_out, 0, n_valid, d_head);
    size_t tmp = c->sort_tmp_bytes;
    SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->d_sort_tmp, tmp, d_head, d_rank, int(n_valid), st));
    uint32_t last_flag = 0, last_rank = 0;
    SO_CUDA_TRY(cudaMemcpyAsync(&last_flag, d_head + n_valid - 1, 4, cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaMemcpyAsync(&last_rank, d_rank + n_valid - 1, 4, cudaMemcpyDeviceToHost, st));
    k_voxel_centroid<<<(n_valid + 255) / 256, 256, 0, st>>>(c->d_scan, c->d_skeys_out, c->d_svals_out, d_rank, 0, n_valid, c->d_scan_sorted);
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    *n_out = last_rank + last_flag;
    c->launches += 10;
    SO_CUDA_TRY(cudaGetLastError());
    return SO_OK;
}

}  // namespace so

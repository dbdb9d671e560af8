// so_features.cu -- edge features of a ring-ordered raw scan (so_scan_extract_edges), sm_90a.
//
// Fills the edgePoints cloud that featureExtraction::extractFeatures publishes empty (featureExtraction.cpp:429-436) with LOAM's
// edge selection (Zhang & Singh, RSS 2014, §V-A, in the form of A-LOAM's scanRegistration, with LOAM's occlusion and parallel-beam
// rejection).  DESIGN.md §9 holds the definition; tests/edge_features_numpy.py restates it.  Every float operation is rounded on its
// own (__fadd_rn / __fmul_rn / ...: no contraction), sums left to right as the definition writes them.
//
//   k_edge_keys     one thread per record: validity, key ring << 32 | ordered time bits (invalid: kInvalidKey), value = index
//   (stable radix sort: (ring, time, input index) order)
//   k_edge_rings    one thread per sorted position: gather the point, ring bounds and the ring list, clear the marks
//   k_edge_curv     one thread per point: curvature, occlusion and parallel-beam marks (all write 1), the candidate key
//                   (ring, sector, ~curvature bits) and the reach of its neighbour marks
//   (stable radix sort: candidates by (ring, sector, curvature descending, position ascending))
//   k_edge_walk     one warp per ring, sectors in order, 32 candidates at a time resolved in registers
//   (exclusive scan of the accepted flags)  k_edge_scatter  compaction into (ring, position) order
// The buffers are Ctx::feat, never the scan buffers; the optional voxel filter is cloud_voxel_filter (so_map.cu).
#include <algorithm>
#include <cmath>

#include <cub/cub.cuh>

#include "so_ctx.cuh"

namespace so {

namespace {

constexpr uint64_t kInvalidKey = uint64_t(1) << 48;        // after every (ring, time) key
constexpr int kCandBits = 51;                               // ring 16 | sector 3 | ~curvature 32
constexpr uint64_t kNoCand = uint64_t(1) << kCandBits;      // after every candidate key
constexpr uint32_t kRings = 65536;
constexpr int kWalkBlocks = 256, kWalkThreads = 128;

// float bits in an order that sorts like the value; -0 is taken as +0
__device__ __forceinline__ uint32_t ordered_bits(float t) {
    const uint32_t u = t == 0.f ? 0u : __float_as_uint(t);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

template <bool kAligned>
__device__ __forceinline__ float ld_f32(const unsigned char* p) {
    if (kAligned) return *reinterpret_cast<const float*>(p);
    return __uint_as_float(uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24));
}
template <bool kAligned>
__device__ __forceinline__ uint32_t ld_u16(const unsigned char* p) {
    if (kAligned) return *reinterpret_cast<const uint16_t*>(p);
    return uint32_t(p[0]) | (uint32_t(p[1]) << 8);
}

__device__ __forceinline__ float n2(float x, float y, float z) { return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)); }
__device__ __forceinline__ float n2(float4 a) { return n2(a.x, a.y, a.z); }
__device__ __forceinline__ float gap2(float4 a, float4 b) { return n2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)); }   // |a - b|^2

template <bool kAligned>
__global__ void __launch_bounds__(256) k_edge_keys(const unsigned char* __restrict__ raw, uint32_t n, uint32_t stride, uint32_t toff, uint32_t roff,
                                                   float min_r2, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned char* r = raw + size_t(i) * stride;
    const float x = ld_f32<kAligned>(r), y = ld_f32<kAligned>(r + 4), z = ld_f32<kAligned>(r + 8), t = ld_f32<kAligned>(r + toff);
    const bool ok = isfinite(x) && isfinite(y) && isfinite(z) && isfinite(t) && n2(x, y, z) > min_r2;
    keys[i] = ok ? (uint64_t(ld_u16<kAligned>(r + roff)) << 32) | ordered_bits(t) : kInvalidKey;
    vals[i] = i;
}

template <bool kAligned>
__global__ void __launch_bounds__(256) k_edge_rings(const unsigned char* __restrict__ raw, uint32_t n, uint32_t stride, uint32_t toff,
                                                    const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, float4* __restrict__ pts,
                                                    uint32_t* __restrict__ ring_tab, uint8_t* __restrict__ excl, uint32_t* __restrict__ sel) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    excl[p] = 0;
    sel[p] = 0;
    const uint64_t key = keys[p];
    if (key >= kInvalidKey) return;
    const unsigned char* r = raw + size_t(vals[p]) * stride;
    pts[p] = make_float4(ld_f32<kAligned>(r), ld_f32<kAligned>(r + 4), ld_f32<kAligned>(r + 8), ld_f32<kAligned>(r + toff));
    const uint32_t ring = uint32_t(key >> 32);
    if (p == 0 || uint32_t(keys[p - 1] >> 32) != ring) {
        ring_tab[ring] = p;
        ring_tab[2 * kRings + atomicAdd(&ring_tab[3 * kRings], 1u)] = ring;      // list order does not matter: rings are independent
    }
    if (p == n - 1 || uint32_t(keys[p + 1] >> 32) != ring) ring_tab[kRings + ring] = p + 1;    // an invalid key never equals a ring
}

__global__ void __launch_bounds__(256) k_edge_curv(const float4* __restrict__ pts, const uint64_t* __restrict__ keys, uint32_t n,
                                                   const uint32_t* __restrict__ ring_tab, float thr, uint8_t* __restrict__ excl,
                                                   uint8_t* __restrict__ reach, uint64_t* __restrict__ ckeys, uint32_t* __restrict__ cvals) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    cvals[p] = p;
    uint64_t ckey = kNoCand;
    const uint64_t key = keys[p];
    if (key < kInvalidKey) {
        const uint32_t ring = uint32_t(key >> 32), lo = ring_tab[ring], m = ring_tab[kRings + ring] - lo, k = p - lo;
        const float4* q = pts + lo;
        if (k >= 5 && k + 6 <= m) {                                   // 5 <= k <= m-6
            const float4 qk = q[k];
            float sx = q[k - 5].x, sy = q[k - 5].y, sz = q[k - 5].z;
#pragma unroll
            for (int o = -4; o <= 5; ++o) {
                if (o == 0) continue;
                const float4 v = q[int(k) + o];
                sx = __fadd_rn(sx, v.x); sy = __fadd_rn(sy, v.y); sz = __fadd_rn(sz, v.z);
            }
            const float c = n2(__fsub_rn(sx, __fmul_rn(10.f, qk.x)), __fsub_rn(sy, __fmul_rn(10.f, qk.y)), __fsub_rn(sz, __fmul_rn(10.f, qk.z)));
            const float4 qp = q[k - 1], qn = q[k + 1];
            const float lim = __fmul_rn(0.0002f, n2(qk));                          // parallel beam
            if (gap2(qk, qp) > lim && gap2(qn, qk) > lim) excl[lo + k] = 1;
            if (k + 7 <= m) {                                                       // 5 <= k <= m-7
                if (gap2(qn, qk) > 0.1f) {                                          // occlusion
                    const float ra = __fsqrt_rn(n2(qk)), rb = __fsqrt_rn(n2(qn));
                    if (ra > rb) {
                        const float ex = __fsub_rn(qn.x, __fdiv_rn(__fmul_rn(qk.x, rb), ra)), ey = __fsub_rn(qn.y, __fdiv_rn(__fmul_rn(qk.y, rb), ra)),
                                    ez = __fsub_rn(qn.z, __fdiv_rn(__fmul_rn(qk.z, rb), ra));
                        if (__fdiv_rn(__fsqrt_rn(n2(ex, ey, ez)), rb) < 0.1f)
                            for (uint32_t u = k - 5; u <= k; ++u) excl[lo + u] = 1;
                    } else {
                        const float ex = __fsub_rn(__fdiv_rn(__fmul_rn(qn.x, ra), rb), qk.x), ey = __fsub_rn(__fdiv_rn(__fmul_rn(qn.y, ra), rb), qk.y),
                                    ez = __fsub_rn(__fdiv_rn(__fmul_rn(qn.z, ra), rb), qk.z);
                        if (__fdiv_rn(__fsqrt_rn(n2(ex, ey, ez)), ra) < 0.1f)
                            for (uint32_t u = k + 1; u <= k + 6; ++u) excl[lo + u] = 1;
                    }
                }
                if (m >= 17 && c > thr) {                                           // a candidate of sector j (NaN never is)
                    const uint32_t a = 5, span = m - 11;                            // z - a with z = m - 6
                    uint32_t j = 0;
                    while (j < 5 && k >= a + span * (j + 1) / 6) ++j;
                    uint32_t fwd = 0, bwd = 0;
                    for (uint32_t l = 1; l <= 5 && !(gap2(q[k + l], q[k + l - 1]) > 0.05f); ++l) fwd = l;
                    for (uint32_t l = 1; l <= 5 && !(gap2(q[k - l], q[k - l + 1]) > 0.05f); ++l) bwd = l;
                    reach[p] = uint8_t((bwd << 4) | fwd);
                    ckey = (uint64_t(ring) << 35) | (uint64_t(j) << 32) | uint64_t(~__float_as_uint(c));
                }
            }
        }
    }
    ckeys[p] = ckey;
}

// first index in [lo, hi) whose key is >= v (keys ascending), the whole warp searching 32 ways per step
__device__ __forceinline__ uint32_t warp_lower_bound(const uint64_t* keys, uint32_t lo, uint32_t hi, uint64_t v, uint32_t lane) {
    while (hi - lo > 32) {
        const uint32_t step = (hi - lo) / 32;
        const uint32_t below = __popc(__ballot_sync(0xffffffffu, keys[lo + step * (lane + 1) - 1] < v));
        const uint32_t nhi = below < 32 ? lo + step * (below + 1) : hi;
        lo += step * below;
        hi = nhi;
    }
    return lo + __popc(__ballot_sync(0xffffffffu, lo + lane < hi && keys[lo + lane] < v));
}

// One warp per ring (rings strided over the grid's warps), its six sectors in order.  A sector's candidates come 32 at a time in
// (curvature descending, position ascending) order; lane t's candidate is accepted when it is not excluded -- by the marks in memory
// or by an earlier lane of the chunk -- and the sector has room; its marks [p - bwd, p + fwd] then reach the later lanes in
// registers and everything after the chunk through excl (ordered by __syncwarp).
__global__ void __launch_bounds__(kWalkThreads) k_edge_walk(const uint64_t* __restrict__ ckeys, const uint32_t* __restrict__ cvals, uint32_t n,
                                                            const uint32_t* __restrict__ ring_tab, uint8_t* excl, const uint8_t* __restrict__ reach,
                                                            uint32_t* __restrict__ sel, int max_per_sector) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t n_rings = ring_tab[3 * kRings];
    for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_rings; w += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t ring = ring_tab[2 * kRings + w];
        if (ring_tab[kRings + ring] - ring_tab[ring] < 17) continue;
        uint32_t b = warp_lower_bound(ckeys, 0, n, uint64_t(ring) << 35, lane);
        for (uint32_t j = 0; j < 6; ++j) {
            const uint32_t e = warp_lower_bound(ckeys, b, n, (uint64_t(ring) << 35) | (uint64_t(j + 1) << 32), lane);
            int count = 0;
            for (uint32_t s = b; s < e && count < max_per_sector; s += 32) {
                const bool has = s + lane < e;
                const uint32_t p = has ? cvals[s + lane] : 0u;
                bool ex = !has || excl[p];
                const uint32_t rc = has ? reach[p] : 0u, plo = p - (rc >> 4), phi = p + (rc & 15);
                bool acc = false;
                const uint32_t nv = min(32u, e - s);
                for (uint32_t t = 0; t < nv && count < max_per_sector; ++t) {
                    if (!__shfl_sync(0xffffffffu, int(!ex), t)) continue;
                    const uint32_t tlo = __shfl_sync(0xffffffffu, plo, t), thi = __shfl_sync(0xffffffffu, phi, t);
                    acc |= lane == t;
                    ex |= p >= tlo && p <= thi;
                    ++count;
                }
                if (acc) {
                    sel[p] = 1;
                    for (uint32_t u = plo; u <= phi; ++u) excl[u] = 1;
                }
                __syncwarp();
            }
            b = e;
        }
    }
}

__global__ void __launch_bounds__(256) k_edge_scatter(const float4* __restrict__ pts, const uint32_t* __restrict__ sel, const uint32_t* __restrict__ rank,
                                                      uint32_t n, float4* __restrict__ out, uint32_t* __restrict__ n_out) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    if (p == n - 1) *n_out = rank[p] + sel[p];
    if (sel[p]) out[rank[p]] = pts[p];
}

// Every buffer for n points of raw_bytes of records
int features_reserve(Ctx* c, size_t n, size_t raw_bytes) {
    Ctx::Feat& F = c->feat;
    int rc = F.d_raw.reserve(raw_bytes);
    if (!rc) rc = F.d_ring.reserve(3 * size_t(kRings) + 4);
    if (rc) return rc;
    if (n > F.d_pts.cap()) {                       // the per-point buffers grow together: every old one goes before the first new one
        for (int k = 0; k < 2; ++k) { F.d_keys[k].reset(); F.d_vals[k].reset(); }
        F.d_pts.reset(); F.d_excl.reset(); F.d_reach.reset(); F.d_sel.reset(); F.d_rank.reset(); F.d_out.reset(); F.d_vout.reset();
        F.d_tmp.reset();
    }
    for (int k = 0; k < 2 && !rc; ++k) {
        rc = F.d_keys[k].reserve(n);
        if (!rc) rc = F.d_vals[k].reserve(n);
    }
    if (!rc) rc = F.d_pts.reserve(n);
    if (!rc) rc = F.d_excl.reserve(n);
    if (!rc) rc = F.d_reach.reserve(n);
    if (!rc) rc = F.d_sel.reserve(n);
    if (!rc) rc = F.d_rank.reserve(n);
    if (!rc) rc = F.d_out.reserve(n);
    if (!rc) rc = F.d_vout.reserve(n);
    if (rc) return rc;
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, F.d_keys[0].get(), F.d_keys[1].get(), F.d_vals[0].get(), F.d_vals[1].get(), int(n), 0, 64);
    cub::DeviceScan::ExclusiveSum(nullptr, b, F.d_sel.get(), F.d_rank.get(), int(n));
    return F.d_tmp.reserve(std::max(a, b) + 256);
}

// records already in F.d_raw -> F.d_out[0..*n_out) (then F.d_vout with a voxel leaf); *out_dev = the cloud to download
int extract_edges(Ctx* c, uint32_t n, uint32_t stride, uint32_t toff, uint32_t roff, bool aligned, const so_edge_opts& o, const float4** out_dev,
                  uint32_t* n_out) {
    Ctx::Feat& F = c->feat;
    cudaStream_t st = c->stream;
    const uint32_t grid = (n + 255) / 256;
    const float min_r2 = o.min_range * o.min_range;
    uint32_t* ctl = F.d_ring + 3 * kRings;
    SO_CUDA_TRY(cudaMemsetAsync(ctl, 0, 4 * sizeof(uint32_t), st));
    if (aligned) k_edge_keys<true><<<grid, 256, 0, st>>>(F.d_raw, n, stride, toff, roff, min_r2, F.d_keys[0], F.d_vals[0]);
    else k_edge_keys<false><<<grid, 256, 0, st>>>(F.d_raw, n, stride, toff, roff, min_r2, F.d_keys[0], F.d_vals[0]);
    size_t tmp = F.d_tmp.cap();
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(F.d_tmp, tmp, F.d_keys[0].get(), F.d_keys[1].get(), F.d_vals[0].get(), F.d_vals[1].get(), int(n), 0, 49, st));
    if (aligned) k_edge_rings<true><<<grid, 256, 0, st>>>(F.d_raw, n, stride, toff, F.d_keys[1], F.d_vals[1], F.d_pts, F.d_ring, F.d_excl, F.d_sel);
    else k_edge_rings<false><<<grid, 256, 0, st>>>(F.d_raw, n, stride, toff, F.d_keys[1], F.d_vals[1], F.d_pts, F.d_ring, F.d_excl, F.d_sel);
    k_edge_curv<<<grid, 256, 0, st>>>(F.d_pts, F.d_keys[1], n, F.d_ring, o.edge_threshold, F.d_excl, F.d_reach, F.d_keys[0], F.d_vals[0]);
    tmp = F.d_tmp.cap();
    SO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(F.d_tmp, tmp, F.d_keys[0].get(), F.d_keys[1].get(), F.d_vals[0].get(), F.d_vals[1].get(), int(n), 0, kCandBits + 1, st));
    k_edge_walk<<<kWalkBlocks, kWalkThreads, 0, st>>>(F.d_keys[1], F.d_vals[1], n, F.d_ring, F.d_excl, F.d_reach, F.d_sel, o.max_per_sector);
    tmp = F.d_tmp.cap();
    SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(F.d_tmp, tmp, F.d_sel.get(), F.d_rank.get(), int(n), st));
    k_edge_scatter<<<grid, 256, 0, st>>>(F.d_pts, F.d_sel, F.d_rank, n, F.d_out, ctl + 1);
    c->launches += 7;            // five kernels, two sorts and a scan counted one each; timed_launch_end counts the eighth
    uint32_t m = 0;
    SO_CUDA_TRY(cudaMemcpyAsync(&m, ctl + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    *out_dev = F.d_out;
    *n_out = m;
    if (o.voxel_leaf > 0.f && m) {
        const VoxelBufs vb{F.d_keys[0], F.d_keys[1], F.d_vals[0], F.d_vals[1], F.d_tmp, F.d_tmp.cap()};
        const int rc = cloud_voxel_filter(c, F.d_out, m, o.voxel_leaf, vb, F.d_vout, n_out);
        if (rc) return rc;
        *out_dev = F.d_vout;
    }
    return SO_OK;
}

}  // namespace

}  // namespace so

using namespace so;

extern "C" {

int so_scan_extract_edges(so_ctx* ctx, const void* points, size_t n, size_t stride, size_t toff, size_t roff, const so_edge_opts* opts,
                          float* out_xyzi, size_t cap, size_t* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || (!points && n) || !n_out || (!out_xyzi && cap)) return fail(SO_ERR_ARG, "bad args");
    if (stride < 12 || stride > UINT32_MAX || toff + 4 > stride || roff + 2 > stride) return fail(SO_ERR_ARG, "the record stride does not hold x, y, z, the time and the ring");
    if (toff < 12 || roff < 12) return fail(SO_ERR_ARG, "the time or the ring overlaps x, y, z");
    if (toff < roff + 2 && roff < toff + 4) return fail(SO_ERR_ARG, "the time and the ring overlap");
    so_edge_opts o = opts ? *opts : so_edge_opts{};
    for (float v : {o.min_range, o.edge_threshold, o.voxel_leaf})
        if (!std::isfinite(v) || v < 0.f) return fail(SO_ERR_ARG, "so_edge_opts: min_range, edge_threshold and voxel_leaf must be finite and >= 0");
    if (o.max_per_sector < 0) return fail(SO_ERR_ARG, "so_edge_opts: max_per_sector must be >= 0");
    if (o.edge_threshold == 0.f) o.edge_threshold = 0.1f;
    if (o.max_per_sector == 0) o.max_per_sector = 20;
    if (n > c->scan_cap) return fail(SO_ERR_CAPACITY, "cloud larger than the scan buffers (max_scan_points)");
    *n_out = 0;
    if (n == 0) return SO_OK;
    SO_CUDA_TRY(cudaSetDevice(c->device));
    int rc = features_reserve(c, n, n * stride);
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemcpyAsync(c->feat.d_raw, points, n * stride, cudaMemcpyHostToDevice, c->stream));
    count_h2d(c, n * stride);
    const bool aligned = stride % 4 == 0 && toff % 4 == 0 && roff % 2 == 0;
    const float4* out_dev = nullptr;
    uint32_t m = 0;
    timed_launch_begin(c);
    rc = extract_edges(c, uint32_t(n), uint32_t(stride), uint32_t(toff), uint32_t(roff), aligned, o, &out_dev, &m);
    timed_launch_end(c, 3, 1);
    if (rc) return rc;
    *n_out = m;
    const size_t ncopy = std::min<size_t>(m, cap);
    if (ncopy) {
        SO_CUDA_TRY(cudaMemcpyAsync(out_xyzi, out_dev, ncopy * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
        count_d2h(c, ncopy * sizeof(float4));
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    return SO_OK;
}

}  // extern "C"

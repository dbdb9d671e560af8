// so_reloc.cu -- global localization search (so_localize_global*): occupancy bitmap of the surf map (and of its block archive, read
// in place, for whole_map searches), cube dilation, the occupancy pyramid, and the branch-and-bound scoring and traversal of x/y/z
// voxel shifts x yaw steps of the scan.  The host side (score-point selection, suppression, refinement through register_core)
// lives in so_global.cu.
//
// Everything here is integer-valued once a point has been put into a voxel, and the voxel of a point is computed with
// explicitly rounded FP64 operations (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn: no FMA contraction), so a numpy
// restatement reproduces every score exactly.
#include <cub/cub.cuh>

#include "so_ctx.cuh"

namespace so {

namespace {

// qrot (so_internal.cuh) with every operation rounded on its own, in the same order
__device__ __forceinline__ void qrot_rn(const double q[4], const double v[3], double o[3]) {
    double ux = __dsub_rn(__dmul_rn(q[1], v[2]), __dmul_rn(q[2], v[1]));
    double uy = __dsub_rn(__dmul_rn(q[2], v[0]), __dmul_rn(q[0], v[2]));
    double uz = __dsub_rn(__dmul_rn(q[0], v[1]), __dmul_rn(q[1], v[0]));
    ux = __dadd_rn(ux, ux); uy = __dadd_rn(uy, uy); uz = __dadd_rn(uz, uz);
    o[0] = __dadd_rn(__dadd_rn(v[0], __dmul_rn(q[3], ux)), __dsub_rn(__dmul_rn(q[1], uz), __dmul_rn(q[2], uy)));
    o[1] = __dadd_rn(__dadd_rn(v[1], __dmul_rn(q[3], uy)), __dsub_rn(__dmul_rn(q[2], ux), __dmul_rn(q[0], uz)));
    o[2] = __dadd_rn(__dadd_rn(v[2], __dmul_rn(q[3], uz)), __dsub_rn(__dmul_rn(q[0], uy), __dmul_rn(q[1], ux)));
}

// The voxel of a score point rotated by a hypothesis yaw's quaternion, relative to the hypothesis translation:
// floor(qrot(q, v) / res) per axis: the entries of the branch-and-bound offset table.
__device__ __forceinline__ int3 reloc_voxel(const float4 v, const double q[4], double res) {
    const double vd[3] = {double(v.x), double(v.y), double(v.z)};
    double r[3];
    qrot_rn(q, vd, r);
    return make_int3(int(floor(__ddiv_rn(r[0], res))), int(floor(__ddiv_rn(r[1], res))), int(floor(__ddiv_rn(r[2], res))));
}

// One pass of the separable cube dilation, one thread per bitmap word: axis 0 ORs the word shifted by 1..d bits both ways (with the
// neighbouring words' carries), axes 1 and 2 OR the words d rows / planes away.  The padding bits past bx stay zero.
__global__ void __launch_bounds__(256) k_reloc_dilate(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, RelocGrid g, int d, int axis) {
    const size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const size_t total = size_t(g.by) * g.bz * g.wpr;
    if (idx >= total) return;
    const uint32_t wi = uint32_t(idx % g.wpr);
    const size_t row = idx / g.wpr;
    uint32_t r = in[idx];
    if (axis == 0) {
        const uint32_t cur = r, prev = wi ? in[idx - 1] : 0u, next = wi + 1 < uint32_t(g.wpr) ? in[idx + 1] : 0u;
        for (int s = 1; s <= d; ++s) r |= (cur >> s) | (next << (32 - s)) | (cur << s) | (prev >> (32 - s));
        if (wi + 1 == uint32_t(g.wpr) && (g.bx & 31)) r &= (1u << (g.bx & 31)) - 1u;
    } else if (axis == 1) {
        const int y = int(row % g.by);
        for (int s = -d; s <= d; ++s)
            if (s && y + s >= 0 && y + s < g.by) r |= in[idx + ptrdiff_t(s) * g.wpr];
    } else {
        const int z = int(row / g.by);
        for (int s = -d; s <= d; ++s)
            if (s && z + s >= 0 && z + s < g.bz) r |= in[idx + ptrdiff_t(s) * g.by * g.wpr];
    }
    out[idx] = r;
}

// ---------------------------------------------------------------------------------------------- branch and bound
// Bounding box of the surf store: per-thread min / max, a warp reduction, one atomic per warp and axis.
__global__ void __launch_bounds__(256) k_map_bounds(const float4* __restrict__ pts, uint32_t n, uint32_t* __restrict__ b) {
    uint32_t lo[3] = {~0u, ~0u, ~0u}, hi[3] = {0u, 0u, 0u};
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 p = pts[i];
        const uint32_t v[3] = {float_order(p.x), float_order(p.y), float_order(p.z)};
        for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], v[a]); hi[a] = max(hi[a], v[a]); }
    }
    for (int a = 0; a < 3; ++a) {
        lo[a] = __reduce_min_sync(0xffffffffu, lo[a]);
        hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
    }
    if ((threadIdx.x & 31) == 0)
        for (int a = 0; a < 3; ++a) { atomicMin(b + a, lo[a]); atomicMax(b + 3 + a, hi[a]); }
}

// The box voxel of a map coordinate along one axis, floor((m - lo) / res), every operation rounded on its own.  Every raster goes
// through it, so the window's points and the archive's land in the same voxels.
__device__ __forceinline__ double box_voxel(float m, double lo, double res) { return floor(__ddiv_rn(__dsub_rn(double(m), lo), res)); }

// One thread per surf-store point: the box voxel per axis; points inside the window W set their bit, shifted to W's origin.
__global__ void __launch_bounds__(256) k_bnb_raster(const float4* __restrict__ pts, uint32_t n, RelocGrid g, BnbPyramid w, uint32_t* __restrict__ bits) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[i];
    const double fx = box_voxel(p.x, g.lo[0], g.res);
    const double fy = box_voxel(p.y, g.lo[1], g.res);
    const double fz = box_voxel(p.z, g.lo[2], g.res);
    if (!(fx >= double(w.x0) && fx < double(w.x0 + w.wx) && fy >= double(w.y0) && fy < double(w.y0 + w.wy) &&
          fz >= double(w.z0) && fz < double(w.z0 + w.wz))) return;
    const uint32_t x = uint32_t(fx) - uint32_t(w.x0), y = uint32_t(fy) - uint32_t(w.y0), z = uint32_t(fz) - uint32_t(w.z0);
    atomicOr(bits + (size_t(z) * w.wy + y) * w.wpr[0] + (x >> 5), 1u << (x & 31));
}

// The archive's pool read in place, segment by segment (the walk of k_seg_gather): CTA (s, y) takes every gridDim.y-th run of
// blockDim.x points of live segment s, so that a large block spreads over several CTAs.  The pool's holes (restored blocks, stale
// points) are never read.  Bounds: k_map_bounds' reduction over those points.
__global__ void __launch_bounds__(256) k_seg_bounds(const float4* __restrict__ pool, const GatherSeg* __restrict__ segs, uint32_t* __restrict__ b) {
    const GatherSeg s = segs[blockIdx.x];
    uint32_t lo[3] = {~0u, ~0u, ~0u}, hi[3] = {0u, 0u, 0u};
    for (uint32_t j = blockIdx.y * blockDim.x + threadIdx.x; j < s.n; j += gridDim.y * blockDim.x) {
        const float4 p = pool[s.src + j];
        const uint32_t v[3] = {float_order(p.x), float_order(p.y), float_order(p.z)};
        for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], v[a]); hi[a] = max(hi[a], v[a]); }
    }
    for (int a = 0; a < 3; ++a) {
        lo[a] = __reduce_min_sync(0xffffffffu, lo[a]);
        hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
    }
    if ((threadIdx.x & 31) == 0)
        for (int a = 0; a < 3; ++a) { atomicMin(b + a, lo[a]); atomicMax(b + 3 + a, hi[a]); }
}

// Raster: k_bnb_raster's voxel and window test for every point of the live segments
__global__ void __launch_bounds__(256) k_seg_raster(const float4* __restrict__ pool, const GatherSeg* __restrict__ segs, RelocGrid g, BnbPyramid w,
                                                    uint32_t* __restrict__ bits) {
    const GatherSeg s = segs[blockIdx.x];
    for (uint32_t j = blockIdx.y * blockDim.x + threadIdx.x; j < s.n; j += gridDim.y * blockDim.x) {
        const float4 p = pool[s.src + j];
        const double fx = box_voxel(p.x, g.lo[0], g.res);
        const double fy = box_voxel(p.y, g.lo[1], g.res);
        const double fz = box_voxel(p.z, g.lo[2], g.res);
        if (!(fx >= double(w.x0) && fx < double(w.x0 + w.wx) && fy >= double(w.y0) && fy < double(w.y0 + w.wy) &&
              fz >= double(w.z0) && fz < double(w.z0 + w.wz))) continue;
        const uint32_t x = uint32_t(fx) - uint32_t(w.x0), y = uint32_t(fy) - uint32_t(w.y0), z = uint32_t(fz) - uint32_t(w.z0);
        atomicOr(bits + (size_t(z) * w.wy + y) * w.wpr[0] + (x >> 5), 1u << (x & 31));
    }
}

// Bits x .. x+31 of a row of wpr words (x may be negative); bits outside the row read 0.
__device__ __forceinline__ uint32_t row_bits(const uint32_t* __restrict__ row, int wpr, int x) {
    const int q = x >> 5, s = x & 31;
    const uint32_t a = (q >= 0 && q < wpr) ? row[q] : 0u;
    const uint32_t b = (q + 1 >= 0 && q + 1 < wpr) ? row[q + 1] : 0u;
    return s ? (a >> s) | (b << (32 - s)) : a;
}

// Level L+1 from level L, one thread per word: B_{L+1}(x, y) = B_L(x, y) | B_L(x+s, y) | B_L(x, y+s) | B_L(x+s, y+s) with s = 2^L.
// Level L+1 starts s voxels lower than level L on both axes, so its word w reads level L at bit 32w - s and (word-aligned) 32w.
__global__ void __launch_bounds__(256) k_bnb_level(BnbPyramid p, int L, uint32_t* __restrict__ pyr) {
    const int s = 1 << L;
    const int xw = p.wx + 2 * s - 1, yw = p.wy + 2 * s - 1, ys = p.wy + s - 1;
    const int wpr = p.wpr[L + 1], wprs = p.wpr[L];
    const size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= size_t(p.wz) * yw * wpr) return;
    const int w = int(idx % wpr);
    const size_t row = idx / wpr;
    const int y = int(row % yw), z = int(row / yw);
    const uint32_t* src = pyr + p.off[L];
    uint32_t r = 0;
    for (int ly = y - s; ly <= y; ly += s) {
        if (ly < 0 || ly >= ys) continue;
        const uint32_t* srow = src + (size_t(z) * ys + ly) * wprs;
        r |= row_bits(srow, wprs, 32 * w - s) | row_bits(srow, wprs, 32 * w);
    }
    if (w + 1 == wpr && (xw & 31)) r &= (1u << (xw & 31)) - 1u;
    pyr[p.off[L + 1] + idx] = r;
}

// Offset table, one thread per (yaw m, score point): the box voxel {x, y} of hypothesis shift (0, 0, 0), and its z relative to W's
// first plane (z shift k reads plane z + k of W).
__global__ void __launch_bounds__(256) k_bnb_offsets(const float4* __restrict__ spts, int n_pts, const double* __restrict__ q_yaw, RelocGrid g,
                                                     int z0, int4* __restrict__ off) {
    const size_t t = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= size_t(g.nyaw) * n_pts) return;
    const int p = int(t % n_pts), m = int(t / n_pts);
    const double q[4] = {q_yaw[4 * m], q_yaw[4 * m + 1], q_yaw[4 * m + 2], q_yaw[4 * m + 3]};
    const int3 w = reloc_voxel(spts[p], q, g.res);
    off[t] = make_int4(w.x + g.e, w.y + g.e, w.z + g.e - z0, 0);
}

// Node bound, one warp per node, lanes striding over the score points, one integer warp sum:
// U = sum_p B_L[o_p + (i0, j0)], the key (65535 - U) << 32 | lin(m, k, j0, i0).  Statistics: one atomic per CTA.
__global__ void __launch_bounds__(256) k_bnb_score(RelocGrid g, BnbPyramid p, const uint32_t* __restrict__ pyr, const int4* __restrict__ off,
                                                   int n_pts, int level, const uint64_t* __restrict__ parents, uint64_t first, uint32_t n,
                                                   BnbCtl* __restrict__ ctl, uint64_t* __restrict__ out) {
    __shared__ unsigned long long s_cnt[2];
    if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t kstar = ctl->kstar;
    const int lane = threadIdx.x & 31;
    const int s = 1 << level;
    const int ox = p.x0 - (s - 1), oy = p.y0 - (s - 1), xw = p.wx + s - 1, yw = p.wy + s - 1, wpr = p.wpr[level];
    const uint32_t* bits = pyr + p.off[level];
    const uint32_t nx = uint32_t(g.nx), ny = uint32_t(g.ny), nz = uint32_t(g.nz);
    const uint32_t nbx = (nx + uint32_t(s) - 1) >> level, nby = (ny + uint32_t(s) - 1) >> level;
    unsigned long long scored = 0, discarded = 0;
    for (uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < n; c += (gridDim.x * blockDim.x) >> 5) {
        uint32_t i0, j0, k, m;
        bool live = true;
        if (parents) {
            const uint64_t pk = parents[c >> 2];
            uint32_t lin = uint32_t(pk);
            i0 = lin % nx + ((c & 1u) << level); lin /= nx;
            j0 = lin % ny + (((c >> 1) & 1u) << level); lin /= ny;
            k = lin % nz; m = lin / nz;
            live = pk <= kstar && i0 < nx && j0 < ny;
        } else {
            uint64_t r = first + c;
            i0 = uint32_t(r % nbx) << level; r /= nbx;
            j0 = uint32_t(r % nby) << level; r /= nby;
            k = uint32_t(r % nz); m = uint32_t(r / nz);
        }
        uint64_t key = kBnbNone;
        if (live) {                                                 // warp-uniform
            const int4* o = off + size_t(m) * size_t(n_pts);
            uint32_t cnt = 0;
            for (int q = lane; q < n_pts; q += 32) {
                const int4 v = __ldg(o + q);
                const int x = v.x + int(i0) - ox, y = v.y + int(j0) - oy, z = v.z + int(k);
                if (uint32_t(z) < uint32_t(p.wz) && uint32_t(x) < uint32_t(xw) && uint32_t(y) < uint32_t(yw))
                    cnt += (__ldg(bits + (size_t(z) * yw + y) * wpr + (x >> 5)) >> (x & 31)) & 1u;
            }
            cnt = __reduce_add_sync(0xffffffffu, cnt);
            const uint64_t lin = ((uint64_t(m) * nz + k) * ny + j0) * nx + i0;
            key = (uint64_t(65535u - cnt) << 32) | lin;
            ++scored;
            if (key > kstar) { key = kBnbNone; ++discarded; }
        }
        if (lane == 0) out[c] = key;
    }
    if (lane == 0 && scored) { atomicAdd(&s_cnt[0], scored); atomicAdd(&s_cnt[1], discarded); }
    __syncthreads();
    if (threadIdx.x == 0 && s_cnt[0]) { atomicAdd(&ctl->scored[level], s_cnt[0]); atomicAdd(&ctl->discarded[level], s_cnt[1]); }
}

// One thread per level: binary search of the first key above K* in the level's sorted, not yet expanded nodes.
__global__ void k_bnb_trim(BnbTrim t, const uint64_t* __restrict__ nodes, BnbCtl* __restrict__ ctl) {
    const int l = threadIdx.x;
    if (l < 1 || l > t.lmax) return;
    const uint64_t ks = ctl->kstar;
    const uint64_t* a = nodes + t.base[l];
    uint64_t lo = t.head[l], hi = t.cnt[l];
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (a[mid] <= ks) lo = mid + 1; else hi = mid;
    }
    ctl->cnt[l] = lo;
    hi = t.cnt[l];                              // the nodes cut here, not those already discarded when scored (kBnbNone, at the end)
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (a[mid] != kBnbNone) lo = mid + 1; else hi = mid;
    }
    ctl->discarded[l] += lo - ctl->cnt[l];
}

}  // namespace

uint32_t* launch_reloc_dilate(const RelocGrid& g, int d, uint32_t* a, uint32_t* b, cudaStream_t st) {
    const size_t total = size_t(g.by) * g.bz * g.wpr;
    const uint32_t grid = uint32_t((total + 255) / 256);
    k_reloc_dilate<<<grid, 256, 0, st>>>(a, b, g, d, 0);
    k_reloc_dilate<<<grid, 256, 0, st>>>(b, a, g, d, 1);
    k_reloc_dilate<<<grid, 256, 0, st>>>(a, b, g, d, 2);
    return b;
}

void launch_map_bounds(const float4* pts, uint32_t n, uint32_t* d_bounds, cudaStream_t st) {
    if (n) k_map_bounds<<<std::min<uint32_t>((n + 255) / 256, 1024), 256, 0, st>>>(pts, n, d_bounds);
}

void launch_bnb_raster(const float4* pts, uint32_t n, const RelocGrid& g, const BnbPyramid& p, uint32_t* bits, cudaStream_t st) {
    if (n) k_bnb_raster<<<(n + 255) / 256, 256, 0, st>>>(pts, n, g, p, bits);
}

// CTAs per segment: enough for the largest one at 8 points per thread, at most 64
static dim3 seg_grid(uint32_t n_segs, uint32_t max_n) { return dim3(n_segs, std::min<uint32_t>(64, std::max<uint32_t>(1, (max_n + 2047) / 2048))); }

void launch_seg_bounds(const float4* pool, const GatherSeg* segs, uint32_t n_segs, uint32_t max_n, uint32_t* d_bounds, cudaStream_t st) {
    if (n_segs) k_seg_bounds<<<seg_grid(n_segs, max_n), 256, 0, st>>>(pool, segs, d_bounds);
}

void launch_seg_raster(const float4* pool, const GatherSeg* segs, uint32_t n_segs, uint32_t max_n, const RelocGrid& g, const BnbPyramid& p,
                       uint32_t* bits, cudaStream_t st) {
    if (n_segs) k_seg_raster<<<seg_grid(n_segs, max_n), 256, 0, st>>>(pool, segs, g, p, bits);
}

void launch_bnb_levels(const BnbPyramid& p, uint32_t* pyr, cudaStream_t st) {
    for (int L = 0; L < p.lmax; ++L) {
        const size_t words = size_t(p.wz) * size_t(p.wy + (2 << L) - 1) * size_t(p.wpr[L + 1]);
        k_bnb_level<<<uint32_t((words + 255) / 256), 256, 0, st>>>(p, L, pyr);
    }
}

void launch_bnb_offsets(const float4* spts, int n_pts, const double* d_q, const RelocGrid& g, const BnbPyramid& p, int4* off, cudaStream_t st) {
    const size_t total = size_t(g.nyaw) * size_t(n_pts);
    if (total) k_bnb_offsets<<<uint32_t((total + 255) / 256), 256, 0, st>>>(spts, n_pts, d_q, g, p.z0, off);
}

void launch_bnb_score(const RelocGrid& g, const BnbPyramid& p, const uint32_t* pyr, const int4* off, int n_pts, int level,
                      const uint64_t* parents, uint64_t first, uint32_t n, BnbCtl* ctl, uint64_t* out, cudaStream_t st) {
    if (n) k_bnb_score<<<std::min<uint32_t>((n + 7) / 8, 132 * 16), 256, 0, st>>>(g, p, pyr, off, n_pts, level, parents, first, n, ctl, out);
}

void launch_bnb_trim(const BnbTrim& t, const uint64_t* nodes, BnbCtl* ctl, cudaStream_t st) {
    k_bnb_trim<<<1, kBnbLevels, 0, st>>>(t, nodes, ctl);
}

// the node keys: score bits 32..47, index bits 0..31, and bit 48 that only kBnbNone sets
size_t bnb_sort_bytes(size_t n) {
    size_t b = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, b, (const uint64_t*)nullptr, (uint64_t*)nullptr, int(n), 0, 49);
    return b;
}

int bnb_sort(void* tmp, size_t tmp_bytes, const uint64_t* in, uint64_t* out, size_t n, cudaStream_t st) {
    SO_CUDA_TRY(cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, in, out, int(n), 0, 49, st));
    return SO_OK;
}

}  // namespace so

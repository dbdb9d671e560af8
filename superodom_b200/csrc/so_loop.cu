// so_loop.cu -- loop detection over the keyframe store (so_loop_candidates, so_keyframe_descriptors): a Scan Context descriptor per
// keyframe (G. Kim, A. Kim, IROS 2018) and an exhaustive, rotation-aware search of a query against every eligible keyframe.
//
// No reference counterpart.  Three kernels (DESIGN.md, "Loop detection"):
//   - k_loop_describe: one CTA per keyframe.  The image is built in shared memory with an atomicMax on the bits of the float cell
//     values (all >= 0, so the bits order as the values and the image does not depend on the order of the atomics), then written out
//     with its column norms.
//   - k_loop_search: one CTA per (query, tile of kLoopTile candidates), the query image and norms in shared memory, a warp per
//     candidate with its lanes over the shifts.  Writes each pair's best (distance, shift, n_pairs) to a pair table.
//   - k_loop_topk: one CTA per query, k rounds of a block-wide minimum of (distance, id) above the last one taken.
// The arithmetic is FP64 without contractible multiply-adds, in a fixed order, so that a numpy restatement takes the same roundings.
#include <algorithm>
#include <cfloat>
#include <cmath>

#include "so_ctx.cuh"

namespace so {

constexpr double kPiL = 3.141592653589793;
constexpr int kLoopMaxRings = 64, kLoopMaxSectors = 360, kLoopMaxK = 64;
constexpr int kLoopSearchThreads = 256;                       // 8 warps
constexpr int kLoopTile = 32;                                 // candidates per search CTA: 4 per warp
constexpr int kLoopDescThreads = 512;
constexpr size_t kLoopPairCap = size_t(1) << 20;              // pair-table entries of one query chunk (16 MiB)

struct LoopGrid { int32_t rings, sectors; double max_range, h, sector_w; };
struct DescSeg { uint64_t first; uint32_t n, id; double L[9]; };   // keyframe id: pool[first .. first + n), levelled by L (row-major)
struct LoopPair { double d; int32_t id, shift, n_pairs, pad; };
struct LoopQuery { int32_t q, lo, count; };                        // query q's candidates: ids [lo, lo + count) but q

__device__ __forceinline__ double row3(const double* L, int r, double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dmul_rn(L[3 * r], x), __dmul_rn(L[3 * r + 1], y)), __dmul_rn(L[3 * r + 2], z));
}

__global__ void __launch_bounds__(kLoopDescThreads) k_loop_describe(const float4* __restrict__ pool, const DescSeg* __restrict__ segs,
                                                                    LoopGrid g, float* __restrict__ desc, double* __restrict__ norm) {
    extern __shared__ uint32_t img[];                          // [rings][sectors] float bits
    const DescSeg& s = segs[blockIdx.x];
    const int cells = g.rings * g.sectors;
    for (int i = threadIdx.x; i < cells; i += blockDim.x) img[i] = 0u;
    __syncthreads();
    const float4* pts = pool + s.first;
    for (uint32_t i = threadIdx.x; i < s.n; i += blockDim.x) {
        const float4 p = pts[i];
        if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) continue;
        const double x = p.x, y = p.y, z = p.z;
        const double vx = row3(s.L, 0, x, y, z), vy = row3(s.L, 1, x, y, z), vz = row3(s.L, 2, x, y, z);
        const double rho = hypot(vx, vy);
        if (!(rho < g.max_range)) continue;
        const int ring = min(int(floor(__dmul_rn(__ddiv_rn(rho, g.max_range), double(g.rings)))), g.rings - 1);
        double az = atan2(vy, vx);
        if (az >= kPiL) az = __dsub_rn(az, 2.0 * kPiL);              // [-pi, pi), as free_pixel folds it
        const int sector = min(int(floor(__ddiv_rn(__dadd_rn(az, kPiL), g.sector_w))), g.sectors - 1);
        const float v = __double2float_rn(__dadd_rn(vz, g.h));
        if (v > 0.f) atomicMax(img + ring * g.sectors + sector, __float_as_uint(v));
    }
    __syncthreads();
    float* out = desc + size_t(s.id) * cells;
    for (int i = threadIdx.x; i < cells; i += blockDim.x) out[i] = __uint_as_float(img[i]);
    for (int j = threadIdx.x; j < g.sectors; j += blockDim.x) {
        double acc = 0.0;
        for (int r = 0; r < g.rings; ++r) {
            const double v = __uint_as_float(img[r * g.sectors + j]);
            acc = __dadd_rn(acc, __dmul_rn(v, v));
        }
        norm[size_t(s.id) * g.sectors + j] = sqrt(acc);
    }
}

// pairs[qi * stride + u]: query queries[blockIdx.y] against every candidate b of its range [lo, lo + count) but itself
__global__ void __launch_bounds__(kLoopSearchThreads) k_loop_search(const float* __restrict__ desc, const double* __restrict__ norm,
                                                                    const LoopQuery* __restrict__ queries, int rings, int sectors,
                                                                    LoopPair* __restrict__ pairs, size_t stride) {
    extern __shared__ double sm[];
    double* qn = sm;                                           // [sectors]
    float* qd = reinterpret_cast<float*>(sm + sectors);        // [rings][sectors]
    const LoopQuery Q = queries[blockIdx.y];
    const int32_t q = Q.q, m = Q.count;
    const int32_t first = blockIdx.x * kLoopTile;
    if (first >= m) return;
    const int cells = rings * sectors;
    for (int i = threadIdx.x; i < cells; i += blockDim.x) qd[i] = desc[size_t(q) * cells + i];
    for (int i = threadIdx.x; i < sectors; i += blockDim.x) qn[i] = norm[size_t(q) * sectors + i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int t = warp; t < kLoopTile; t += kLoopSearchThreads / 32) {
        const int32_t u = first + t;
        if (u >= m) break;
        const int32_t b = Q.lo + u;
        if (b == q) continue;                                  // k_loop_topk skips it
        const float* cd = desc + size_t(b) * cells;
        const double* cn = norm + size_t(b) * sectors;
        double best = HUGE_VAL;
        int best_s = 0, best_n = 0;
        for (int s = lane; s < sectors; s += 32) {
            double sum = 0.0;
            int np = 0;
            int col = s;
            for (int j = 0; j < sectors; ++j, col = (col + 1 == sectors) ? 0 : col + 1) {
                const double na = qn[j], nb = __ldg(cn + col);
                if (na == 0.0 || nb == 0.0) continue;
                double dot = 0.0;
                for (int r = 0; r < rings; ++r)
                    dot = __dadd_rn(dot, __dmul_rn(double(qd[r * sectors + j]), double(__ldg(cd + r * sectors + col))));
                sum = __dadd_rn(sum, __ddiv_rn(dot, __dmul_rn(na, nb)));
                ++np;
            }
            const double d = np ? __dsub_rn(1.0, __ddiv_rn(sum, double(np))) : 1.0;
            if (d < best) { best = d; best_s = s; best_n = np; }
        }
        for (int o = 16; o; o >>= 1) {                         // (distance, shift) minimum over the lanes
            const double od = __shfl_xor_sync(0xffffffffu, best, o);
            const int os = __shfl_xor_sync(0xffffffffu, best_s, o), on = __shfl_xor_sync(0xffffffffu, best_n, o);
            if (od < best || (od == best && os < best_s)) { best = od; best_s = os; best_n = on; }
        }
        if (lane == 0) pairs[size_t(blockIdx.y) * stride + u] = LoopPair{best, b, best_s, best_n, 0};
    }
}

__device__ __forceinline__ bool key_less(double d0, int32_t i0, double d1, int32_t i1) { return d0 < d1 || (d0 == d1 && i0 < i1); }

// top[qi * k .. + k): the k smallest (distance, id) of the query's row, ascending; id -1 past the eligible count
__global__ void __launch_bounds__(256) k_loop_topk(const LoopPair* __restrict__ pairs, size_t stride, const LoopQuery* __restrict__ queries,
                                                   int k, LoopPair* __restrict__ top) {
    __shared__ double wd[8];
    __shared__ int32_t wi[8];
    __shared__ LoopPair last;
    const LoopQuery Q = queries[blockIdx.x];
    const LoopPair* row = pairs + size_t(blockIdx.x) * stride;
    LoopPair* out = top + size_t(blockIdx.x) * k;
    double ld = -HUGE_VAL;
    int32_t li = -1;
    for (int t = 0; t < k; ++t) {
        double bd = HUGE_VAL;
        int32_t bi = INT32_MAX;
        for (int32_t j = threadIdx.x; j < Q.count; j += blockDim.x) {
            const int32_t b = Q.lo + j;
            if (b == Q.q) continue;
            const double d = row[j].d;
            if (key_less(ld, li, d, b) && key_less(d, b, bd, bi)) { bd = d; bi = b; }
        }
        for (int o = 16; o; o >>= 1) {
            const double od = __shfl_xor_sync(0xffffffffu, bd, o);
            const int32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (key_less(od, oi, bd, bi)) { bd = od; bi = oi; }
        }
        if ((threadIdx.x & 31) == 0) { wd[threadIdx.x >> 5] = bd; wi[threadIdx.x >> 5] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < int(blockDim.x >> 5); ++w)
                if (key_less(wd[w], wi[w], bd, bi)) { bd = wd[w]; bi = wi[w]; }
            last = bi == INT32_MAX ? LoopPair{1.0, -1, 0, 0, 0} : row[bi - Q.lo];
            out[t] = last;
        }
        __syncthreads();
        if (last.id < 0) {                                     // fewer than k eligible: the rest are unused slots
            for (int u = t + 1 + threadIdx.x; u < k; u += blockDim.x) out[u] = last;
            return;
        }
        ld = last.d; li = last.id;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------------------------ host side
static void loop_defaults(so_loop_opts* o) {
    *o = so_loop_opts{};
    o->rings = 20; o->sectors = 60; o->max_range = 80.0; o->height_offset = 2.0; o->exclude_recent = 30;
}

static int loop_check(const Ctx* c, const so_loop_opts* o) {
    if (!o) return fail(SO_ERR_ARG, "loop detection: NULL opts");
    if (!c->kf.cap_frames) return fail(SO_ERR_ARG, "loop detection needs a keyframe store (so_keyframe_reserve)");
    if (o->rings < 1 || o->rings > kLoopMaxRings) return fail(SO_ERR_ARG, "so_loop_opts: rings must be in 1..64");
    if (o->sectors < 2 || o->sectors > kLoopMaxSectors) return fail(SO_ERR_ARG, "so_loop_opts: sectors must be in 2..360");
    if (!(std::isfinite(o->max_range) && o->max_range > 0)) return fail(SO_ERR_ARG, "so_loop_opts: max_range must be finite and positive");
    if (!std::isfinite(o->height_offset)) return fail(SO_ERR_ARG, "so_loop_opts: height_offset must be finite");
    if (o->exclude_recent < 0) return fail(SO_ERR_ARG, "so_loop_opts: exclude_recent must be >= 0");
    return SO_OK;
}

static int check_loop_ids(const KeyframeStore& s, const int32_t* ids, size_t n) {
    if (n && !ids) return fail(SO_ERR_ARG, "bad args");
    for (size_t i = 0; i < n; ++i)
        if (ids[i] < 0 || size_t(ids[i]) >= s.frames()) return fail(SO_ERR_ARG, "keyframe id out of range");
    return SO_OK;
}

static size_t cells_of(const so_loop_opts& o) { return size_t(o.rings) * size_t(o.sectors); }

static bool same_descriptor(const so_loop_opts& a, const so_loop_opts& b) {
    return a.rings == b.rings && a.sectors == b.sectors && a.max_range == b.max_range && a.height_offset == b.height_offset;
}

int loop_table_alloc(const KeyframeStore& s, size_t cap_frames, DeviceBuffer<float>* desc, DeviceBuffer<double>* norm) {
    if (!s.desc_opts.rings || !cap_frames) return SO_OK;
    const size_t cells = cells_of(s.desc_opts), sec = size_t(s.desc_opts.sectors), keep = s.frames();   // a table holds cap_frames >= frames
    DeviceBuffer<float> d;
    DeviceBuffer<double> m;
    if (d.reserve(cap_frames * cells) || m.reserve(cap_frames * sec)) {
        cudaGetLastError();
        return fail(SO_ERR_CUDA, "so_keyframe_reserve: cudaMalloc of the loop descriptor table failed");
    }
    if (keep && (cudaMemcpy(d, s.d_desc, keep * cells * sizeof(float), cudaMemcpyDeviceToDevice) != cudaSuccess ||
                 cudaMemcpy(m, s.d_desc_norm, keep * sec * sizeof(double), cudaMemcpyDeviceToDevice) != cudaSuccess))
        return fail(SO_ERR_CUDA, "so_keyframe_reserve: copy of the loop descriptors failed");
    *desc = std::move(d);
    *norm = std::move(m);
    return SO_OK;
}

// Levelling matrix L = Rz(-psi) R of a pose (row-major): R from the normalised quaternion, cos / sin psi as R00 / h and R10 / h with
// h = sqrt(R00^2 + R10^2), so psi = atan2(R10, R00) without a trigonometric call (psi = 0 when h = 0)
static void levelling(const double* pose, double L[9]) {
    const double* q = pose + 3;
    const double nq = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double x = q[0] / nq, y = q[1] / nq, z = q[2] / nq, w = q[3] / nq;
    const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                         2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                         2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
    const double h = std::sqrt(R[0] * R[0] + R[3] * R[3]);
    const double cs = h > 0 ? R[0] / h : 1.0, sn = h > 0 ? R[3] / h : 0.0;
    for (int k = 0; k < 3; ++k) {
        L[k] = cs * R[k] + sn * R[3 + k];
        L[3 + k] = cs * R[3 + k] - sn * R[k];
        L[6 + k] = R[6 + k];
    }
}

static LoopGrid grid_of(const so_loop_opts& o) {
    return LoopGrid{o.rings, o.sectors, o.max_range, o.height_offset, (2.0 * kPiL) / double(o.sectors)};
}

static int loop_events(Ctx* c) {
    for (Event& e : c->kfs.ev_loop) if (!e) { int rc = e.create(); if (rc) return rc; }
    return SO_OK;
}

static double elapsed_ms(cudaEvent_t a, cudaEvent_t b) { float ms = 0.f; cudaEventElapsedTime(&ms, a, b); return double(ms); }

// Every keyframe of ids[0..n) without a valid descriptor for o described (the table first set up for o); *n_described of them
static int loop_describe(Ctx* c, const int32_t* ids, size_t n, const so_loop_opts& o, uint64_t* n_described, double* ms) {
    KeyframeStore& s = c->kf;
    const size_t cells = cells_of(o);
    *n_described = 0; *ms = 0.0;
    if (!s.desc_opts.rings || !same_descriptor(s.desc_opts, o)) {       // other options: every descriptor is invalid
        s.desc_ok.assign(s.desc_ok.size(), 0);
        if (!s.desc_opts.rings || s.desc_opts.rings != o.rings || s.desc_opts.sectors != o.sectors) {
            SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
            s.d_desc.reset(); s.d_desc_norm.reset();                  // at the new size, so the old table goes first
            s.desc_opts = so_loop_opts{};                             // no table until both allocations succeed
            int rc = s.d_desc.reserve(s.cap_frames * cells);
            if (!rc) rc = s.d_desc_norm.reserve(s.cap_frames * size_t(o.sectors));
            if (rc) return rc;
        }
        s.desc_opts = o;
    }
    s.desc_ok.resize(s.frames(), 0);
    std::vector<DescSeg> segs;
    for (size_t i = 0; i < n; ++i) {
        const int32_t id = ids[i];
        if (s.desc_ok[id]) continue;
        s.desc_ok[id] = 2;                                            // listed once
        DescSeg g{};
        g.first = s.off[0][id]; g.n = uint32_t(s.off[0][id + 1] - g.first); g.id = uint32_t(id);
        levelling(s.poses.data() + 7 * size_t(id), g.L);
        segs.push_back(g);
    }
    if (segs.empty()) return SO_OK;
    for (const DescSeg& g : segs) s.desc_ok[g.id] = 0;                // valid only once the kernel has run
    KeyframeScratch& k = c->kfs;
    int rc = k.d_dsegs.reserve(segs.size());
    if (!rc) rc = loop_events(c);
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemcpyAsync(k.d_dsegs, segs.data(), segs.size() * sizeof(DescSeg), cudaMemcpyHostToDevice, c->stream));
    const int smem = int(cells * sizeof(uint32_t));
    SO_CUDA_TRY(cudaFuncSetAttribute(k_loop_describe, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    SO_CUDA_TRY(cudaEventRecord(k.ev_loop[0], c->stream));
    k_loop_describe<<<uint32_t(segs.size()), kLoopDescThreads, smem, c->stream>>>(s.d_pool[0], k.d_dsegs, grid_of(o), s.d_desc, s.d_desc_norm);
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaEventRecord(k.ev_loop[1], c->stream));
    SO_CUDA_TRY(cudaEventSynchronize(k.ev_loop[1]));                  // the segment list's host copy goes out of scope
    c->launches++;
    for (const DescSeg& g : segs) s.desc_ok[g.id] = 1;
    *n_described = segs.size();
    *ms = elapsed_ms(k.ev_loop[0], k.ev_loop[1]);
    return SO_OK;
}

// Each query against its candidates qs[i] (LoopQuery); the pair table of a chunk of queries is as wide as its longest range
static int loop_search(Ctx* c, const std::vector<LoopQuery>& qs, const so_loop_opts& o, int k, so_loop_candidate* out, double* ms) {
    KeyframeStore& s = c->kf;
    KeyframeScratch& ks = c->kfs;
    const size_t n = qs.size();
    size_t max_m = 0;
    for (const LoopQuery& q : qs) max_m = std::max(max_m, size_t(q.count));
    int rc = ks.d_queries.reserve(std::max<size_t>(n, 1));
    if (!rc) rc = ks.d_pairs.reserve(std::max(kLoopPairCap, std::max<size_t>(max_m, 1)));
    if (!rc) rc = ks.d_top.reserve(std::max<size_t>(n * size_t(k), 1));
    if (!rc) rc = loop_events(c);
    if (rc) return rc;
    SO_CUDA_TRY(cudaMemcpyAsync(ks.d_queries, qs.data(), n * sizeof(LoopQuery), cudaMemcpyHostToDevice, c->stream));
    const int smem = int(size_t(o.sectors) * sizeof(double) + cells_of(o) * sizeof(float));
    SO_CUDA_TRY(cudaFuncSetAttribute(k_loop_search, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    SO_CUDA_TRY(cudaEventRecord(ks.ev_loop[2], c->stream));
    for (size_t a = 0; a < n;) {                                      // query chunks whose pair table fits ks.d_pairs
        size_t b = a, stride = 0;
        while (b < n && b - a < 65535) {
            const size_t st = std::max(stride, std::max<size_t>(size_t(qs[b].count), 1));
            if ((b - a + 1) * st > ks.d_pairs.cap()) break;
            stride = st; ++b;
        }
        const uint32_t nq = uint32_t(b - a), tiles = uint32_t((stride + kLoopTile - 1) / kLoopTile);
        k_loop_search<<<dim3(tiles, nq), kLoopSearchThreads, smem, c->stream>>>(s.d_desc, s.d_desc_norm, ks.d_queries + a, o.rings,
                                                                               o.sectors, ks.d_pairs, stride);
        k_loop_topk<<<nq, 256, 0, c->stream>>>(ks.d_pairs, stride, ks.d_queries + a, k, ks.d_top + a * size_t(k));
        c->launches += 2;
        a = b;
    }
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaEventRecord(ks.ev_loop[3], c->stream));
    std::vector<LoopPair> top(n * size_t(k));
    SO_CUDA_TRY(cudaMemcpyAsync(top.data(), ks.d_top, top.size() * sizeof(LoopPair), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    *ms = elapsed_ms(ks.ev_loop[2], ks.ev_loop[3]);
    const double step = (2.0 * kPiL) / double(o.sectors);
    for (size_t i = 0; i < top.size(); ++i) {
        const LoopPair& p = top[i];
        so_loop_candidate& r = out[i];
        r.query = qs[i / size_t(k)].q;
        r.id = p.id;
        r.distance = p.d; r.shift = p.shift; r.n_pairs = p.n_pairs;
        double yaw = double(p.shift) * step;
        if (yaw > kPiL) yaw -= 2.0 * kPiL;
        r.yaw = p.id < 0 ? 0.0 : yaw;
    }
    return SO_OK;
}

}  // namespace so

// =================================================================================================== C ABI
using namespace so;

extern "C" {

void so_loop_opts_defaults(so_loop_opts* opts) { if (opts) loop_defaults(opts); }

int so_loop_candidates(so_ctx* ctx, const int32_t* queries, size_t n, const so_loop_opts* opts, int32_t k, so_loop_candidate* out,
                       so_loop_stats* stats) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    { int rc = loop_check(c, opts); if (rc) return rc; }
    if (k < 1 || k > kLoopMaxK) return fail(SO_ERR_ARG, "so_loop_candidates: k must be in 1..64");
    if (n && !out) return fail(SO_ERR_ARG, "so_loop_candidates: NULL out");
    { int rc = check_loop_ids(c->kf, queries, n); if (rc) return rc; }
    SO_CUDA_TRY(cudaSetDevice(c->device));
    // every keyframe a query is compared with: the queries and ids 0 .. the largest eligible count
    int32_t top = 0;
    std::vector<LoopQuery> qs(n);
    for (size_t i = 0; i < n; ++i) {
        qs[i] = LoopQuery{queries[i], 0, std::max(queries[i] - opts->exclude_recent, 0)};
        top = std::max(top, qs[i].count);
    }
    std::vector<int32_t> need(queries, queries + n);
    for (int32_t i = 0; i < top; ++i) need.push_back(i);
    so_loop_stats st{};
    int rc = loop_describe(c, need.data(), need.size(), *opts, &st.n_described, &st.time_describe_ms);
    if (!rc && n) rc = loop_search(c, qs, *opts, k, out, &st.time_search_ms);
    if (rc) return rc;
    if (stats) *stats = st;
    return SO_OK;
}

int so_loop_candidates_range(so_ctx* ctx, const int32_t* queries, size_t n, const so_loop_opts* opts, int32_t id_begin, int32_t id_end,
                             int32_t k, so_loop_candidate* out, so_loop_stats* stats) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    { int rc = loop_check(c, opts); if (rc) return rc; }
    if (k < 1 || k > kLoopMaxK) return fail(SO_ERR_ARG, "so_loop_candidates_range: k must be in 1..64");
    if (n && !out) return fail(SO_ERR_ARG, "so_loop_candidates_range: NULL out");
    if (id_begin < 0 || id_end < id_begin) return fail(SO_ERR_ARG, "so_loop_candidates_range: the range must have 0 <= id_begin <= id_end");
    if (size_t(id_end) > c->kf.frames()) return fail(SO_ERR_ARG, "so_loop_candidates_range: id_end past the keyframes the store holds");
    { int rc = check_loop_ids(c->kf, queries, n); if (rc) return rc; }
    SO_CUDA_TRY(cudaSetDevice(c->device));
    std::vector<LoopQuery> qs(n);
    for (size_t i = 0; i < n; ++i) qs[i] = LoopQuery{queries[i], id_begin, id_end - id_begin};
    std::vector<int32_t> need(queries, queries + n);
    for (int32_t i = id_begin; i < id_end; ++i) need.push_back(i);
    so_loop_stats st{};
    int rc = loop_describe(c, need.data(), need.size(), *opts, &st.n_described, &st.time_describe_ms);
    if (!rc && n) rc = loop_search(c, qs, *opts, k, out, &st.time_search_ms);
    if (rc) return rc;
    if (stats) *stats = st;
    return SO_OK;
}

int so_keyframe_descriptors(so_ctx* ctx, const int32_t* ids, size_t n, const so_loop_opts* opts, float* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    { int rc = loop_check(c, opts); if (rc) return rc; }
    if (n && !out) return fail(SO_ERR_ARG, "so_keyframe_descriptors: NULL out");
    { int rc = check_loop_ids(c->kf, ids, n); if (rc) return rc; }
    SO_CUDA_TRY(cudaSetDevice(c->device));
    uint64_t described = 0;
    double ms = 0.0;
    int rc = loop_describe(c, ids, n, *opts, &described, &ms);
    if (rc) return rc;
    const size_t cells = cells_of(*opts);
    for (size_t i = 0; i < n; ++i)
        SO_CUDA_TRY(cudaMemcpyAsync(out + i * cells, c->kf.d_desc + size_t(ids[i]) * cells, cells * sizeof(float), cudaMemcpyDeviceToHost,
                                    c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SO_OK;
}

}  // extern "C"

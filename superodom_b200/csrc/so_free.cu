// so_free.cu -- free-space clearing (so_map_clear_free_space*): remove the map points a scan saw clearly past.
//
// No reference counterpart: LocalMap::addSurfPointCloud only adds points, so anything that moved stays in the map.  The rule is a
// visibility test against a range image of the scan (DESIGN.md §2): one thread per scan point builds the image (k_range_image, an
// atomicMin on the bits of the float range -- positive floats order as unsigned ints, so the image does not depend on the order of the
// atomics), one thread per window map point tests it (k_free_mark), and the store drops the marked points through a stable compaction
// and the existing index stage (map_compact, so_map.cu).
#include <cmath>

#include <cub/cub.cuh>

#include "so_free.cuh"
#include "so_free_rule.h"

namespace so {

__global__ void __launch_bounds__(256) k_range_image(const float4* __restrict__ pts, uint32_t n, FreeGrid g, uint32_t* __restrict__ img,
                                                     FreeCounters* __restrict__ cnt) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    bool in = false, first = false;
    if (i < n) {
        const float4 p = pts[i];
        if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
            const double x = p.x, y = p.y, z = p.z;
            const double r = norm3(x, y, z);
            int row, col;
            if (r > 0.0 && free_pixel(g, x, y, z, &row, &col)) {
                in = true;
                first = atomicMin(img + size_t(row) * g.W + col, __float_as_uint(float(r))) == kUnknown;
            }
        }
    }
    warp_count(&cnt->image_points, in);
    warp_count(&cnt->pixels_hit, first);
}

// keep[i] = 0 when window point i is removed
__global__ void __launch_bounds__(256) k_free_mark(const float4* __restrict__ pts, uint32_t n, FreeGrid g, FreePose P,
                                                   const uint32_t* __restrict__ img, uint8_t* __restrict__ keep,
                                                   uint32_t* __restrict__ cand_ctr, uint32_t* __restrict__ rem_ctr) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    bool cand = false, rem = false;
    if (i < n) {
        rem = free_decide(g, P, pts[i], img, &cand);
        keep[i] = rem ? 0 : 1;
    }
    warp_count(cand_ctr, cand);
    warp_count(rem_ctr, rem);
}

// ------------------------------------------------------------------------------------------------------------------ keyframes
// so_map_clear_free_space_keyframes: the clearing of every selected keyframe at once.  One keyframe's decision on a map point reads
// only its own image and that point, so a point goes when any keyframe removes it.  Keyframes are imaged a tile at a time (kFreeTileBytes
// of images), the keep flags carry from tile to tile, and each store that lost points is compacted once at the end.
struct FreeOrigin { int32_t o[3]; };
// keep flags of the keyframe form: 0 removed, 1 kept, 3 kept and a candidate of some keyframe already (counted once)
constexpr uint8_t kKeep = 1, kKeepCand = 3;

// The range images of one tile, one thread per keyframe point read in place from the pool; image j at imgs + j * W * H.  Each pixel
// keeps its minimum as k_range_image keeps it.
__global__ void __launch_bounds__(256) k_range_images(const float4* __restrict__ pool, const KfImgSeg* __restrict__ segs, uint32_t n_segs,
                                                      uint32_t n, FreeGrid g, uint32_t* __restrict__ imgs, FreeKfCounters* __restrict__ cnt) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    bool in = false, first = false;
    if (i < n) {
        uint32_t lo = 0, hi = n_segs;                                   // the last entry that starts at or before i holds it
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (segs[mid].start <= i) lo = mid; else hi = mid; }
        const KfImgSeg sg = segs[lo];
        const float4 p = pool[sg.src + (i - sg.start)];
        if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
            const double x = p.x, y = p.y, z = p.z;
            const double r = norm3(x, y, z);
            int row, col;
            if (r > 0.0 && free_pixel(g, x, y, z, &row, &col)) {
                in = true;
                uint32_t* img = imgs + size_t(lo) * size_t(g.W) * size_t(g.H);
                first = atomicMin(img + size_t(row) * g.W + col, __float_as_uint(float(r))) == kUnknown;
            }
        }
    }
    warp_count64(&cnt->image_points, in);
    warp_count64(&cnt->pixels_hit, first);
}

// The tile's keyframes that can reach window block blockIdx.x (so_free_rule.h), in tile order: their count into count[b] (list ==
// nullptr), or the keyframes themselves into list[off[b] ..).  Blocks without points in a carved store get none.
constexpr int kCullThreads = 128;
__global__ void __launch_bounds__(kCullThreads) k_kf_cull(const int32_t* __restrict__ surf_count, const int32_t* __restrict__ edge_count,
                                                          FreeOrigin o, const FreePose* __restrict__ poses, uint32_t n_e, double max_range,
                                                          uint32_t* __restrict__ count, const uint32_t* __restrict__ off,
                                                          uint32_t* __restrict__ list) {
    __shared__ uint32_t s_warp[kCullThreads / 32];
    const int b = blockIdx.x;
    const bool active = (surf_count && surf_count[b] > 0) || (edge_count && edge_count[b] > 0);
    uint32_t base = 0;
    if (active) {
        double lo[3], hi[3];
        free_block_box(b, o.o, lo, hi);
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (uint32_t j0 = 0; j0 < n_e; j0 += kCullThreads) {
            const uint32_t j = j0 + threadIdx.x;
            const bool f = j < n_e && free_block_in_reach(lo, hi, poses[j].t, max_range);
            const unsigned bal = __ballot_sync(0xffffffffu, f);
            if (lane == 0) s_warp[warp] = __popc(bal);
            __syncthreads();
            uint32_t before = 0, total = 0;
            for (int w = 0; w < kCullThreads / 32; ++w) { before += w < warp ? s_warp[w] : 0; total += s_warp[w]; }
            if (f && list) list[off[b] + base + before + __popc(bal & ((1u << lane) - 1u))] = j;
            base += total;
            __syncthreads();
        }
    }
    if (!list && threadIdx.x == 0) count[b] = base;
}

// One pass of a tile over the store's sorted copy (w = the point's id, so a CTA's points share a block): each point still kept is
// tested against its block's keyframes in tile order, up to the first that removes it.  cand / rem count the points that became a
// candidate / were removed in this pass.
__global__ void __launch_bounds__(256) k_kf_free_mark(const float4* __restrict__ sorted, uint32_t n, FreeOrigin o, FreeGrid g,
                                                      const FreePose* __restrict__ poses, const uint32_t* __restrict__ imgs,
                                                      const uint32_t* __restrict__ off, const uint32_t* __restrict__ list,
                                                      uint8_t* __restrict__ keep, unsigned long long* __restrict__ cand_ctr,
                                                      unsigned long long* __restrict__ rem_ctr) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    bool new_cand = false, rem = false;
    if (i < n) {
        const float4 p = sorted[i];
        const uint32_t id = __float_as_uint(p.w);
        const uint8_t was = keep[id];
        const int b = was ? free_grid_block(p.x, p.y, p.z, o.o) : -1;
        if (b >= 0) {
            bool cand = false;
            const size_t px = size_t(g.W) * size_t(g.H);
            for (uint32_t k = off[b], e = off[b + 1]; k < e && !rem; ++k) {
                const uint32_t j = list[k];
                rem = free_decide(g, poses[j], p, imgs + size_t(j) * px, &cand);
            }
            new_cand = cand && was == kKeep;
            if (rem) keep[id] = 0;
            else if (new_cand) keep[id] = kKeepCand;
        }
    }
    warp_count64(cand_ctr, new_cand);
    warp_count64(rem_ctr, rem);
}

// ------------------------------------------------------------------------------------------------------------------ host side
void free_space_defaults(so_free_space* o) {
    o->az_res_deg = 0.4f; o->el_res_deg = 0.4f;
    o->el_min_deg = -23.f; o->el_max_deg = 23.f;
    o->dilate = 2;
    o->margin = 0.3f; o->margin_rel = 0.02f;
    o->min_range = 0.5f; o->max_range = 60.f;
}

int free_space_check(const so_free_space* o, int stores, const double pose[7]) {
    if (!o || !pose) return fail(SO_ERR_ARG, "so_map_clear_free_space: NULL opts or pose");
    if (!finite_pose(pose)) return fail(SO_ERR_ARG, "so_map_clear_free_space: pose not finite (or a zero quaternion)");
    if (stores < 1 || stores > 3) return fail(SO_ERR_ARG, "so_map_clear_free_space: stores must be 1 (surf), 2 (edge) or 3 (both)");
    if (!(std::isfinite(o->az_res_deg) && o->az_res_deg > 0 && std::isfinite(o->el_res_deg) && o->el_res_deg > 0))
        return fail(SO_ERR_ARG, "so_free_space: az_res_deg and el_res_deg must be finite and positive");
    if (!(std::isfinite(o->el_min_deg) && std::isfinite(o->el_max_deg) && o->el_max_deg > o->el_min_deg))
        return fail(SO_ERR_ARG, "so_free_space: el_max_deg must be finite and above a finite el_min_deg");
    const double W = std::ceil(360.0 / double(o->az_res_deg)), H = std::ceil((double(o->el_max_deg) - double(o->el_min_deg)) / double(o->el_res_deg));
    if (!(W * H <= double(1 << 24))) return fail(SO_ERR_ARG, "so_free_space: the range image exceeds 2^24 pixels");
    if (o->dilate < 0 || o->dilate > 4) return fail(SO_ERR_ARG, "so_free_space: dilate must be in 0..4");
    if (!(std::isfinite(o->margin) && o->margin >= 0 && std::isfinite(o->margin_rel) && o->margin_rel >= 0))
        return fail(SO_ERR_ARG, "so_free_space: margin and margin_rel must be finite and non-negative");
    if (!(o->min_range < o->max_range)) return fail(SO_ERR_ARG, "so_free_space: min_range must be below max_range");
    return SO_OK;
}

// Every selected store built (and, for the registered form, the surf store whose tail holds the scan): a pending origin or
// resolution change is applied first, as the inserts apply it
int free_space_prepare(Ctx* c, int stores) {
    if ((stores & 1) && c->surf.dirty) { int rc = map_rebuild(c, c->surf); if (rc) return rc; }
    if ((stores & 2) && c->edge.dirty) { int rc = map_rebuild(c, c->edge); if (rc) return rc; }
    return SO_OK;
}

int free_space_reserve_points(Ctx* c, size_t n) { return c->fs.d_pts.reserve(std::max<size_t>(n, 1)); }

void launch_range_image(const float4* pts, uint32_t n, const FreeGrid& g, uint32_t* img, FreeCounters* cnt, cudaStream_t st) {
    if (n) k_range_image<<<(n + 255) / 256, 256, 0, st>>>(pts, n, g, img, cnt);
}

void launch_range_images(const float4* pool, const KfImgSeg* segs, uint32_t n_segs, uint32_t n, const FreeGrid& g, uint32_t* imgs,
                         FreeKfCounters* cnt, cudaStream_t st) {
    if (n) k_range_images<<<(n + 255) / 256, 256, 0, st>>>(pool, segs, n_segs, n, g, imgs, cnt);
}

FreeGrid free_grid(const so_free_space& o) {
    FreeGrid g{};
    g.az_res = double(o.az_res_deg) * (kPiD / 180.0); g.el_res = double(o.el_res_deg) * (kPiD / 180.0);
    g.el_min = double(o.el_min_deg) * (kPiD / 180.0); g.el_max = double(o.el_max_deg) * (kPiD / 180.0);
    g.W = int(std::ceil(360.0 / double(o.az_res_deg)));
    g.H = int(std::ceil((double(o.el_max_deg) - double(o.el_min_deg)) / double(o.el_res_deg)));
    g.d = o.dilate;
    g.margin = o.margin; g.margin_rel = o.margin_rel; g.min_range = o.min_range; g.max_range = o.max_range;
    return g;
}

FreePose free_pose(const double pose[7]) {
    FreePose P{};
    const double* q = pose + 3;
    const double nq = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double x = q[0] / nq, y = q[1] / nq, z = q[2] / nq, w = q[3] / nq;
    const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                         2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                         2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
    for (int k = 0; k < 9; ++k) P.R[k] = R[k];
    for (int k = 0; k < 3; ++k) P.t[k] = pose[k];
    return P;
}

int free_space_clear(Ctx* c, int stores, const float4* d_pts, uint32_t n_pts, const double pose[7], const so_free_space& o,
                     so_free_space_result* out) {
    cudaStream_t st = c->stream;
    const FreeGrid g = free_grid(o);
    const FreePose P = free_pose(pose);
    const size_t M = c->cfg.max_map_points;
    int rc = c->fs.d_img.reserve(size_t(g.W) * g.H);
    if (!rc) rc = c->fs.d_keep.reserve(2 * M);
    if (!rc) rc = c->fs.d_cnt.reserve(1);
    if (!rc) rc = c->fs.h_cnt.reserve(1);
    if (rc) return rc;
    MapStore* ms[2] = {&c->surf, &c->edge};
    timed_launch_begin(c);
    SO_CUDA_TRY(cudaMemsetAsync(c->fs.d_img, 0xFF, size_t(g.W) * g.H * sizeof(uint32_t), st));
    SO_CUDA_TRY(cudaMemsetAsync(c->fs.d_cnt, 0, sizeof(FreeCounters), st));
    if (n_pts) { k_range_image<<<(n_pts + 255) / 256, 256, 0, st>>>(d_pts, n_pts, g, c->fs.d_img, c->fs.d_cnt); c->launches++; }
    for (int k = 0; k < 2; ++k) {
        if (!(stores & (1 << k)) || ms[k]->n == 0) continue;
        k_free_mark<<<(ms[k]->n + 255) / 256, 256, 0, st>>>(ms[k]->d_xyzi, ms[k]->n, g, P, c->fs.d_img, c->fs.d_keep + k * M,
                                                            &c->fs.d_cnt->cand[k], &c->fs.d_cnt->removed[k]);
        c->launches++;
    }
    SO_CUDA_TRY(cudaMemcpyAsync(c->fs.h_cnt, c->fs.d_cnt, sizeof(FreeCounters), cudaMemcpyDeviceToHost, st));
    c->launches += 1;                                                   // the two memsets
    timed_launch_end(c, 3);
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    const FreeCounters h = *c->fs.h_cnt;
    for (int k = 0; k < 2; ++k) {
        if (!(stores & (1 << k)) || h.removed[k] == 0) continue;       // nothing removed: the store is not touched
        timed_launch_begin(c);
        rc = map_compact(c, *ms[k], c->fs.d_keep + k * M, ms[k]->n - h.removed[k], &c->fs.d_cnt->selected);
        timed_launch_end(c, 3);
        if (rc) return rc;
    }
    if (out) {
        *out = so_free_space_result{};
        out->n_image_points = h.image_points;
        out->n_pixels_hit = h.pixels_hit;
        for (int k = 0; k < 2; ++k) {
            if (!(stores & (1 << k))) continue;
            out->n_candidates += h.cand[k];
            out->n_removed += h.removed[k];
        }
        out->n_after[0] = c->surf.n; out->n_after[1] = c->edge.n;
    }
    return SO_OK;
}

int free_space_clear_keyframes(Ctx* c, Ctx* src, const int32_t* ids, size_t n_ids, const double* poses7, int stores, const so_free_space& o,
                               so_free_space_keyframes_result* out) {
    cudaStream_t st = c->stream;
    const KeyframeStore& kf = src->kf;
    const FreeGrid g = free_grid(o);
    const size_t px = size_t(g.W) * size_t(g.H);
    const size_t per_tile = std::max<size_t>(kFreeTileBytes / (px * sizeof(uint32_t)), 1);
    // the tiles: runs of consecutive entries, at most per_tile images and fewer than 2^31 points each
    std::vector<KfImgSeg> segs(n_ids);
    std::vector<FreePose> poses(n_ids);
    std::vector<size_t> tile_first{0};
    std::vector<uint32_t> tile_points;
    uint64_t at = 0;
    for (size_t i = 0; i < n_ids; ++i) {
        const uint64_t first = kf.off[0][ids[i]], n = kf.off[0][ids[i] + 1] - first;
        if (i > tile_first.back() && (i - tile_first.back() == per_tile || at + n >= (uint64_t(1) << 31))) {
            tile_points.push_back(uint32_t(at));
            tile_first.push_back(i);
            at = 0;
        }
        if (n >= (uint64_t(1) << 31)) return fail(SO_ERR_CAPACITY, "so_map_clear_free_space_keyframes: a keyframe of 2^31 points or more");
        segs[i] = KfImgSeg{first, uint32_t(at), uint32_t(n)};
        poses[i] = free_pose(poses7 + 7 * i);
        at += n;
    }
    tile_points.push_back(uint32_t(at));
    tile_first.push_back(n_ids);
    const size_t n_tiles = tile_points.size();
    size_t widest = 0;
    for (size_t t = 0; t < n_tiles; ++t) widest = std::max(widest, tile_first[t + 1] - tile_first[t]);
    const size_t M = c->cfg.max_map_points;
    auto& f = c->fs;
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, kNumBlocks + 1);
    int rc = f.d_img.reserve(widest * px);
    if (!rc) rc = f.d_keep.reserve(2 * M);
    if (!rc) rc = f.d_kseg.reserve(n_ids);
    if (!rc) rc = f.d_kpose.reserve(n_ids);
    if (!rc) rc = f.d_ccount.reserve(kNumBlocks + 1);
    if (!rc) rc = f.d_coff.reserve(kNumBlocks + 1);
    if (!rc) rc = f.d_clist.reserve(size_t(kNumBlocks) * widest);
    if (!rc) rc = f.d_tmp.reserve(scan_bytes + 256);
    if (!rc) rc = f.d_kcnt.reserve(1);
    if (!rc) rc = f.h_kcnt.reserve(1);
    if (!rc && !f.ev[0]) rc = f.ev[0].create();
    if (!rc && !f.ev[1]) rc = f.ev[1].create();
    if (rc) return rc;
    if (src != c) SO_CUDA_TRY(cudaStreamSynchronize(src->stream));     // the keyframes have landed in src's pool
    SO_CUDA_TRY(cudaMemcpyAsync(f.d_kseg, segs.data(), n_ids * sizeof(KfImgSeg), cudaMemcpyHostToDevice, st));
    SO_CUDA_TRY(cudaMemcpyAsync(f.d_kpose, poses.data(), n_ids * sizeof(FreePose), cudaMemcpyHostToDevice, st));
    MapStore* ms[2] = {&c->surf, &c->edge};
    const bool carve[2] = {(stores & 1) && ms[0]->n > 0, (stores & 2) && ms[1]->n > 0};
    const FreeOrigin org{{c->origin[0], c->origin[1], c->origin[2]}};
    SO_CUDA_TRY(cudaEventRecord(f.ev[0], st));
    SO_CUDA_TRY(cudaMemsetAsync(f.d_kcnt, 0, sizeof(FreeKfCounters), st));
    SO_CUDA_TRY(cudaMemsetAsync(f.d_ccount, 0, (kNumBlocks + 1) * sizeof(uint32_t), st));
    c->launches += 2;
    for (int k = 0; k < 2; ++k)
        if (carve[k]) { SO_CUDA_TRY(cudaMemsetAsync(f.d_keep + k * M, kKeep, ms[k]->n, st)); c->launches++; }
    for (size_t t = 0; t < n_tiles; ++t) {
        const size_t a = tile_first[t];
        const uint32_t n_e = uint32_t(tile_first[t + 1] - a), n_pts = tile_points[t];
        SO_CUDA_TRY(cudaMemsetAsync(f.d_img, 0xFF, n_e * px * sizeof(uint32_t), st));
        c->launches++;
        if (n_pts) {
            k_range_images<<<(n_pts + 255) / 256, 256, 0, st>>>(kf.d_pool[0], f.d_kseg + a, n_e, n_pts, g, f.d_img, f.d_kcnt);
            c->launches++;
        }
        if (!carve[0] && !carve[1]) continue;
        const int32_t* cnt_s = carve[0] ? ms[0]->d_block_count.get() : nullptr;
        const int32_t* cnt_e = carve[1] ? ms[1]->d_block_count.get() : nullptr;
        k_kf_cull<<<kNumBlocks, kCullThreads, 0, st>>>(cnt_s, cnt_e, org, f.d_kpose + a, n_e, g.max_range, f.d_ccount, nullptr, nullptr);
        size_t tmp = f.d_tmp.cap();
        SO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(f.d_tmp.get(), tmp, f.d_ccount.get(), f.d_coff.get(), kNumBlocks + 1, st));
        k_kf_cull<<<kNumBlocks, kCullThreads, 0, st>>>(cnt_s, cnt_e, org, f.d_kpose + a, n_e, g.max_range, nullptr, f.d_coff, f.d_clist);
        c->launches += 3;
        for (int k = 0; k < 2; ++k) {
            if (!carve[k]) continue;
            k_kf_free_mark<<<(ms[k]->n + 255) / 256, 256, 0, st>>>(ms[k]->d_sorted, ms[k]->n, org, g, f.d_kpose + a, f.d_img, f.d_coff,
                                                                   f.d_clist, f.d_keep + k * M, &f.d_kcnt->cand[k], &f.d_kcnt->removed[k]);
            c->launches++;
        }
    }
    SO_CUDA_TRY(cudaMemcpyAsync(f.h_kcnt, f.d_kcnt, sizeof(FreeKfCounters), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    const FreeKfCounters h = *f.h_kcnt;
    for (int k = 0; k < 2; ++k) {
        if (!carve[k] || h.removed[k] == 0) continue;                  // nothing removed: the store is not touched
        rc = map_compact(c, *ms[k], f.d_keep + k * M, ms[k]->n - uint32_t(h.removed[k]), &f.d_kcnt->selected);
        if (rc) return rc;
    }
    SO_CUDA_TRY(cudaEventRecord(f.ev[1], st));
    SO_CUDA_TRY(cudaEventSynchronize(f.ev[1]));
    float ms_dev = 0.f;
    SO_CUDA_TRY(cudaEventElapsedTime(&ms_dev, f.ev[0], f.ev[1]));
    if (out) {
        *out = so_free_space_keyframes_result{};
        out->n_keyframes = n_ids;
        out->n_image_points = h.image_points;
        out->n_pixels_hit = h.pixels_hit;
        for (int k = 0; k < 2; ++k) {
            if (!(stores & (1 << k))) continue;
            out->n_candidates += h.cand[k];
            out->n_removed += h.removed[k];
        }
        out->n_after[0] = c->surf.n; out->n_after[1] = c->edge.n;
        out->n_tiles = n_tiles;
        out->time_ms = ms_dev;
    }
    return SO_OK;
}

}  // namespace so

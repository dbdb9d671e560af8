// so_verify.cu -- loop verification (so_loop_verify): align a keyframe against each loop candidate's submap and score the alignment by
// overlap and visibility conflicts, so that a look-alike place does not become a pose-graph edge.
//
// No reference counterpart.  Per candidate the submap and the alignment are the existing calls (so_map_from_keyframes,
// so_register_keyframes), made on the caller's scratch context; the scores are new kernels: k_verify_overlap (the in-block 1-NN
// of so_knn per query point, bounded by the inlier radius), and two counting passes of the free-space rule (so_free.cuh, k_verify_conflict)
// -- the submap against the query's range image, the query against the submap keyframes' images.  Nothing is removed from either map.
#include <algorithm>
#include <cmath>
#include <vector>

#include "so_free.cuh"
#include "so_free_rule.h"
#include "so_knn.cuh"
#include "so_verify_rule.h"

namespace so {

// Device counters of one candidate, read back once
struct VerifyCounters {
    FreeCounters img;                              // k_range_image of the query's image
    FreeKfCounters kimg;                           // k_range_images of the submap keyframes' images
    uint32_t n_query, n_inliers;                   // finite query points, inliers
    uint32_t cand_map, conflict_map;               // submap points the query's image observes / sees clearly past
    uint32_t cand_query, conflict_query;           // query points some submap keyframe's image observes / sees clearly past
    double sum_d2;                                 // sum of the inliers' d^2 (k_verify_sum)
};

constexpr int kVerifyThreads = 64;                 // as k_knn (so_icp.cu): the search's shared candidate list is kBufCap x this
constexpr int kVerifySumThreads = 256;

// One thread per query point: its nearest point of its own 50 m block within max_d2, exactly as k_knn<1> finds it (so_knn).  Inliers
// and finite points are counted; each CTA writes the sum of its inliers' d^2 in FP64, reduced in a fixed tree, to partials[blockIdx.x].
// (8 CTAs per SM: without that bound ptxas holds the search to 48 registers and spills.)
__global__ void __launch_bounds__(kVerifyThreads, 8) k_verify_overlap(MapView m, const float4* __restrict__ q, uint32_t n, float max_d2,
                                                                  double* __restrict__ partials, VerifyCounters* __restrict__ cnt) {
    __shared__ uint32_t s_buf[kBufCap * kVerifyThreads];
    __shared__ double s_sum[kVerifyThreads];
    const uint32_t i = blockIdx.x * kVerifyThreads + threadIdx.x;
    bool finite = false, hit = false;
    double d2 = 0.0;
    if (i < n) {
        const float4 p = q[i];
        finite = isfinite(p.x) && isfinite(p.y) && isfinite(p.z);
        QueryCell qc;
        qc.slot = -1;
        if (finite) locate(m, p.x, p.y, p.z, qc);
        if (qc.slot >= 0) {
            TopK<1> tk;
            tk.init(max_d2);
            knn_search<1>(BlockGrid(m, qc.slot), m, qc, p.x, p.y, p.z, max_d2, s_buf, tk);
            hit = tk.id[0] != 0xFFFFFFFFu;
            if (hit) d2 = double(tk.d2[0]);
        }
    }
    warp_count(&cnt->n_query, finite);
    warp_count(&cnt->n_inliers, hit);
    s_sum[threadIdx.x] = d2;
    __syncthreads();
#pragma unroll
    for (int h = kVerifyThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) s_sum[threadIdx.x] += s_sum[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) partials[blockIdx.x] = s_sum[0];
}

// The sum of partials[0..n) in index order: thread t sums its contiguous run in order, thread 0 the runs in order
__global__ void __launch_bounds__(kVerifySumThreads) k_verify_sum(const double* __restrict__ partials, uint32_t n, double* __restrict__ out) {
    __shared__ double s_run[kVerifySumThreads];
    const uint32_t per = (n + kVerifySumThreads - 1) / kVerifySumThreads;
    const uint32_t a = threadIdx.x * per, e = min(n, a + per);
    double v = 0.0;
    for (uint32_t k = a; k < e; ++k) v += partials[k];
    s_run[threadIdx.x] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int k = 0; k < kVerifySumThreads; ++k) t += s_run[k];
        *out = t;
    }
}

// The finite points pts[0..n) against n_img range images (image j at imgs + j * W * H, pose poses[j]), in order up to the first that
// sees past the point: the decision of k_free_mark (one image) and k_kf_free_mark (every keyframe), counted only
__global__ void __launch_bounds__(256) k_verify_conflict(const float4* __restrict__ pts, uint32_t n, FreeGrid g,
                                                               const FreePose* __restrict__ poses, const uint32_t* __restrict__ imgs,
                                                               uint32_t n_img, uint32_t* __restrict__ cand_ctr,
                                                               uint32_t* __restrict__ conflict_ctr) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    bool cand = false, rem = false;
    if (i < n) {
        const float4 p = pts[i];
        if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
            const size_t px = size_t(g.W) * size_t(g.H);
            const uint32_t* img = imgs;
            for (uint32_t j = 0; j < n_img && !rem; ++j, img += px) rem = free_decide(g, poses[j], p, img, &cand);
        }
    }
    warp_count(cand_ctr, cand);
    warp_count(conflict_ctr, rem);
}

// ------------------------------------------------------------------------------------------------------------------ host side
constexpr int kVerifyMaxHalfWindow = 8;

static int verify_check(const Ctx* c, const so_loop_candidate* cands, size_t n, const so_loop_verify_opts& o) {
    const KeyframeStore& kf = c->kf;
    const int64_t frames = int64_t(kf.frames());
    if (o.half_window < 0 || o.half_window > kVerifyMaxHalfWindow) return fail(SO_ERR_ARG, "so_loop_verify: half_window must be in 0..8");
    if (o.exclude_recent < 0) return fail(SO_ERR_ARG, "so_loop_verify: exclude_recent must be >= 0");
    if (o.id_end >= 0 && (o.id_begin < 0 || o.id_end < o.id_begin || o.id_end > frames))
        return fail(SO_ERR_ARG, "so_loop_verify: the id range must satisfy 0 <= id_begin <= id_end <= the keyframes held");
    { int rc = icp_opts_check(o.icp); if (rc) return rc; }
    const float bound = float(o.inlier_dist * o.inlier_dist);
    if (!(std::isfinite(o.inlier_dist) && o.inlier_dist > 0 && std::isfinite(bound) && bound > 0))
        return fail(SO_ERR_ARG, "so_loop_verify: inlier_dist must be finite and positive");
    static const double kIdentity[7] = {0, 0, 0, 0, 0, 0, 1};
    { int rc = free_space_check(&o.image, 1, kIdentity); if (rc) return rc; }
    const FreeGrid g = free_grid(o.image);
    if (double(2 * o.half_window + 1) * double(g.W) * double(g.H) * sizeof(uint32_t) > double(kFreeTileBytes))
        return fail(SO_ERR_ARG, "so_loop_verify: the submap's range images exceed 256 MiB");
    if (!(o.min_overlap >= 0 && o.min_overlap <= 1) || !(o.max_conflict >= 0 && o.max_conflict <= 1))
        return fail(SO_ERR_ARG, "so_loop_verify: min_overlap and max_conflict must be in [0, 1]");
    for (size_t i = 0; i < n; ++i) {
        const so_loop_candidate& cd = cands[i];
        if (cd.query < 0 || cd.query >= frames) return fail(SO_ERR_ARG, "so_loop_verify: a query keyframe the store does not hold");
        if (cd.id == -1) continue;
        if (cd.id < 0 || cd.id >= frames) return fail(SO_ERR_ARG, "so_loop_verify: a candidate keyframe the store does not hold");
        if (cd.id == cd.query) return fail(SO_ERR_ARG, "so_loop_verify: a candidate equal to its query");
        if (!verify_eligible(verify_range(cd.query, o.id_begin, o.id_end, o.exclude_recent), cd.query, cd.id))
            return fail(SO_ERR_ARG, "so_loop_verify: a candidate outside the eligible ids");
    }
    return SO_OK;
}

static int verify_one(Ctx* c, Ctx* s, const so_loop_candidate& cd, const so_loop_verify_opts& o, so_loop_verify_result* out) {
    *out = so_loop_verify_result{};
    out->query = cd.query;
    out->id = cd.id;
    if (cd.id == -1) { out->skipped = 1; return SO_OK; }
    const KeyframeStore& kf = c->kf;
    const int32_t qid = cd.query, id = cd.id;
    // 1. the submap: the eligible ids around the candidate, at their current poses
    const VerifyRange range = verify_range(qid, o.id_begin, o.id_end, o.exclude_recent);
    std::vector<int32_t> ids;
    std::vector<double> poses;
    for (int64_t k = int64_t(id) - o.half_window; k <= int64_t(id) + o.half_window; ++k) {
        if (k < 0 || !verify_eligible(range, qid, int32_t(k))) continue;
        ids.push_back(int32_t(k));
        poses.insert(poses.end(), kf.poses.begin() + 7 * k, kf.poses.begin() + 7 * (k + 1));
    }
    const double* xc = kf.poses.data() + 7 * size_t(id);
    const double* xq = kf.poses.data() + 7 * size_t(qid);
    Ctx::Verify& v = s->ver;
    cudaStream_t st = s->stream;
    SO_CUDA_TRY(cudaEventRecord(v.ev[0], st));
    so_ctx* hc = reinterpret_cast<so_ctx*>(c);
    so_ctx* hs = reinterpret_cast<so_ctx*>(s);
    int rc = so_map_set_origin(hs, xc, nullptr);
    if (!rc) rc = so_map_from_keyframes(hs, hc, ids.data(), ids.size(), poses.data(), 1);
    if (rc) return rc;
    // 2. the alignment from the candidate's prior
    double prior[7];
    loop_prior(xc, xq, cd.yaw, prior);
    rc = so_register_keyframes(hs, hc, &qid, 1, prior, &o.icp, &out->reg);
    if (rc < 0) return rc;
    rc = ensure_maps(s);
    if (rc) return rc;
    loop_relative(xc, out->reg.pose, out->rel7);
    out->n_submap_keyframes = int32_t(ids.size());
    out->n_submap_points = s->surf.n;
    // 3. and 4. the scores, on scratch's stream
    const uint64_t first = kf.off[0][qid];
    const uint32_t nq = uint32_t(kf.off[0][qid + 1] - first);
    const FreeGrid g = free_grid(o.image);
    const size_t px = size_t(g.W) * size_t(g.H);
    const uint32_t n_img = uint32_t(ids.size());
    std::vector<KfImgSeg> segs(n_img);
    std::vector<FreePose> kposes(n_img + 1);                           // the submap keyframes', then the query's at reg.pose
    uint32_t at = 0;
    for (uint32_t j = 0; j < n_img; ++j) {
        const uint64_t f = kf.off[0][ids[j]];
        const uint32_t m = uint32_t(kf.off[0][ids[j] + 1] - f);
        segs[j] = KfImgSeg{f, at, m};
        kposes[j] = free_pose(poses.data() + 7 * size_t(j));
        at += m;
    }
    kposes[n_img] = free_pose(out->reg.pose);
    const uint32_t grid = (nq + kVerifyThreads - 1) / kVerifyThreads;
    rc = v.d_q.reserve(std::max<uint32_t>(nq, 1));
    if (!rc) rc = v.d_img.reserve((1 + n_img) * px);
    if (!rc) rc = v.d_kseg.reserve(std::max<uint32_t>(n_img, 1));
    if (!rc) rc = v.d_kpose.reserve(n_img + 1);
    if (!rc) rc = v.d_partials.reserve(std::max<uint32_t>(grid, 1));
    if (!rc) rc = v.d_cnt.reserve(1);
    if (!rc) rc = v.h_cnt.reserve(1);
    if (rc) return rc;
    const float4* q_raw = kf.d_pool[0] + first;
    VerifyCounters* dc = v.d_cnt;
    SO_CUDA_TRY(cudaMemsetAsync(dc, 0, sizeof(VerifyCounters), st));
    SO_CUDA_TRY(cudaMemsetAsync(v.d_img, 0xFF, (1 + n_img) * px * sizeof(uint32_t), st));
    s->launches += 2;
    if (n_img) SO_CUDA_TRY(cudaMemcpyAsync(v.d_kseg, segs.data(), n_img * sizeof(KfImgSeg), cudaMemcpyHostToDevice, st));
    SO_CUDA_TRY(cudaMemcpyAsync(v.d_kpose, kposes.data(), (n_img + 1) * sizeof(FreePose), cudaMemcpyHostToDevice, st));
    if (nq) {                                                          // the query at reg.pose, as so_keyframe_download(reg.pose) places it
        SO_CUDA_TRY(cudaMemcpyAsync(v.d_q, q_raw, size_t(nq) * sizeof(float4), cudaMemcpyDeviceToDevice, st));
        launch_transform(v.d_q, nq, out->reg.pose, st);
        k_verify_overlap<<<grid, kVerifyThreads, 0, st>>>(map_view(s, s->surf), v.d_q, nq, float(o.inlier_dist * o.inlier_dist),
                                                          v.d_partials, dc);
        k_verify_sum<<<1, kVerifySumThreads, 0, st>>>(v.d_partials, grid, &dc->sum_d2);
        s->launches += 3;
    }
    launch_range_image(q_raw, nq, g, v.d_img, &dc->img, st);
    launch_range_images(kf.d_pool[0], v.d_kseg, n_img, at, g, v.d_img + px, &dc->kimg, st);
    s->launches += (nq ? 1 : 0) + (at ? 1 : 0);
    if (s->surf.n) {
        k_verify_conflict<<<(s->surf.n + 255) / 256, 256, 0, st>>>(s->surf.d_xyzi, s->surf.n, g, v.d_kpose + n_img, v.d_img, 1,
                                                                  &dc->cand_map, &dc->conflict_map);
        s->launches++;
    }
    if (nq && n_img) {
        k_verify_conflict<<<(nq + 255) / 256, 256, 0, st>>>(v.d_q, nq, g, v.d_kpose, v.d_img + px, n_img, &dc->cand_query,
                                                            &dc->conflict_query);
        s->launches++;
    }
    SO_CUDA_TRY(cudaGetLastError());
    SO_CUDA_TRY(cudaMemcpyAsync(v.h_cnt, dc, sizeof(VerifyCounters), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaEventRecord(v.ev[1], st));
    SO_CUDA_TRY(cudaEventSynchronize(v.ev[1]));
    float ms = 0.f;
    SO_CUDA_TRY(cudaEventElapsedTime(&ms, v.ev[0], v.ev[1]));
    // 5. the scores and the decision
    const VerifyCounters h = *v.h_cnt;
    out->n_query_points = h.n_query;
    out->n_inliers = h.n_inliers;
    out->overlap = h.n_query ? double(h.n_inliers) / double(h.n_query) : 0.0;
    out->rmse = h.n_inliers ? std::sqrt(h.sum_d2 / double(h.n_inliers)) : 0.0;
    out->n_cand_query = h.cand_query;
    out->n_conflict_query = h.conflict_query;
    out->n_cand_map = h.cand_map;
    out->n_conflict_map = h.conflict_map;
    out->conflict_query = verify_fraction(h.conflict_query, h.cand_query);
    out->conflict_map = verify_fraction(h.conflict_map, h.cand_map);
    out->accepted = verify_accept(out->reg.status, out->overlap, out->conflict_query, out->conflict_map, o.min_overlap, o.max_conflict);
    out->time_ms = ms;
    return SO_OK;
}

}  // namespace so

// =================================================================================================== C ABI
using namespace so;

extern "C" {

void so_loop_prior(const double cand7[7], const double query7[7], double yaw, double out7[7]) {
    if (cand7 && query7 && out7) loop_prior(cand7, query7, yaw, out7);
}

void so_loop_verify_opts_defaults(so_loop_verify_opts* o) {
    if (!o) return;
    *o = so_loop_verify_opts{};
    o->half_window = 2;
    o->id_begin = 0;
    o->id_end = -1;
    o->exclude_recent = 30;
    o->icp.max_icp_iters = 20;
    o->icp.lm_max_iterations = 4;
    o->inlier_dist = 0.5;
    free_space_defaults(&o->image);
    o->min_overlap = 0.5;
    o->max_conflict = 0.05;
}

int so_loop_verify(so_ctx* ctx, so_ctx* scratch, const so_loop_candidate* cands, size_t n, const so_loop_verify_opts* opts,
                   so_loop_verify_result* out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    Ctx* s = reinterpret_cast<Ctx*>(scratch);
    if (!c || !s || !opts || (n && (!cands || !out))) return fail(SO_ERR_ARG, "bad args");
    if (c == s) return fail(SO_ERR_ARG, "so_loop_verify: scratch must be another context than ctx");
    if (c->device != s->device) return fail(SO_ERR_ARG, "so_loop_verify: the two contexts are on different devices");
    if (!c->kf.cap_frames) return fail(SO_ERR_ARG, "so_loop_verify needs a keyframe store in ctx (so_keyframe_reserve)");
    { int rc = verify_check(c, cands, n, *opts); if (rc) return rc; }
    if (n == 0) return SO_OK;
    bool any = false;
    for (size_t i = 0; i < n; ++i) any |= cands[i].id != -1;
    if (any) {
        SO_CUDA_TRY(cudaSetDevice(s->device));
        for (int k = 0; k < 2; ++k)
            if (!s->ver.ev[k]) { int rc = s->ver.ev[k].create(); if (rc) return rc; }
    }
    for (size_t i = 0; i < n; ++i) {
        int rc = verify_one(c, s, cands[i], *opts, out + i);
        if (rc) return rc;
    }
    return SO_OK;
}

}  // extern "C"

// so_global.cu -- global localization against the prior map, host side: defaults and limits of the search, score points and yaw
// quaternions, the branch-and-bound search (kernels in so_reloc.cu), suppression and refinement of the best hypotheses through
// register_scans (window by window over the block archive for whole_map searches), and the so_localize_* / so_map_bounds* entry
// points of the C ABI.
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstring>

#include "so_ctx.cuh"

namespace so {

// The score of so_localize_global is an integer function of a few double-precision expressions evaluated on the host (score-point
// ranges, the yaw quaternions) and on the device (voxel of every point).  The host ones are compiled without FMA contraction so that
// a numpy restatement, which never contracts, reproduces them bit for bit on any host architecture.
#if defined(__GNUC__) && !defined(__clang__)
#define SO_NO_FP_CONTRACT __attribute__((optimize("fp-contract=off")))
#else
#define SO_NO_FP_CONTRACT
#endif

struct GlobalPlan {
    so_global_opts o{};                    // defaults applied
    RelocGrid g{};
    int32_t I = 0, J = 0, K = 0;           // index of the centre along each shift axis
    int32_t m_off = 0;                     // yaw index of the centre's yaw (0 for the full circle)
    double dpsi = 0.0;                     // yaw step actually used
    uint64_t n_hyp = 0, bitmap_words = 0;
    bool whole = false;                    // whole_map = 1 with the archive on: search the archive too, refine window by window
};

// Defaults, argument checks and the grid of so_localize_global (host only).  Capacity errors return with the plan filled in.
// Limits: 2^24 hypotheses and a whole-box bitmap of at most 2^32 bits; bnb: those of so_localize_global_bnb instead (2^32
// hypotheses, no bitmap limit).
static int global_plan(const so_global_opts* in, GlobalPlan* P, bool bnb = false) {
    if (!in) return fail(SO_ERR_ARG, "null so_global_opts");
    so_global_opts o = *in;
    if (o.res == 0) o.res = 0.25;
    if (o.yaw_step == 0) o.yaw_step = 2.0 * M_PI / 180.0;
    if (o.max_range == 0) o.max_range = 40.0;
    if (o.score_points == 0) o.score_points = 1024;
    if (o.dilate == 0) o.dilate = 1;
    if (o.k == 0) o.k = 16;
    if (o.nms_xy == 0) o.nms_xy = 1.0;
    if (o.nms_yaw == 0) o.nms_yaw = 10.0 * M_PI / 180.0;
    auto nonneg = [](double v) { return std::isfinite(v) && v >= 0.0; };
    auto pos = [](double v) { return std::isfinite(v) && v > 0.0; };
    if (!nonneg(o.half_x) || !nonneg(o.half_y) || !nonneg(o.half_z)) return fail(SO_ERR_ARG, "search half-extents must be finite and >= 0");
    if (!nonneg(o.yaw_half)) return fail(SO_ERR_ARG, "yaw_half must be finite and >= 0");
    if (!pos(o.res) || !pos(o.yaw_step) || !pos(o.max_range)) return fail(SO_ERR_ARG, "res, yaw_step and max_range must be finite and > 0");
    if (!nonneg(o.nms_xy) || !nonneg(o.nms_yaw)) return fail(SO_ERR_ARG, "nms_xy and nms_yaw must be finite and >= 0");
    if (o.score_points < 1 || o.score_points > 4096) return fail(SO_ERR_ARG, "score_points must be in [1, 4096]");
    if (o.k < 1 || o.k > 64) return fail(SO_ERR_ARG, "k must be in [1, 64]");
    if (o.dilate < 1 || o.dilate > 8) return fail(SO_ERR_ARG, "dilate must be in [1, 8]");
    if (o.whole_map != 0 && o.whole_map != 1) return fail(SO_ERR_ARG, "whole_map must be 0 or 1");
    P->o = o;
    const double Id = std::floor(o.half_x / o.res), Jd = std::floor(o.half_y / o.res), Kd = std::floor(o.half_z / o.res);
    const double ed = std::ceil(o.max_range / o.res);
    const bool full = o.yaw_half >= M_PI;
    const double Md = full ? 0.0 : std::floor(o.yaw_half / o.yaw_step);
    double nyaw = full ? std::floor(2.0 * M_PI / o.yaw_step + 0.5) : 2.0 * Md + 1.0;
    if (nyaw < 1.0) nyaw = 1.0;
    const double lim = double(1 << 24);
    if (Id > lim || Jd > lim || Kd > lim || ed > lim || nyaw > lim) return fail(SO_ERR_CAPACITY, "search region too large (more than 2^24 hypotheses)");
    RelocGrid& g = P->g;
    P->I = int32_t(Id); P->J = int32_t(Jd); P->K = int32_t(Kd); P->m_off = int32_t(Md);
    g.nx = 2 * P->I + 1; g.ny = 2 * P->J + 1; g.nz = 2 * P->K + 1; g.nyaw = int32_t(nyaw);
    g.e = int32_t(ed);
    g.res = o.res;
    P->dpsi = full ? 2.0 * M_PI / nyaw : o.yaw_step;
    const double hyp = double(g.nx) * g.ny * g.nz * g.nyaw;
    const double words = std::ceil((double(g.nx) + 2.0 * g.e) / 32.0) * (double(g.ny) + 2.0 * g.e) * (double(g.nz) + 2.0 * g.e);
    P->n_hyp = hyp < 1.8e19 ? uint64_t(hyp) : UINT64_MAX;
    P->bitmap_words = words < 1.8e19 ? uint64_t(words) : UINT64_MAX;
    if (bnb) {
        if (hyp > 4294967296.0) return fail(SO_ERR_CAPACITY, "more than 2^32 hypotheses");
    } else {
        if (hyp > lim) return fail(SO_ERR_CAPACITY, "more than 2^24 hypotheses");
        if (words * 32.0 > 4294967296.0) return fail(SO_ERR_CAPACITY, "occupancy bitmap above 2^32 bits");
    }
    g.bx = g.nx + 2 * g.e; g.by = g.ny + 2 * g.e; g.bz = g.nz + 2 * g.e; g.wpr = (g.bx + 31) / 32;
    return SO_OK;
}

static void plan_dims(const GlobalPlan& P, int32_t dims[4]) { dims[0] = P.g.nx; dims[1] = P.g.ny; dims[2] = P.g.nz; dims[3] = P.g.nyaw; }

// A hypothesis key, as the search writes it: (65535 - score) << 32 | linear index, so that the ascending order is score
// descending, then index ascending.
static int32_t key_score(uint64_t key) { return int32_t(65535u - uint32_t(key >> 32)); }
static uint32_t key_index(uint64_t key) { return uint32_t(key & 0xffffffffu); }

// The scan side of the search: the points that are scored, the centre's rotation split into yaw and roll/pitch, one quaternion per
// hypothesis yaw.
struct GlobalScan {
    std::vector<float4> pts;               // score points, cloud order
    double t[3], lo[3], yaw_c, q_rp[4];     // centre position, bitmap corner (RelocGrid::lo)
    std::vector<double> q;                 // [nyaw][4] q_z(yaw_m) (x) q_rp
    std::vector<double> yaw;               // [nyaw] yaw_m
};

// finite, within max_range (double squared range), then shouldProcessPoint capped at score_points (so_sampling_indices' rule)
SO_NO_FP_CONTRACT static void select_score_points(const void* xyzi, size_t n, size_t stride, size_t ioff, const so_global_opts& o, GlobalScan* S) {
    std::vector<float4> near;
    near.reserve(n);
    const double r2max = o.max_range * o.max_range;
    const unsigned char* p = static_cast<const unsigned char*>(xyzi);
    for (size_t i = 0; i < n; ++i, p += stride) {
        const float4 v = read_point(p, stride, ioff);
        if (!std::isfinite(v.x) || !std::isfinite(v.y) || !std::isfinite(v.z)) continue;
        const double x = v.x, y = v.y, z = v.z;
        const double xx = x * x, yy = y * y, zz = z * z;
        if ((xx + yy) + zz > r2max) continue;
        near.push_back(v);
    }
    std::vector<uint32_t> idx(near.size());
    size_t k = 0;
    so_sampling_indices(uint32_t(near.size()), o.score_points, idx.data(), idx.size(), &k);
    S->pts.resize(k);
    for (size_t j = 0; j < k; ++j) S->pts[j] = near[idx[j]];
}

SO_NO_FP_CONTRACT static void qmul_nc(const double a[4], const double b[4], double o[4]) {    // qmul (so_internal.cuh), uncontracted
    const double a3b0 = a[3] * b[0], a0b3 = a[0] * b[3], a1b2 = a[1] * b[2], a2b1 = a[2] * b[1];
    const double a3b1 = a[3] * b[1], a1b3 = a[1] * b[3], a2b0 = a[2] * b[0], a0b2 = a[0] * b[2];
    const double a3b2 = a[3] * b[2], a2b3 = a[2] * b[3], a0b1 = a[0] * b[1], a1b0 = a[1] * b[0];
    const double a3b3 = a[3] * b[3], a0b0 = a[0] * b[0], a1b1 = a[1] * b[1], a2b2 = a[2] * b[2];
    o[0] = ((a3b0 + a0b3) + a1b2) - a2b1;
    o[1] = ((a3b1 + a1b3) + a2b0) - a0b2;
    o[2] = ((a3b2 + a2b3) + a0b1) - a1b0;
    o[3] = ((a3b3 - a0b0) - a1b1) - a2b2;
}

// q_c = q_z(yaw_c) (x) q_rp with yaw_c tf2's getRPY yaw of the normalised centre rotation; hypothesis yaw m is yaw_c + (m - m_off) dpsi
SO_NO_FP_CONTRACT static void yaw_quaternions(const GlobalPlan& P, const double center[7], GlobalScan* S) {
    const double x = center[3], y = center[4], z = center[5], w = center[6];
    const double xx = x * x, yy = y * y, zz = z * z, ww = w * w;
    const double nrm = std::sqrt(((xx + yy) + zz) + ww);
    const double qc[4] = {x / nrm, y / nrm, z / nrm, w / nrm};
    double roll, pitch;
    tf2_get_rpy(qc, &roll, &pitch, &S->yaw_c);
    const double h = -S->yaw_c * 0.5;
    const double qz_inv[4] = {0.0, 0.0, std::sin(h), std::cos(h)};
    qmul_nc(qz_inv, qc, S->q_rp);
    const int32_t shift[3] = {P.I, P.J, P.K};
    for (int a = 0; a < 3; ++a) {
        S->t[a] = center[a];
        const double reach = double(shift[a] + P.g.e) * P.g.res;
        S->lo[a] = center[a] - reach;
    }
    S->q.resize(size_t(P.g.nyaw) * 4);
    S->yaw.resize(P.g.nyaw);
    for (int32_t m = 0; m < P.g.nyaw; ++m) {
        const double psi = S->yaw_c + double(m - P.m_off) * P.dpsi;
        const double hm = psi * 0.5;
        const double qz[4] = {0.0, 0.0, std::sin(hm), std::cos(hm)};
        S->yaw[m] = psi;
        qmul_nc(qz, S->q_rp, S->q.data() + 4 * m);
    }
}

// Upload the score points and yaw quaternions on the context stream (the buffers allocated or grown on demand)
static int global_upload(Ctx* c, const GlobalScan& S) {
    Ctx::Bnb& R = c->bnb;
    int rc = R.d_pts.reserve(kRelocMaxPoints);
    if (!rc) rc = R.d_q.reserve(S.q.size());
    if (rc) return rc;
    cudaStream_t st = c->stream;
    if (!S.pts.empty()) SO_CUDA_TRY(cudaMemcpyAsync(R.d_pts, S.pts.data(), S.pts.size() * sizeof(float4), cudaMemcpyHostToDevice, st));
    SO_CUDA_TRY(cudaMemcpyAsync(R.d_q, S.q.data(), S.q.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    count_h2d(c, S.pts.size() * sizeof(float4) + S.q.size() * sizeof(double));
    return SO_OK;
}

// The surf archive's live segments into the same raster (whole_map searches; after ensure_maps, which may change the directory)
static int archive_raster(Ctx* c, const RelocGrid& g, const BnbPyramid& w, uint32_t* bits) {
    uint32_t n_segs = 0, max_n = 0;
    int rc = archive_segments(c, c->surf, &n_segs, &max_n);
    if (rc) return rc;
    launch_seg_raster(c->surf.arc.d_pool, c->surf.arc.d_segs, n_segs, max_n, g, w, bits, c->stream);
    c->launches += n_segs ? 1 : 0;
    return SO_OK;
}

static int global_check_args(Ctx* c, const void* xyzi, size_t n, size_t stride, const double center[7], const so_global_opts* gopts, GlobalPlan* P,
                             bool bnb = false) {
    if (!c || !center || !gopts || (!xyzi && n) || stride < 12) return fail(SO_ERR_ARG, "bad args");
    for (int a = 0; a < 7; ++a) if (!std::isfinite(center[a])) return fail(SO_ERR_ARG, "centre pose is not finite");
    if (center[3] == 0 && center[4] == 0 && center[5] == 0 && center[6] == 0) return fail(SO_ERR_ARG, "centre quaternion is zero");
    int rc = global_plan(gopts, P, bnb);
    if (rc) return rc;
    if (n > c->cfg.max_scan_points) return fail(SO_ERR_CAPACITY, "scan larger than so_config.max_scan_points");
    P->whole = P->o.whole_map == 1 && c->surf.arc.d_pool.cap() != 0;        // archive off: the window is the whole map
    return SO_OK;
}

// Everything after the search: suppression over the sorted key prefix pref[0..n_pref), refinement of the kept candidates, winner
// selection.  The candidates register in groups of one window each: for whole_map searches the window so_map_shift(prior) would
// leave from the current origin O0 (groups ordered by their best-ranked member, the window moved to each in turn, and on return
// left at the winner's, or at O0 when there is none); otherwise the current window, one group in rank order.
static int global_refine(Ctx* c, const GlobalPlan& P, const GlobalScan& S, const uint64_t* pref, size_t n_pref, const void* xyzi, size_t n,
                         size_t stride, size_t ioff, const so_icp_opts* opts, so_global_candidate* cands, size_t cap, so_global_result* out,
                         std::chrono::steady_clock::time_point t0, std::chrono::steady_clock::time_point t1) {
    out->best_score = n_pref ? key_score(pref[0]) : 0;
    // greedy suppression in rank order: drop a hypothesis within nms_xy (x/y distance) AND nms_yaw (wrapped) of a kept one
    struct Cand { double prior[7]; double yaw; int32_t score; };
    std::vector<Cand> kept;
    const RelocGrid& g = P.g;
    for (size_t r = 0; r < n_pref && int32_t(kept.size()) < P.o.k; ++r) {
        const int32_t score = key_score(pref[r]);
        if (score == 0) break;
        uint32_t lin = key_index(pref[r]);
        const int32_t i = int32_t(lin % uint32_t(g.nx)); lin /= uint32_t(g.nx);
        const int32_t j = int32_t(lin % uint32_t(g.ny)); lin /= uint32_t(g.ny);
        const int32_t k = int32_t(lin % uint32_t(g.nz));
        const int32_t m = int32_t(lin / uint32_t(g.nz));
        Cand cd;
        cd.prior[0] = S.t[0] + double(i - P.I) * g.res;
        cd.prior[1] = S.t[1] + double(j - P.J) * g.res;
        cd.prior[2] = S.t[2] + double(k - P.K) * g.res;
        std::memcpy(cd.prior + 3, S.q.data() + 4 * m, 4 * sizeof(double));
        cd.yaw = S.yaw[m];
        cd.score = score;
        bool suppressed = false;
        for (const Cand& o : kept) {
            const double dx = cd.prior[0] - o.prior[0], dy = cd.prior[1] - o.prior[1];
            const double dyaw = std::fabs(std::remainder(cd.yaw - o.yaw, 2.0 * M_PI));
            if (dx * dx + dy * dy <= P.o.nms_xy * P.o.nms_xy && dyaw <= P.o.nms_yaw) { suppressed = true; break; }
        }
        if (!suppressed) kept.push_back(cd);
    }
    // the whole cloud goes to the scan buffer (so_map_add_registered_scan inserts it afterwards), once per batch slot
    c->prefiltered_n = SIZE_MAX;
    c->reg.valid = false;
    int rc = upload_cloud(c, xyzi, n, stride, ioff, c->d_scan);
    if (rc) return rc;
    c->reg = RegisteredScan{};
    c->reg.n = uint32_t(n);
    const size_t n_cand = kept.size();
    out->n_candidates = int32_t(n_cand);
    std::vector<so_icp_result> res(n_cand);
    const int32_t o0[3] = {c->origin[0], c->origin[1], c->origin[2]};       // the search applied any pending origin change
    std::vector<std::array<int32_t, 3>> win(n_cand, std::array<int32_t, 3>{o0[0], o0[1], o0[2]});
    if (P.whole) for (size_t k = 0; k < n_cand; ++k) shift_origin(o0, kept[k].prior, win[k].data(), nullptr);
    std::vector<std::vector<size_t>> groups;                                 // candidate indices per window, rank order
    for (size_t k = 0; k < n_cand; ++k) {
        size_t gi = 0;
        while (gi < groups.size() && win[groups[gi][0]] != win[k]) ++gi;
        if (gi == groups.size()) groups.emplace_back();
        groups[gi].push_back(k);
    }
    if (n_cand) {
        const size_t B = std::min<size_t>(c->max_batch, n_cand);
        for (size_t s = 1; s < B && n; ++s)
            SO_CUDA_TRY(cudaMemcpyAsync(c->d_scan + s * n, c->d_scan, n * sizeof(float4), cudaMemcpyDeviceToDevice, c->stream));
        std::vector<uint32_t> npts(B, uint32_t(n));
        RegisterRequest q;                                    // the candidate registrations leave no rows in a pose sink
        q.src = RegisterRequest::Source::DEVICE; q.scans = c->d_scan; q.n_points = npts.data(); q.opts = opts; q.sink_rows = false;
        for (const std::vector<size_t>& grp : groups) {
            if (P.whole) { rc = move_window(c, win[grp[0]].data()); if (rc) return rc; }   // the map moves; d_scan does not
            std::vector<double> priors(7 * grp.size());
            std::vector<so_icp_result> gres(grp.size());
            for (size_t j = 0; j < grp.size(); ++j) std::memcpy(priors.data() + 7 * j, kept[grp[j]].prior, 7 * sizeof(double));
            for (size_t s0 = 0; s0 < grp.size(); s0 += B) {
                q.n_scans = std::min(B, grp.size() - s0); q.poses = priors.data() + 7 * s0; q.results = gres.data() + s0;
                rc = register_scans(c, q);
                if (rc) return rc;
            }
            for (size_t j = 0; j < grp.size(); ++j) res[grp[j]] = gres[j];
        }
    }
    if (P.whole) out->n_windows = int32_t(groups.size());
    // winner: most SUCCESS correspondences in the final ICP iteration, then the lower final cost, then the better rank
    int32_t winner = -1;
    bool all_nef = n_cand > 0;
    auto final_cost = [](const so_icp_result& r) { return r.n_iterations > 0 ? r.iter_cost[r.n_iterations - 1] : HUGE_VAL; };
    for (size_t q = 0; q < n_cand; ++q) {
        const so_icp_result& r = res[q];
        all_nef &= r.status == SO_STATUS_NOT_ENOUGH_FEATURES;
        if (r.status != SO_OK) continue;
        if (winner < 0) { winner = int32_t(q); continue; }
        const so_icp_result& b = res[winner];
        if (r.hist_reject_plane[SO_MATCH_SUCCESS] > b.hist_reject_plane[SO_MATCH_SUCCESS] ||
            (r.hist_reject_plane[SO_MATCH_SUCCESS] == b.hist_reject_plane[SO_MATCH_SUCCESS] && final_cost(r) < final_cost(b)))
            winner = int32_t(q);
    }
    if (P.whole) { rc = move_window(c, winner >= 0 ? win[winner].data() : o0); if (rc) return rc; }
    for (size_t q = 0; q < std::min(n_cand, cap); ++q) {
        so_global_candidate& o = cands[q];
        std::memset(&o, 0, sizeof(o));
        std::memcpy(o.prior, kept[q].prior, sizeof(o.prior));
        o.score = kept[q].score;
        o.n_success = res[q].hist_reject_plane[SO_MATCH_SUCCESS];
        o.cost = res[q].n_iterations > 0 ? res[q].iter_cost[res[q].n_iterations - 1] : 0.0;
        std::memcpy(o.pose, res[q].pose, sizeof(o.pose));
        o.status = res[q].status;
    }
    out->winner = winner;
    if (winner >= 0) {
        out->status = SO_OK;
        out->icp = res[winner];
        std::memcpy(out->pose, res[winner].pose, sizeof(out->pose));
    } else {
        out->status = all_nef ? SO_STATUS_NOT_ENOUGH_FEATURES : SO_STATUS_NO_CORRESPONDENCES;
    }
    const auto t2 = std::chrono::steady_clock::now();
    out->time_refine_ms = std::chrono::duration<double, std::milli>(t2 - t1).count();
    out->time_total_ms = std::chrono::duration<double, std::milli>(t2 - t0).count();
    return out->status;
}

// ---------------------------------------------------------------------------------------------- branch and bound
// The search yields the P smallest keys of every hypothesis, ascending (the sorted prefix of a dense scoring), from an occupancy
// pyramid of the map (memory: the map's window of the search box, per level) and a batched depth-first traversal (memory:
// kBnbRoot + 4C keys per level), so neither grows with the hypothesis count.  See DESIGN.md §4.

// Lmax: the smallest L >= 1 whose root level fits kBnbRoot nodes, or at which one root tile covers every x/y shift (the root is
// then scored in chunks of kBnbRoot).
static uint64_t bnb_level_nodes(const RelocGrid& g, int L) {
    const uint64_t s = (1ull << L) - 1;
    return uint64_t(g.nyaw) * uint64_t(g.nz) * ((uint64_t(g.nx) + s) >> L) * ((uint64_t(g.ny) + s) >> L);
}

static int bnb_lmax(const RelocGrid& g) {
    for (int L = 1;; ++L) {
        const uint64_t s = (1ull << L) - 1;
        if ((((uint64_t(g.nx) + s) >> L) == 1 && ((uint64_t(g.ny) + s) >> L) == 1) || bnb_level_nodes(g, L) <= uint64_t(kBnbRoot)) return L;
    }
}

static_assert(SO_BNB_LEVELS == kBnbLevels, "so_bnb_stats holds one entry per pyramid level");

// 16-byte offset entries for every (yaw, score point): a host-decidable cap
constexpr double kBnbTableBytes = double(1u << 30);

static int bnb_check_table(const GlobalPlan& P, const GlobalScan& S) {
    if (double(P.g.nyaw) * double(S.pts.size()) * 16.0 > kBnbTableBytes) return fail(SO_ERR_CAPACITY, "offset table above 1 GiB");
    return SO_OK;
}

static int bnb_alloc(Ctx* c) {
    Ctx::Bnb& B = c->bnb;
    int rc = SO_OK;
    for (Event& e : B.ev) if (!rc && !e) rc = e.create();
    if (!rc) rc = B.d_nodes.reserve(size_t(kBnbRoot) + size_t(kBnbLevels - 2) * 4 * kBnbBatch);
    if (!rc) rc = B.d_unsorted.reserve(size_t(std::max(kBnbRoot, 4 * kBnbBatch)));
    if (!rc) rc = B.d_merge[0].reserve(kBnbMerge);
    if (!rc) rc = B.d_merge[1].reserve(kBnbMerge);
    if (!rc) rc = B.d_tmp.reserve(std::max(bnb_sort_bytes(kBnbMerge), bnb_sort_bytes(kBnbRoot)) + 256);
    if (!rc) rc = B.d_ctl.reserve(1);
    if (!rc) rc = B.h_ctl.reserve(1);
    if (!rc) rc = B.d_bounds.reserve(6);
    return rc;
}

static float float_from_order(uint32_t o) {
    const uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
    float f;
    std::memcpy(&f, &u, 4);
    return f;
}

// Bounding box of the surf store (whole: and of its archive's live segments), reduced on the device; lo / hi are left alone for an
// empty map.
static int map_bounds(Ctx* c, float lo[3], float hi[3], size_t* n, bool whole = false) {
    { int rc = bnb_alloc(c); if (rc) return rc; }
    { int rc = ensure_maps(c); if (rc) return rc; }
    const bool arc = whole && c->surf.arc.live;
    *n = c->surf.n + (arc ? c->surf.arc.live : 0);
    if (!*n) return SO_OK;
    cudaStream_t st = c->stream;
    SO_CUDA_TRY(cudaMemsetAsync(c->bnb.d_bounds, 0xff, 3 * sizeof(uint32_t), st));
    SO_CUDA_TRY(cudaMemsetAsync(c->bnb.d_bounds + 3, 0, 3 * sizeof(uint32_t), st));
    timed_launch_begin(c);
    launch_map_bounds(c->surf.d_xyzi, c->surf.n, c->bnb.d_bounds, st);
    if (arc) {
        uint32_t n_segs = 0, max_n = 0;
        { int rc = archive_segments(c, c->surf, &n_segs, &max_n); if (rc) return rc; }
        launch_seg_bounds(c->surf.arc.d_pool, c->surf.arc.d_segs, n_segs, max_n, c->bnb.d_bounds, st);
        c->launches += c->surf.n ? 1 : 0;                               // one launch is counted by timed_launch_end
    }
    timed_launch_end(c, 6, 1);
    uint32_t h[6];
    SO_CUDA_TRY(cudaMemcpyAsync(h, c->bnb.d_bounds, sizeof(h), cudaMemcpyDeviceToHost, st));
    count_d2h(c, sizeof(h));
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    for (int a = 0; a < 3; ++a) { lo[a] = float_from_order(h[a]); hi[a] = float_from_order(h[3 + a]); }
    return SO_OK;
}

// The window W and the level layout.  floor((p - lo) / res) with correctly rounded operations is monotonic in p, so the voxels of
// the map's float bounding box bound the voxel of every map point; grown by the dilation and cut to the box, that is W.
SO_NO_FP_CONTRACT static int bnb_layout(const GlobalPlan& P, const double box_lo[3], const float mlo[3], const float mhi[3], size_t n_map,
                                        BnbPyramid* out, uint64_t* words) {
    const RelocGrid& g = P.g;
    BnbPyramid p{};
    p.lmax = bnb_lmax(g);
    const int32_t dims[3] = {g.bx, g.by, g.bz};
    int32_t w0[3] = {0, 0, 0}, wn[3] = {1, 1, 1};
    bool empty = n_map == 0;
    for (int a = 0; a < 3 && !empty; ++a) {
        const double f0 = std::floor((double(mlo[a]) - box_lo[a]) / g.res), f1 = std::floor((double(mhi[a]) - box_lo[a]) / g.res);
        const double v0 = std::max(0.0, f0 - P.o.dilate), v1 = std::min(double(dims[a] - 1), f1 + P.o.dilate);
        if (!(v0 <= v1)) { empty = true; break; }
        w0[a] = int32_t(v0); wn[a] = int32_t(v1 - v0) + 1;
    }
    if (empty) for (int a = 0; a < 3; ++a) { w0[a] = 0; wn[a] = 1; }   // nothing of the map in the box: one voxel, never set
    p.x0 = w0[0]; p.y0 = w0[1]; p.z0 = w0[2]; p.wx = wn[0]; p.wy = wn[1]; p.wz = wn[2];
    uint64_t total = 0;
    for (int L = 0; L <= p.lmax; ++L) {
        const uint64_t xw = uint64_t(p.wx) + (1ull << L) - 1, yw = uint64_t(p.wy) + (1ull << L) - 1, wpr = (xw + 31) / 32;
        if (double(wpr) * 32.0 * double(yw) * double(p.wz) > 4294967296.0) return fail(SO_ERR_CAPACITY, "a pyramid level above 2^32 bits");
        p.wpr[L] = int32_t(wpr);
        p.off[L] = total;
        total += wpr * yw * uint64_t(p.wz);
    }
    *out = p;
    *words = total;
    return SO_OK;
}

// Map bounds -> window -> raster, dilation, levels 1..Lmax, offset table.  Events: ev[0] start, ev[1] after the raster, ev[2] built.
static int bnb_build(Ctx* c, const GlobalPlan& P, const GlobalScan& S, RelocGrid* g_out, BnbPyramid* p_out, uint64_t* pyr_words) {
    Ctx::Bnb& B = c->bnb;
    { int rc = bnb_alloc(c); if (rc) return rc; }
    cudaStream_t st = c->stream;
    SO_CUDA_TRY(cudaEventRecord(B.ev[0], st));
    float mlo[3] = {0, 0, 0}, mhi[3] = {0, 0, 0};
    size_t n_map = 0;
    { int rc = map_bounds(c, mlo, mhi, &n_map, P.whole); if (rc) return rc; }
    RelocGrid g = P.g;
    for (int a = 0; a < 3; ++a) g.lo[a] = S.lo[a];
    BnbPyramid p;
    uint64_t words = 0;
    { int rc = bnb_layout(P, S.lo, mlo, mhi, n_map, &p, &words); if (rc) return rc; }
    const uint64_t w0 = p.off[1];                                   // level 0 words
    { int rc = B.d_pyr.reserve(words); if (rc) return rc; }
    { int rc = B.d_scratch.reserve(w0); if (rc) return rc; }
    const size_t n_off = std::max<size_t>(1, size_t(g.nyaw) * S.pts.size());
    { int rc = B.d_off.reserve(n_off); if (rc) return rc; }
    { int rc = global_upload(c, S); if (rc) return rc; }
    timed_launch_begin(c);
    SO_CUDA_TRY(cudaMemsetAsync(B.d_scratch, 0, w0 * sizeof(uint32_t), st));
    launch_bnb_raster(c->surf.d_xyzi, c->surf.n, g, p, B.d_scratch, st);
    if (P.whole) { int rc = archive_raster(c, g, p, B.d_scratch); if (rc) return rc; }
    timed_launch_end(c, 6, 1);
    SO_CUDA_TRY(cudaEventRecord(B.ev[1], st));
    RelocGrid gw{};                                                 // level 0 as k_reloc_dilate sees it: the window, same dilation
    gw.bx = p.wx; gw.by = p.wy; gw.bz = p.wz; gw.wpr = p.wpr[0];
    timed_launch_begin(c);
    launch_reloc_dilate(gw, P.o.dilate, B.d_scratch, B.d_pyr, st);  // ends in its second buffer: level 0
    c->launches += 2;
    timed_launch_end(c, 6, 1);
    timed_launch_begin(c);
    launch_bnb_levels(p, B.d_pyr, st);
    c->launches += p.lmax > 0 ? p.lmax - 1 : 0;
    timed_launch_end(c, 6, 1);
    timed_launch_begin(c);
    launch_bnb_offsets(B.d_pts, int(S.pts.size()), B.d_q, g, p, B.d_off, st);
    timed_launch_end(c, 6, 1);
    SO_CUDA_TRY(cudaEventRecord(B.ev[2], st));
    SO_CUDA_TRY(cudaGetLastError());
    *g_out = g; *p_out = p; *pyr_words = words;
    return SO_OK;
}

static int bnb_reset_ctl(Ctx* c) {
    Ctx::Bnb& B = c->bnb;
    std::memset(B.h_ctl, 0, sizeof(BnbCtl));
    B.h_ctl->kstar = kBnbNone;
    SO_CUDA_TRY(cudaMemcpyAsync(B.d_ctl, B.h_ctl, sizeof(BnbCtl), cudaMemcpyHostToDevice, c->stream));
    return SO_OK;
}

// The traversal.  Node keys are (65535 - U) << 32 | lin(m, k, j0, i0); a node is discarded when its key is above K*, the P-th
// smallest leaf key found so far.  Each step expands the first C admitted nodes of the finest non-empty level (whose buffer is
// sorted), so the level below is empty when it receives at most 4C children.  keys <- the P smallest hypothesis keys, ascending.
static int bnb_search(Ctx* c, const RelocGrid& g, const BnbPyramid& p, int n_pts, size_t n_keys, uint64_t* keys, uint64_t* steps_out) {
    Ctx::Bnb& B = c->bnb;
    cudaStream_t st = c->stream;
    { int rc = bnb_reset_ctl(c); if (rc) return rc; }
    SO_CUDA_TRY(cudaMemsetAsync(B.d_merge[0], 0xff, n_keys * sizeof(uint64_t), st));
    const int lmax = p.lmax;
    const uint64_t root_n = bnb_level_nodes(g, lmax);
    BnbTrim t{};
    t.lmax = lmax;
    t.base[lmax] = 0;
    for (int l = 1; l < lmax; ++l) t.base[l] = uint64_t(kBnbRoot) + uint64_t(l - 1) * 4 * kBnbBatch;
    uint64_t r0 = 0, steps = 0;
    for (;;) {
        int L = 0;
        for (int l = 1; l <= lmax; ++l) if (t.head[l] < t.cnt[l]) { L = l; break; }
        if (L == 0 && r0 >= root_n) break;
        timed_launch_begin(c);
        if (L == 0) {                                               // every level drained: the next chunk of the root
            const uint32_t nr = uint32_t(std::min<uint64_t>(kBnbRoot, root_n - r0));
            launch_bnb_score(g, p, B.d_pyr, B.d_off, n_pts, lmax, nullptr, r0, nr, B.d_ctl, B.d_unsorted, st);
            { int rc = bnb_sort(B.d_tmp, B.d_tmp.cap(), B.d_unsorted, B.d_nodes + t.base[lmax], nr, st); if (rc) return rc; }
            r0 += nr;
            t.head[lmax] = 0; t.cnt[lmax] = nr;
        } else {
            const uint32_t take = uint32_t(std::min<uint64_t>(kBnbBatch, t.cnt[L] - t.head[L]));
            const uint64_t* parents = B.d_nodes + t.base[L] + t.head[L];
            t.head[L] += take;
            if (L == 1) {                                           // leaves: merge into the running top P
                launch_bnb_score(g, p, B.d_pyr, B.d_off, n_pts, 0, parents, 0, 4 * take, B.d_ctl, B.d_merge[0] + n_keys, st);
                { int rc = bnb_sort(B.d_tmp, B.d_tmp.cap(), B.d_merge[0], B.d_merge[1], n_keys + 4 * take, st); if (rc) return rc; }
                SO_CUDA_TRY(cudaMemcpyAsync(B.d_merge[0], B.d_merge[1], n_keys * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
                SO_CUDA_TRY(cudaMemcpyAsync(&B.d_ctl->kstar, B.d_merge[1] + n_keys - 1, sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
            } else {
                launch_bnb_score(g, p, B.d_pyr, B.d_off, n_pts, L - 1, parents, 0, 4 * take, B.d_ctl, B.d_unsorted, st);
                { int rc = bnb_sort(B.d_tmp, B.d_tmp.cap(), B.d_unsorted, B.d_nodes + t.base[L - 1], 4 * take, st); if (rc) return rc; }
                t.head[L - 1] = 0; t.cnt[L - 1] = 4 * take;
            }
        }
        launch_bnb_trim(t, B.d_nodes, B.d_ctl, st);
        c->launches += 2;
        timed_launch_end(c, 6, 1);
        SO_CUDA_TRY(cudaMemcpyAsync(B.h_ctl, B.d_ctl, sizeof(BnbCtl), cudaMemcpyDeviceToHost, st));
        count_d2h(c, sizeof(BnbCtl));
        SO_CUDA_TRY(cudaStreamSynchronize(st));
        for (int l = 1; l <= lmax; ++l) t.cnt[l] = B.h_ctl->cnt[l];
        ++steps;
    }
    SO_CUDA_TRY(cudaEventRecord(B.ev[3], st));
    SO_CUDA_TRY(cudaMemcpyAsync(keys, B.d_merge[0], n_keys * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    SO_CUDA_TRY(cudaMemcpyAsync(B.h_ctl, B.d_ctl, sizeof(BnbCtl), cudaMemcpyDeviceToHost, st));
    count_d2h(c, n_keys * sizeof(uint64_t) + sizeof(BnbCtl));
    SO_CUDA_TRY(cudaStreamSynchronize(st));
    SO_CUDA_TRY(cudaGetLastError());
    *steps_out = steps;
    return SO_OK;
}

// Build + search: the first min(n_hyp, 64 k) keys of the ascending order of every hypothesis' key, and the statistics.  64 keys per
// candidate asked for leave room for the hypotheses the suppression drops around each kept one.
static int bnb_run(Ctx* c, const GlobalPlan& P, const GlobalScan& S, std::vector<uint64_t>* keys, so_bnb_stats* stats) {
    RelocGrid g;
    BnbPyramid p;
    uint64_t words = 0, steps = 0;
    { int rc = bnb_build(c, P, S, &g, &p, &words); if (rc) return rc; }
    keys->assign(std::min<size_t>(P.n_hyp, size_t(64) * P.o.k), 0);
    { int rc = bnb_search(c, g, p, int(S.pts.size()), keys->size(), keys->data(), &steps); if (rc) return rc; }
    if (stats) {
        const BnbCtl& k = *c->bnb.h_ctl;
        std::memset(stats, 0, sizeof(*stats));
        stats->lmax = p.lmax;
        stats->root_nodes = bnb_level_nodes(g, p.lmax);
        for (int l = 0; l <= p.lmax; ++l) { stats->scored[l] = k.scored[l]; stats->discarded[l] = k.discarded[l]; }
        stats->leaves_scored = k.scored[0];
        stats->steps = steps;
        stats->kstar_score = keys->empty() ? 0 : key_score(keys->back());
        stats->pyramid_bytes = words * sizeof(uint32_t);
        float ms = 0.f;
        cudaEventElapsedTime(&ms, c->bnb.ev[0], c->bnb.ev[2]); stats->time_build_ms = ms;
        cudaEventElapsedTime(&ms, c->bnb.ev[2], c->bnb.ev[3]); stats->time_search_ms = ms;
    }
    return SO_OK;
}

// ---------------------------------------------------------------------------------------------- entry points
// The rest of every entry point's prologue, after its own argument checks: the score points, the offset-table cap (so that its
// capacity error comes before any device work), the device, the yaw quaternions.
static int global_prologue(Ctx* c, const GlobalPlan& P, const void* xyzi, size_t n, size_t stride, size_t ioff, const double center[7],
                           GlobalScan* S) {
    select_score_points(xyzi, n, stride, ioff, P.o, S);
    { int rc = bnb_check_table(P, *S); if (rc) return rc; }
    SO_CUDA_TRY(cudaSetDevice(c->device));
    yaw_quaternions(P, center, S);
    return SO_OK;
}

// so_localize_global (bnb = false) and so_localize_global_bnb, which differ in their limits only: the sorted key prefix from the
// search, then global_refine.  Stage times: the build up to the raster, the rest of the build, and the traversal, with no sort
// (time_sort_ms = 0).
static int localize(Ctx* c, bool bnb, const void* xyzi, size_t n, size_t stride, size_t ioff, const double center[7], const so_global_opts* gopts,
                    const so_icp_opts* opts, so_global_candidate* cands, size_t cap, so_global_result* out, so_bnb_stats* stats) {
    GlobalPlan P;
    int rc = global_check_args(c, xyzi, n, stride, center, gopts, &P, bnb);
    if (rc) return rc;
    if (!opts || !out || (!cands && cap)) return fail(SO_ERR_ARG, "bad args");
    rc = icp_opts_check(*opts);
    if (rc) return rc;
    const auto t0 = std::chrono::steady_clock::now();
    GlobalScan S;
    rc = global_prologue(c, P, xyzi, n, stride, ioff, center, &S);
    if (rc) return rc;
    std::memset(out, 0, sizeof(*out));
    std::memcpy(out->pose, center, 7 * sizeof(double));
    out->winner = -1;
    out->n_hypotheses = P.n_hyp;
    out->n_score_points = int32_t(S.pts.size());
    std::vector<uint64_t> pref;
    rc = bnb_run(c, P, S, &pref, stats);
    if (rc) return rc;
    const auto t1 = std::chrono::steady_clock::now();
    double* stage[3] = {&out->time_raster_ms, &out->time_dilate_ms, &out->time_score_ms};
    for (int s = 0; s < 3; ++s) { float ms = 0.f; cudaEventElapsedTime(&ms, c->bnb.ev[s], c->bnb.ev[s + 1]); *stage[s] = double(ms); }
    return global_refine(c, P, S, pref.data(), pref.size(), xyzi, n, stride, ioff, opts, cands, cap, out, t0, t1);
}

// so_localize_scores (level 0: the score of every hypothesis) and so_localize_bnb_bounds: every node bound of one level, with no
// pruning, in (yaw, z shift, tile y, tile x) order.
static int bnb_dense(Ctx* c, const GlobalPlan& P, const GlobalScan& S, int level, uint16_t* bounds) {
    RelocGrid g;
    BnbPyramid p;
    uint64_t words = 0;
    { int rc = bnb_build(c, P, S, &g, &p, &words); if (rc) return rc; }
    { int rc = bnb_reset_ctl(c); if (rc) return rc; }
    const uint64_t total = bnb_level_nodes(g, level);
    std::vector<uint64_t> buf(kBnbRoot);
    for (uint64_t r0 = 0; r0 < total; r0 += kBnbRoot) {
        const uint32_t nr = uint32_t(std::min<uint64_t>(kBnbRoot, total - r0));
        timed_launch_begin(c);
        launch_bnb_score(g, p, c->bnb.d_pyr, c->bnb.d_off, int(S.pts.size()), level, nullptr, r0, nr, c->bnb.d_ctl, c->bnb.d_unsorted, c->stream);
        timed_launch_end(c, 6, 1);
        SO_CUDA_TRY(cudaMemcpyAsync(buf.data(), c->bnb.d_unsorted, nr * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
        count_d2h(c, nr * sizeof(uint64_t));
        SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
        for (uint32_t i = 0; i < nr; ++i) bounds[r0 + i] = uint16_t(key_score(buf[i]));
    }
    SO_CUDA_TRY(cudaGetLastError());
    return SO_OK;
}

}  // namespace so

// =================================================================================================== C ABI
using namespace so;

extern "C" {

int so_localize_global_size(const so_global_opts* gopts, int32_t dims[4], uint64_t* n_hyp, uint64_t* bitmap_bytes) {
    GlobalPlan P;
    const int rc = global_plan(gopts, &P);
    if (rc == SO_ERR_ARG) return rc;
    if (dims) plan_dims(P, dims);
    if (n_hyp) *n_hyp = P.n_hyp;
    if (bitmap_bytes) *bitmap_bytes = P.bitmap_words < UINT64_MAX / 4 ? P.bitmap_words * 4 : UINT64_MAX;
    return rc;
}

int so_localize_scores(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, const double center[7], const so_global_opts* gopts,
                       uint16_t* scores, size_t cap, int32_t dims[4], int32_t* n_score_points) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    GlobalPlan P;
    int rc = global_check_args(c, xyzi, n, stride, center, gopts, &P);
    if (rc) return rc;
    if (!scores || !dims) return fail(SO_ERR_ARG, "bad args");
    if (cap < P.n_hyp) return fail(SO_ERR_CAPACITY, "score array smaller than the hypothesis count");
    GlobalScan S;
    rc = global_prologue(c, P, xyzi, n, stride, ioff, center, &S);
    if (rc) return rc;
    rc = bnb_dense(c, P, S, 0, scores);
    if (rc) return rc;
    plan_dims(P, dims);
    if (n_score_points) *n_score_points = int32_t(S.pts.size());
    return SO_OK;
}

int so_localize_global(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, const double center[7], const so_global_opts* gopts,
                       const so_icp_opts* opts, so_global_candidate* cands, size_t cap, so_global_result* out) {
    return localize(reinterpret_cast<Ctx*>(ctx), false, xyzi, n, stride, ioff, center, gopts, opts, cands, cap, out, nullptr);
}

int so_localize_global_bnb(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, const double center[7], const so_global_opts* gopts,
                           const so_icp_opts* opts, so_global_candidate* cands, size_t cap, so_global_result* out, so_bnb_stats* stats) {
    return localize(reinterpret_cast<Ctx*>(ctx), true, xyzi, n, stride, ioff, center, gopts, opts, cands, cap, out, stats);
}

int so_localize_bnb_keys(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, const double center[7], const so_global_opts* gopts,
                         uint64_t* keys, size_t cap, size_t* n_keys, so_bnb_stats* stats) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    GlobalPlan P;
    int rc = global_check_args(c, xyzi, n, stride, center, gopts, &P, true);
    if (rc) return rc;
    if ((!keys && cap) || !n_keys) return fail(SO_ERR_ARG, "bad args");
    GlobalScan S;
    rc = global_prologue(c, P, xyzi, n, stride, ioff, center, &S);
    if (rc) return rc;
    std::vector<uint64_t> pref;
    rc = bnb_run(c, P, S, &pref, stats);
    if (rc) return rc;
    std::memcpy(keys, pref.data(), std::min(cap, pref.size()) * sizeof(uint64_t));
    *n_keys = pref.size();
    return SO_OK;
}

int so_localize_bnb_bounds(so_ctx* ctx, const void* xyzi, size_t n, size_t stride, size_t ioff, const double center[7], const so_global_opts* gopts,
                           int level, uint16_t* bounds, size_t cap, int32_t dims[4]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    GlobalPlan P;
    int rc = global_check_args(c, xyzi, n, stride, center, gopts, &P, true);
    if (rc) return rc;
    if ((!bounds && cap) || !dims) return fail(SO_ERR_ARG, "bad args");
    if (level < 0 || level > bnb_lmax(P.g)) return fail(SO_ERR_ARG, "level must be in [0, Lmax]");
    const int32_t s = 1 << level;
    dims[0] = int32_t((int64_t(P.g.nx) + s - 1) >> level); dims[1] = int32_t((int64_t(P.g.ny) + s - 1) >> level);
    dims[2] = P.g.nz; dims[3] = P.g.nyaw;
    if (cap < bnb_level_nodes(P.g, level)) return fail(SO_ERR_CAPACITY, "bound array smaller than the level's node count");
    GlobalScan S;
    rc = global_prologue(c, P, xyzi, n, stride, ioff, center, &S);
    if (rc) return rc;
    return bnb_dense(c, P, S, level, bounds);
}

int so_map_bounds(so_ctx* ctx, float lo[3], float hi[3], size_t* n) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !lo || !hi || !n) return fail(SO_ERR_ARG, "bad args");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    for (int a = 0; a < 3; ++a) lo[a] = hi[a] = 0.f;
    return map_bounds(c, lo, hi, n);
}

int so_map_bounds_all(so_ctx* ctx, float lo[3], float hi[3], size_t* n) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !lo || !hi || !n) return fail(SO_ERR_ARG, "bad args");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    for (int a = 0; a < 3; ++a) lo[a] = hi[a] = 0.f;
    return map_bounds(c, lo, hi, n, true);
}

}  // extern "C"

// so_free.cu -- free-space clearing (so_map_clear_free_space*): remove the map points a scan saw clearly past.
//
// No reference counterpart: LocalMap::addSurfPointCloud only adds points, so anything that moved stays in the map.  The rule is a
// visibility test against a range image of the scan (DESIGN.md §2): one thread per scan point builds the image (k_range_image, an
// atomicMin on the bits of the float range -- positive floats order as unsigned ints, so the image does not depend on the order of the
// atomics), one thread per window map point tests it (k_free_mark), and the store drops the marked points through a stable compaction
// and the existing index stage (map_compact, so_map.cu).
#include <cmath>

#include "so_ctx.cuh"

namespace so {

constexpr uint32_t kUnknown = 0xFFFFFFFFu;     // pixel without a return: above the bits of every positive float (and of +inf)
constexpr double kPiD = 3.141592653589793;

// Image geometry and decision constants, all in double (angles in radians)
struct FreeGrid {
    double az_res, el_res, el_min, el_max;
    int32_t W, H, d, pad;
    double margin, margin_rel, min_range, max_range;
};
struct FreePose { double R[9]; double t[3]; };  // row-major R of the (normalised) pose quaternion; the map point goes to R^T (m - t)

// Device counters of one call, read back once
struct FreeCounters {
    uint32_t image_points, pixels_hit;
    uint32_t cand[2], removed[2];
    uint32_t selected, pad;                     // cub::DeviceSelect's count (not read back: the host knows it)
};

// Pixel of a sensor-frame direction, or false when its elevation is outside [el_min, el_max).  Written without contractible
// multiply-adds, so that a restatement in numpy takes the same roundings.
__device__ __forceinline__ bool free_pixel(const FreeGrid& g, double x, double y, double z, int* row, int* col) {
    double az = atan2(y, x);
    if (az >= kPiD) az = __dsub_rn(az, 2.0 * kPiD);                  // [-pi, pi)
    const double el = atan2(z, hypot(x, y));
    if (!(el >= g.el_min && el < g.el_max)) return false;
    const int r = int(floor(__ddiv_rn(__dsub_rn(el, g.el_min), g.el_res)));
    if (r < 0 || r >= g.H) return false;
    int c = int(floor(__ddiv_rn(__dadd_rn(az, kPiD), g.az_res)));
    if (c > g.W - 1) c = g.W - 1;
    *row = r; *col = c;
    return true;
}

__device__ __forceinline__ double norm3(double x, double y, double z) {
    return sqrt(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}

// warp-aggregated counter increment: one atomic per warp (every lane of the warp calls it)
__device__ __forceinline__ void warp_count(uint32_t* ctr, bool flag) {
    const unsigned b = __ballot_sync(0xffffffffu, flag);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(ctr, uint32_t(__popc(b)));
}

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

// keep[i] = 0 when window point i is removed.  The range test comes before any pixel work.
__global__ void __launch_bounds__(256) k_free_mark(const float4* __restrict__ pts, uint32_t n, FreeGrid g, FreePose P,
                                                   const uint32_t* __restrict__ img, uint8_t* __restrict__ keep,
                                                   uint32_t* __restrict__ cand_ctr, uint32_t* __restrict__ rem_ctr) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    bool cand = false, rem = false;
    if (i < n) {
        const float4 p = pts[i];
        const double dx = __dsub_rn(double(p.x), P.t[0]), dy = __dsub_rn(double(p.y), P.t[1]), dz = __dsub_rn(double(p.z), P.t[2]);
        auto rt = [&](int a) {                                          // row a of R^T (m - t): column a of R
            return __dadd_rn(__dadd_rn(__dmul_rn(dx, P.R[a]), __dmul_rn(dy, P.R[3 + a])), __dmul_rn(dz, P.R[6 + a]));
        };
        const double qx = rt(0), qy = rt(1), qz = rt(2);
        const double rm = norm3(qx, qy, qz);
        int row, col;
        if (rm >= g.min_range && rm <= g.max_range && free_pixel(g, qx, qy, qz, &row, &col) && row - g.d >= 0 && row + g.d < g.H) {
            uint32_t mn = kUnknown;
            bool known = true;
            for (int dr = -g.d; dr <= g.d && known; ++dr) {
                const uint32_t* line = img + size_t(row + dr) * g.W;
                for (int dc = -g.d; dc <= g.d; ++dc) {
                    int c = (col + dc) % g.W;
                    if (c < 0) c += g.W;
                    const uint32_t v = line[c];
                    if (v == kUnknown) { known = false; break; }
                    mn = min(mn, v);
                }
            }
            if (known) {
                cand = true;
                const double thr = __dadd_rn(rm, fmax(g.margin, __dmul_rn(g.margin_rel, rm)));
                rem = double(__uint_as_float(mn)) > thr;
            }
        }
        keep[i] = rem ? 0 : 1;
    }
    warp_count(cand_ctr, cand);
    warp_count(rem_ctr, rem);
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

int free_space_clear(Ctx* c, int stores, const float4* d_pts, uint32_t n_pts, const double pose[7], const so_free_space& o,
                     so_free_space_result* out) {
    cudaStream_t st = c->stream;
    FreeGrid g{};
    g.az_res = double(o.az_res_deg) * (kPiD / 180.0); g.el_res = double(o.el_res_deg) * (kPiD / 180.0);
    g.el_min = double(o.el_min_deg) * (kPiD / 180.0); g.el_max = double(o.el_max_deg) * (kPiD / 180.0);
    g.W = int(std::ceil(360.0 / double(o.az_res_deg)));
    g.H = int(std::ceil((double(o.el_max_deg) - double(o.el_min_deg)) / double(o.el_res_deg)));
    g.d = o.dilate;
    g.margin = o.margin; g.margin_rel = o.margin_rel; g.min_range = o.min_range; g.max_range = o.max_range;
    FreePose P{};
    {
        const double* q = pose + 3;
        const double nq = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        const double x = q[0] / nq, y = q[1] / nq, z = q[2] / nq, w = q[3] / nq;
        const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                             2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                             2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
        for (int k = 0; k < 9; ++k) P.R[k] = R[k];
        for (int k = 0; k < 3; ++k) P.t[k] = pose[k];
    }
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

}  // namespace so

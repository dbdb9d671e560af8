// so_free.cuh -- the visibility test of free-space clearing (DESIGN.md §2), shared by the clearing (so_free.cu) and loop verification
// (so_verify.cu): the range-image geometry, the pixel of a direction, the decision on one map point against one image, the counters.
#pragma once
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

// so_map_clear_free_space_keyframes: tile entry j of the images, pool[src .. src + n) are points start .. start + n of the tile
struct KfImgSeg { uint64_t src; uint32_t start, n; };
struct FreeKfCounters {
    unsigned long long image_points, pixels_hit;
    unsigned long long cand[2], removed[2];
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

__device__ __forceinline__ void warp_count64(unsigned long long* ctr, bool flag) {
    const unsigned b = __ballot_sync(0xffffffffu, flag);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(ctr, (unsigned long long)__popc(b));
}

// The decision on map point p against one image: true when it is removed; *cand when its neighbourhood is fully observed.  The range
// test comes before any pixel work.
__device__ __forceinline__ bool free_decide(const FreeGrid& g, const FreePose& P, const float4 p, const uint32_t* __restrict__ img, bool* cand) {
    const double dx = __dsub_rn(double(p.x), P.t[0]), dy = __dsub_rn(double(p.y), P.t[1]), dz = __dsub_rn(double(p.z), P.t[2]);
    auto rt = [&](int a) {                                              // row a of R^T (m - t): column a of R
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
            *cand = true;
            const double thr = __dadd_rn(rm, fmax(g.margin, __dmul_rn(g.margin_rel, rm)));
            return double(__uint_as_float(mn)) > thr;
        }
    }
    return false;
}

// Host side (so_free.cu): the image geometry of the options, the decision pose of a pose7, and the image kernels.  img / imgs must be
// filled with kUnknown (0xFF bytes) first; each pixel keeps the minimum float range of its points.
FreeGrid free_grid(const so_free_space& o);
FreePose free_pose(const double pose[7]);
// The range image of the sensor-frame points pts[0..n) (k_range_image)
void launch_range_image(const float4* pts, uint32_t n, const FreeGrid& g, uint32_t* img, FreeCounters* cnt, cudaStream_t st);
// The range images of one tile, image j of the points segs[j] names in pool, at imgs + j * W * H (k_range_images); n: the tile's points
void launch_range_images(const float4* pool, const KfImgSeg* segs, uint32_t n_segs, uint32_t n, const FreeGrid& g, uint32_t* imgs,
                         FreeKfCounters* cnt, cudaStream_t st);

}  // namespace so

// CPU test of the keyframe cull of so_map_clear_free_space_keyframes (superodom_b200/csrc/so_free_rule.h): the block bucketing is the
// store's own (grid_block, so_map.cu, restated below), and no culled (block, keyframe) pair holds a map point whose FP64 sensor range, as
// k_free_mark computes it, is at most max_range.  Points are random and adversarial: on block faces, at max_range and one float step
// either side of it, with sensors on and off the grid and rotated.  Build with -ffp-contract=off so that the range takes the kernel's
// roundings.  Prints "ok <pairs tested> <pairs in range> <pairs culled>" and exits 0 on success.
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include "../../superodom_b200/csrc/so_free_rule.h"

#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

// grid_block of so_map.cu, as written there
static int store_block(float x, float y, float z, const int32_t o[3]) {
    auto coord = [](double v, int origin) { int c = int(v / 50.0); if (v < 0) c--; return c + origin; };
    const int gx = coord(double(x) + 25.0, o[0]), gy = coord(double(y) + 25.0, o[1]), gz = coord(double(z) + 25.0, o[2]);
    if (gx >= 0 && gx < 21 && gy >= 0 && gy < 21 && gz >= 0 && gz < 11 && std::isfinite(x) && std::isfinite(y) && std::isfinite(z))
        return gx + 21 * gy + 21 * 21 * gz;
    return -1;
}

struct Pose { double R[9], t[3]; };

// free_pose (so_free.cu): the rotation of the normalised quaternion xyzw
static Pose make_pose(const double t[3], const double q[4]) {
    Pose P;
    const double nq = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double x = q[0] / nq, y = q[1] / nq, z = q[2] / nq, w = q[3] / nq;
    const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                         2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                         2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
    for (int k = 0; k < 9; ++k) P.R[k] = R[k];
    for (int k = 0; k < 3; ++k) P.t[k] = t[k];
    return P;
}

// r_m of free_decide: R^T (m - t) and norm3, one rounding per operation
static double range_of(const Pose& P, const float m[3]) {
    const double dx = double(m[0]) - P.t[0], dy = double(m[1]) - P.t[1], dz = double(m[2]) - P.t[2];
    double q[3];
    for (int a = 0; a < 3; ++a) q[a] = (dx * P.R[a] + dy * P.R[3 + a]) + dz * P.R[6 + a];
    return std::sqrt((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]);
}

int main() {
    using namespace so;
    std::mt19937_64 rng(11);
    std::uniform_real_distribution<double> uni(-1.0, 1.0);
    const int32_t origins[3][3] = {{10, 10, 5}, {-3, 17, 2}, {30, -12, 9}};
    const float max_ranges[3] = {60.f, 25.3f, 130.f};
    size_t tested = 0, in_range = 0, culled = 0, near_edge = 0;

    // the bucketing is the store's
    for (int it = 0; it < 200000; ++it) {
        const int32_t* o = origins[it % 3];
        float p[3];
        for (int a = 0; a < 3; ++a) {
            const double face = 50.0 * double(int(std::floor(uni(rng) * 12))) - 25.0 - 50.0 * o[a] + 50.0 * (a == 2 ? 5 : 10);
            p[a] = float(face);
            for (int s = int(rng() % 7) - 3; s != 0; s += s > 0 ? -1 : 1) p[a] = std::nextafter(p[a], s > 0 ? INFINITY : -INFINITY);
            if (rng() % 4 == 0) p[a] = float(face + 60.0 * uni(rng));
        }
        CHECK(free_grid_block(p[0], p[1], p[2], o) == store_block(p[0], p[1], p[2], o));
    }
    CHECK(free_grid_block(NAN, 0.f, 0.f, origins[0]) == -1 && free_grid_block(0.f, INFINITY, 0.f, origins[0]) == -1);

    auto test_pair = [&](const Pose& P, const float m[3], const int32_t o[3], float max_range) -> bool {
        const int b = free_grid_block(m[0], m[1], m[2], o);
        if (b < 0) return true;
        double lo[3], hi[3];
        free_block_box(b, o, lo, hi);
        const bool reach = free_block_in_reach(lo, hi, P.t, double(max_range));
        const double rm = range_of(P, m);
        ++tested;
        if (rm <= double(max_range)) ++in_range;
        if (!reach) ++culled;
        if (std::fabs(rm - double(max_range)) < 1e-3) ++near_edge;
        return reach || rm > double(max_range);
    };

    for (int it = 0; it < 400000; ++it) {
        const int32_t* o = origins[it % 3];
        const float max_range = max_ranges[(it / 3) % 3];
        // a sensor on the grid (a block corner, face or centre) or anywhere in the window, upright or rotated
        double t[3];
        for (int a = 0; a < 3; ++a) {
            const double base = -50.0 * o[a] + 50.0 * (a == 2 ? 5 : 10);
            const int kind = int(rng() % 3);
            t[a] = kind == 0 ? base + 50.0 * double(int(uni(rng) * 8)) - 25.0
                 : kind == 1 ? base + 50.0 * double(int(uni(rng) * 8)) : base + 400.0 * uni(rng) * (a == 2 ? 0.4 : 1.0);
        }
        double q[4] = {0, 0, 0, 1};
        if (rng() % 2) for (double& v : q) v = uni(rng);
        if (rng() % 8 == 0) { q[0] = q[1] = q[2] = 0; q[3] = -3.0; }  // unnormalised
        const Pose P = make_pose(t, q);
        // a point at max_range from the sensor along a random direction, then moved onto the nearest block face along one axis, and
        // float steps either side of both
        double d[3] = {uni(rng), uni(rng), uni(rng)};
        const double nd = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        float m[3];
        for (int a = 0; a < 3; ++a) m[a] = float(t[a] + double(max_range) * d[a] / nd);
        const int ax = int(rng() % 3);
        if (rng() % 2) {                                              // onto a face: the sensor's reach ends there
            const double f = 50.0 * std::round((double(m[ax]) + 25.0) / 50.0) - 25.0;
            m[ax] = float(f);
            // put the range back at max_range over the other two axes where it can be
            const double rest = double(max_range) * double(max_range) - (f - t[ax]) * (f - t[ax]);
            const int b1 = (ax + 1) % 3, b2 = (ax + 2) % 3;
            const double cur = (double(m[b1]) - t[b1]) * (double(m[b1]) - t[b1]) + (double(m[b2]) - t[b2]) * (double(m[b2]) - t[b2]);
            if (rest > 0 && cur > 0) {
                const double s = std::sqrt(rest / cur);
                m[b1] = float(t[b1] + (double(m[b1]) - t[b1]) * s);
                m[b2] = float(t[b2] + (double(m[b2]) - t[b2]) * s);
            }
        }
        for (int s = -3; s <= 3; ++s) {
            float mm[3] = {m[0], m[1], m[2]};
            const int a = (s + 3 + it) % 3;
            for (int k = 0; k < std::abs(s); ++k) mm[a] = std::nextafter(mm[a], s > 0 ? INFINITY : -INFINITY);
            CHECK(test_pair(P, mm, o, max_range));
        }
    }
    // axis-aligned: the sensor exactly max_range from a face point, the point on the face and one float step into either block
    for (int k = -8; k <= 8; ++k) {
        const int32_t* o = origins[0];
        const float face = float(50.0 * k - 25.0);
        for (float mr : max_ranges) {
            const double t[3] = {double(face) - double(mr), 3.0, 1.0}, q[4] = {0, 0, 0, 1};
            const Pose P = make_pose(t, q);
            for (float x : {face, std::nextafter(face, -INFINITY), std::nextafter(face, INFINITY)}) {
                const float m[3] = {x, 3.f, 1.f};
                CHECK(test_pair(P, m, o, mr));
            }
        }
    }
    // the cull is tight: a block whose nearest face lies a metre past max_range is culled, one just inside is not
    {
        double lo[3], hi[3];
        const int32_t o[3] = {10, 10, 5};
        free_block_box(10 + 21 * 10 + 21 * 21 * 5, o, lo, hi);       // the block around the world origin: [-25, 25)^3
        const double t_out[3] = {25.0 + 61.0, 0, 0}, t_in[3] = {25.0 + 59.9, 0, 0};
        CHECK(!free_block_in_reach(lo, hi, t_out, 60.0));
        CHECK(free_block_in_reach(lo, hi, t_in, 60.0));
        const double t_nan[3] = {NAN, 0, 0};
        CHECK(free_block_in_reach(lo, hi, t_nan, 60.0));
    }
    CHECK(in_range > 1000 && culled > 1000 && near_edge > 1000);
    std::printf("ok %zu %zu %zu\n", tested, in_range, culled);
    return 0;
}

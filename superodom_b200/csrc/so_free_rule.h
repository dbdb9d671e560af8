// so_free_rule.h -- the keyframe cull of so_map_clear_free_space_keyframes (plain C++: shared by the kernels in so_free.cu and a CPU
// test).
//
// A keyframe can remove a map point only when the point's FP64 sensor range r_m (k_free_mark) is at most max_range.  The batched
// clearing tests a (window block, keyframe) pair only when the keyframe's sensor position can lie within max_range of a point the store
// buckets into that block; the cull below must never skip a pair that holds such a point.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>

#ifdef __CUDACC__
#define SO_FR_HD __host__ __device__ __forceinline__
#else
#define SO_FR_HD inline
#endif

namespace so {

constexpr int kFreeW = 21, kFreeH = 21, kFreeD = 11;           // the window's blocks (kW, kH, kD in so_internal.cuh)
constexpr double kFreeBlock = 50.0, kFreeHalfBlock = 25.0;     // block edge and the offset of block 0's lower face (kBlock, kHalfBlock)
// Range images of one tile of keyframes fit this many bytes: 2^26 pixels of 4 bytes, so at least four of the largest image
// free_space_check admits (2^24 pixels) and 648 of the OS1-128 defaults (900 x 115 pixels)
constexpr size_t kFreeTileBytes = size_t(256) << 20;

// Window block of a map point, as the store buckets it (grid_block, so_map.cu: LocalMap.h:594-605 per axis, then the linear index),
// or -1 off the window
SO_FR_HD int free_coord(double v, int origin) {
    int c = int(v / kFreeBlock);
    if (v < 0) c--;
    return c + origin;
}
SO_FR_HD int free_grid_block(float x, float y, float z, const int32_t origin[3]) {
    const int gx = free_coord(double(x) + kFreeHalfBlock, origin[0]), gy = free_coord(double(y) + kFreeHalfBlock, origin[1]),
              gz = free_coord(double(z) + kFreeHalfBlock, origin[2]);
    if (gx >= 0 && gx < kFreeW && gy >= 0 && gy < kFreeH && gz >= 0 && gz < kFreeD && std::isfinite(x) && std::isfinite(y) && std::isfinite(z))
        return gx + kFreeW * gy + kFreeW * kFreeH * gz;
    return -1;
}

// The box of window block b under origin, padded at every face: free_coord's sum and quotient round, so a point at a face can land in
// either neighbour.  Each rounding is relative (2^-53 of a value within 2 (|lo| + |hi| + 50) here); the pad is 10^-9 of that scale.
SO_FR_HD void free_block_box(int b, const int32_t origin[3], double lo[3], double hi[3]) {
    const int g[3] = {b % kFreeW, (b / kFreeW) % kFreeH, b / (kFreeW * kFreeH)};
    for (int a = 0; a < 3; ++a) {
        const double l = double(g[a] - origin[a]) * kFreeBlock - kFreeHalfBlock, h = l + kFreeBlock;
        const double pad = 1e-9 * (std::fabs(l) + std::fabs(h) + kFreeBlock);
        lo[a] = l - pad;
        hi[a] = h + pad;
    }
}

// false only when every point of the (padded) box lies farther than max_range from the sensor position t, with a relative slack of
// 10^-9: every FP64 operation on the way to r_m (differences, the rotation by a normalised quaternion's matrix, norm3) and to the box
// distance here errs by a few 2^-53 of its own scale, far inside that slack.  A NaN distance keeps the pair.
SO_FR_HD bool free_block_in_reach(const double lo[3], const double hi[3], const double t[3], double max_range) {
    double s = 0.0;
    for (int a = 0; a < 3; ++a) {
        const double d = t[a] < lo[a] ? lo[a] - t[a] : (t[a] > hi[a] ? t[a] - hi[a] : 0.0);
        s += d * d;
    }
    return !(std::sqrt(s) > max_range * (1.0 + 1e-9));
}

}  // namespace so

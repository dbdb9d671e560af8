// so_archive.h -- world block keys of the block archive (plain C++: shared by so_map.cu, its kernels and a CPU unit test).
//
// With the archive on, a map store behaves like a LocalMap over an unbounded block grid seen through the 21 x 21 x 11 window.  A
// block is named by its world block coordinate w = g - origin, where g is the grid index grid_block computes; w does not depend on
// the origin.  Blocks the window drops are kept in the archive under the key of w, and come back when the window reaches them again.
#pragma once
#include <cmath>
#include <cstdint>

#ifdef __CUDACC__
#define SO_ARCHIVE_HD __host__ __device__
#else
#define SO_ARCHIVE_HD
#endif

namespace so {
namespace archive {

constexpr int kWinW = 21, kWinH = 21, kWinD = 11;    // the window: LocalMap's laserCloudWidth / Height / Depth
constexpr int kKeyBits = 20;                         // bits per axis of a world key
constexpr int kKeyOff = 1 << (kKeyBits - 1);         // w in [-2^19, 2^19): +-26 214 km at 50 m blocks
constexpr double kBlockM = 50.0, kHalfBlockM = 25.0;
constexpr uint64_t kKeyNone = ~uint64_t(0);

// World block coordinate of one axis, as LocalMap.h:594-605 bins a point (int((v + 25) / 50), minus one below zero, double math on
// the float coordinate): false when v is not finite or its block lies outside the key range.
SO_ARCHIVE_HD inline bool world_axis(float x, int* w) {
    const double v = double(x) + kHalfBlockM;
    if (!(fabs(v) < double(kKeyOff) * kBlockM)) return false;       // also false for NaN and inf
    int c = int(v / kBlockM);
    if (v < 0) c--;
    *w = c;
    return true;
}

// Key of world block w: z, then y, then x, each biased by 2^19 -- numeric order is the window's cube order (x fastest).
SO_ARCHIVE_HD inline uint64_t world_key(int wx, int wy, int wz) {
    return (uint64_t(uint32_t(wz + kKeyOff)) << (2 * kKeyBits)) | (uint64_t(uint32_t(wy + kKeyOff)) << kKeyBits) | uint64_t(uint32_t(wx + kKeyOff));
}

// Key of the block a point falls in, or kKeyNone (not finite, or beyond the key range)
SO_ARCHIVE_HD inline uint64_t point_key(float x, float y, float z) {
    int wx, wy, wz;
    if (!world_axis(x, &wx) || !world_axis(y, &wy) || !world_axis(z, &wz)) return kKeyNone;
    return world_key(wx, wy, wz);
}

inline void unpack_key(uint64_t key, int w[3]) {
    const uint64_t m = (uint64_t(1) << kKeyBits) - 1;
    w[0] = int(key & m) - kKeyOff;
    w[1] = int((key >> kKeyBits) & m) - kKeyOff;
    w[2] = int((key >> (2 * kKeyBits)) & m) - kKeyOff;
}

// Whether world block w lies in the window of `origin` (grid index g = w + origin inside 21 x 21 x 11)
inline bool in_window(const int w[3], const int32_t origin[3]) {
    const int g[3] = {w[0] + origin[0], w[1] + origin[1], w[2] + origin[2]};
    return g[0] >= 0 && g[0] < kWinW && g[1] >= 0 && g[1] < kWinH && g[2] >= 0 && g[2] < kWinD;
}

// The window of `origin` as 21 * 11 key ranges [lo, hi], one per (z, y) row of blocks, in key order: a sorted directory finds the
// archived blocks the window covers with one lookup per row, whatever the archive holds.  f(lo, hi) is called for every row.
template <class F>
inline void window_rows(const int32_t origin[3], F&& f) {
    for (int gz = 0; gz < kWinD; ++gz)
        for (int gy = 0; gy < kWinH; ++gy) {
            const int wy = gy - origin[1], wz = gz - origin[2], wx0 = -origin[0];
            f(world_key(wx0, wy, wz), world_key(wx0 + kWinW - 1, wy, wz));
        }
}

}  // namespace archive
}  // namespace so

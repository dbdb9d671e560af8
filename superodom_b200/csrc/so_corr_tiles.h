// so_corr_tiles.h -- where the solve's correspondence record keeps a scan's points (plain C++: shared by the kernels in so_icp.cu /
// so_motion.cu, the host code in so_api.cu and a CPU test).
//
// The record is three arrays of kCorrTile-point tiles (the plane solution or {n, d}, the weight, the scan point); the evaluation kernels
// copy a scan's tiles with one cp.async.bulk per array and tile, which needs every span to start 16 B-aligned.  So every scan starts on
// a tile of its own: scan s of a batch (s counted from the batch's first scan, whose points start at offset 0) with its first point at
// offset[s] in the scan buffer starts at tile ceil(offset[s] / kCorrTile) + s.  The "+ s" pays for the partial last tile of every scan
// before it, so the rule needs no prefix sum, and a buffer of corr_tile_cap(points, scans) tiles holds any batch of that many points.
#pragma once
#include <cstddef>
#include <cstdint>

#ifdef __CUDACC__
#define SO_CT_HD __host__ __device__ __forceinline__
#else
#define SO_CT_HD inline
#endif

namespace so {

constexpr uint32_t kCorrTile = 256;            // points per tile: the CTA width of the evaluation kernels (kThreads)

// First record slot of scan s (its point i is at slot corr_first(s, offset) + i)
SO_CT_HD size_t corr_first(uint32_t s, uint32_t offset) {
    return ((size_t(offset) + (kCorrTile - 1)) / kCorrTile + s) * kCorrTile;
}

// Tiles that hold every batch of at most `points` points in at most `scans` scans
SO_CT_HD size_t corr_tile_cap(size_t points, size_t scans) { return (points + kCorrTile - 1) / kCorrTile + scans; }

}  // namespace so

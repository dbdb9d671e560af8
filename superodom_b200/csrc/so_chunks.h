// so_chunks.h -- how a batch of registrations is cut into chunks (plain C++: shared by so_api.cu and a CPU unit test).
//
// A chunk is a run of consecutive scans whose kernels are launched together; even chunks run on the context stream, odd ones on
// the auxiliary stream, and with host input chunk k+1 is copied (copy stream) while chunk k computes.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

namespace so {

constexpr size_t kMaxChunks = 16;        // one upload event per chunk (Ctx::ev_copy)

// Bounds b[0] = 0 < b[1] < ... < b[m] = n_scans of the m <= kMaxChunks chunks of a batch.
//   profiling      : one chunk (every launch is timed on its own)
//   chunk_override : that many equal chunks (SO_CHUNKS, tuning aid)
//   host scans     : chunks that GROW -- 8, 16, 40, 64, then doubling (cumulative bounds 8, 24, 64, 128, 256, ...).  The one upload
//                    nothing can hide is chunk 0's, so it is short; every later chunk is uploaded (copy stream, back to back) while
//                    the chunks before it compute, and it can be large because that computing takes longer than its copy.  On an
//                    H100 80GB HBM3 (700 W limit, scripts/ab_step.py, 256-scan calls) this rule gives 7 805 scans/s end to end,
//                    one chunk 6 078, 4 / 8 equal chunks 7 394 / 7 478.  No chunk but the first two is shorter than 8 scans.
//   device scans   : two chunks (one per stream) from 16 scans on, else one.
inline std::vector<uint32_t> chunk_bounds(size_t n_scans, bool host_input, bool profiling, int chunk_override) {
    std::vector<uint32_t> b;
    if (n_scans == 0) return {0u, 0u};
    if (profiling) return {0u, uint32_t(n_scans)};
    if (chunk_override > 0) {
        const size_t m = size_t(chunk_override) < kMaxChunks ? size_t(chunk_override) : kMaxChunks;
        for (size_t k = 0; k <= m; ++k) b.push_back(uint32_t(k * n_scans / m));
        return b;
    }
    if (host_input && n_scans >= 32) {
        b = {0u, 8u, 24u};
        for (size_t e = 64; e < n_scans && b.size() < kMaxChunks; e *= 2) b.push_back(uint32_t(e));
        if (n_scans - b.back() < 8) b.pop_back();           // no sliver at the end
        b.push_back(uint32_t(n_scans));
        return b;
    }
    if (n_scans >= 16) return {0u, uint32_t(n_scans / 2), uint32_t(n_scans)};
    return {0u, uint32_t(n_scans)};
}

}  // namespace so

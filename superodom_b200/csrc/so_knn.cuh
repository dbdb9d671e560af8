// so_knn.cuh -- the neighbour search of the ICP path: exact k-NN inside the query's 50 m block of the sorted hash grid.
//
// Replaces nanoflann::Octree::knnNeighbors (flann/octree.h:1004-1055) as called by LocalMap::nearestKSearchSurf
// (LidarProcess/LocalMap.h:481-525) from LidarSLAM::findNearestNeighbors (src/LidarProcess/LidarSlam.cpp:720-747).
//
// Lists are kept ascending by (d2, id); d2 carries the reference's rounding float(double sum of squares) (flann/octree.h:95-102).
// Sentinel id 0xFFFFFFFF marks empty slots; d2 slots start at `bound` so that the NEIGHBORS_TOO_FAR gate (d2 > 3*planeRes,
// LidarSlam.cpp:741) doubles as the search radius.
//
// The search is a three-round SELECT (all loops do the same kind of work in every lane):
//   1. bound : a value-only min/max network over the 2x2x2 cells nearest the query gives U, an upper bound on the k-th neighbour
//              distance (skipped when the previous ICP iteration's neighbours already provide one);
//   2. gather: pruned walk of the search cube with the fixed bound U; the few candidates with approx d2 <= U are only recorded
//              (into a per-lane shared-memory list) -- no divergent insertion in the hot loop;
//   3. refine: the recorded candidates get the reference's exact d2 rounding and are ordered by (d2, id).
// The result is identical to an exhaustive in-block search with the same ordering: every true neighbour has approx d2 <= U
// (U carries a 4e-6 relative margin over the FP32 evaluation error of 4e-7).
//
// The walks read the cell table and the map points straight from global memory (L1 / L2).  Queries arrive ordered by cell
// (scan_order_key), so the lanes of a warp walk the same or neighbouring cell rows.
#pragma once
#include "so_icp.cuh"
#include "so_graph_rule.h"

namespace so {

template <int K>
struct TopK {
    float d2[K]; uint32_t id[K]; uint32_t pos[K];
    __device__ __forceinline__ void init(float bound) {
#pragma unroll
        for (int j = 0; j < K; ++j) { d2[j] = bound; id[j] = 0xFFFFFFFFu; pos[j] = 0; }
    }
    __device__ __forceinline__ float worst() const { return d2[K - 1]; }
    // Insert (d, i, p) if it precedes the current last entry in (d2, id) order.  The shift is a branch-free select
    // network: in a warp some lane inserts at almost every candidate step, so this path runs ~once per step at low lane
    // occupancy and its length, not its frequency, is what matters.
    __device__ __forceinline__ void offer(float d, uint32_t i, uint32_t p) {
        if (d < d2[K - 1] || (d == d2[K - 1] && i < id[K - 1])) {
            bool lt[K];                     // lt[j]: candidate precedes slot j
#pragma unroll
            for (int j = 0; j < K - 1; ++j) lt[j] = d < d2[j] || (d == d2[j] && i < id[j]);
            lt[K - 1] = true;
#pragma unroll
            for (int j = K - 1; j > 0; --j) {
                // slot j takes slot j-1 when the candidate precedes slot j-1, the candidate when it lands exactly here
                d2[j] = lt[j - 1] ? d2[j - 1] : (lt[j] ? d : d2[j]);
                id[j] = lt[j - 1] ? id[j - 1] : (lt[j] ? i : id[j]);
                pos[j] = lt[j - 1] ? pos[j - 1] : (lt[j] ? p : pos[j]);
            }
            d2[0] = lt[0] ? d : d2[0];
            id[0] = lt[0] ? i : id[0];
            pos[0] = lt[0] ? p : pos[0];
        }
    }
    __device__ __forceinline__ int count() const {
        int c = 0;
#pragma unroll
        for (int j = 0; j < K; ++j) c += (id[j] != 0xFFFFFFFFu);
        return c;
    }
};

struct QueryCell {
    int32_t slot;        // block slot or -1
    int32_t c[3];        // cell inside the block
    float f[3];          // offset of the query inside its cell, metres, in [0, cs]
    int32_t nblock;      // points in the block
};

// LocalMap::nearestKSearchSurf block lookup (LocalMap.h:488-507) + cell inside the block.
__device__ __forceinline__ void locate(const MapView& m, float qx, float qy, float qz, QueryCell& qc) {
    const float q[3] = {qx, qy, qz};
    int g[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double v = double(q[a]) + kHalfBlock;
        int b = int(v / kBlock);
        if (v < 0) b--;
        g[a] = b + m.origin[a];
        const double u = (v - kBlock * double(b)) * m.inv_cs;
        int c = int(u);
        c = c < 0 ? 0 : (c > m.nb - 1 ? m.nb - 1 : c);
        qc.c[a] = c;
        const float f = float(u - double(c)) * m.cs;
        qc.f[a] = fminf(fmaxf(f, 0.f), m.cs);
    }
    const bool ok = g[0] >= 0 && g[0] < kW && g[1] >= 0 && g[1] < kH && g[2] >= 0 && g[2] < kD;
    qc.slot = -1; qc.nblock = 0;
    if (ok) {
        const int lin = g[0] + kW * g[1] + kW * kH * g[2];
        qc.slot = __ldg(&m.block_slot[lin]);
        qc.nblock = __ldg(&m.block_count[lin]);
    }
}

// Order of the queries: cell-linear (x fastest) inside the block, blocks by slot, so that consecutive queries -- the lanes of a
// warp -- walk the same cell rows.  scan_key_space: the number of distinct keys.
__host__ __device__ inline uint64_t scan_key_space(int n_slots, int nb) {
    return uint64_t(n_slots) * uint64_t(nb) * uint64_t(nb) * uint64_t(nb);
}
__device__ __forceinline__ uint32_t scan_order_key(const MapView& m, const QueryCell& qc) {
    return uint32_t(qc.slot) * uint32_t(m.nb * m.nb * m.nb) + uint32_t((qc.c[2] * m.nb + qc.c[1]) * m.nb + qc.c[0]);
}

__device__ __forceinline__ float approx_d2(const float4 c, float qx, float qy, float qz) {
    const float dx = qx - c.x, dy = qy - c.y, dz = qz - c.z;
    return fmaf(dx, dx, fmaf(dy, dy, dz * dz));
}
__device__ __forceinline__ float exact_d2(const float4 c, float qx, float qy, float qz) {      // flann/octree.h:95-102
    const float dx = qx - c.x, dy = qy - c.y, dz = qz - c.z;
    return float(double(dx) * double(dx) + double(dy) * double(dy) + double(dz) * double(dz));
}

// The query's block: row(): candidate span [t, end) of cells xlo..xhi of row (zz, yy), as positions in the sorted map;
// load(t): the point at position t.
struct BlockGrid {
    const float4* pts; const uint32_t* cell_start; uint32_t base; int nb;
    __device__ __forceinline__ BlockGrid(const MapView& m, int slot)
        : pts(m.pts), cell_start(m.cell_start), base(uint32_t(slot) * uint32_t(m.nb) * uint32_t(m.nb) * uint32_t(m.nb)), nb(m.nb) {}
    __device__ __forceinline__ void row(int zz, int yy, int xlo, int xhi, uint32_t& t, uint32_t& end) const {
        const uint32_t r = base + uint32_t(zz * nb + yy) * uint32_t(nb);
        t = __ldg(&cell_start[r + xlo]);
        end = __ldg(&cell_start[r + xhi + 1]);
    }
    __device__ __forceinline__ float4 load(uint32_t t) const { return __ldg(&pts[t]); }
};

// ------------------------------------------------------------------------------------------------------------------
// Walks.  Distance (not squared) from the query to the slab / row `d` cells away along one axis: {f + cs, f, 0, g, g + cs} for
// d = -2..2 (rings <= 2 by construction of the grid: cells are >= half the search radius), generic beyond.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float axis_gap(int d, float f, float g, float cs) {
    const int ad = d < 0 ? -d : d;
    const float side = d < 0 ? f : g;
    return d == 0 ? 0.f : (ad <= 2 ? side + (ad == 2 ? cs : 0.f) : side + float(ad - 1) * cs);
}

// f(candidate, its position in the sorted map) for every position of [t, end).  Four candidates per trip with the tail predicated:
// the loads of a short span (most rows hold 1-3 points) are issued together instead of one per trip of a remainder loop; a lane
// past the end evaluates a far-away dummy that fails every test
template <class F>
__device__ __forceinline__ void for_span(const BlockGrid& g, uint32_t t, uint32_t end, F&& f) {
    const float4 far = make_float4(3.0e18f, 3.0e18f, 3.0e18f, 0.f);
    for (; t < end; t += 4) {
        const float4 c0 = g.load(t);
        const float4 c1 = t + 1 < end ? g.load(t + 1) : far;
        const float4 c2 = t + 2 < end ? g.load(t + 2) : far;
        const float4 c3 = t + 3 < end ? g.load(t + 3) : far;
        f(c0, t); f(c1, t + 1); f(c2, t + 2); f(c3, t + 3);
    }
}

// Pruned walk of the cube of R rings around the query's cell, clipped to its block (LocalMap.h:488-507), for a FIXED bound U:
// a row / cell is skipped when its lower bound on the distance exceeds U (with a 1e-4 margin).  Slabs and rows in natural order
// (the bound does not change during the walk, so the order is irrelevant).
template <class F>
__device__ __forceinline__ void walk_cube(const BlockGrid& g, int nb, float cs, const QueryCell& qc, float U, int R, F&& f) {
    const float fx = qc.f[0], fy = qc.f[1], fz = qc.f[2];
    const float gx = cs - fx, gy = cs - fy, gz = cs - fz;
    const int cx = qc.c[0], cy = qc.c[1], cz = qc.c[2];
    const float Um = U * 1.0001f;
#pragma unroll 1
    for (int oz = -R; oz <= R; ++oz) {
        const int zz = cz + oz;
        if (zz < 0 || zz >= nb) continue;
        const float lz = axis_gap(oz, fz, gz, cs);
        const float lz2 = lz * lz;
        if (lz2 > Um) continue;
#pragma unroll 1
        for (int oy = -R; oy <= R; ++oy) {
            const int yy = cy + oy;
            if (yy < 0 || yy >= nb) continue;
            const float ly = axis_gap(oy, fy, gy, cs);
            const float lb = fmaf(ly, ly, lz2);
            if (lb > Um) continue;
            // x extent of the row, branch-free for the rings that exist by construction (R <= 2); each step outwards needs the step before it
            const bool l1 = cx >= 1 && fmaf(fx, fx, lb) <= Um;
            const bool l2 = l1 && R >= 2 && cx >= 2 && fmaf(fx + cs, fx + cs, lb) <= Um;
            const bool r1 = cx + 1 < nb && fmaf(gx, gx, lb) <= Um;
            const bool r2 = r1 && R >= 2 && cx + 2 < nb && fmaf(gx + cs, gx + cs, lb) <= Um;
            int xlo = cx - int(l1) - int(l2), xhi = cx + int(r1) + int(r2);
            if (R > 2) {                                     // generic tail (not reached with the grids map_cells_per_block builds)
                if (l2) for (int k = 3; k <= R; ++k) { const float lx = fx + float(k - 1) * cs; if (cx - k < 0 || fmaf(lx, lx, lb) > Um) break; xlo = cx - k; }
                if (r2) for (int k = 3; k <= R; ++k) { const float lx = gx + float(k - 1) * cs; if (cx + k > nb - 1 || fmaf(lx, lx, lb) > Um) break; xhi = cx + k; }
            }
            uint32_t t, end;
            g.row(zz, yy, xlo, xhi, t, end);
            for_span(g, t, end, f);
        }
    }
}

// The 2 x 2 x 2 cells nearest the query (its own cell and, per axis, the neighbour on the side the query leans to), clipped to the
// block: ANY candidate subset yields a valid upper bound on the k-th neighbour distance, and this one holds the true neighbours
// almost always (it covers >= cs/2 around the query in every direction) at 8/27 of the cells and 4/9 of the rows of the full ring.
template <class F>
__device__ __forceinline__ void walk_octant(const BlockGrid& g, int nb, float cs, const QueryCell& qc, F&& f) {
    const float h = 0.5f * cs;
    const int cx = qc.c[0], cy = qc.c[1], cz = qc.c[2];
    const int sx = qc.f[0] < h ? -1 : 1, sy = qc.f[1] < h ? -1 : 1, sz = qc.f[2] < h ? -1 : 1;
    const int x0 = max(min(cx, cx + sx), 0), x1 = min(max(cx, cx + sx), nb - 1);
#pragma unroll
    for (int iz = 0; iz < 2; ++iz) {
        const int zz = cz + (iz ? sz : 0);
        if (zz < 0 || zz >= nb) continue;
#pragma unroll
        for (int iy = 0; iy < 2; ++iy) {
            const int yy = cy + (iy ? sy : 0);
            if (yy < 0 || yy >= nb) continue;
            uint32_t t, end;
            g.row(zz, yy, x0, x1, t, end);
            for_span(g, t, end, f);
        }
    }
}

// Recorded candidates per query before round 2 falls back to direct insertion.
constexpr int kBufCap = 24;

// Rounds 1 and 2 of the select search.  s_buf: [kBufCap][blockDim.x] positions, column = this thread.  u_seed < 0: no seed.
// `bound`: neighbours farther than this (squared) are not wanted; tk must have been initialised with it.  Complete for
// d2 <= min(bound, (R*cs)^2).  On return tk.pos holds positions in the sorted map.
// OCT: round 1 over the 2x2x2 nearest cells (measured: -7 % on scans, whose lanes sit in different cells anyway) or over the 27
// cells of ring 1 (dense query sets such as cfg5: lanes that share a cell then read the same rows; the octant splits them, +10 %).
// Round 1 returns U; unless seeded it sets *anchor to the position of the nearest candidate it saw (0xFFFFFFFF: none).
template <int K, bool OCT>
__device__ __forceinline__ float knn_bound(const BlockGrid& g, const MapView& m, const QueryCell& qc, float qx, float qy, float qz, float u_seed, float bound,
                                           uint32_t* anchor) {
    float U;
    if (u_seed >= 0.f) U = u_seed * 1.000004f;
    else {
        *anchor = 0xFFFFFFFFu;
        float a[K];                                                            // K smallest approx d2 so far, ascending
#pragma unroll
        for (int j = 0; j < K; ++j) a[j] = bound;
        auto net = [&](const float4 c, uint32_t e) {
            const float d = approx_d2(c, qx, qy, qz);
            if (d < a[0]) *anchor = e;
#pragma unroll
            for (int j = K - 1; j > 0; --j) a[j] = fminf(a[j], fmaxf(a[j - 1], d));
            a[0] = fminf(a[0], d);
        };
        // (measured and not kept for dense query sets: the bound from the query's own cell alone -- cfg5 2.83 ms against 2.72 ms; a
        // tight bound saves more in round 2 than a short round 1 saves)
        if (OCT) walk_octant(g, m.nb, m.cs, qc, net);
        else walk_cube(g, m.nb, m.cs, qc, bound, 1, net);
        U = a[K - 1] * 1.000004f;
    }
    return fminf(U, bound * 1.000004f);
}

template <int K>
__device__ __forceinline__ void knn_gather(const BlockGrid& g, const MapView& m, const QueryCell& qc, float qx, float qy, float qz, float U,
                                           uint32_t* s_buf, TopK<K>& tk) {
    int cnt = 0;
    const int stride = blockDim.x;
    walk_cube(g, m.nb, m.cs, qc, U, m.R, [&](const float4 c, uint32_t e) {
        if (approx_d2(c, qx, qy, qz) <= U) {
            if (cnt < kBufCap) { s_buf[cnt * stride + threadIdx.x] = e; ++cnt; }
            else tk.offer(exact_d2(c, qx, qy, qz), __float_as_uint(c.w), e);     // overflow (dense cluster inside U): insert directly
        }
    });
    for (int k = 0; k < cnt; ++k) {
        const uint32_t e = s_buf[k * stride + threadIdx.x];
        const float4 c = g.load(e);
        tk.offer(exact_d2(c, qx, qy, qz), __float_as_uint(c.w), e);
    }
}

template <int K, bool OCT>
__device__ __forceinline__ void knn_select(const BlockGrid& g, const MapView& m, const QueryCell& qc, float qx, float qy, float qz, float u_seed, float bound,
                                           uint32_t* s_buf, TopK<K>& tk) {
    uint32_t anchor = 0xFFFFFFFFu;
    const float U = knn_bound<K, OCT>(g, m, qc, qx, qy, qz, u_seed, bound, &anchor);
    knn_gather<K>(g, m, qc, qx, qy, qz, U, s_buf, tk);
}

// ------------------------------------------------------------------------------------------------------------------
// Neighbour graph (k_knn_scan): row a of MapView::graph holds the positions of the kGraphK nearest in-block points of map point a
// (a excluded, (d2, id) order, exact_d2), radius[a] = 0.99999 sqrt(d2 of the last of them): every in-block point p with
// |a - p| < radius[a] is in the row.  A block with at most kGraphK other points puts all of them in the row, radius +inf; a point
// its own search does not return (more than kGraphK duplicates with smaller ids) gets radius 0 (never certifies).
//
// Certificate: a query q with round-1 bound U and an anchor a in its block.  Every point the select search could return lies within
// sqrt(U) of q (U bounds the 5th distance, walk filter approx_d2 <= U), so within sqrt(U) + |q - a| of a; when that is below
// radius[a], {a} + row a holds all of them, and ranking those few candidates gives exactly the select search's result: the same
// top-5 in (d2, id) order over any candidate set between the true five and the block.  Error budget: approx_d2, exact_d2 and the
// float square roots are within ~5e-7 of the true distances; the 0.99999 in radius is 20 times that.  A NaN or infinite term
// fails the test (the comparison is false), so such queries take round 2.
// ------------------------------------------------------------------------------------------------------------------
// Anchor a certifies the query: then knn_graph_rank gives the select search's result.
__device__ __forceinline__ bool graph_certified(const MapView& m, uint32_t a, float qx, float qy, float qz, float U) {
    return graph_certifies(U, exact_d2(__ldg(&m.pts[a]), qx, qy, qz), __ldg(&m.graph_radius[a]));
}

// Ranks {a} + row a into tk (a certified anchor).
template <int K>
__device__ __forceinline__ void knn_graph_rank(const MapView& m, uint32_t a, float qx, float qy, float qz, float U, TopK<K>& tk) {
    const float4 ca = __ldg(&m.pts[a]);
    tk.offer(exact_d2(ca, qx, qy, qz), __float_as_uint(ca.w), a);
    const uint4* row = m.graph + size_t(a) * (kGraphK / 4);
    const float4 far = make_float4(3.0e18f, 3.0e18f, 3.0e18f, 0.f);
    auto one = [&](const float4 c, uint32_t e) {
        if (approx_d2(c, qx, qy, qz) <= U) tk.offer(exact_d2(c, qx, qy, qz), __float_as_uint(c.w), e);
    };
#pragma unroll 1
    for (int j = 0; j < kGraphK / 4; ++j) {
        const uint4 e = __ldg(row + j);                  // empty slots (0xFFFFFFFF) only in blocks of <= kGraphK points: a dummy that fails the filter
        const float4 c0 = e.x != 0xFFFFFFFFu ? __ldg(&m.pts[e.x]) : far;
        const float4 c1 = e.y != 0xFFFFFFFFu ? __ldg(&m.pts[e.y]) : far;
        const float4 c2 = e.z != 0xFFFFFFFFu ? __ldg(&m.pts[e.z]) : far;
        const float4 c3 = e.w != 0xFFFFFFFFu ? __ldg(&m.pts[e.w]) : far;
        one(c0, e.x); one(c1, e.y); one(c2, e.z); one(c3, e.w);
    }
}

// Unpruned cube [c-R, c+R]^3 clipped to the block (fallback rings of the exact, unbounded search).
template <int K>
__device__ __forceinline__ void knn_cube(const MapView& m, const QueryCell& qc, float qx, float qy, float qz, int R, TopK<K>& tk) {
    const BlockGrid g(m, qc.slot);
    const int nb = m.nb;
    const int xlo = max(qc.c[0] - R, 0), xhi = min(qc.c[0] + R, nb - 1);
    for (int zz = max(qc.c[2] - R, 0); zz <= min(qc.c[2] + R, nb - 1); ++zz)
        for (int yy = max(qc.c[1] - R, 0); yy <= min(qc.c[1] + R, nb - 1); ++yy) {
            uint32_t t, end;
            g.row(zz, yy, xlo, xhi, t, end);
            // cheap FP32 filter (relative error < 4e-7), then the reference's exact rounding for real contenders; four loads in flight
            for_span(g, t, end, [&](const float4 c, uint32_t e) {
                if (approx_d2(c, qx, qy, qz) <= tk.worst() * 1.000002f) tk.offer(exact_d2(c, qx, qy, qz), __float_as_uint(c.w), e);
            });
        }
}

// In-block k-NN, radius-bounded (max_d2 > 0) or exact (max_d2 <= 0).  The select walk is complete up to min(bound, (R*cs)^2);
// wider / unbounded searches then grow an unpruned cube until the k-th distance is provably final.  On return tk.pos holds
// positions of the sorted map.
template <int K>
__device__ __forceinline__ void knn_search(const BlockGrid& g, const MapView& m, const QueryCell& qc, float qx, float qy, float qz, float max_d2,
                                           uint32_t* s_buf, TopK<K>& tk) {
    const bool bounded = max_d2 > 0.f;
    int R = m.R;
    const float ring_d2 = float(R) * m.cs * float(R) * m.cs;
    bool done = false;
    if (bounded && max_d2 <= ring_d2) { tk.init(max_d2); knn_select<K, false>(g, m, qc, qx, qy, qz, -1.f, max_d2, s_buf, tk); done = true; }
    else if (!bounded) {
        tk.init(ring_d2 * 0.999f);
        knn_select<K, false>(g, m, qc, qx, qy, qz, -1.f, ring_d2 * 0.999f, s_buf, tk);
        done = tk.count() == K;                                      // K neighbours inside the guaranteed-complete radius
    } else { const float r = sqrtf(max_d2); while (float(R) * m.cs < r && R < m.nb) ++R; }
    while (!done) {
        tk.init(bounded ? max_d2 : FLT_MAX);
        knn_cube<K>(m, qc, qx, qy, qz, R, tk);
        if (bounded) break;
        float reach = FLT_MAX;
        bool covers = true;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (qc.c[a] - R > 0) { covers = false; reach = fminf(reach, qc.f[a] + float(R) * m.cs); }
            if (qc.c[a] + R < m.nb - 1) { covers = false; reach = fminf(reach, (m.cs - qc.f[a]) + float(R) * m.cs); }
        }
        if (covers) break;
        if (tk.count() == K && tk.worst() < reach * reach * 0.999f) break;
        R = (R < 4) ? R + 1 : R * 2;
    }
}

}  // namespace so

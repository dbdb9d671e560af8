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
// The walks read the map through a GRID POLICY:
//   GlobalGrid : cell table and points straight from global memory (L1 / L2), any query anywhere;
//   TileGrid   : a CTA-shared tile in shared memory.  Queries arrive in BRICK order (8x8x8 cells), so the 128 queries of a CTA sit
//                in a small box of cells; the rows of that box grown by two rings are contiguous float4 spans of the sorted map,
//                which the CTA copies with one cp.async.bulk (TMA, 1-D) per row onto an mbarrier, next to a 16-bit local cell
//                table.  Row headers then cost two 16-bit LDS instead of the index arithmetic + two global loads of the
//                global walk, candidates come by LDS.128, and the bulk copies of a tile overlap the other CTAs' searches.
//                CTAs whose box does not fit (sparse far-range returns, block faces) fall back to GlobalGrid as a whole.
#pragma once
#include "so_icp.cuh"

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
    // offer() that also tracks `next`: the smallest d2 among everything offered that did NOT end up in the list (candidates that
    // lose, and entries a better candidate pushes out) -- a lower bound on the (K+1)-th neighbour distance among the offered
    __device__ __forceinline__ void offer_track(float d, uint32_t i, uint32_t p, float& next) {
        const bool enters = d < d2[K - 1] || (d == d2[K - 1] && i < id[K - 1]);
        next = fminf(next, enters ? d2[K - 1] : d);
        offer(d, i, p);
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

// Order of the queries: cells grouped into 8x8x8 BRICKS (x fastest, both among the bricks of a block and inside a brick), so that
// any run of consecutive queries stays inside a compact box of cells -- what makes a CTA-shared candidate tile small.
constexpr int kBrickShift = 3, kBrickCells = 512;
__host__ __device__ inline uint32_t bricks_per_axis(int nb) { return uint32_t((nb + 7) >> kBrickShift); }
__host__ __device__ inline uint64_t scan_key_space(int n_slots, int nb) {
#if !SO_KNN_TILE
    return uint64_t(n_slots) * uint64_t(nb) * uint64_t(nb) * uint64_t(nb);
#endif
    const uint64_t r = bricks_per_axis(nb);
    return uint64_t(n_slots) * r * r * r * kBrickCells;
}
__device__ __forceinline__ uint32_t scan_order_key(const MapView& m, const QueryCell& qc) {
#if !SO_KNN_TILE
    return uint32_t(qc.slot) * uint32_t(m.nb * m.nb * m.nb) + uint32_t((qc.c[2] * m.nb + qc.c[1]) * m.nb + qc.c[0]);      // cell-linear, x fastest
#endif
    const uint32_t r = bricks_per_axis(m.nb);
    const uint32_t brick = ((uint32_t(qc.c[2]) >> kBrickShift) * r + (uint32_t(qc.c[1]) >> kBrickShift)) * r + (uint32_t(qc.c[0]) >> kBrickShift);
    const uint32_t within = ((uint32_t(qc.c[2]) & 7u) << 6) | ((uint32_t(qc.c[1]) & 7u) << 3) | (uint32_t(qc.c[0]) & 7u);
    return (uint32_t(qc.slot) * r * r * r + brick) * kBrickCells + within;
}

__device__ __forceinline__ float approx_d2(const float4 c, float qx, float qy, float qz) {
    const float dx = qx - c.x, dy = qy - c.y, dz = qz - c.z;
    return fmaf(dx, dx, fmaf(dy, dy, dz * dz));
}
__device__ __forceinline__ float exact_d2(const float4 c, float qx, float qy, float qz) {      // flann/octree.h:95-102
    const float dx = qx - c.x, dy = qy - c.y, dz = qz - c.z;
    return float(double(dx) * double(dx) + double(dy) * double(dy) + double(dz) * double(dz));
}

// ------------------------------------------------------------------------------------------------------------------
// Grid policies.  row(): candidate span [t, end) of cells xlo..xhi of row (zz, yy) of the query's block; load(t): candidate t;
// entry(t): what the select records for it; load_entry / pos_of: the candidate / its position in the sorted map from an entry.
// ------------------------------------------------------------------------------------------------------------------
struct GlobalGrid {
    const float4* pts; const uint32_t* cell_start; uint32_t base; int nb;
    __device__ __forceinline__ GlobalGrid(const MapView& m, int slot)
        : pts(m.pts), cell_start(m.cell_start), base(uint32_t(slot) * uint32_t(m.nb) * uint32_t(m.nb) * uint32_t(m.nb)), nb(m.nb) {}
    __device__ __forceinline__ void row(int zz, int yy, int xlo, int xhi, uint32_t& t, uint32_t& end, uint32_t& tag) const {
        const uint32_t r = base + uint32_t(zz * nb + yy) * uint32_t(nb);
        t = __ldg(&cell_start[r + xlo]);
        end = __ldg(&cell_start[r + xhi + 1]);
        tag = 0;
    }
    __device__ __forceinline__ float4 load(uint32_t t) const { return __ldg(&pts[t]); }
    __device__ __forceinline__ uint32_t entry(uint32_t t, uint32_t) const { return t; }
    __device__ __forceinline__ float4 load_entry(uint32_t e) const { return __ldg(&pts[e]); }
    __device__ __forceinline__ uint32_t pos_of(uint32_t e) const { return e; }
};

// SO_KNN_TILE = 1 builds the TMA-tiled search (brick query order, 128 queries per CTA, tile with global fallback); 0 (default) the
// global-memory search (cell-linear query order, 256 queries per CTA).  Both give bit-identical results.  Measured on an H100 80GB HBM3
// (700 W limit, scripts/ab_knn.py, 64 cfg2 scans = 8.4 M queries per launch): tiled 1.45 ms, global 1.05-1.07 ms per launch.
// The search is bound by per-candidate instructions (distance,
// min/max network, record), which a tile does not remove; what it removes (row headers: index arithmetic + two cell-table loads,
// ~30 % of the instructions) is paid back by the tile build (box reduction, row scan, cell table, ~250 warp-instructions and eight
// barriers per 128 queries, with the bulk-copy latency exposed at 6 CTAs per SM) and by the brick order, whose 8-cell runs
// lose part of the row coherence the cell-linear order gives the lanes of a warp.
#ifndef SO_KNN_TILE
#define SO_KNN_TILE 0
#endif
#ifndef SO_KNN_THREADS
#define SO_KNN_THREADS 64          // H100 (as above): 32 -> 1.08, 64 -> 1.05-1.07, 128 -> 1.07, 256 -> 1.11 ms per launch
#endif
constexpr int kTileThreads = SO_KNN_TILE ? 128 : SO_KNN_THREADS;      // queries per CTA of the search kernels
#ifndef SO_TILE_PTS
#define SO_TILE_PTS 1024
#endif
constexpr int kTilePts = SO_TILE_PTS;  // candidate points a tile holds (16 B each)
constexpr int kTileRows = 256;         // (y, z) rows of a tile: two per thread
constexpr int kTileCells = 3072;       // entries of the local cell table (rows x (width + 1))
constexpr int kTileMinQueries = 24;    // CTAs with fewer searchable queries are not worth a tile

struct TileSmem {
    alignas(128) float4 pts[kTilePts];
    uint16_t cell[kTileCells];         // local cell table: cell[r * w1 + x] = first tile point of cell x0 + x in tile row r; [.. + w] = end
    int32_t delta[kTileRows];          // position in the sorted map = tile index + delta[row]
    alignas(8) unsigned long long mbar;
    int32_t red[kTileThreads / 32][8]; // per-warp box partials
    int32_t box[8];                    // lo[3], hi[3], slot (or -2: mixed), searchable queries
    uint32_t wsum[kTileThreads / 32];
    uint32_t total;
};

struct TileGrid {
    const float4* pts; const uint16_t* cell; const int32_t* delta;
    int x0, y0, z0, w1, ny;
    __device__ __forceinline__ void row(int zz, int yy, int xlo, int xhi, uint32_t& t, uint32_t& end, uint32_t& tag) const {
        const int r = (zz - z0) * ny + (yy - y0);
        const uint16_t* c = cell + r * w1 - x0;
        t = c[xlo];
        end = c[xhi + 1];
        tag = uint32_t(r) << 16;
    }
    __device__ __forceinline__ float4 load(uint32_t t) const { return pts[t]; }
    __device__ __forceinline__ uint32_t entry(uint32_t t, uint32_t tag) const { return t | tag; }      // tile index < 65536
    __device__ __forceinline__ float4 load_entry(uint32_t e) const { return pts[e & 0xFFFFu]; }
    __device__ __forceinline__ uint32_t pos_of(uint32_t e) const { return uint32_t(int32_t(e & 0xFFFFu) + delta[e >> 16]); }
};

// ---- mbarrier / bulk-copy primitives (PTX ISA: mbarrier, cp.async.bulk) ----------------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(arrivals) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "SO_MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra SO_MBAR_DONE;\n"
        "bra SO_MBAR_WAIT;\n"
        "SO_MBAR_DONE:\n"
        "}\n" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
// 1-D TMA: `bytes` (multiple of 16) from global to shared memory, completion counted on the mbarrier
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_global, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst_smem)),
                 "l"(src_global), "r"(bytes), "r"(smem_addr(bar))
                 : "memory");
}

// Build the CTA's tile.  Must be called by all kTileThreads threads; `valid`: this thread has a searchable query at qc.
// Returns false (nothing staged) when the CTA does not qualify; the caller then searches through GlobalGrid.
__device__ __forceinline__ bool build_tile(const MapView& m, TileSmem& ts, bool valid, const QueryCell& qc, TileGrid& tg) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // ---- box of the CTA's queries (cells), their common block
    {
        const int lo0 = __reduce_min_sync(full, valid ? qc.c[0] : 0x7fffffff), hi0 = __reduce_max_sync(full, valid ? qc.c[0] : -1);
        const int lo1 = __reduce_min_sync(full, valid ? qc.c[1] : 0x7fffffff), hi1 = __reduce_max_sync(full, valid ? qc.c[1] : -1);
        const int lo2 = __reduce_min_sync(full, valid ? qc.c[2] : 0x7fffffff), hi2 = __reduce_max_sync(full, valid ? qc.c[2] : -1);
        const int smin = __reduce_min_sync(full, valid ? qc.slot : 0x7fffffff), smax = __reduce_max_sync(full, valid ? qc.slot : -1);
        const int nv = __popc(__ballot_sync(full, valid));
        if (lane == 0) {
            ts.red[warp][0] = lo0; ts.red[warp][1] = lo1; ts.red[warp][2] = lo2; ts.red[warp][3] = hi0; ts.red[warp][4] = hi1; ts.red[warp][5] = hi2;
            ts.red[warp][6] = (smin == smax || nv == 0) ? smin : -2;      // 0x7fffffff: no query in this warp
            ts.red[warp][7] = nv;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {-1, -1, -1}, slot = 0x7fffffff, nv = 0;
#pragma unroll
        for (int w = 0; w < kTileThreads / 32; ++w) {
#pragma unroll
            for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], ts.red[w][a]); hi[a] = max(hi[a], ts.red[w][3 + a]); }
            const int sw = ts.red[w][6];
            if (sw != 0x7fffffff) slot = (slot == 0x7fffffff || slot == sw) ? sw : -2;
            nv += ts.red[w][7];
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) { ts.box[a] = lo[a]; ts.box[3 + a] = hi[a]; }
        ts.box[6] = slot; ts.box[7] = nv;
    }
    __syncthreads();
    const int slot = ts.box[6];
    if (slot < 0 || slot == 0x7fffffff || ts.box[7] < kTileMinQueries) return false;
    const int nb = m.nb, R = 2;
    const int x0 = max(ts.box[0] - R, 0), x1 = min(ts.box[3] + R, nb - 1);
    const int y0 = max(ts.box[1] - R, 0), y1 = min(ts.box[4] + R, nb - 1);
    const int z0 = max(ts.box[2] - R, 0), z1 = min(ts.box[5] + R, nb - 1);
    const int w1 = x1 - x0 + 2, ny = y1 - y0 + 1, nz = z1 - z0 + 1, rows = ny * nz;
    if (rows > kTileRows || rows * w1 > kTileCells) return false;
    // ---- row spans (two rows per thread), exclusive scan of their sizes
    const uint32_t base = uint32_t(slot) * uint32_t(nb) * uint32_t(nb) * uint32_t(nb);
    uint32_t gs[2], cnt[2], off[2], rowbase[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int r = int(threadIdx.x) + k * kTileThreads;
        gs[k] = 0; cnt[k] = 0; rowbase[k] = 0;
        if (r < rows) {
            const int rz = r / ny, ry = r - rz * ny;
            rowbase[k] = base + uint32_t((z0 + rz) * nb + (y0 + ry)) * uint32_t(nb);
            gs[k] = __ldg(&m.cell_start[rowbase[k] + x0]);
            cnt[k] = __ldg(&m.cell_start[rowbase[k] + x1 + 1]) - gs[k];
        }
    }
    uint32_t carry = 0;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        uint32_t v = cnt[k];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(full, v, o); if (lane >= o) v += u; }
        if (lane == 31) ts.wsum[warp] = v;
        __syncthreads();
        uint32_t before = carry;
#pragma unroll
        for (int w = 0; w < kTileThreads / 32; ++w) { const uint32_t s = ts.wsum[w]; if (w < warp) before += s; carry += s; }
        off[k] = before + v - cnt[k];
        __syncthreads();
    }
    const uint32_t total = carry;                                       // identical in every thread
    if (total > uint32_t(kTilePts)) return false;
    // ---- one bulk copy per non-empty row onto the mbarrier; the local cell table meanwhile
    if (threadIdx.x == 0) { mbar_init(&ts.mbar, 1); mbar_arrive_expect_tx(&ts.mbar, total * 16u); }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int r = int(threadIdx.x) + k * kTileThreads;
        if (r < rows) {
            if (cnt[k]) bulk_copy_g2s(&ts.pts[off[k]], m.pts + gs[k], cnt[k] * 16u, &ts.mbar);
            const int32_t dl = int32_t(gs[k]) - int32_t(off[k]);
            ts.delta[r] = dl;
            const uint32_t* cs = m.cell_start + rowbase[k] + x0;
            uint16_t* out = ts.cell + r * w1;
            out[0] = uint16_t(off[k]);
            for (int x = 1; x < w1 - 1; ++x) out[x] = uint16_t(int32_t(__ldg(cs + x)) - dl);
            out[w1 - 1] = uint16_t(off[k] + cnt[k]);
        }
    }
    __syncthreads();
    mbar_wait(&ts.mbar, 0);
    tg.pts = ts.pts; tg.cell = ts.cell; tg.delta = ts.delta;
    tg.x0 = x0; tg.y0 = y0; tg.z0 = z0; tg.w1 = w1; tg.ny = ny;
    return true;
}

// ------------------------------------------------------------------------------------------------------------------
// Walks.  Distance (not squared) from the query to the slab / row `d` cells away along one axis: {f + cs, f, 0, g, g + cs} for
// d = -2..2 (rings <= 2 by construction of the grid: cells are >= half the search radius), generic beyond.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float axis_gap(int d, float f, float g, float cs) {
    const int ad = d < 0 ? -d : d;
    const float side = d < 0 ? f : g;
    return d == 0 ? 0.f : (ad <= 2 ? side + (ad == 2 ? cs : 0.f) : side + float(ad - 1) * cs);
}

// four candidates per trip with the tail predicated: the loads of a short span (most rows hold 1-3 points) are issued together
// instead of one per trip of a remainder loop; a lane past the end evaluates a far-away dummy that fails every test
template <class Grid, class F>
__device__ __forceinline__ void for_span(const Grid& g, uint32_t t, uint32_t end, uint32_t tag, F&& f) {
    const float4 far = make_float4(3.0e18f, 3.0e18f, 3.0e18f, 0.f);
    for (; t < end; t += 4) {
        const float4 c0 = g.load(t);
        const float4 c1 = t + 1 < end ? g.load(t + 1) : far;
        const float4 c2 = t + 2 < end ? g.load(t + 2) : far;
        const float4 c3 = t + 3 < end ? g.load(t + 3) : far;
        f(c0, g.entry(t, tag)); f(c1, g.entry(t + 1, tag)); f(c2, g.entry(t + 2, tag)); f(c3, g.entry(t + 3, tag));
    }
}

// Pruned walk of the cube of R rings around the query's cell, clipped to its block (LocalMap.h:488-507), for a FIXED bound U:
// a row / cell is skipped when its lower bound on the distance exceeds U (with a 1e-4 margin).  Slabs and rows in natural order
// (the bound does not change during the walk, so the order is irrelevant).
template <class Grid, class F>
__device__ __forceinline__ void walk_cube(const Grid& g, int nb, float cs, const QueryCell& qc, float U, int R, F&& f) {
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
            uint32_t t, end, tag;
            g.row(zz, yy, xlo, xhi, t, end, tag);
            for_span(g, t, end, tag, f);
        }
    }
}

// The 2 x 2 x 2 cells nearest the query (its own cell and, per axis, the neighbour on the side the query leans to), clipped to the
// block: ANY candidate subset yields a valid upper bound on the k-th neighbour distance, and this one holds the true neighbours
// almost always (it covers >= cs/2 around the query in every direction) at 8/27 of the cells and 4/9 of the rows of the full ring.
template <class Grid, class F>
__device__ __forceinline__ void walk_octant(const Grid& g, int nb, float cs, const QueryCell& qc, F&& f) {
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
            uint32_t t, end, tag;
            g.row(zz, yy, x0, x1, t, end, tag);
            for_span(g, t, end, tag, f);
        }
    }
}

#ifndef SO_BUF_CAP
#define SO_BUF_CAP 24
#endif
#ifndef SO_R1_OCTANT
#define SO_R1_OCTANT 1            // scans (k_knn_scan): 1 = round 1 over the 2x2x2 nearest cells, 0 = over the 27 cells of ring 1
#endif
constexpr int kBufCap = SO_BUF_CAP;          // recorded candidates per query before round 2 falls back to direct insertion

// s_buf: [kBufCap][blockDim.x] entries, column = this thread.  u_seed < 0: no seed.  `bound`: neighbours farther than this (squared)
// are not wanted; tk must have been initialised with it.  Complete for d2 <= min(bound, (R*cs)^2).  On return tk.pos holds ENTRIES
// of the grid policy (g.pos_of() turns them into positions of the sorted map).
// OCT: round 1 over the 2x2x2 nearest cells (measured: -7 % on scans, whose lanes sit in different cells anyway) or over the 27
// cells of ring 1 (dense query sets such as cfg5: lanes that share a cell then read the same rows; the octant splits them, +10 %).
// *next_lb (optional): receives a lower bound on the squared distance from the query to every point of its block that is NOT in
// the returned list (the best loser among the examined candidates, or the bound U beyond which nothing was examined).
template <int K, bool OCT, class Grid>
__device__ __forceinline__ void knn_select(const Grid& g, const MapView& m, const QueryCell& qc, float qx, float qy, float qz, float u_seed, float bound,
                                           uint32_t* s_buf, TopK<K>& tk, float* next_lb = nullptr) {
    float U;
    if (u_seed >= 0.f) U = u_seed * 1.000004f;
    else {
        float a[K];                                                            // K smallest approx d2 so far, ascending
#pragma unroll
        for (int j = 0; j < K; ++j) a[j] = bound;
        auto net = [&](const float4 c, uint32_t) {
            const float d = approx_d2(c, qx, qy, qz);
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
    U = fminf(U, bound * 1.000004f);
    int cnt = 0;
    float next = FLT_MAX;
    const int stride = blockDim.x;
    walk_cube(g, m.nb, m.cs, qc, U, m.R, [&](const float4 c, uint32_t e) {
        if (approx_d2(c, qx, qy, qz) <= U) {
            if (cnt < kBufCap) { s_buf[cnt * stride + threadIdx.x] = e; ++cnt; }
            else tk.offer_track(exact_d2(c, qx, qy, qz), __float_as_uint(c.w), e, next);    // overflow (dense cluster inside U): insert directly
        }
    });
    for (int k = 0; k < cnt; ++k) {
        const uint32_t e = s_buf[k * stride + threadIdx.x];
        const float4 c = g.load_entry(e);
        tk.offer_track(exact_d2(c, qx, qy, qz), __float_as_uint(c.w), e, next);
    }
    // every block point with FP32 d2 <= U was offered; one that was not has true d2 > U (1 - 4e-7)
    if (next_lb) *next_lb = fminf(next, U) * (1.f - 2e-6f);
}

// Unpruned cube [c-R, c+R]^3 clipped to the block (fallback rings of the exact, unbounded search), global memory.
template <int K>
__device__ __forceinline__ void knn_cube(const MapView& m, const QueryCell& qc, float qx, float qy, float qz, int R, TopK<K>& tk) {
    const GlobalGrid g(m, qc.slot);
    const int nb = m.nb;
    const int xlo = max(qc.c[0] - R, 0), xhi = min(qc.c[0] + R, nb - 1);
    for (int zz = max(qc.c[2] - R, 0); zz <= min(qc.c[2] + R, nb - 1); ++zz)
        for (int yy = max(qc.c[1] - R, 0); yy <= min(qc.c[1] + R, nb - 1); ++yy) {
            uint32_t t, end, tag;
            g.row(zz, yy, xlo, xhi, t, end, tag);
            // cheap FP32 filter (relative error < 4e-7), then the reference's exact rounding for real contenders; four loads in flight
            for_span(g, t, end, tag, [&](const float4 c, uint32_t e) {
                if (approx_d2(c, qx, qy, qz) <= tk.worst() * 1.000002f) tk.offer(exact_d2(c, qx, qy, qz), __float_as_uint(c.w), e);
            });
        }
}

// In-block k-NN, radius-bounded (max_d2 > 0) or exact (max_d2 <= 0).  The select walk is complete up to min(bound, (R*cs)^2);
// wider / unbounded searches then grow an unpruned cube until the k-th distance is provably final.  On return tk.pos holds
// positions of the sorted map.
template <int K, class Grid>
__device__ __forceinline__ void knn_search(const Grid& g, const MapView& m, const QueryCell& qc, float qx, float qy, float qz, float max_d2,
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
    if (done) {
#pragma unroll
        for (int j = 0; j < K; ++j) if (tk.id[j] != 0xFFFFFFFFu) tk.pos[j] = g.pos_of(tk.pos[j]);
    }
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

// so_reloc.cu -- global localization search (so_localize_global): occupancy bitmap of the surf map, cube dilation, exhaustive
// scoring of x/y/z voxel shifts x yaw steps of the scan, and the key sort that ranks the hypotheses.  The host side (score-point
// selection, suppression, refinement through register_core) lives in so_api.cu.
//
// Everything here is integer-valued once a point has been put into a voxel, and the voxel of a point is computed with
// explicitly rounded FP64 operations (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn: no FMA contraction), so a numpy
// restatement reproduces every score exactly.
#include <cub/cub.cuh>

#include "so_ctx.cuh"

namespace so {

namespace {

// qrot (so_internal.cuh) with every operation rounded on its own, in the same order
__device__ __forceinline__ void qrot_rn(const double q[4], const double v[3], double o[3]) {
    double ux = __dsub_rn(__dmul_rn(q[1], v[2]), __dmul_rn(q[2], v[1]));
    double uy = __dsub_rn(__dmul_rn(q[2], v[0]), __dmul_rn(q[0], v[2]));
    double uz = __dsub_rn(__dmul_rn(q[0], v[1]), __dmul_rn(q[1], v[0]));
    ux = __dadd_rn(ux, ux); uy = __dadd_rn(uy, uy); uz = __dadd_rn(uz, uz);
    o[0] = __dadd_rn(__dadd_rn(v[0], __dmul_rn(q[3], ux)), __dsub_rn(__dmul_rn(q[1], uz), __dmul_rn(q[2], uy)));
    o[1] = __dadd_rn(__dadd_rn(v[1], __dmul_rn(q[3], uy)), __dsub_rn(__dmul_rn(q[2], ux), __dmul_rn(q[0], uz)));
    o[2] = __dadd_rn(__dadd_rn(v[2], __dmul_rn(q[3], uz)), __dsub_rn(__dmul_rn(q[0], uy), __dmul_rn(q[1], ux)));
}

// One thread per surf-store point: w = floor((m - lo) / res) per axis; points inside the box set their bit.
__global__ void __launch_bounds__(256) k_reloc_raster(const float4* __restrict__ pts, uint32_t n, RelocGrid g, uint32_t* __restrict__ bits) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[i];
    const double fx = floor(__ddiv_rn(__dsub_rn(double(p.x), g.lo[0]), g.res));
    const double fy = floor(__ddiv_rn(__dsub_rn(double(p.y), g.lo[1]), g.res));
    const double fz = floor(__ddiv_rn(__dsub_rn(double(p.z), g.lo[2]), g.res));
    if (!(fx >= 0.0 && fx < double(g.bx) && fy >= 0.0 && fy < double(g.by) && fz >= 0.0 && fz < double(g.bz))) return;
    const uint32_t x = uint32_t(fx), y = uint32_t(fy), z = uint32_t(fz);
    atomicOr(bits + (size_t(z) * g.by + y) * g.wpr + (x >> 5), 1u << (x & 31));
}

// One pass of the separable cube dilation, one thread per bitmap word: axis 0 ORs the word shifted by 1..d bits both ways (with the
// neighbouring words' carries), axes 1 and 2 OR the words d rows / planes away.  The padding bits past bx stay zero.
__global__ void __launch_bounds__(256) k_reloc_dilate(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, RelocGrid g, int d, int axis) {
    const size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const size_t total = size_t(g.by) * g.bz * g.wpr;
    if (idx >= total) return;
    const uint32_t wi = uint32_t(idx % g.wpr);
    const size_t row = idx / g.wpr;
    uint32_t r = in[idx];
    if (axis == 0) {
        const uint32_t cur = r, prev = wi ? in[idx - 1] : 0u, next = wi + 1 < uint32_t(g.wpr) ? in[idx + 1] : 0u;
        for (int s = 1; s <= d; ++s) r |= (cur >> s) | (next << (32 - s)) | (cur << s) | (prev >> (32 - s));
        if (wi + 1 == uint32_t(g.wpr) && (g.bx & 31)) r &= (1u << (g.bx & 31)) - 1u;
    } else if (axis == 1) {
        const int y = int(row % g.by);
        for (int s = -d; s <= d; ++s)
            if (s && y + s >= 0 && y + s < g.by) r |= in[idx + ptrdiff_t(s) * g.wpr];
    } else {
        const int z = int(row / g.by);
        for (int s = -d; s <= d; ++s)
            if (s && z + s >= 0 && z + s < g.bz) r |= in[idx + ptrdiff_t(s) * g.by * g.wpr];
    }
    out[idx] = r;
}

// One CTA per (tile of kRelocRows y shifts, z shift, yaw).  Prologue: every score point rotated by the yaw's quaternion and put
// into its voxel, stored as {x0, y0, z row base} so that hypothesis (i, j) reads bit x0 + i of row (zbase + y0 + j).  Main loop:
// a warp takes 32 consecutive x shifts of one y shift, so each step reads one or two bitmap words (L1 / L2 resident).  Output:
// the sort key (65535 - score) << 32 | linear index, which orders hypotheses by score descending, then index ascending.
__global__ void __launch_bounds__(kRelocThreads) k_reloc_score(const float4* __restrict__ spts, int n_pts, const double* __restrict__ q_yaw,
                                                                RelocGrid g, const uint32_t* __restrict__ bits, uint64_t* __restrict__ keys) {
    extern __shared__ int4 s_off[];
    const int j0 = blockIdx.x * kRelocRows, k = blockIdx.y, m = blockIdx.z;
    const double q[4] = {q_yaw[4 * m], q_yaw[4 * m + 1], q_yaw[4 * m + 2], q_yaw[4 * m + 3]};
    for (int p = threadIdx.x; p < n_pts; p += blockDim.x) {
        const float4 v = spts[p];
        const double vd[3] = {double(v.x), double(v.y), double(v.z)};
        double r[3];
        qrot_rn(q, vd, r);
        const int wx = int(floor(__ddiv_rn(r[0], g.res))), wy = int(floor(__ddiv_rn(r[1], g.res))), wz = int(floor(__ddiv_rn(r[2], g.res)));
        const int z = wz + k + g.e;
        int4 o;
        o.x = wx + g.e;
        o.y = (z >= 0 && z < g.bz) ? wy + g.e : -(1 << 29);         // a z outside the box: every lookup of this point misses
        o.z = (z >= 0 && z < g.bz) ? z * g.by : 0;
        o.w = 0;
        s_off[p] = o;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nxc = (g.nx + 31) >> 5;
    for (int item = warp; item < nxc * kRelocRows; item += kRelocThreads / 32) {
        const int j = j0 + item / nxc, i = (item % nxc) * 32 + lane;
        if (j >= g.ny) continue;                                    // warp-uniform
        uint32_t cnt = 0;
#pragma unroll 4
        for (int p = 0; p < n_pts; ++p) {
            const int4 o = s_off[p];
            const int y = o.y + j, x = o.x + i;
            if (uint32_t(y) < uint32_t(g.by) && uint32_t(x) < uint32_t(g.bx)) {
                const uint32_t w = __ldg(bits + size_t(o.z + y) * g.wpr + uint32_t(x >> 5));
                cnt += (w >> (x & 31)) & 1u;
            }
        }
        if (i < g.nx) {
            const uint32_t lin = ((uint32_t(m) * g.nz + k) * g.ny + j) * g.nx + i;
            keys[lin] = (uint64_t(65535u - cnt) << 32) | lin;
        }
    }
}

}  // namespace

void launch_reloc_raster(const float4* pts, uint32_t n, const RelocGrid& g, uint32_t* bits, cudaStream_t st) {
    if (n) k_reloc_raster<<<(n + 255) / 256, 256, 0, st>>>(pts, n, g, bits);
}

uint32_t* launch_reloc_dilate(const RelocGrid& g, int d, uint32_t* a, uint32_t* b, cudaStream_t st) {
    const size_t total = size_t(g.by) * g.bz * g.wpr;
    const uint32_t grid = uint32_t((total + 255) / 256);
    k_reloc_dilate<<<grid, 256, 0, st>>>(a, b, g, d, 0);
    k_reloc_dilate<<<grid, 256, 0, st>>>(b, a, g, d, 1);
    k_reloc_dilate<<<grid, 256, 0, st>>>(a, b, g, d, 2);
    return b;
}

int launch_reloc_score(const float4* spts, int n_pts, const double* d_q, const RelocGrid& g, const uint32_t* bits, uint64_t* keys, cudaStream_t st) {
    const size_t smem = size_t(n_pts > 0 ? n_pts : 1) * sizeof(int4);
    SO_CUDA_TRY(cudaFuncSetAttribute(k_reloc_score, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kRelocMaxPoints * sizeof(int4))));
    const dim3 grid((g.ny + kRelocRows - 1) / kRelocRows, g.nz, g.nyaw);
    k_reloc_score<<<grid, kRelocThreads, smem, st>>>(spts, n_pts, d_q, g, bits, keys);
    return SO_OK;
}

// cub radix sort of the keys: score bits 32..47 and index bits 0..23 (the keys are unique, so the order is fully determined)
size_t reloc_sort_bytes(size_t n) {
    size_t b = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, b, (const uint64_t*)nullptr, (uint64_t*)nullptr, int(n), 0, 48);
    return b;
}

int reloc_sort(void* tmp, size_t tmp_bytes, const uint64_t* in, uint64_t* out, size_t n, cudaStream_t st) {
    SO_CUDA_TRY(cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, in, out, int(n), 0, 48, st));
    return SO_OK;
}

}  // namespace so

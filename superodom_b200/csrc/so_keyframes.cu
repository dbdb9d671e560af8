// so_keyframes.cu -- keyframes for a loop-closing back end: registered scans kept on the device with their poses (so_keyframe_*),
// keyframes of an earlier session imported from the host (so_keyframe_import), and the map rebuilt from them at corrected poses
// (so_map_from_keyframes; its kernels are in so_map.cu).
#include <algorithm>
#include <cstring>

#include "so_ctx.cuh"

namespace so {

static size_t held(const KeyframeStore& s, int store) { return s.off[store].empty() ? 0 : size_t(s.off[store].back()); }

// Both pools and the frame table at once: new pools are allocated and filled before the old ones go, so a failure changes nothing
static int keyframes_reserve(Ctx* c, size_t cap_points, size_t cap_frames) {
    KeyframeStore& s = c->kf;
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (cap_points == 0 && cap_frames == 0) {
        s = KeyframeStore{};
        return SO_OK;
    }
    if (cap_frames < s.frames() || cap_points < held(s, 0) || cap_points < held(s, 1))
        return fail(SO_ERR_ARG, "so_keyframe_reserve: capacity below what the store holds");
    DeviceBuffer<float> desc;
    DeviceBuffer<double> norm;
    if (cap_frames != s.cap_frames) { int rc = loop_table_alloc(s, cap_frames, &desc, &norm); if (rc) return rc; }
    if (cap_points != s.cap_points) {
        DeviceBuffer<float4> pool[2];
        for (int k = 0; k < 2; ++k) {
            if (pool[k].reserve(std::max<size_t>(cap_points, 1))) {
                cudaGetLastError();
                return fail(SO_ERR_CUDA, "so_keyframe_reserve: cudaMalloc of a keyframe pool failed");
            }
            if (held(s, k) && cudaMemcpy(pool[k], s.d_pool[k], held(s, k) * sizeof(float4), cudaMemcpyDeviceToDevice) != cudaSuccess)
                return fail(SO_ERR_CUDA, "so_keyframe_reserve: copy of the keyframes failed");
        }
        for (int k = 0; k < 2; ++k) s.d_pool[k] = std::move(pool[k]);
        s.cap_points = cap_points;
    }
    if (desc) {                                                        // the descriptor table follows the frame table
        s.d_desc = std::move(desc);
        s.d_desc_norm = std::move(norm);
    }
    for (int k = 0; k < 2; ++k) if (s.off[k].empty()) s.off[k].push_back(0);
    s.cap_frames = cap_frames;
    return SO_OK;
}

static int check_ids(const KeyframeStore& s, const int32_t* ids, size_t n) {
    if (n && !ids) return fail(SO_ERR_ARG, "bad args");
    for (size_t i = 0; i < n; ++i)
        if (ids[i] < 0 || size_t(ids[i]) >= s.frames()) return fail(SO_ERR_ARG, "keyframe id out of range");
    return SO_OK;
}

// The keyframes ids[0..n) of src as registration input on dst's device: their surf clouds back to back, read in place when the ids are
// consecutive (the pool holds them back to back), else gathered into dst's scratch
int keyframe_scans(Ctx* dst, Ctx* src, const int32_t* ids, size_t n, const float4** scans, std::vector<uint32_t>* n_points) {
    const KeyframeStore& s = src->kf;
    int rc = check_ids(s, ids, n);
    if (rc) return rc;
    n_points->resize(n);
    bool consecutive = true;
    size_t total = 0;
    for (size_t i = 0; i < n; ++i) {
        (*n_points)[i] = uint32_t(s.off[0][ids[i] + 1] - s.off[0][ids[i]]);
        total += (*n_points)[i];
        if (i && ids[i] != ids[i - 1] + 1) consecutive = false;
    }
    SO_CUDA_TRY(cudaStreamSynchronize(src->stream));                   // the keyframes have landed in src's pool
    if (consecutive) { *scans = s.d_pool[0] + (n ? s.off[0][ids[0]] : 0); return SO_OK; }
    KeyframeScratch& k = dst->kfs;
    rc = k.d_raw.reserve(std::max<size_t>(total, 1));
    if (rc) return rc;
    size_t at = 0;
    for (size_t i = 0; i < n; ++i) {
        if ((*n_points)[i])
            SO_CUDA_TRY(cudaMemcpyAsync(k.d_raw + at, s.d_pool[0] + s.off[0][ids[i]], size_t((*n_points)[i]) * sizeof(float4), cudaMemcpyDeviceToDevice,
                                        dst->stream));
        at += (*n_points)[i];
    }
    *scans = k.d_raw;
    return SO_OK;
}

}  // namespace so

// =================================================================================================== C ABI
using namespace so;

extern "C" {

int so_keyframe_reserve(so_ctx* ctx, size_t cap_points, size_t cap_frames) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    if ((cap_points == 0) != (cap_frames == 0)) return fail(SO_ERR_ARG, "so_keyframe_reserve: cap_points and cap_frames are both 0 or both > 0");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    return keyframes_reserve(c, cap_points, cap_frames);
}

int so_keyframe_add_registered(so_ctx* ctx, const double pose[7], int32_t* id) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose) return fail(SO_ERR_ARG, "bad args");
    KeyframeStore& s = c->kf;
    if (!s.cap_frames) return fail(SO_ERR_ARG, "so_keyframe_add_registered needs a keyframe store (so_keyframe_reserve)");
    if (!finite_pose(pose)) return fail(SO_ERR_ARG, "so_keyframe_add_registered: pose must be finite with a non-zero quaternion");
    const RegisteredScan& r = c->reg;
    if (!r.valid || r.n == 0 || (r.n_edge && !r.edge_valid))
        return fail(SO_ERR_ARG, "so_keyframe_add_registered needs a preceding single-scan so_register* of a non-empty scan (and nothing that reuses the scan or edge buffers in between)");
    if (s.frames() >= s.cap_frames || held(s, 0) + r.n > s.cap_points || held(s, 1) + r.n_edge > s.cap_points)
        return fail(SO_ERR_CAPACITY, "keyframe store full: grow it with so_keyframe_reserve");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    const uint32_t n[2] = {r.n, r.n_edge};
    for (int k = 0; k < 2; ++k)
        if (n[k]) { int rc = put_registered_scan(c, k == 1, s.d_pool[k] + held(s, k), pose); if (rc) return rc; }
    SO_CUDA_TRY(cudaGetLastError());
    for (int k = 0; k < 2; ++k) s.off[k].push_back(s.off[k].back() + n[k]);
    if (id) *id = int32_t(s.frames());
    s.poses.insert(s.poses.end(), pose, pose + 7);
    return SO_OK;
}

int so_keyframe_import(so_ctx* ctx, const void* surf_xyzi, size_t n_surf, const void* edge_xyzi, size_t n_edge, size_t stride_bytes,
                       size_t intensity_offset, const double pose[7], int32_t* id) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !pose || (n_surf && !surf_xyzi) || (n_edge && !edge_xyzi)) return fail(SO_ERR_ARG, "bad args");
    if (stride_bytes < 12) return fail(SO_ERR_ARG, "so_keyframe_import: stride_bytes must be >= 12");
    KeyframeStore& s = c->kf;
    if (!s.cap_frames) return fail(SO_ERR_ARG, "so_keyframe_import needs a keyframe store (so_keyframe_reserve)");
    if (!finite_pose(pose)) return fail(SO_ERR_ARG, "so_keyframe_import: pose must be finite with a non-zero quaternion");
    if (s.frames() >= s.cap_frames || n_surf > s.cap_points - held(s, 0) || n_edge > s.cap_points - held(s, 1))
        return fail(SO_ERR_CAPACITY, "keyframe store full: grow it with so_keyframe_reserve");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    const void* src[2] = {surf_xyzi, edge_xyzi};
    const size_t n[2] = {n_surf, n_edge};
    for (int k = 0; k < 2; ++k) {                                      // verbatim, as so_keyframe_download(id, k, NULL) returns them
        int rc = upload_cloud(c, src[k], n[k], stride_bytes, intensity_offset, s.d_pool[k] + held(s, k));
        if (rc) return rc;
    }
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));                    // the host clouds may go once this returns
    for (int k = 0; k < 2; ++k) s.off[k].push_back(s.off[k].back() + n[k]);
    if (id) *id = int32_t(s.frames());
    s.poses.insert(s.poses.end(), pose, pose + 7);
    return SO_OK;
}

int so_keyframe_info(so_ctx* ctx, size_t* n_frames, size_t* n_points, size_t* n_edge_points) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return fail(SO_ERR_ARG, "null ctx");
    if (n_frames) *n_frames = c->kf.frames();
    if (n_points) *n_points = held(c->kf, 0);
    if (n_edge_points) *n_edge_points = held(c->kf, 1);
    return SO_OK;
}

int so_keyframe_poses(so_ctx* ctx, double* out7, size_t cap, size_t* n) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !n || (!out7 && cap)) return fail(SO_ERR_ARG, "bad args");
    const size_t f = c->kf.frames();
    if (out7) std::memcpy(out7, c->kf.poses.data(), std::min(cap, f) * 7 * sizeof(double));
    *n = f;
    return SO_OK;
}

int so_keyframe_download(so_ctx* ctx, int32_t id, int store, const double pose7[7], float* out_xyzi, size_t cap, size_t* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !n_out || (store != 0 && store != 1) || (!out_xyzi && cap)) return fail(SO_ERR_ARG, "bad args");
    KeyframeStore& s = c->kf;
    { int rc = check_ids(s, &id, 1); if (rc) return rc; }
    if (pose7 && !finite_pose(pose7)) return fail(SO_ERR_ARG, "so_keyframe_download: pose must be finite with a non-zero quaternion");
    SO_CUDA_TRY(cudaSetDevice(c->device));
    const size_t first = s.off[store][id], n = s.off[store][id + 1] - first, m = std::min(n, cap);
    *n_out = n;
    if (!m) return SO_OK;
    const float4* src = s.d_pool[store] + first;
    if (pose7) {                                                       // k_transform_points, as the rebuild transforms it
        KeyframeScratch& k = c->kfs;
        int rc = k.d_raw.reserve(n);
        if (rc) return rc;
        SO_CUDA_TRY(cudaMemcpyAsync(k.d_raw, src, n * sizeof(float4), cudaMemcpyDeviceToDevice, c->stream));
        launch_transform(k.d_raw, uint32_t(n), pose7, c->stream);
        c->launches++;
        src = k.d_raw;
    }
    SO_CUDA_TRY(cudaMemcpyAsync(out_xyzi, src, m * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    SO_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SO_OK;
}

int so_map_from_keyframes(so_ctx* dst_ctx, so_ctx* src_ctx, const int32_t* ids, size_t n_ids, const double* poses7, int stores) {
    Ctx* d = reinterpret_cast<Ctx*>(dst_ctx);
    Ctx* s = reinterpret_cast<Ctx*>(src_ctx);
    if (!d || !s || (n_ids && !poses7) || stores < 1 || stores > 3) return fail(SO_ERR_ARG, "bad args");
    if (d->device != s->device) return fail(SO_ERR_ARG, "so_map_from_keyframes: the two contexts are on different devices");
    const KeyframeStore& kf = s->kf;
    { int rc = check_ids(kf, ids, n_ids); if (rc) return rc; }
    for (size_t i = 0; i < n_ids; ++i)
        if (!finite_pose(poses7 + 7 * i)) return fail(SO_ERR_ARG, "so_map_from_keyframes: poses must be finite with a non-zero quaternion");
    SO_CUDA_TRY(cudaSetDevice(d->device));
    if (s != d) SO_CUDA_TRY(cudaStreamSynchronize(s->stream));        // the keyframes have landed in src's pools
    MapStore* ms[2] = {&d->surf, &d->edge};
    KfBuild b[2];
    for (int k = 0; k < 2; ++k) {                                      // filter and check both stores before either changes
        if (!(stores & (1 << k))) continue;
        std::vector<KfSeg> segs(n_ids);
        uint64_t total = 0;
        for (size_t i = 0; i < n_ids; ++i) {
            const uint64_t first = kf.off[k][ids[i]], n = kf.off[k][ids[i] + 1] - first;
            segs[i].src = first; segs[i].start = uint32_t(total); segs[i].n = uint32_t(n);
            std::memcpy(segs[i].pose, poses7 + 7 * i, sizeof(segs[i].pose));
            total += n;
        }
        if (total >= (uint64_t(1) << 31)) return fail(SO_ERR_CAPACITY, "so_map_from_keyframes: 2^31 points or more selected");
        int rc = keyframe_map_filter(d, *ms[k], k, segs.data(), uint32_t(n_ids), uint32_t(total), kf.d_pool[k], &b[k]);
        if (rc) return rc;
    }
    for (int k = 0; k < 2; ++k) {
        if (!(stores & (1 << k))) continue;
        int rc = keyframe_map_commit(d, *ms[k], k, b[k]);
        if (rc) return rc;
    }
    if (s == d)                                                        // the rebuild after a correction: the keyframes' poses move with it
        for (size_t i = 0; i < n_ids; ++i) {                           // and the loop descriptors of those that moved go stale (host only)
            double* p = d->kf.poses.data() + 7 * size_t(ids[i]);
            if (std::memcmp(p, poses7 + 7 * i, 7 * sizeof(double)) && size_t(ids[i]) < d->kf.desc_ok.size()) d->kf.desc_ok[ids[i]] = 0;
            std::memcpy(p, poses7 + 7 * i, 7 * sizeof(double));
        }
    return SO_OK;
}

int so_map_clear_free_space_keyframes(so_ctx* dst_ctx, so_ctx* src_ctx, const int32_t* ids, size_t n_ids, const double* poses7, int stores,
                                      const so_free_space* opts, so_free_space_keyframes_result* result) {
    Ctx* d = reinterpret_cast<Ctx*>(dst_ctx);
    Ctx* s = reinterpret_cast<Ctx*>(src_ctx);
    if (!d || !s || (n_ids && (!ids || !poses7))) return fail(SO_ERR_ARG, "bad args");
    static const double kIdentity[7] = {0, 0, 0, 0, 0, 0, 1};          // the options and stores alone: every pose is checked below
    { int rc = free_space_check(opts, stores, kIdentity); if (rc) return rc; }
    if (d->device != s->device) return fail(SO_ERR_ARG, "so_map_clear_free_space_keyframes: the two contexts are on different devices");
    if (!s->kf.cap_frames) return fail(SO_ERR_ARG, "so_map_clear_free_space_keyframes needs a keyframe store in src (so_keyframe_reserve)");
    { int rc = check_ids(s->kf, ids, n_ids); if (rc) return rc; }
    for (size_t i = 0; i < n_ids; ++i)
        if (!finite_pose(poses7 + 7 * i)) return fail(SO_ERR_ARG, "so_map_clear_free_space_keyframes: poses must be finite with a non-zero quaternion");
    if (n_ids == 0) {
        if (result) { *result = so_free_space_keyframes_result{}; result->n_after[0] = d->surf.n; result->n_after[1] = d->edge.n; }
        return SO_OK;
    }
    SO_CUDA_TRY(cudaSetDevice(d->device));
    int rc = free_space_prepare(d, stores);
    return rc ? rc : free_space_clear_keyframes(d, s, ids, n_ids, poses7, stores, *opts, result);
}

}  // extern "C"

// =============================================================================
// superodom_b200/KeyframeIO.hpp -- dependency-free writer and reader of a mapping
// session's keyframes, so that a later session can be joined to it
// (LocalMap::saveKeyframes / loadKeyframes in LidarSlam.hpp; INTEGRATION.md,
// "Sessions").  One file holds one session:
//
//   offset 0   "SOKF"                      magic, 4 bytes
//          4   uint32 version              1
//          8   uint64 n_keyframes
//         16   uint64 n_edges
//         24   n_keyframes x { float64 pose7[7]; uint64 n_surf; uint64 n_edge; }
//              then, keyframe by keyframe, n_surf then n_edge points of
//              float32 {x, y, z, intensity} (sensor frame, compensated: what
//              so_keyframe_download(id, store, NULL) returns)
//              then n_edges so_pose_edge records { int32 i, j; float64 z[7],
//              sqrt_info[36], cauchy; } (360 bytes each): the session's graph
//
// Every field is little-endian and fixed-width, whatever the host.  The reader
// checks the whole layout against the file's size before it allocates anything
// from a count in the file: a truncated or padded file, counts that overflow or
// exceed the file, a bad magic or version and non-finite poses are rejected.
// Same convention as PcdIO.hpp: true / false + a message, never throws.
// =============================================================================
#pragma once
#include <array>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <string>
#include <utility>
#include <vector>

#include "../superodom_b200.h"

namespace super_odometry {
namespace b200 {

// One session's keyframes (id order) and graph edges.  Keyframe k's surf and edge clouds are float4 rows of surf[k] and edge[k].
struct KeyframeSession {
    std::vector<std::array<double, 7>> poses;
    std::vector<std::vector<float>> surf, edge;
    std::vector<so_pose_edge> edges;
};

namespace kfio_detail {

constexpr char kMagic[4] = {'S', 'O', 'K', 'F'};
constexpr uint32_t kVersion = 1;
constexpr uint64_t kHeaderBytes = 24, kFrameBytes = 7 * 8 + 2 * 8, kPointBytes = 16, kEdgeBytes = 2 * 4 + (7 + 36 + 1) * 8;

inline void put_u32(std::vector<unsigned char>& b, uint32_t v) { for (int k = 0; k < 4; ++k) b.push_back(static_cast<unsigned char>(v >> (8 * k))); }
inline void put_u64(std::vector<unsigned char>& b, uint64_t v) { for (int k = 0; k < 8; ++k) b.push_back(static_cast<unsigned char>(v >> (8 * k))); }
inline void put_f64(std::vector<unsigned char>& b, double v) { uint64_t u; std::memcpy(&u, &v, 8); put_u64(b, u); }
inline void put_f32(std::vector<unsigned char>& b, float v) { uint32_t u; std::memcpy(&u, &v, 4); put_u32(b, u); }
inline uint32_t get_u32(const unsigned char* p) { uint32_t v = 0; for (int k = 0; k < 4; ++k) v |= uint32_t(p[k]) << (8 * k); return v; }
inline uint64_t get_u64(const unsigned char* p) { uint64_t v = 0; for (int k = 0; k < 8; ++k) v |= uint64_t(p[k]) << (8 * k); return v; }
inline double get_f64(const unsigned char* p) { const uint64_t u = get_u64(p); double v; std::memcpy(&v, &u, 8); return v; }
inline float get_f32(const unsigned char* p) { const uint32_t u = get_u32(p); float v; std::memcpy(&v, &u, 4); return v; }

inline bool fail(std::string* err, const std::string& msg) { if (err) *err = msg; return false; }

}  // namespace kfio_detail

// Writes s to path.  false (and *err) when the session is inconsistent or the file cannot be written.
inline bool writeKeyframeSession(const std::string& path, const KeyframeSession& s, std::string* err = nullptr) {
    using namespace kfio_detail;
    const size_t n = s.poses.size();
    if (s.surf.size() != n || s.edge.size() != n) return fail(err, "writeKeyframeSession: one surf and one edge cloud per pose");
    std::vector<unsigned char> b;
    b.insert(b.end(), kMagic, kMagic + 4);
    put_u32(b, kVersion);
    put_u64(b, n);
    put_u64(b, s.edges.size());
    for (size_t k = 0; k < n; ++k) {
        if (s.surf[k].size() % 4 || s.edge[k].size() % 4) return fail(err, "writeKeyframeSession: clouds are float4 rows");
        for (double v : s.poses[k]) put_f64(b, v);
        put_u64(b, s.surf[k].size() / 4);
        put_u64(b, s.edge[k].size() / 4);
    }
    for (size_t k = 0; k < n; ++k) {
        for (float v : s.surf[k]) put_f32(b, v);
        for (float v : s.edge[k]) put_f32(b, v);
    }
    for (const so_pose_edge& e : s.edges) {
        put_u32(b, uint32_t(e.i)); put_u32(b, uint32_t(e.j));
        for (double v : e.z) put_f64(b, v);
        for (double v : e.sqrt_info) put_f64(b, v);
        put_f64(b, e.cauchy);
    }
    std::ofstream f(path.c_str(), std::ios::binary | std::ios::trunc);
    if (!f.good()) return fail(err, "writeKeyframeSession: cannot open " + path);
    f.write(reinterpret_cast<const char*>(b.data()), std::streamsize(b.size()));
    f.close();
    if (!f.good()) return fail(err, "writeKeyframeSession: write to " + path + " failed");
    return true;
}

// Reads path into *out (replaced only on success).
inline bool readKeyframeSession(const std::string& path, KeyframeSession* out, std::string* err = nullptr) {
    using namespace kfio_detail;
    std::ifstream f(path.c_str(), std::ios::binary);
    if (!f.good()) return fail(err, "readKeyframeSession: cannot open " + path);
    f.seekg(0, std::ios::end);
    const std::streamoff end = f.tellg();
    if (end < 0) return fail(err, "readKeyframeSession: cannot size " + path);
    const uint64_t size = uint64_t(end);
    f.seekg(0, std::ios::beg);
    if (size < kHeaderBytes) return fail(err, "readKeyframeSession: truncated header");
    unsigned char h[kHeaderBytes];
    if (!f.read(reinterpret_cast<char*>(h), kHeaderBytes)) return fail(err, "readKeyframeSession: truncated header");
    if (std::memcmp(h, kMagic, 4)) return fail(err, "readKeyframeSession: bad magic");
    if (get_u32(h + 4) != kVersion) return fail(err, "readKeyframeSession: unsupported version " + std::to_string(get_u32(h + 4)));
    const uint64_t n = get_u64(h + 8), m = get_u64(h + 16);
    // each count bounded by the bytes left before it is multiplied, so no product below can wrap
    uint64_t left = size - kHeaderBytes;
    if (n > left / kFrameBytes) return fail(err, "readKeyframeSession: keyframe count exceeds the file");
    left -= n * kFrameBytes;
    if (m > left / kEdgeBytes) return fail(err, "readKeyframeSession: edge count exceeds the file");
    left -= m * kEdgeBytes;
    std::vector<unsigned char> table(size_t(n * kFrameBytes));
    if (n && !f.read(reinterpret_cast<char*>(table.data()), std::streamsize(table.size()))) return fail(err, "readKeyframeSession: truncated table");
    KeyframeSession s;
    s.poses.resize(size_t(n));
    std::vector<uint64_t> counts(size_t(2 * n));
    uint64_t points = 0;
    for (uint64_t k = 0; k < n; ++k) {
        const unsigned char* p = table.data() + k * kFrameBytes;
        for (int t = 0; t < 7; ++t) {
            s.poses[k][t] = get_f64(p + 8 * t);
            if (!std::isfinite(s.poses[k][t])) return fail(err, "readKeyframeSession: keyframe " + std::to_string(k) + " has a non-finite pose");
        }
        const std::array<double, 7>& q = s.poses[k];
        if (!(q[3] * q[3] + q[4] * q[4] + q[5] * q[5] + q[6] * q[6] > 0.0))
            return fail(err, "readKeyframeSession: keyframe " + std::to_string(k) + " has a zero quaternion");
        for (int c = 0; c < 2; ++c) {
            const uint64_t v = get_u64(p + 56 + 8 * c);
            if (v > left / kPointBytes - points) return fail(err, "readKeyframeSession: point counts exceed the file");
            points += v;
            counts[2 * k + c] = v;
        }
    }
    if (points * kPointBytes != left) return fail(err, "readKeyframeSession: the file size does not match its counts");
    std::vector<unsigned char> body(size_t(left + m * kEdgeBytes));
    if (!body.empty() && !f.read(reinterpret_cast<char*>(body.data()), std::streamsize(body.size()))) return fail(err, "readKeyframeSession: truncated body");
    const unsigned char* p = body.data();
    s.surf.resize(size_t(n));
    s.edge.resize(size_t(n));
    for (uint64_t k = 0; k < n; ++k)
        for (int c = 0; c < 2; ++c) {
            std::vector<float>& dst = c ? s.edge[k] : s.surf[k];
            dst.resize(size_t(4 * counts[2 * k + c]));
            for (float& v : dst) { v = get_f32(p); p += 4; }
        }
    s.edges.resize(size_t(m));
    for (so_pose_edge& e : s.edges) {
        e.i = int32_t(get_u32(p)); e.j = int32_t(get_u32(p + 4)); p += 8;
        for (double& v : e.z) { v = get_f64(p); p += 8; }
        for (double& v : e.sqrt_info) { v = get_f64(p); p += 8; }
        e.cauchy = get_f64(p); p += 8;
    }
    *out = std::move(s);
    return true;
}

}  // namespace b200
}  // namespace super_odometry

// Drives extractEdgeFeatures (include/superodom_b200/FeatureExtraction.hpp) on point_os::PointcloudXYZITR records the way the
// feature-extraction node would fill edgePoints.  Input: binary file from tests/test_edge_features.py {int32 n, float voxel_leaf,
// n records of 32 bytes}; output: int32 count, then {x, y, z, intensity} per edge point, as raw floats.
#include <cstdio>
#include <memory>
#include <vector>

#include "superodom_b200/FeatureExtraction.hpp"

namespace so = super_odometry::b200;

struct PointXYZITR {        // point_os::PointcloudXYZITR layout: x,y,z,pad | intensity, time, ring | pad -> 32 bytes
    float x, y, z, pad0;
    float intensity, time;
    uint16_t ring, pad1;
    float pad2;
};
struct PointXYZI { float x, y, z, pad0; float intensity, pad1[3]; };
template <class P> struct CloudT {
    std::vector<P> points;
    size_t size() const { return points.size(); }
};

static bool rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }

int main(int argc, char** argv) {
    static_assert(sizeof(PointXYZITR) == 32, "layout");
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    int32_t n = 0;
    float leaf = 0.f;
    if (!rd(f, &n, 4) || !rd(f, &leaf, 4)) return 2;
    auto raw = std::make_shared<CloudT<PointXYZITR>>();
    raw->points.resize(n);
    if (n && !rd(f, raw->points.data(), size_t(n) * sizeof(PointXYZITR))) return 2;
    fclose(f);
    size_t stride = 0, toff = 0, roff = 0;
    so::raw_point_layout<PointXYZITR>(&stride, &toff, &roff);
    if (stride != 32 || toff != 20 || roff != 24) return 3;
    so::Context ctx;
    ctx.cfg.max_scan_points = 1u << 18;
    ctx.cfg.max_map_points = 1024;
    try {
        ctx.ensure(0.1f, 0.2f);
        auto edges = std::make_shared<CloudT<PointXYZI>>();
        so_edge_opts opts{};
        opts.voxel_leaf = leaf;
        so::extractEdgeFeatures(ctx, raw, edges, opts);
        FILE* o = fopen(argv[2], "wb");
        if (!o) return 2;
        const int32_t k = int32_t(edges->size());
        fwrite(&k, 4, 1, o);
        for (const auto& p : edges->points) { const float v[4] = {p.x, p.y, p.z, p.intensity}; fwrite(v, 4, 4, o); }
        fclose(o);
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    return 0;
}

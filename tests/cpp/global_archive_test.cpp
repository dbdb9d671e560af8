// Drives LidarSLAM::globalLocalizeInWholeMap (include/superodom_b200/LidarSlam.hpp) in localization-mode order: setArchive ->
// setOrigin -> loadPriorMap -> globalLocalizeInWholeMap, then prints the result.
// Input (little endian): int32 n_map, n_scan, iters, cap; float plane_res; uint64 archive capacity; double origin position[3],
// centre[7]; so_global_opts (half_x / half_y are ignored); n_map then n_scan float4 {x, y, z, intensity} points.
// Output: "status winner" and the seven pose values (%.17g), then last_T_w_lidar, then "lmax leaves_scored steps n_windows", then
// the map origin afterwards.
#include <cstdio>
#include <memory>
#include <vector>

#include "superodom_b200/LidarSlam.hpp"

namespace so = super_odometry::b200;

struct PointXYZI {          // pcl::PointXYZI layout: 32-byte stride, intensity at byte 16
    float x, y, z, pad0;
    float intensity, pad1[3];
};
struct Cloud {
    std::vector<PointXYZI> points;
    size_t size() const { return points.size(); }
};
using CloudPtr = std::shared_ptr<Cloud>;

static bool rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }

static bool read_cloud(FILE* f, int32_t n, Cloud& c) {
    std::vector<float> xyzi(size_t(n) * 4);
    if (n && !rd(f, xyzi.data(), xyzi.size() * 4)) return false;
    c.points.resize(size_t(n));
    for (int32_t i = 0; i < n; ++i) {
        PointXYZI& p = c.points[size_t(i)];
        p.x = xyzi[4 * i]; p.y = xyzi[4 * i + 1]; p.z = xyzi[4 * i + 2]; p.pad0 = 1.f; p.intensity = xyzi[4 * i + 3];
    }
    return true;
}

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: global_archive_test case.bin\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror("open"); return 2; }
    int32_t n_map = 0, n_scan = 0, iters = 0, cap = 0;
    float plane_res = 0;
    uint64_t archive_cap = 0;
    double origin_at[7] = {0, 0, 0, 0, 0, 0, 1}, centre[7];
    so_global_opts opts;
    if (!rd(f, &n_map, 4) || !rd(f, &n_scan, 4) || !rd(f, &iters, 4) || !rd(f, &cap, 4) || !rd(f, &plane_res, 4) ||
        !rd(f, &archive_cap, 8) || !rd(f, origin_at, 3 * sizeof(double)) || !rd(f, centre, sizeof(centre)) || !rd(f, &opts, sizeof(opts)))
        return 2;
    Cloud map;
    CloudPtr scan = std::make_shared<Cloud>();
    if (!read_cloud(f, n_map, map) || !read_cloud(f, n_scan, *scan)) return 2;
    fclose(f);
    so::LidarSLAM slam(0, 1u << 22, 1u << 18);
    slam.localMap.lineRes_ = 0.1f;
    slam.localMap.planeRes_ = plane_res;
    slam.LocalizationICPMaxIter = size_t(iters);
    slam.OptSet.max_surface_features = cap;
    slam.OptSet.yaw_ratio = 0.f;
    try {
        slam.localMap.setArchive(size_t(archive_cap));
        slam.localMap.setOrigin(so::Transformd::from_pose7(origin_at).pos);
        slam.localMap.loadPriorMap(map);
        const int rc = slam.globalLocalizeInWholeMap(scan, so::Transformd::from_pose7(centre), opts);
        double out[7], last[7];
        slam.T_w_lidar.to_pose7(out);
        slam.last_T_w_lidar.to_pose7(last);
        printf("%d %d", rc, slam.last_global.winner);
        for (double v : out) printf(" %.17g", v);
        printf("\n");
        for (double v : last) printf(" %.17g", v);
        printf("\n%d %llu %llu %d\n", slam.last_bnb.lmax, (unsigned long long)slam.last_bnb.leaves_scored,
               (unsigned long long)slam.last_bnb.steps, slam.last_global.n_windows);
        int32_t o[3];
        if (so_map_get_origin(slam.context.h, o) != SO_OK) return 1;
        printf("%d %d %d\n", o[0], o[1], o[2]);
    } catch (const so::Error& e) {
        fprintf(stderr, "shim error: %s\n", e.what());
        return 1;
    }
    return 0;
}

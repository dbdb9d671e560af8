// Within-scan motion compensation with an edge cloud through the shim: slam.Undistortion = APPROXIMATED (mode 1) or OPTIMIZED (mode 2),
// per-point time in the intensity of both clouds.  Otherwise as undistort_test.cpp.  Arguments: case.bin rotation(0|1) map.bin mode.
// Input: a binary file written by tests/test_undistortion_edges.py; output: one line of %.17g numbers per scan on stdout, and the
// whole map (so_map_download mode 0, both stores) as float32 x y z intensity records in map.bin.
#include <cstdio>
#include <cstdlib>
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

static bool read_cloud(FILE* f, CloudPtr& c) {
    int32_t n = 0;
    if (!rd(f, &n, 4)) return false;
    std::vector<float> xyzi(size_t(n) * 4);
    if (!rd(f, xyzi.data(), xyzi.size() * 4)) return false;
    c = std::make_shared<Cloud>();
    c->points.resize(n);
    for (int i = 0; i < n; ++i) {
        PointXYZI& p = c->points[i];
        p.x = xyzi[4 * i]; p.y = xyzi[4 * i + 1]; p.z = xyzi[4 * i + 2]; p.pad0 = 1.f; p.intensity = xyzi[4 * i + 3];
    }
    return true;
}

int main(int argc, char** argv) {
    if (argc < 5) { fprintf(stderr, "usage: undistort_edges_test case.bin rotation map.bin mode\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror("open"); return 2; }
    int32_t n_scans = 0, max_iters = 0, cap = 0;
    float plane_res = 0;
    if (!rd(f, &n_scans, 4) || !rd(f, &max_iters, 4) || !rd(f, &cap, 4) || !rd(f, &plane_res, 4)) return 2;
    static_assert(sizeof(PointXYZI) == 32, "layout");
    so::LidarSLAM slam(0, 1u << 21, 1u << 17);
    slam.localMap.lineRes_ = 0.1f;
    slam.localMap.planeRes_ = plane_res;
    slam.LocalizationICPMaxIter = size_t(max_iters);
    slam.OptSet.max_surface_features = cap;
    slam.OptSet.yaw_ratio = 0.f;
    slam.Undistortion = atoi(argv[4]) == 2 ? so::LidarSLAM::OPTIMIZED : so::LidarSLAM::APPROXIMATED;
    slam.UndistortRotation = atoi(argv[2]) != 0;
    try {
        for (int s = 0; s < n_scans; ++s) {
            double pose[7];
            if (!rd(f, pose, sizeof(pose))) return 2;
            CloudPtr surf, edge;
            if (!read_cloud(f, surf) || !read_cloud(f, edge)) return 2;
            const so::Transformd prior = so::Transformd::from_pose7(pose);
            // OPTIMIZED: the motion prior Localization derives (printed so that the C ABI replay can pass the same bits)
            const so::Transformd D0 = slam.undistort_has_prev ? slam.undistort_prev_pose.inverse() * prior : so::Transformd();
            slam.Localization(s > 0, so::LidarSLAM::PredictionSource::IMU_ORIENTATION, prior, edge, surf, 0.1 * s);
            double out[7];
            slam.T_w_lidar.to_pose7(out);
            printf("%d", s);
            for (double v : out) printf(" %.17g", v);
            const int last = slam.last_result.n_iterations > 0 ? slam.last_result.n_iterations - 1 : 0;
            printf(" %d %zu %d %d", slam.stats.n_iterations, slam.localMap.size(), slam.last_result.iter_n_edge[last], slam.last_result.status);
            double d0[7], dm[7];
            D0.to_pose7(d0);
            slam.LastMotion.to_pose7(dm);
            for (double v : d0) printf(" %.17g", v);
            for (double v : dm) printf(" %.17g", v);
            printf("\n");
        }
        size_t n = slam.localMap.size(), got = 0;
        std::vector<float> map(std::max<size_t>(n, 1) * 4);
        if (so_map_download(slam.context.h, 0, nullptr, map.data(), n, &got) != SO_OK || got != n) { fprintf(stderr, "download\n"); return 1; }
        FILE* g = fopen(argv[3], "wb");
        if (!g || fwrite(map.data(), 4, n * 4, g) != n * 4) { perror("map.bin"); return 1; }
        fclose(g);
    } catch (const so::Error& e) {
        fprintf(stderr, "shim error: %s\n", e.what());
        return 1;
    }
    fclose(f);
    return 0;
}

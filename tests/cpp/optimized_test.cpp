// Within-scan motion estimated by the registration through the shim: slam.Undistortion = OPTIMIZED, per-point time in intensity.
// Otherwise as undistort_test.cpp.  Arguments: case.bin info (OptimizedMotionInformation, all six).  Each scan's line also carries
// the motion prior the shim forms (undistort_prev_pose^-1 * position, recomputed here with the same Transformd operations) and
// LastMotion, so that the caller can repeat the call through the C ABI.  Exercises the reference-surface shim the way laserMapping does:
//   slam.localMap.planeRes_ = ...; slam.LocalizationICPMaxIter = ...; slam.OptSet.max_surface_features = ...;
//   slam.Localization(false, ...)  -> first scan initialises the map
//   slam.Localization(true, ...)   -> ICP + map insert, repeated
// Input: a binary file written by tests/test_cpp_shim.py; output: one line of %.17g numbers per scan on stdout.
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

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: optimized_test case.bin info\n"); return 2; }
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
    slam.Undistortion = so::LidarSLAM::OPTIMIZED;
    for (double& v : slam.OptimizedMotionInformation) v = atof(argv[2]);
    CloudPtr edge = std::make_shared<Cloud>();          // featureExtraction publishes an empty edge cloud
    try {
        for (int s = 0; s < n_scans; ++s) {
            int32_t n = 0;
            double pose[7];
            if (!rd(f, &n, 4) || !rd(f, pose, sizeof(pose))) return 2;
            std::vector<float> xyzi(size_t(n) * 4);
            if (!rd(f, xyzi.data(), xyzi.size() * 4)) return 2;
            CloudPtr surf = std::make_shared<Cloud>();
            surf->points.resize(n);
            for (int i = 0; i < n; ++i) {
                PointXYZI& p = surf->points[i];
                p.x = xyzi[4 * i]; p.y = xyzi[4 * i + 1]; p.z = xyzi[4 * i + 2]; p.pad0 = 1.f; p.intensity = xyzi[4 * i + 3];
            }
            const so::Transformd prior = so::Transformd::from_pose7(pose);
            double d0[7];
            (slam.undistort_prev_pose.inverse() * prior).to_pose7(d0);
            slam.Localization(s > 0, so::LidarSLAM::PredictionSource::IMU_ORIENTATION, prior, edge, surf, 0.1 * s);
            double out[7];
            slam.T_w_lidar.to_pose7(out);
            printf("%d", s);
            for (double v : out) printf(" %.17g", v);
            printf(" %d %d %zu %.17g %.17g %d %d %d", slam.stats.n_iterations, slam.stats.laser_cloud_surf_from_map_num, slam.localMap.size(),
                   slam.LocalizationUncertainty.PositionError, slam.stats.uncertainty_x, slam.localMap.origin_.x(), slam.pos_in_localmap.x(),
                   slam.PlaneFeatureHistogramObs[6]);
            double dl[7];
            slam.LastMotion.to_pose7(dl);
            for (double v : d0) printf(" %.17g", v);
            for (double v : dl) printf(" %.17g", v);
            printf("\n");
        }
        Cloud all = slam.localMap.getAllLocalMap<Cloud>();
        Cloud near = slam.localMap.get5x5LocalMap<Cloud>(slam.pos_in_localmap);
        printf("map %zu %zu\n", all.size(), near.size());
    } catch (const so::Error& e) {
        fprintf(stderr, "shim error: %s\n", e.what());
        return 1;
    }
    fclose(f);
    return 0;
}

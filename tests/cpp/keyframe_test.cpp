// Loop closure through the shim (include/superodom_b200/LidarSlam.hpp), the way a node drives it:
//   slam.localMap.reserveKeyframes(points, frames)
//   slam.Localization(...) then slam.addKeyframe()             -> every registered scan kept with its pose
//   submap.buildFromKeyframes(slam.localMap, first ids, poses)  -> a loop-verification submap in a second context
//   slam.alignKeyframes(submap, {last id}, {its pose})          -> the loop constraint (pose, cov)
//   slam.rebuildFromKeyframes(corrected)                        -> the map rebuilt from every keyframe
// Input: the binary case file of shim_test (scans and priors; the first scan initialises the map and is not a keyframe).
// stdout: "kf <id> <pose7>" per keyframe, "loop <status> <pose7>", then "rebuilt <keyframes> <map points> <T_w_lidar pose7>".
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

#include "superodom_b200/LidarSlam.hpp"

namespace so = super_odometry::b200;

struct PointXYZI { float x, y, z, pad0; float intensity, pad1[3]; };
struct Cloud { std::vector<PointXYZI> points; size_t size() const { return points.size(); } };
using CloudPtr = std::shared_ptr<Cloud>;

static bool rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }
static void put(const so::Transformd& t) { double p[7]; t.to_pose7(p); for (double v : p) printf(" %.17g", v); }

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: keyframe_test case.bin\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror("open"); return 2; }
    int32_t n_scans = 0, max_iters = 0, cap = 0;
    float plane_res = 0;
    if (!rd(f, &n_scans, 4) || !rd(f, &max_iters, 4) || !rd(f, &cap, 4) || !rd(f, &plane_res, 4)) return 2;
    so::LidarSLAM slam(0, 1u << 21, 1u << 17);
    slam.localMap.lineRes_ = 0.1f;
    slam.localMap.planeRes_ = plane_res;
    slam.LocalizationICPMaxIter = size_t(max_iters);
    slam.OptSet.max_surface_features = cap;
    slam.OptSet.yaw_ratio = 0.f;
    so::Context sub_ctx;
    so::LocalMap submap(&sub_ctx);
    submap.planeRes_ = plane_res;
    CloudPtr edge = std::make_shared<Cloud>();
    try {
        slam.localMap.reserveKeyframes(size_t(n_scans) << 17, size_t(n_scans));
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
            slam.Localization(s > 0, so::LidarSLAM::PredictionSource::IMU_ORIENTATION, so::Transformd::from_pose7(pose), edge, surf, 0.1 * s);
            if (s > 0) {
                const int32_t id = slam.addKeyframe();
                printf("kf %d", id);
                put(slam.T_w_lidar);
                printf("\n");
            }
        }
        std::vector<so::Transformd> poses = slam.keyframePoses();
        if (poses.size() < 3) { fprintf(stderr, "need at least 4 scans\n"); return 2; }
        const int32_t last = int32_t(poses.size()) - 1;
        submap.buildFromKeyframes(slam.localMap, {0, 1}, {poses[0], poses[1]});
        const std::vector<so_icp_result> r = slam.alignKeyframes(submap, {last}, {poses[last]});
        printf("loop %d", r[0].status);
        put(so::Transformd::from_pose7(r[0].pose));
        printf("\n");
        poses[last] = so::Transformd::from_pose7(r[0].pose);
        slam.rebuildFromKeyframes(poses);
        printf("rebuilt %zu %zu", slam.keyframePoses().size(), slam.localMap.size());
        put(slam.T_w_lidar);
        printf("\n");
    } catch (const so::Error& e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}

// Loop detection through the shim (include/superodom_b200/LidarSlam.hpp), the way a node drives it:
//   slam.Localization(...) then slam.addKeyframe()              -> every registered scan kept with its pose
//   slam.loopCandidates(last, k)                                 -> the best Scan Context matches of the last keyframe
//   slam.loopPrior(best), submap.buildFromKeyframes(...)         -> the alignment prior and a submap around the candidate
//   slam.alignKeyframes(submap, {last}, {prior})                 -> the loop constraint
// Input: the binary case file of shim_test (scans and priors; the first scan initialises the map and is not a keyframe); argv[2]:
// exclude_recent.  stdout: "kf <id> <pose7>" per keyframe, "cand <query> <id> <distance> <shift> <n_pairs> <yaw>" per candidate,
// "prior <pose7>", then "loop <status> <pose7>".
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
    if (argc < 3) { fprintf(stderr, "usage: loop_test case.bin exclude_recent\n"); return 2; }
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
    slam.loopOpts.exclude_recent = atoi(argv[2]);
    slam.loopOpts.max_range = 30.0;
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
        const std::vector<so::Transformd> poses = slam.keyframePoses();
        const int32_t last = int32_t(poses.size()) - 1;
        const std::vector<so_loop_candidate> c = slam.loopCandidates(last, 3);
        for (const so_loop_candidate& x : c) printf("cand %d %d %.17g %d %d %.17g\n", x.query, x.id, x.distance, x.shift, x.n_pairs, x.yaw);
        if (c.empty() || c[0].id < 0) { fprintf(stderr, "no candidate\n"); return 1; }
        const so::Transformd prior = slam.loopPrior(c[0]);
        printf("prior");
        put(prior);
        printf("\n");
        submap.buildFromKeyframes(slam.localMap, {c[0].id}, {poses[size_t(c[0].id)]});
        const std::vector<so_icp_result> r = slam.alignKeyframes(submap, {last}, {prior});
        printf("loop %d", r[0].status);
        put(so::Transformd::from_pose7(r[0].pose));
        printf("\n");
    } catch (const so::Error& e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}

// isDegenerate and DegeneracyAware through the shim.  Arguments: case.bin pos_threshold ori_threshold aware (0/1).  Input as
// optimized_test.cpp (written by tests/test_degeneracy_shim.py); the scans register with Undistortion == NONE.  Output: one line per
// scan of %.17g numbers: s, T_w_lidar pose7, isDegenerate, last_result.pos_inv_cond, last_result.ori_inv_cond, last_result.status,
// last_degeneracy.flags_pos, last_degeneracy.flags_ori, last_degeneracy.icp.pose_opt[7].
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
    if (argc < 5) { fprintf(stderr, "usage: degeneracy_test case.bin pos_threshold ori_threshold aware\n"); return 2; }
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
    slam.Pos_degeneracy_threshold = float(atof(argv[2]));
    slam.Ori_degeneracy_threshold = float(atof(argv[3]));
    slam.DegeneracyAware = atoi(argv[4]) != 0;
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
            slam.Localization(s > 0, so::LidarSLAM::PredictionSource::IMU_ORIENTATION, so::Transformd::from_pose7(pose), edge, surf, 0.1 * s);
            double out[7];
            slam.T_w_lidar.to_pose7(out);
            printf("%d", s);
            for (double v : out) printf(" %.17g", v);
            printf(" %d %.17g %.17g %d %d %d", slam.isDegenerate ? 1 : 0, slam.last_result.pos_inv_cond, slam.last_result.ori_inv_cond,
                   slam.last_result.status, slam.last_degeneracy.flags_pos, slam.last_degeneracy.flags_ori);
            for (double v : slam.last_degeneracy.icp.pose_opt) printf(" %.17g", v);
            printf("\n");
        }
    } catch (const so::Error& e) {
        fprintf(stderr, "shim error: %s\n", e.what());
        return 1;
    }
    fclose(f);
    return 0;
}

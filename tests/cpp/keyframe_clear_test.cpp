// Free-space clearing after a loop-closure rebuild, through the shim (include/superodom_b200/LidarSlam.hpp):
//   slam.Localization(...) with ClearFreeSpace on, then slam.addKeyframe()   -> every registered scan kept with its pose
//   slam.rebuildFromKeyframes(corrected, opts)                                -> the map rebuilt, then cleared against every keyframe
// Usage: keyframe_clear_test case.bin map.bin
// case.bin: int32 n_scans, then per scan int32 n, double pose[7] (the prior; the first scan initialises the map there and is not a
// keyframe), float xyzi[n][4].  The corrected poses are the keyframes' own poses moved by (0.05, -0.03, 0) m.
// stdout: "kf <id> <corrected pose7>" per keyframe, then "clear <n_keyframes> <removed> <surf after> <edge after> <tiles>";
// map.bin: the final surf + edge map (getAllLocalMap) as float xyzi.
#include <cstdio>
#include <memory>
#include <vector>

#include "superodom_b200/LidarSlam.hpp"

namespace so = super_odometry::b200;

struct PointXYZI { float x, y, z, pad0; float intensity, pad1[3]; };
struct Cloud { std::vector<PointXYZI> points; size_t size() const { return points.size(); } };
using CloudPtr = std::shared_ptr<Cloud>;

static bool rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: keyframe_clear_test case.bin map.bin\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror("open"); return 2; }
    int32_t n_scans = 0;
    if (!rd(f, &n_scans, 4)) return 2;
    so::LidarSLAM slam(0, 1u << 21, 1u << 17);
    slam.localMap.lineRes_ = 0.1f;
    slam.localMap.planeRes_ = 0.2f;
    slam.LocalizationICPMaxIter = 5;
    slam.OptSet.max_surface_features = 0;
    slam.ClearFreeSpace = true;
    slam.FreeSpaceOpts.az_res_deg = 0.4f;                 // VLP-16 image: one row per beam
    slam.FreeSpaceOpts.el_res_deg = 2.f;
    slam.FreeSpaceOpts.el_min_deg = -16.f;
    slam.FreeSpaceOpts.el_max_deg = 16.f;
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
            if (s > 0) slam.addKeyframe();
        }
        std::vector<so::Transformd> corrected = slam.keyframePoses();
        for (size_t i = 0; i < corrected.size(); ++i) {
            double p[7];
            corrected[i].to_pose7(p);
            p[0] += 0.05; p[1] -= 0.03;
            corrected[i] = so::Transformd::from_pose7(p);
            corrected[i].to_pose7(p);
            printf("kf %zu", i);
            for (double v : p) printf(" %.17g", v);
            printf("\n");
        }
        slam.rebuildFromKeyframes(corrected, slam.FreeSpaceOpts);
        const so_free_space_keyframes_result& r = slam.last_keyframe_clear;
        printf("clear %llu %llu %llu %llu %llu\n", (unsigned long long)r.n_keyframes, (unsigned long long)r.n_removed,
               (unsigned long long)r.n_after[0], (unsigned long long)r.n_after[1], (unsigned long long)r.n_tiles);
        Cloud all = slam.localMap.getAllLocalMap<Cloud>();
        FILE* o = fopen(argv[2], "wb");
        if (!o) { perror("open"); return 2; }
        for (const PointXYZI& p : all.points) { const float v[4] = {p.x, p.y, p.z, p.intensity}; fwrite(v, 4, 4, o); }
        fclose(o);
    } catch (const so::Error& e) {
        fprintf(stderr, "shim error: %s\n", e.what());
        return 1;
    }
    fclose(f);
    return 0;
}

// The block archive through the shim (include/superodom_b200/LidarSlam.hpp, PcdIO.hpp), in localization mode's order:
//   localMap.setArchive(cap); localMap.setOrigin(start); readPointCloud(prior.pcd); localMap.loadPriorMap(prior)
// then the window moves away and back (shiftMap), and getWholeMap + writePointCloud save the map for the next session.
// Usage: archive_shim_test prior.pcd out.pcd x_far; stdout: "<window points> <archive points> <whole-map points>" after the load,
// after the far shift and after the return, one line each.
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

#include "superodom_b200/LidarSlam.hpp"
#include "superodom_b200/PcdIO.hpp"

namespace so = super_odometry::b200;

struct PointXYZI { float x, y, z, pad0; float intensity, pad1[3]; };
struct Cloud { std::vector<PointXYZI> points; size_t size() const { return points.size(); } };

int main(int argc, char** argv) {
    if (argc < 4) { fprintf(stderr, "usage: archive_shim_test prior.pcd out.pcd x_far\n"); return 2; }
    so::LidarSLAM slam(0, 1u << 20, 1u << 16);
    slam.localMap.planeRes_ = 0.4f;
    try {
        slam.localMap.setArchive(size_t(1) << 22);
        slam.localMap.setOrigin(so::Vector3d(0, 0, 0));
        auto prior = std::make_shared<Cloud>();
        if (!so::readPointCloud(argv[1], prior)) return 1;
        slam.localMap.loadPriorMap(*prior);
        auto line = [&]() {
            printf("%zu %zu %zu\n", slam.localMap.size(), slam.localMap.archiveSize(), slam.localMap.getWholeMap<Cloud>().size());
        };
        line();
        slam.localMap.shiftMap(so::Vector3d(std::atof(argv[3]), 0, 0));
        line();
        slam.localMap.shiftMap(so::Vector3d(0, 0, 0));
        line();
        if (!so::writePointCloud(argv[2], slam.localMap.getWholeMap<Cloud>())) return 1;
    } catch (const so::Error& e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}

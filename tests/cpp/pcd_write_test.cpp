// Round trip of include/superodom_b200/PcdIO.hpp: raw float records {x, y, z, intensity} (argv[1]) -> writePointCloud (argv[2]) ->
// readPointCloud -> raw floats (argv[3]).  Exit code 3 when the cloud read back differs from the one written, bit for bit.
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include "superodom_b200/PcdIO.hpp"

struct PointXYZI { float x, y, z, pad0; float intensity, pad1[3]; };
struct Cloud { std::vector<PointXYZI> points; size_t size() const { return points.size(); } };

int main(int argc, char** argv) {
    if (argc < 4) return 2;
    FILE* in = fopen(argv[1], "rb");
    if (!in) return 2;
    Cloud cloud;
    float v[4];
    while (fread(v, 4, 4, in) == 4) { PointXYZI p{}; p.x = v[0]; p.y = v[1]; p.z = v[2]; p.intensity = v[3]; cloud.points.push_back(p); }
    fclose(in);
    if (!super_odometry::b200::writePointCloud(argv[2], cloud)) return 1;
    auto back = std::make_shared<Cloud>();
    if (!super_odometry::b200::readPointCloud(argv[2], back)) return 1;
    if (back->size() != cloud.size()) return 3;
    for (size_t i = 0; i < cloud.size(); ++i) {
        const PointXYZI &a = cloud.points[i], &b = back->points[i];
        if (std::memcmp(&a.x, &b.x, 12) || std::memcmp(&a.intensity, &b.intensity, 4)) return 3;
    }
    FILE* o = fopen(argv[3], "wb");
    if (!o) return 2;
    for (const auto& p : back->points) { const float w[4] = {p.x, p.y, p.z, p.intensity}; fwrite(w, 4, 4, o); }
    fclose(o);
    return 0;
}

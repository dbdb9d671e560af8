// Two sessions joined through the shim (include/superodom_b200/LidarSlam.hpp), the way INTEGRATION.md's "Sessions" drives it:
//   session A: Localization() + addKeyframe() per scan, then localMap.saveKeyframes(file, A's odometry edges)
//   session B, in a frame T_BW away: the same, then localMap.loadKeyframes(file) -> A's ids after B's
//   loopCandidatesIn(B's newest, k, A's ids) -> loopPrior -> alignKeyframes against a submap of A's candidate
//   optimizeKeyframes(B's odometry + A's edges + the cross edge, A constant, from B moved into A's frame by the loop result)
//   mergeKeyframes(corrected, B's newest)
// Input: shim_test's case file with B's frame (pose7, doubles) after its header.  Argument 2: the session file to write.
// stdout: "a_last <pose7>", "loaded <first> <count>", "candidate <id> <distance>", "merged <T_w_lidar pose7>", "map <points>".
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "superodom_b200/LidarSlam.hpp"

namespace so = super_odometry::b200;

struct PointXYZI { float x, y, z, pad0; float intensity, pad1[3]; };
struct Cloud { std::vector<PointXYZI> points; size_t size() const { return points.size(); } };
using CloudPtr = std::shared_ptr<Cloud>;

static bool rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }
static void put(const char* tag, const so::Transformd& t) {
    double p[7];
    t.to_pose7(p);
    printf("%s", tag);
    for (double v : p) printf(" %.17g", v);
    printf("\n");
}

static so_pose_edge edge(int32_t i, int32_t j, const so::Transformd& z, double w_t, double w_r, double cauchy) {
    so_pose_edge e{};
    e.i = i; e.j = j;
    z.to_pose7(e.z);
    for (int k = 0; k < 6; ++k) e.sqrt_info[k * 7] = k < 3 ? w_t : w_r;
    e.cauchy = cauchy;
    return e;
}

static void configure(so::LidarSLAM& slam, float plane_res, int max_iters, int cap) {
    slam.localMap.lineRes_ = 0.1f;
    slam.localMap.planeRes_ = plane_res;
    slam.LocalizationICPMaxIter = size_t(max_iters);
    slam.OptSet.max_surface_features = cap;
    slam.OptSet.yaw_ratio = 0.f;
}

// Every scan localized from its prior (moved by `frame`) and kept as a keyframe after the first; -> the odometry edges
static std::vector<so_pose_edge> drive(so::LidarSLAM& slam, const std::vector<CloudPtr>& scans, const std::vector<so::Transformd>& priors,
                                       const so::Transformd& frame) {
    CloudPtr edge_cloud = std::make_shared<Cloud>();
    slam.localMap.reserveKeyframes(scans.size() << 17, 2 * scans.size());
    for (size_t s = 0; s < scans.size(); ++s) {
        slam.Localization(s > 0, so::LidarSLAM::PredictionSource::IMU_ORIENTATION, frame * priors[s], edge_cloud, scans[s], 0.1 * double(s));
        if (s > 0) slam.addKeyframe();
    }
    const std::vector<so::Transformd> p = slam.keyframePoses();
    std::vector<so_pose_edge> edges;
    for (size_t i = 0; i + 1 < p.size(); ++i) edges.push_back(edge(int32_t(i), int32_t(i + 1), p[i].inverse() * p[i + 1], 20.0, 57.0, 0.0));
    return edges;
}

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: session_test case.bin session.sokf\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror("open"); return 2; }
    int32_t n_scans = 0, max_iters = 0, cap = 0;
    float plane_res = 0;
    double frame7[7];
    if (!rd(f, &n_scans, 4) || !rd(f, &max_iters, 4) || !rd(f, &cap, 4) || !rd(f, &plane_res, 4) || !rd(f, frame7, sizeof(frame7))) return 2;
    std::vector<CloudPtr> scans;
    std::vector<so::Transformd> priors;
    for (int s = 0; s < n_scans; ++s) {
        int32_t n = 0;
        double pose[7];
        if (!rd(f, &n, 4) || !rd(f, pose, sizeof(pose))) return 2;
        std::vector<float> xyzi(size_t(n) * 4);
        if (!rd(f, xyzi.data(), xyzi.size() * 4)) return 2;
        CloudPtr c = std::make_shared<Cloud>();
        c->points.resize(size_t(n));
        for (int i = 0; i < n; ++i) {
            PointXYZI& p = c->points[size_t(i)];
            p.x = xyzi[4 * i]; p.y = xyzi[4 * i + 1]; p.z = xyzi[4 * i + 2]; p.pad0 = 1.f; p.intensity = xyzi[4 * i + 3];
        }
        scans.push_back(c);
        priors.push_back(so::Transformd::from_pose7(pose));
    }
    try {
        {   // session A, in its own frame, saved
            so::LidarSLAM a(0, 1u << 21, 1u << 17);
            configure(a, plane_res, max_iters, cap);
            const std::vector<so_pose_edge> edges = drive(a, scans, priors, so::Transformd());
            put("a_last", a.keyframePoses().back());
            a.localMap.saveKeyframes(argv[2], edges);
        }
        so::LidarSLAM b(0, 1u << 21, 1u << 17);
        configure(b, plane_res, max_iters, cap);
        std::vector<so_pose_edge> edges = drive(b, scans, priors, so::Transformd::from_pose7(frame7));
        const int32_t live = int32_t(b.keyframePoses().size()) - 1;
        const so::LocalMap::LoadedKeyframes A = b.localMap.loadKeyframes(argv[2]);
        printf("loaded %d %d\n", A.first, A.count);
        b.loopOpts.max_range = 20.0;
        const so_loop_candidate c = b.loopCandidatesIn(live, 3, A.first, A.first + A.count)[0];
        printf("candidate %d %.17g\n", c.id, c.distance);
        if (c.id < 0) { fprintf(stderr, "no candidate\n"); return 1; }
        const std::vector<so::Transformd> est = b.keyframePoses();
        so::Context sub_ctx;
        so::LocalMap submap(&sub_ctx);
        submap.planeRes_ = plane_res;
        submap.setOrigin(est[size_t(c.id)].pos);
        submap.buildFromKeyframes(b.localMap, {c.id}, {est[size_t(c.id)]});
        const so_icp_result r = b.alignKeyframes(submap, {live}, {b.loopPrior(c)})[0];
        if (r.status != 0) { fprintf(stderr, "alignment status %d\n", r.status); return 1; }
        const so::Transformd aligned = so::Transformd::from_pose7(r.pose);
        for (so_pose_edge e : A.edges) { e.i += A.first; e.j += A.first; edges.push_back(e); }
        edges.push_back(edge(c.id, live, est[size_t(c.id)].inverse() * aligned, 20.0, 286.0, 1.0));
        std::vector<uint8_t> constant(est.size(), 0);
        std::vector<so::Transformd> init = est;
        const so::Transformd C0 = aligned * est[size_t(live)].inverse();
        for (size_t i = 0; i < est.size(); ++i) {
            if (int32_t(i) >= A.first) constant[i] = 1;
            else init[i] = C0 * est[i];
        }
        so_pose_graph_opts opts;
        so_pose_graph_opts_defaults(&opts);
        const so::LidarSLAM::GraphSolution sol = b.optimizeKeyframes(edges, constant, opts, init);
        b.mergeKeyframes(sol.poses, live);
        put("merged", b.T_w_lidar);
        printf("map %zu\n", b.localMap.size());
    } catch (const so::Error& e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}

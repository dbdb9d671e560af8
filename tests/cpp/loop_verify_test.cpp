// Loop verification through the shim (include/superodom_b200/LidarSlam.hpp), the way a loop-closing back end drives it:
//   slam.localMap.loadKeyframes(file)                            -> a session's keyframes (sensor-frame clouds, drifted poses)
//   slam.loopCandidates(query, 5)                                -> the best Scan Context matches of the query
//   slam.verifyLoop(scratch, candidates)                         -> each candidate aligned and scored; the first accepted one is the loop
//   slam.optimizeKeyframes(odometry + loop edges, ...)           -> the corrected poses
//   slam.rebuildFromKeyframes(corrected)                         -> the map rebuilt at them
// argv[1]: the session file (KeyframeIO.hpp), argv[2]: the query keyframe.  stdout: "cand <id> <distance>" per candidate, "verify <id>
// <skipped> <accepted> <status> <overlap> <conflict_query> <conflict_map> <rel7>" per result, "loop <id>", "graph <termination>",
// "pose <id> <pose7>" per keyframe, then "map <points>".
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "superodom_b200/LidarSlam.hpp"

namespace so = super_odometry::b200;

static void put(const double* p, int n) { for (int k = 0; k < n; ++k) printf(" %.17g", p[k]); }

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: loop_verify_test session.bin query\n"); return 2; }
    const int32_t query = atoi(argv[2]);
    so::LidarSLAM slam(0, 1u << 21, 1u << 18);
    slam.localMap.lineRes_ = 0.1f;
    slam.localMap.planeRes_ = 0.2f;
    slam.loopOpts.rings = 20; slam.loopOpts.sectors = 60; slam.loopOpts.max_range = 20.0; slam.loopOpts.height_offset = 2.0;
    slam.loopOpts.exclude_recent = 30;
    slam.loopVerifyOpts.image.el_res_deg = 2.f;                        // VLP-16
    slam.loopVerifyOpts.image.el_min_deg = -16.f;
    slam.loopVerifyOpts.image.el_max_deg = 16.f;
    so::Context sub_ctx;
    sub_ctx.cfg.max_map_points = 1u << 21;
    sub_ctx.cfg.max_scan_points = 1u << 18;
    so::LocalMap scratch(&sub_ctx);
    scratch.lineRes_ = 0.1f;
    scratch.planeRes_ = 0.2f;
    try {
        slam.localMap.reserveKeyframes(size_t(query + 1) << 15, size_t(query + 1));
        const so::LocalMap::LoadedKeyframes kf = slam.localMap.loadKeyframes(argv[1]);
        if (kf.count != query + 1) { fprintf(stderr, "expected %d keyframes, got %d\n", query + 1, kf.count); return 1; }
        const std::vector<so_loop_candidate> c = slam.loopCandidates(query, 5);
        for (const so_loop_candidate& x : c) printf("cand %d %.17g\n", x.id, x.distance);
        const std::vector<so_loop_verify_result> v = slam.verifyLoop(scratch, c);
        int loop = -1;
        for (const so_loop_verify_result& r : v) {
            printf("verify %d %d %d %d %.17g %.17g %.17g", r.id, r.skipped, r.accepted, r.reg.status, r.overlap, r.conflict_query, r.conflict_map);
            put(r.rel7, 7);
            printf("\n");
            if (loop < 0 && r.accepted) loop = int(&r - v.data());
        }
        printf("loop %d\n", loop < 0 ? -1 : v[size_t(loop)].id);
        if (loop < 0) { fprintf(stderr, "no candidate accepted\n"); return 1; }
        // odometry between consecutive keyframes, the verified loop between the candidate and the query; keyframe 0 held
        const std::vector<so::Transformd> est = slam.keyframePoses();
        auto edge = [](int32_t i, int32_t j, const so::Transformd& z, double st, double sr) {
            so_pose_edge e{};
            e.i = i; e.j = j;
            z.to_pose7(e.z);
            for (int k = 0; k < 6; ++k) e.sqrt_info[7 * k] = k < 3 ? 1.0 / st : 1.0 / sr;
            return e;
        };
        const double deg = 3.141592653589793 / 180.0;
        std::vector<so_pose_edge> edges;
        for (int32_t i = 0; i < query; ++i) edges.push_back(edge(i, i + 1, est[size_t(i)].inverse() * est[size_t(i) + 1], 0.05, 1.0 * deg));
        const so_loop_verify_result& r = v[size_t(loop)];
        edges.push_back(edge(r.id, query, so::Transformd::from_pose7(r.rel7), 0.05, 0.2 * deg));
        std::vector<uint8_t> constant(est.size(), 0);
        constant[0] = 1;
        so_pose_graph_opts go{};
        so_pose_graph_opts_defaults(&go);
        const so::LidarSLAM::GraphSolution g = slam.optimizeKeyframes(edges, constant, go);
        printf("graph %d\n", g.result.termination);
        slam.rebuildFromKeyframes(g.poses);
        const std::vector<so::Transformd> after = slam.keyframePoses();
        for (size_t i = 0; i < after.size(); ++i) {
            double p[7];
            after[i].to_pose7(p);
            printf("pose %zu", i);
            put(p, 7);
            printf("\n");
        }
        printf("map %zu\n", slam.localMap.size());
    } catch (const so::Error& e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}

// include/superodom_b200/KeyframeIO.hpp from the command line (tests/test_sessions_cpu.py):
//   keyframe_io_test copy IN OUT   read IN, print "ok <keyframes> <edges> <points>", write it back to OUT; exit 1 with the reader's
//                                  message on stderr when IN is rejected
#include <cstdio>
#include <string>

#include "superodom_b200/KeyframeIO.hpp"

int main(int argc, char** argv) {
    using namespace super_odometry::b200;
    if (argc != 4 || std::string(argv[1]) != "copy") { std::fprintf(stderr, "usage: keyframe_io_test copy IN OUT\n"); return 2; }
    KeyframeSession s;
    std::string err;
    if (!readKeyframeSession(argv[2], &s, &err)) { std::fprintf(stderr, "%s\n", err.c_str()); return 1; }
    size_t points = 0;
    for (size_t k = 0; k < s.poses.size(); ++k) points += (s.surf[k].size() + s.edge[k].size()) / 4;
    std::printf("ok %zu %zu %zu\n", s.poses.size(), s.edges.size(), points);
    if (!writeKeyframeSession(argv[3], s, &err)) { std::fprintf(stderr, "%s\n", err.c_str()); return 1; }
    return 0;
}

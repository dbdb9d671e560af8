// so_graph_rule.h -- the neighbour graph's certificate and build rule (plain C++: shared by the kernels, so_map.cu and a CPU test).
//
// Row a of the graph holds the kGraphK nearest in-block points of map point a; radius[a] = kGraphRadiusScale x the distance to the
// last of them, below which the row holds every in-block point (so_knn.cuh, knn_graph_rank).
#pragma once
#include <cmath>
#include <cstddef>

#ifdef __CUDACC__
#define SO_HD __host__ __device__ __forceinline__
#else
#define SO_HD inline
#endif

namespace so {

#ifndef SO_KNN_GRAPH_K
#define SO_KNN_GRAPH_K 16
#endif
constexpr int kGraphK = SO_KNN_GRAPH_K;
static_assert(kGraphK % 4 == 0, "rows are read as uint4");
// A registration call builds the graph when its queries number at least this many times the store's points.  The build costs one
// exact in-block (kGraphK + 1)-NN search per map point, a few times one query's search; a call of 8 queries per map point searches
// each of them once per ICP iteration (3-20), so it repays the build within the call.  Single scans and the live loop (~2 000
// queries against a map of 10^5-10^6 points) never reach it.
constexpr size_t kGraphQueriesPerPoint = 8;
// The distances the certificate compares (approx_d2, exact_d2, float square roots) are within ~5e-7 of the true ones; 1e-5 is
// twenty times that.
constexpr float kGraphRadiusScale = 0.99999f;

// mode: 1 forced on, -1 off, 0 the rule
SO_HD bool graph_build_due(int mode, size_t queries, size_t map_points) {
    return map_points > 0 && mode >= 0 && (mode > 0 || queries >= kGraphQueriesPerPoint * map_points);
}

// Query q with bound U (every neighbour the search can return lies within sqrt(U)) and anchor a at squared distance qa2 from q:
// every such neighbour lies within sqrt(U) + |q - a| of a, so inside a's row when that is below radius[a].  NaN or infinite terms
// fail (the comparison is false).
SO_HD bool graph_certifies(float U, float qa2, float radius) {
    return sqrtf(U) + sqrtf(qa2) + 1e-12f < radius;
}

}  // namespace so

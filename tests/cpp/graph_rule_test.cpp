// CPU test of the neighbour graph's build rule and certificate (superodom_b200/csrc/so_graph_rule.h): the rule's thresholds, and on
// random clouds that every point within sqrt(U) of a certified query lies in its anchor's row, with distances rounded as the kernels
// round them.  Prints "ok" and exits 0 on success.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include "../../superodom_b200/csrc/so_graph_rule.h"

#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

static float exact_d2(const float* a, const float* b) {
    const float dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
    return float(double(dx) * double(dx) + double(dy) * double(dy) + double(dz) * double(dz));
}

int main() {
    using namespace so;
    // build rule
    CHECK(!graph_build_due(0, 8 * 1000 - 1, 1000));
    CHECK(graph_build_due(0, 8 * 1000, 1000));
    CHECK(graph_build_due(0, 256 * 131072, 1010000));             // a 256-scan call of 131 k-point scans on a 1 M-point map
    CHECK(!graph_build_due(0, 2001, 100000));                      // a single decimated scan
    CHECK(!graph_build_due(0, 1u << 30, 0));
    CHECK(graph_build_due(1, 0, 1));
    CHECK(!graph_build_due(-1, size_t(1) << 40, 1));
    // certificate: strict, and false for NaN / infinite terms; +inf radius certifies every finite query
    CHECK(graph_certifies(0.01f, 0.01f, 0.3f));
    CHECK(!graph_certifies(0.01f, 0.01f, 0.2f));
    CHECK(!graph_certifies(NAN, 0.f, INFINITY));
    CHECK(!graph_certifies(0.f, NAN, INFINITY));
    CHECK(!graph_certifies(0.f, INFINITY, INFINITY));
    CHECK(graph_certifies(0.5f, 0.5f, INFINITY));
    CHECK(!graph_certifies(0.f, 0.f, 0.f));
    // soundness on random clouds (one block): rows and radii as k_knn_graph builds them, queries near map points
    std::mt19937 rng(7);
    std::uniform_real_distribution<float> uni(-2.f, 2.f), small(-0.3f, 0.3f);
    int certified = 0;
    for (int trial = 0; trial < 40; ++trial) {
        const int n = 60 + trial * 10;
        std::vector<float> p(3 * n);
        for (auto& v : p) v = uni(rng);
        for (int i = 0; i < n / 10; ++i) for (int a = 0; a < 3; ++a) p[3 * (n - 1 - i) + a] = p[3 * i + a];   // duplicates
        for (int q = 0; q < 200; ++q) {
            const int a = int(rng() % n);
            const float qq[3] = {p[3 * a] + small(rng), p[3 * a + 1] + small(rng), p[3 * a + 2] + small(rng)};
            std::vector<std::pair<float, int>> da, dq;                                // (d2, id) from the anchor / the query
            for (int i = 0; i < n; ++i) { if (i != a) da.push_back({exact_d2(&p[3 * a], &p[3 * i]), i}); dq.push_back({exact_d2(qq, &p[3 * i]), i}); }
            std::sort(da.begin(), da.end());
            std::sort(dq.begin(), dq.end());
            const float radius = int(da.size()) <= kGraphK ? INFINITY : kGraphRadiusScale * std::sqrt(da[kGraphK - 1].first);
            const float U = dq[4].first * 1.000004f;                                  // the search's bound: at least the 5th d2
            if (!graph_certifies(U, exact_d2(qq, &p[3 * a]), radius)) continue;
            ++certified;
            std::vector<int> row;
            for (int j = 0; j < std::min<int>(kGraphK, int(da.size())); ++j) row.push_back(da[j].second);
            row.push_back(a);
            for (const auto& c : dq) if (c.first <= U) CHECK(std::find(row.begin(), row.end(), c.second) != row.end());
        }
    }
    CHECK(certified > 1000);
    std::printf("ok %d\n", certified);
    return 0;
}

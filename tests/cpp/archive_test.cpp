// CPU unit test of the block archive's key and window logic (superodom_b200/csrc/so_archive.h): world blocks of points (negative
// coordinates, block faces, non-finite values, the key range), key packing and order, window membership and the window's rows.
#include <cmath>
#include <cstdio>
#include <limits>
#include <set>
#include <vector>

#include "so_archive.h"

using namespace so::archive;

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL line %d: %s\n", __LINE__, #c); ++fails; } } while (0)

// LocalMap.h:594-605 with origin 0, as the device bins a point: int((x + 25) / 50), minus one below zero, in double
static int ref_block(float x) { const double v = double(x) + 25.0; int c = int(v / 50.0); if (v < 0) c--; return c; }

int main() {
    // world block of an axis: the device's binning, including its faces and negative side
    for (float x : {0.f, 24.99f, 25.f, -25.f, -25.0001f, -75.f, -74.9f, 1234.5f, -1234.5f, 1e6f, -1e6f, -24.9999f}) {
        int w = 0;
        CHECK(world_axis(x, &w));
        CHECK(w == ref_block(x));
    }
    int w = 0;
    CHECK(!world_axis(std::numeric_limits<float>::quiet_NaN(), &w));
    CHECK(!world_axis(std::numeric_limits<float>::infinity(), &w));
    CHECK(!world_axis(-std::numeric_limits<float>::infinity(), &w));
    CHECK(!world_axis(3e7f, &w) && !world_axis(-3e7f, &w));          // beyond 2^19 blocks
    CHECK(world_axis(2.6e7f, &w) && w < kKeyOff && w == ref_block(2.6e7f));
    CHECK(world_axis(-2.6e7f, &w) && w >= -kKeyOff && w == ref_block(-2.6e7f));
    CHECK(point_key(0.f, std::nanf(""), 0.f) == kKeyNone);

    // packing: a round trip over negative and positive blocks, and key order = (z, y, x) order
    const int vals[] = {-kKeyOff, -70000, -3, -1, 0, 1, 2, 19, 70000, kKeyOff - 1};
    std::vector<std::pair<std::vector<int>, uint64_t>> all;
    for (int x : vals) for (int y : vals) for (int z : vals) {
        const uint64_t k = world_key(x, y, z);
        int u[3];
        unpack_key(k, u);
        CHECK(u[0] == x && u[1] == y && u[2] == z);
        CHECK(k != kKeyNone && k < (uint64_t(1) << 60));
        all.push_back({{z, y, x}, k});
    }
    for (size_t i = 0; i < all.size(); ++i)
        for (size_t j = 0; j < all.size(); j += 37) CHECK((all[i].first < all[j].first) == (all[i].second < all[j].second));
    CHECK(point_key(-30.f, 80.f, -1.f) == world_key(-1, 2, 0) && point_key(-80.f, 80.f, -30.f) == world_key(-2, 2, -1));

    // window membership: grid index g = w + origin in 21 x 21 x 11; the window's rows cover exactly its blocks, in key order
    const int32_t origins[][3] = {{10, 10, 5}, {0, 0, 0}, {-37, 12, 4}, {65, -20, 9}, {3, 17, -2}};
    for (const auto& o : origins) {
        std::set<uint64_t> inside;
        for (int gz = -2; gz < kWinD + 2; ++gz)
            for (int gy = -2; gy < kWinH + 2; ++gy)
                for (int gx = -2; gx < kWinW + 2; ++gx) {
                    const int b[3] = {gx - o[0], gy - o[1], gz - o[2]};
                    const bool in = gx >= 0 && gx < kWinW && gy >= 0 && gy < kWinH && gz >= 0 && gz < kWinD;
                    CHECK(in_window(b, o) == in);
                    if (in) inside.insert(world_key(b[0], b[1], b[2]));
                }
        CHECK(inside.size() == size_t(kWinW * kWinH * kWinD));
        std::set<uint64_t> covered;
        uint64_t prev_hi = 0;
        int rows = 0;
        window_rows(o, [&](uint64_t lo, uint64_t hi) {
            CHECK(lo <= hi && (rows == 0 || lo > prev_hi));
            prev_hi = hi;
            ++rows;
            for (uint64_t k : inside) if (k >= lo && k <= hi) covered.insert(k);
            int a[3], b[3];
            unpack_key(lo, a); unpack_key(hi, b);
            CHECK(in_window(a, o) && in_window(b, o) && b[0] - a[0] == kWinW - 1 && a[1] == b[1] && a[2] == b[2]);
        });
        CHECK(rows == kWinH * kWinD && covered == inside);
    }
    // a shift by one block along +x: the window keeps 20 of 21 columns; the leaving and entering columns are the two faces
    {
        const int32_t o0[3] = {10, 10, 5}, o1[3] = {9, 10, 5};        // the origin decreases when the sensor moves towards +x
        int leave = 0, enter = 0;
        for (int z = -20; z < 20; ++z) for (int y = -30; y < 30; ++y) for (int x = -30; x < 30; ++x) {
            const int b[3] = {x, y, z};
            if (in_window(b, o0) && !in_window(b, o1)) { ++leave; CHECK(x == -10); }
            if (!in_window(b, o0) && in_window(b, o1)) { ++enter; CHECK(x == 11); }
        }
        CHECK(leave == kWinH * kWinD && enter == kWinH * kWinD);
    }
    std::printf(fails ? "FAILED %d\n" : "ok\n", fails);
    return fails ? 1 : 0;
}

// The host rule of so_loop_verify (superodom_b200/csrc/so_verify_rule.h) at its edges: the accept rule at each threshold, the conflict
// fraction without candidates, the eligible submap ids, and loop_relative against a composition written out by hand.  Prints "ok"
// and exits 0 when every check holds.
#include <cmath>
#include <cstdio>

#include "../../superodom_b200/csrc/so_verify_rule.h"

static int failures = 0;
#define CHECK(cond)                                                                 \
    do {                                                                            \
        if (!(cond)) { std::printf("FAIL line %d: %s\n", __LINE__, #cond); ++failures; } \
    } while (0)

int main() {
    using namespace so;
    // the decision: >= min_overlap and <= max_conflict, both fractions, status 0 only
    CHECK(verify_accept(0, 0.5, 0.05, 0.05, 0.5, 0.05));                    // every value at its threshold
    CHECK(!verify_accept(0, std::nextafter(0.5, 0.0), 0.0, 0.0, 0.5, 0.05));
    CHECK(!verify_accept(0, 1.0, std::nextafter(0.05, 1.0), 0.0, 0.5, 0.05));
    CHECK(!verify_accept(0, 1.0, 0.0, std::nextafter(0.05, 1.0), 0.5, 0.05));
    for (int status = 1; status <= 3; ++status) CHECK(!verify_accept(status, 1.0, 0.0, 0.0, 0.5, 0.05));
    CHECK(!verify_accept(0, std::nan(""), 0.0, 0.0, 0.5, 0.05));
    CHECK(verify_accept(0, 0.0, 1.0, 1.0, 0.0, 1.0));                       // the loosest thresholds accept any converged alignment
    CHECK(!verify_accept(0, 1.0, 0.0, 0.0, 1.0 + 1e-12, 0.0) && verify_accept(0, 1.0, 0.0, 0.0, 1.0, 0.0));
    // fractions: zero candidates read 0, which passes any max_conflict
    CHECK(verify_fraction(0, 0) == 0.0);
    CHECK(verify_fraction(3, 0) == 0.0);
    CHECK(verify_fraction(1, 4) == 0.25);
    CHECK(verify_accept(0, 0.5, verify_fraction(0, 0), verify_fraction(0, 0), 0.5, 0.0));
    // eligible ids: below query - exclude_recent, or a range without the query
    const VerifyRange a = verify_range(40, 0, -1, 30);
    CHECK(a.begin == 0 && a.end == 10);
    CHECK(verify_eligible(a, 40, 0) && verify_eligible(a, 40, 9) && !verify_eligible(a, 40, 10) && !verify_eligible(a, 40, -1));
    const VerifyRange b = verify_range(5, 0, -1, 30);
    CHECK(b.begin == 0 && b.end == 0 && !verify_eligible(b, 5, 0));
    const VerifyRange c = verify_range(3, 2, 8, 30);
    CHECK(c.begin == 2 && c.end == 8 && verify_eligible(c, 3, 2) && !verify_eligible(c, 3, 3) && verify_eligible(c, 3, 7) &&
          !verify_eligible(c, 3, 8) && !verify_eligible(c, 3, 1));
    // loop_relative: X^-1 P for X = (t, yaw 90 deg), P = X * (1, 0, 0; yaw 10 deg) -> (1, 0, 0; yaw 10 deg)
    const double s45 = std::sin(M_PI / 4), c45 = std::cos(M_PI / 4);
    const double X[7] = {3.0, -2.0, 0.5, 0.0, 0.0, s45, c45};
    const double s5 = std::sin(M_PI / 36), c5 = std::cos(M_PI / 36);
    double qp[4];
    const double qz[4] = {0.0, 0.0, s5, c5};
    verify_qmul(X + 3, qz, qp);
    const double P[7] = {3.0, -1.0, 0.5, qp[0], qp[1], qp[2], qp[3]};
    double Z[7];
    loop_relative(X, P, Z);
    CHECK(std::fabs(Z[0] - 1.0) < 1e-14 && std::fabs(Z[1]) < 1e-14 && std::fabs(Z[2]) < 1e-14);
    CHECK(std::fabs(Z[3]) < 1e-14 && std::fabs(Z[4]) < 1e-14 && std::fabs(Z[5] - s5) < 1e-14 && std::fabs(Z[6] - c5) < 1e-14);
    // loop_prior: a level query and candidate, yaw 0 -> the candidate's position with the candidate's heading
    double prior[7];
    const double Q[7] = {10.0, 10.0, 1.0, 0.0, 0.0, 0.0, 1.0};
    loop_prior(X, Q, 0.0, prior);
    CHECK(prior[0] == 3.0 && prior[1] == -2.0 && prior[2] == 0.5);
    CHECK(std::fabs(prior[5] - s45) < 1e-15 && std::fabs(prior[6] - c45) < 1e-15 && prior[3] == 0.0 && prior[4] == 0.0);
    if (failures) return 1;
    std::printf("ok\n");
    return 0;
}

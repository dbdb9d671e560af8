// The trust-region rules (superodom_b200/csrc/so_trust_region_rule.h) at their edges: every exit test at its threshold and one ulp
// beyond, the step quality, the radius update at its cap and at the 1/3 floor, the decrease factor, when the diagonal is reused, the
// diagonal clamp, and exits 4 and 5, which no solve of the library reaches.  Prints "ok" and then each constant the numpy restatement
// also states, as "NAME hexfloat", and exits 0 when every check holds.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <limits>

#include "../../superodom_b200/csrc/so_trust_region_rule.h"

static int failures = 0;
#define CHECK(cond)                                                                 \
    do {                                                                            \
        if (!(cond)) { std::printf("FAIL line %d: %s\n", __LINE__, #cond); ++failures; } \
    } while (0)

// The members the rules read and write, under IcpState's names
struct State {
    double radius = 0.0, decrease_factor = 0.0, x_norm = 0.0, gmax = 0.0, cost = 0.0;
    int32_t lm_iter = 0, lm_max_iterations = 0, num_successful = 0, num_unsuccessful = 0, reuse_diagonal = 0, consecutive_invalid = 0,
            termination = 0;
};

static State start(int32_t lm_max_iterations) {
    State s;
    s.lm_max_iterations = lm_max_iterations;
    s.gmax = 1.0;
    so::tr_iteration_zero(s);
    return s;
}

// The top of the loop: count the last step, then the three exits in their order; -1 when the solve goes on to a step
static int top_of_loop(State& s, bool step_successful) {
    using namespace so;
    tr_count(s, step_successful);
    if (tr_at_limit(s)) return kTermIterations;
    if (tr_gradient_small(s)) return kTermGradient;
    if (tr_radius_small(s)) return kTermRadius;
    s.lm_iter++;
    return -1;
}

int main() {
    using namespace so;
    const double inf = std::numeric_limits<double>::infinity(), nan = std::nan("");

    // IterationZero
    State s = start(4);
    CHECK(s.radius == 1e4 && s.decrease_factor == 2.0 && s.reuse_diagonal == 0);

    // the exits before a step: each at its threshold, and one ulp (one iteration) short of it
    s.lm_iter = 4; CHECK(tr_at_limit(s));
    s.lm_iter = 3; CHECK(!tr_at_limit(s));
    s.lm_iter = 5; CHECK(tr_at_limit(s));
    s.gmax = 1e-10; CHECK(tr_gradient_small(s));
    s.gmax = std::nextafter(1e-10, inf); CHECK(!tr_gradient_small(s));
    s.gmax = 0.0; CHECK(tr_gradient_small(s));
    s.gmax = nan; CHECK(!tr_gradient_small(s));
    s.radius = 1e-32; CHECK(tr_radius_small(s));
    s.radius = std::nextafter(1e-32, inf); CHECK(!tr_radius_small(s));

    // the exits on a candidate: |step| <= 1e-8 (|x| + 1e-8), given |step|^2 (sqrt(x * x) == x), |cost change| <= 1e-6 cost, either sign
    s.x_norm = 3.0;
    const double step_max = 1e-8 * (3.0 + 1e-8), step_beyond = std::nextafter(step_max, inf);
    CHECK(tr_parameter_small(s, step_max * step_max));
    CHECK(!tr_parameter_small(s, step_beyond * step_beyond));
    s.x_norm = 0.0;
    const double step_min = 1e-8 * 1e-8, step_min_beyond = std::nextafter(step_min, inf);
    CHECK(tr_parameter_small(s, step_min * step_min) && !tr_parameter_small(s, step_min_beyond * step_min_beyond));
    CHECK(tr_parameter_small(s, 0.0) && !tr_parameter_small(s, nan));
    s.cost = 2.5;
    const double change_max = 1e-6 * 2.5;
    CHECK(tr_function_small(s, change_max) && tr_function_small(s, -change_max));
    CHECK(!tr_function_small(s, std::nextafter(change_max, inf)) && !tr_function_small(s, -std::nextafter(change_max, inf)));

    // step quality: a step is accepted strictly above 1e-3
    CHECK(tr_step_rejected(1e-3));
    CHECK(!tr_step_rejected(std::nextafter(1e-3, inf)));
    CHECK(tr_step_rejected(nan) && tr_step_rejected(-inf) && !tr_step_rejected(inf));

    // a valid step: solved, and a positive model cost change
    CHECK(tr_step_valid(true, std::numeric_limits<double>::denorm_min()));
    CHECK(!tr_step_valid(true, 0.0) && !tr_step_valid(true, -0.0) && !tr_step_valid(true, nan) && !tr_step_valid(false, 1.0));

    // the radius after an accepted step: radius / max(1/3, 1 - (2 rd - 1)^3), at most 1e16
    s = start(4);
    tr_accepted(s, 0.5);
    CHECK(s.radius == 1e4);                                          // 1 - 0^3 = 1
    s = start(4);
    tr_accepted(s, 0.9);                                             // 1 - 0.8^3 = 0.488, above the floor
    CHECK(s.radius == 1e4 / (1.0 - 0.8 * 0.8 * 0.8));
    const double floored[] = {0.95, 1.0, 2.0};                       // 1 - t^3 = 0.271, 0, -26: the floor, three times the radius
    for (double rd : floored) {
        s = start(4);
        tr_accepted(s, rd);
        CHECK(s.radius == 1e4 / (1.0 / 3.0));
    }
    s.radius = 3e15; tr_accepted(s, 1.0);
    CHECK(s.radius == 3e15 / (1.0 / 3.0) && s.radius < 1e16);
    s.radius = 5e15; tr_accepted(s, 1.0);
    CHECK(s.radius == 1e16);                                         // capped
    tr_accepted(s, 1.0);
    CHECK(s.radius == 1e16);
    tr_accepted(s, 0.5);
    CHECK(s.radius == 1e16);

    // the decrease factor doubles over consecutive rejections and an acceptance resets it; the diagonal is kept after a rejection
    // and recomputed after an acceptance
    s = start(4);
    tr_rejected(s);
    CHECK(s.radius == 5e3 && s.decrease_factor == 4.0 && s.reuse_diagonal == 1);
    tr_rejected(s);
    CHECK(s.radius == 1250.0 && s.decrease_factor == 8.0 && s.reuse_diagonal == 1);
    tr_rejected(s);
    CHECK(s.radius == 156.25 && s.decrease_factor == 16.0);
    tr_accepted(s, 0.5);
    CHECK(s.radius == 156.25 && s.decrease_factor == 2.0 && s.reuse_diagonal == 0);
    tr_rejected(s);
    CHECK(s.radius == 78.125 && s.decrease_factor == 4.0 && s.reuse_diagonal == 1);

    // an invalid step keeps the diagonal
    s = start(4);
    CHECK(s.reuse_diagonal == 0 && !tr_invalid_step(s) && s.reuse_diagonal == 1);

    // the LM diagonal clamp [1e-6, 1e32]; a NaN diagonal takes the lower bound
    CHECK(tr_lm_diagonal(1e-6) == 1e-6 && tr_lm_diagonal(std::nextafter(1e-6, 0.0)) == 1e-6);
    CHECK(tr_lm_diagonal(std::nextafter(1e-6, inf)) == std::nextafter(1e-6, inf));
    CHECK(tr_lm_diagonal(0.0) == 1e-6 && tr_lm_diagonal(-1.0) == 1e-6 && tr_lm_diagonal(-inf) == 1e-6);
    CHECK(tr_lm_diagonal(1e32) == 1e32 && tr_lm_diagonal(std::nextafter(1e32, inf)) == 1e32 && tr_lm_diagonal(inf) == 1e32);
    CHECK(tr_lm_diagonal(std::nextafter(1e32, 0.0)) == std::nextafter(1e32, 0.0));
    CHECK(tr_lm_diagonal(1.5) == 1.5);
    CHECK(tr_lm_diagonal(nan) == 1e-6);

    // exit 4: from 1e4 the radius falls by 2, 4, 8, ...; after 14 rejections it is 1e4 / 2^105 ~ 2.5e-28, after 15 it is
    // 1e4 / 2^120 ~ 7.5e-33 and the radius test ends the solve, at 15 LM iterations
    s = start(16);
    int term = top_of_loop(s, false);
    while (term < 0) {
        tr_rejected(s);
        term = top_of_loop(s, false);
    }
    CHECK(term == kTermRadius && s.lm_iter == 15 && s.num_unsuccessful == 16 && s.num_successful == 0);
    CHECK(s.radius == 1e4 / std::ldexp(1.0, 120) && s.radius <= 1e-32 && s.radius * std::ldexp(1.0, 15) > 1e-32);
    // with 15 LM iterations the iteration limit, tested first, ends it instead
    s = start(15);
    term = top_of_loop(s, false);
    while (term < 0) {
        tr_rejected(s);
        term = top_of_loop(s, false);
    }
    CHECK(term == kTermIterations && s.lm_iter == 15 && tr_radius_small(s));

    // exit 5: four invalid steps halve the radius four times, a valid step resets the count, five in a row end the solve
    s = start(16);
    for (int k = 0; k < 4; ++k) CHECK(!tr_invalid_step(s));
    CHECK(s.consecutive_invalid == 4 && s.radius == 625.0);
    tr_valid_step(s);
    CHECK(s.consecutive_invalid == 0 && s.radius == 625.0);
    for (int k = 0; k < 4; ++k) CHECK(!tr_invalid_step(s));
    CHECK(s.consecutive_invalid == 4 && s.radius == 625.0 / 16.0);
    CHECK(tr_invalid_step(s));
    CHECK(s.consecutive_invalid == 5 && s.radius == 625.0 / 16.0);    // the fifth ends the solve without halving

    if (failures) return 1;
    std::printf("ok\n");
    const struct { const char* name; double value; } constants[] = {
        {"FUNCTION_TOL", kTrFunctionTol}, {"GRADIENT_TOL", kTrGradientTol}, {"PARAMETER_TOL", kTrParameterTol},
        {"MIN_REL_DECREASE", kTrMinRelativeDecrease}, {"MIN_LM_DIAG", kTrMinLmDiagonal}, {"MAX_LM_DIAG", kTrMaxLmDiagonal},
        {"MAX_RADIUS", kTrMaxRadius}, {"MIN_RADIUS", kTrMinRadius},
    };
    for (const auto& c : constants) std::printf("%s %a\n", c.name, c.value);
    return 0;
}

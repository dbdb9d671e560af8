// so_trust_region_rule.h -- the trust-region rules every solve of the library follows (plain C++: shared by the device loop of
// so_trust_region.cuh, the pose graph's host loop in so_pose_graph.cu and a CPU test).
//
// The values are Ceres 2.0.0's defaults, which the reference's ceres::Solve runs with: Solver::Options (function, gradient and
// parameter tolerances, min_relative_decrease, initial and maximum trust-region radius, min_trust_region_radius,
// max_num_consecutive_invalid_steps, min/max_lm_diagonal), TrustRegionMinimizer (the exits and their order, the step quality) and
// LevenbergMarquardtStrategy (the radius and decrease-factor updates, the diagonal clamp, when the diagonal is reused).
//
// The rules read and write a state S by member name: radius, decrease_factor, reuse_diagonal, consecutive_invalid, lm_iter,
// lm_max_iterations, num_successful, num_unsuccessful, gmax, x_norm, cost (IcpState on the device).  They are predicates and updates
// only: each loop keeps its own control flow and, at every exit, sets the termination code itself.
#pragma once
#include <cmath>

#ifdef __CUDACC__
#define SO_TR_HD __host__ __device__ __forceinline__
#else
#define SO_TR_HD inline
#endif

namespace so {

constexpr double kTrFunctionTol = 1e-6;
constexpr double kTrGradientTol = 1e-10;
constexpr double kTrParameterTol = 1e-8;
constexpr double kTrMinRelativeDecrease = 1e-3;     // a step of lower quality is rejected
constexpr double kTrInitialRadius = 1e4;
constexpr double kTrMaxRadius = 1e16;
constexpr double kTrMinRadius = 1e-32;
constexpr double kTrRadiusDivisorFloor = 1.0 / 3.0; // an accepted step grows the radius at most threefold
constexpr double kTrInitialDecreaseFactor = 2.0;    // a rejection divides the radius by the decrease factor, then doubles it
constexpr double kTrInvalidRadiusFactor = 0.5;
constexpr int kTrMaxConsecutiveInvalid = 5;
constexpr double kTrMinLmDiagonal = 1e-6;
constexpr double kTrMaxLmDiagonal = 1e32;

// Termination codes (so_icp_result.iter_lm_termination, so_pose_graph_result.termination)
enum : int {
    kTermIterations = 0,    // lm_max_iterations reached
    kTermGradient = 1,      // gmax <= kTrGradientTol
    kTermParameter = 2,     // ParameterToleranceReached
    kTermFunction = 3,      // FunctionToleranceReached
    kTermRadius = 4,        // radius <= kTrMinRadius
    kTermInvalid = 5,       // kTrMaxConsecutiveInvalid invalid steps in a row
};

// IterationZero: the strategy's starting radius and decrease factor; the first step computes the diagonal
template <class S>
SO_TR_HD void tr_iteration_zero(S& s) {
    s.radius = kTrInitialRadius; s.decrease_factor = kTrInitialDecreaseFactor; s.reuse_diagonal = 0;
}

// FinalizeIterationAndCheckIfMinimizerCanContinue: iteration 0 and every step not accepted count as unsuccessful
template <class S>
SO_TR_HD void tr_count(S& s, bool step_successful) {
    if (step_successful) s.num_successful++; else s.num_unsuccessful++;
}

// The exits tested before each step, in this order
template <class S>
SO_TR_HD bool tr_at_limit(const S& s) { return s.lm_iter >= s.lm_max_iterations; }
template <class S>
SO_TR_HD bool tr_gradient_small(const S& s) { return s.gmax <= kTrGradientTol; }
template <class S>
SO_TR_HD bool tr_radius_small(const S& s) { return s.radius <= kTrMinRadius; }

// The LM diagonal of one column from the diagonal of the scaled H
SO_TR_HD double tr_lm_diagonal(double h) { return std::fmin(std::fmax(h, kTrMinLmDiagonal), kTrMaxLmDiagonal); }

// A step is valid when its linear solve succeeded with finite values and the model predicts a decrease
SO_TR_HD bool tr_step_valid(bool solved, double model_cost_change) { return solved && model_cost_change > 0.0; }

// HandleInvalidStep: counts the step; true when it is the kTrMaxConsecutiveInvalid-th in a row (the solve ends with kTermInvalid),
// otherwise the radius is halved and the diagonal kept
template <class S>
SO_TR_HD bool tr_invalid_step(S& s) {
    if (++s.consecutive_invalid >= kTrMaxConsecutiveInvalid) return true;
    s.radius *= kTrInvalidRadiusFactor; s.reuse_diagonal = 1;
    return false;
}
template <class S>
SO_TR_HD void tr_valid_step(S& s) { s.consecutive_invalid = 0; }

// The exits tested on a valid step's candidate, in this order: the step norm (from its square) against |x|, the cost change against
// the cost.  The step norm's square root is taken here, and the step quality test below is stated as the rejection, because in
// these forms the device loop compiles to the SASS it had with the tests written out in place (a predicate on the step norm as an
// argument, or on the acceptance, changes the step kernels' branch layout; scripts/sass_compare.py shows it).
template <class S>
SO_TR_HD bool tr_parameter_small(const S& s, double step_norm2) {
    return std::sqrt(step_norm2) <= kTrParameterTol * (s.x_norm + kTrParameterTol);
}
template <class S>
SO_TR_HD bool tr_function_small(const S& s, double cost_change) { return std::fabs(cost_change) <= kTrFunctionTol * s.cost; }

// The step quality test on cost change / model cost change: a step not above kTrMinRelativeDecrease (or NaN) is rejected
SO_TR_HD bool tr_step_rejected(double relative_decrease) { return !(relative_decrease > kTrMinRelativeDecrease); }

// StepAccepted: the radius grows or shrinks with the step quality, at most threefold and up to kTrMaxRadius; the next step
// recomputes the diagonal
template <class S>
SO_TR_HD void tr_accepted(S& s, double relative_decrease) {
    const double t = 2.0 * relative_decrease - 1.0;
    s.radius = std::fmin(kTrMaxRadius, s.radius / std::fmax(kTrRadiusDivisorFloor, 1.0 - t * t * t));
    s.decrease_factor = kTrInitialDecreaseFactor; s.reuse_diagonal = 0;
}

// StepRejected: the radius falls by the decrease factor, which doubles; the diagonal is kept
template <class S>
SO_TR_HD void tr_rejected(S& s) {
    s.radius = s.radius / s.decrease_factor; s.decrease_factor *= 2.0; s.reuse_diagonal = 1;
}

}  // namespace so

// so_verify_rule.h -- the host arithmetic of loop verification (so_loop_verify, so_verify.cu): the alignment prior of a candidate
// (so_loop_prior), the relative pose a loop edge carries, the eligible submap ids and the accept rule.  Plain C++, so that a CPU test
// compiles it.
#pragma once
#include <cmath>
#include <cstdint>

namespace so {

// Heading psi = atan2(R10, R00) of quaternion {x, y, z, w} (normalised first), as the Scan Context descriptor levels a keyframe
inline double verify_heading(const double q[4]) {
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
    return std::atan2(2 * (x * y + z * w), 1 - 2 * (y * y + z * z));
}

// out = a * b (Hamilton product, {x, y, z, w})
inline void verify_qmul(const double a[4], const double b[4], double out[4]) {
    const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    const double y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    const double z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
    out[0] = x; out[1] = y; out[2] = z; out[3] = w;
}

// The alignment prior of a loop candidate: the candidate's position, and the query's orientation turned about the world z axis by
// psi_cand + yaw - psi_query, which gives the candidate's heading plus yaw and keeps the query's roll and pitch
inline void loop_prior(const double cand7[7], const double query7[7], double yaw, double out7[7]) {
    const double turn = verify_heading(cand7 + 3) + yaw - verify_heading(query7 + 3);
    const double qz[4] = {0.0, 0.0, std::sin(turn / 2), std::cos(turn / 2)};
    double q[4];
    verify_qmul(qz, query7 + 3, q);
    for (int k = 0; k < 3; ++k) out7[k] = cand7[k];
    for (int k = 0; k < 4; ++k) out7[3 + k] = q[k];
}

// z = X^-1 * P (X's quaternion normalised first): the measurement of a loop edge from keyframe X to the aligned pose P
inline void loop_relative(const double x7[7], const double p7[7], double z7[7]) {
    const double n = std::sqrt(x7[3] * x7[3] + x7[4] * x7[4] + x7[5] * x7[5] + x7[6] * x7[6]);
    const double xi[4] = {-x7[3] / n, -x7[4] / n, -x7[5] / n, x7[6] / n};
    const double d[4] = {p7[0] - x7[0], p7[1] - x7[1], p7[2] - x7[2], 0.0};
    double t[4], r[4];
    verify_qmul(xi, d, t);                                               // conj(q) (p - x) q: the difference in X's frame
    const double q[4] = {-xi[0], -xi[1], -xi[2], xi[3]};
    verify_qmul(t, q, r);
    for (int k = 0; k < 3; ++k) z7[k] = r[k];
    verify_qmul(xi, p7 + 3, r);
    for (int k = 0; k < 4; ++k) z7[3 + k] = r[k];
}

// The ids a submap of query may use: [begin, end) without the query itself; end < 0 selects [0, query - exclude_recent), the ids
// so_loop_candidates searches
struct VerifyRange { int32_t begin, end; };
inline VerifyRange verify_range(int32_t query, int32_t id_begin, int32_t id_end, int32_t exclude_recent) {
    if (id_end < 0) {
        const int64_t e = int64_t(query) - int64_t(exclude_recent);
        return VerifyRange{0, int32_t(e > 0 ? e : 0)};
    }
    return VerifyRange{id_begin, id_end};
}
inline bool verify_eligible(const VerifyRange& r, int32_t query, int32_t id) { return id >= r.begin && id < r.end && id != query; }

// A conflict fraction: conflicts over candidates, 0 without candidates
inline double verify_fraction(uint64_t conflicts, uint64_t candidates) {
    return candidates ? double(conflicts) / double(candidates) : 0.0;
}

// The decision: the registration converged (status 0), the overlap reaches min_overlap and neither conflict fraction exceeds max_conflict
inline bool verify_accept(int32_t status, double overlap, double conflict_query, double conflict_map, double min_overlap, double max_conflict) {
    return status == 0 && overlap >= min_overlap && conflict_query <= max_conflict && conflict_map <= max_conflict;
}

}  // namespace so

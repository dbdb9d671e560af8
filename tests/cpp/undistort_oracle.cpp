// CPU oracle for within-scan motion compensation (UndistortionMode::APPROXIMATED, so_register_undistort*): the oracle's own
// translation unit compiled unchanged, plus two entry points that restate the definition (DESIGN.md §3) on the CPU:
//   orc_undistort_points    pInit of a cloud at T_cur = pose
//   orc_register_undistort  orc_register's ICP loop (surf cloud only) with pInit, recomputed from the CURRENT estimate at the
//                           start of every ICP iteration, in place of the sensor-frame points
// Built by tests/undistort_oracle.py with the oracle's flags (-ffp-contract=off: every product and sum rounded on its own, the
// order the device kernels use explicitly).
#include "../../oracle/so_oracle.cpp"

namespace orc_und {

static void qmul(const double a[4], const double b[4], double o[4]) {
    o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    o[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    o[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
    o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}
static void qrot(const double q[4], const double v[3], double o[3]) {
    double ux = q[1] * v[2] - q[2] * v[1], uy = q[2] * v[0] - q[0] * v[2], uz = q[0] * v[1] - q[1] * v[0];
    ux += ux; uy += uy; uz += uz;
    o[0] = v[0] + q[3] * ux + (q[1] * uz - q[2] * uy);
    o[1] = v[1] + q[3] * uy + (q[2] * ux - q[0] * uz);
    o[2] = v[2] + q[3] * uz + (q[0] * uy - q[1] * ux);
}

struct Delta { double q[4], t[3], th, inv; };

// D = T_prev^-1 * T_cur; th < 0 marks Eigen's linear slerp branch (|dot(identity, q_D)| >= 1 - eps)
static Delta delta(const double prev[7], const double cur[7]) {
    Delta D;
    const double qpc[4] = {-prev[3], -prev[4], -prev[5], prev[6]};
    double q[4];
    qmul(qpc, cur + 3, q);
    const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    const double s = 1.0 / std::sqrt(n2);
    for (int k = 0; k < 4; ++k) D.q[k] = q[k] * s;
    const double d[3] = {cur[0] - prev[0], cur[1] - prev[1], cur[2] - prev[2]};
    qrot(qpc, d, D.t);
    const double ad = std::fabs(D.q[3]);
    if (ad >= 1.0 - 2.220446049250313e-16) { D.th = -1.0; D.inv = 0.0; }
    else { D.th = std::acos(ad); D.inv = 1.0 / std::sin(D.th); }
    return D;
}

static void point(const Delta& D, double dt, int rotation, const float* p, float tau, float out[3]) {
    const double a = std::isfinite(tau) ? double(tau) / dt : 0.0;
    const double v[3] = {double(p[0]), double(p[1]), double(p[2])};
    double o[3] = {v[0], v[1], v[2]};
    if (rotation) {
        double s0, s1;
        if (D.th < 0.0) { s0 = 1.0 - a; s1 = a; }
        else { s0 = std::sin((1.0 - a) * D.th) * D.inv; s1 = std::sin(a * D.th) * D.inv; }
        if (D.q[3] < 0.0) s1 = -s1;
        const double qi[4] = {s0 * 0.0 + s1 * D.q[0], s0 * 0.0 + s1 * D.q[1], s0 * 0.0 + s1 * D.q[2], s0 + s1 * D.q[3]};
        qrot(qi, v, o);
    }
    for (int k = 0; k < 3; ++k) out[k] = float(o[k] + a * D.t[k]);
}

}  // namespace orc_und

extern "C" {

// xyzt: n records of stride_floats floats, x y z first and the time at float time_col; out: n x 3
void orc_undistort_points(const float* xyzt, size_t n, size_t stride_floats, size_t time_col, const double pose[7], const double prev_pose[7],
                          double dt, int rotation, float* out) {
    const orc_und::Delta D = orc_und::delta(prev_pose, pose);
    for (size_t i = 0; i < n; ++i) orc_und::point(D, dt, rotation, xyzt + i * stride_floats, xyzt[i * stride_floats + time_col], out + 3 * i);
}

// orc_register_full without the edge branch, pInit in place of the scan at every iteration.  Records: x y z intensity (stride >= 4),
// time at float time_col.
int orc_register_undistort(void* m, const float* scan_xyzi, size_t n, size_t stride_floats, size_t time_col, const double pose_in[7],
                           const double prev_pose[7], double dt, int rotation, const orc_opts* opt, orc_result* out) {
    using namespace orc;
    auto* M = static_cast<Map*>(m);
    std::memset(out, 0, sizeof(*out));
    double T[7], T0[7], last_T[7];
    std::memcpy(T, pose_in, sizeof(T)); std::memcpy(T0, pose_in, sizeof(T)); std::memcpy(last_T, pose_in, sizeof(T));
    std::memcpy(out->pose, T, sizeof(T)); std::memcpy(out->pose_opt, T, sizeof(T));
    out->scan_surf_num = int32_t(n);
    int32_t ijk[3];
    if (!opt->skip_map_checks) orc_map_shift(m, T, ijk);
    else for (int a = 0; a < 3; ++a) ijk[a] = block_coord(T[a] + kHalfBlock, M->origin[a]);
    out->pos_in_localmap[0] = ijk[0]; out->pos_in_localmap[1] = ijk[1]; out->pos_in_localmap[2] = ijk[2];
    out->map_surf_5x5 = orc_map_counts_5x5(m, ijk);
    out->map_edge_5x5 = orc_map_edge_counts_5x5(m, ijk);
    if (!(out->map_surf_5x5 > 50)) { out->status = 1; return 1; }
    const int max_iters = std::min<int>(opt->max_icp_iters, ORC_MAX_ICP_ITERS);
    std::vector<Corr> corr(n);
    std::vector<float> pinit(n * 4);
    Evaluator E; { const double a = double(std::sqrt(3 * opt->plane_res)); E.a2 = a * a; const double al = double(std::sqrt(3 * opt->line_res)); E.a2_line = al * al; }
    bool have_cov = false;
    for (int it = 0; it < max_iters; ++it) {
        const orc_und::Delta D = orc_und::delta(prev_pose, T);                 // the estimate the previous iteration left
        for (size_t i = 0; i < n; ++i) {
            const float* p = scan_xyzi + i * stride_floats;
            orc_und::point(D, dt, rotation, p, p[time_col], &pinit[4 * i]);
            pinit[4 * i + 3] = p[3];
        }
        for (int k = 0; k < 7; ++k) out->hist_reject_line[k] = 0;
        E.edges.clear();
        correspond_all(*M, pinit.data(), n, 4, T, opt->plane_res, opt->max_surface_features, opt->knn_mode, opt->n_threads, corr.data(), out->hist_obs, out->hist_reject_plane);
        E.blocks.clear();
        for (size_t i = 0; i < n; ++i) if (corr[i].status == SUCCESS) E.blocks.push_back(&corr[i]);
        E.prior.on = false;
        double prev[7]; std::memcpy(prev, T, sizeof(T));
        double params[7]; std::memcpy(params, T, sizeof(T));
        SolveSummary S = ceres_solve(E, params, opt->lm_max_iterations);
        std::memcpy(T, params, sizeof(T));
        out->iter_n_surf[it] = int32_t(E.blocks.size()); out->iter_n_edge[it] = 0;
        rel_motion(prev, T, &out->iter_dtrans[it], &out->iter_drot[it]);
        out->iter_lm_steps[it] = S.iterations; out->iter_lm_successful[it] = S.num_successful_steps; out->iter_lm_termination[it] = S.termination; out->iter_cost[it] = S.final_cost;
        out->n_iterations = it + 1;
        if (S.num_successful_steps == 1 || it == max_iters - 1) {
            if (!E.blocks.empty()) { ceres_covariance(E, T, out->cov); have_cov = true; }
            break;
        }
    }
    if (have_cov) {
        double P[9], O[9], w[3], V[9];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { P[i * 3 + j] = out->cov[i * 6 + j]; O[i * 3 + j] = out->cov[(i + 3) * 6 + (j + 3)]; }
        sym_eig(3, P, w, V);
        out->pos_err = std::sqrt(w[2]); out->pos_dir[0] = V[2]; out->pos_dir[1] = V[5]; out->pos_dir[2] = V[8];
        out->pos_inv_cond = std::sqrt(w[0]) / std::sqrt(w[2]);
        sym_eig(3, O, w, V);
        out->ori_err_deg = std::sqrt(w[2]) / M_PI * 180.; out->ori_dir[0] = V[2]; out->ori_dir[1] = V[5]; out->ori_dir[2] = V[8];
        out->ori_inv_cond = std::sqrt(w[0]) / std::sqrt(w[2]);
    } else if (out->n_iterations > 0 && out->iter_n_surf[out->n_iterations - 1] == 0) out->status = 2;
    std::memcpy(out->pose_opt, T, sizeof(T));
    manual_yaw_correction(last_T, T, double(opt->yaw_ratio));
    rel_motion(T0, T, &out->total_translation, &out->total_rotation);
    rel_motion(last_T, T, &out->translation_from_last, &out->rotation_from_last);
    std::memcpy(out->pose, T, sizeof(T));
    return out->status;
}

}  // extern "C"

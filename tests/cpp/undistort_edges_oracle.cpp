// CPU oracle for within-scan motion compensation with an edge cloud (so_register_undistort_edges): undistort_oracle.cpp (the oracle's
// translation unit, unchanged, and the pInit restatement) plus
//   orc_register_undistort_edges  orc_register_full's ICP loop with pInit, recomputed from the CURRENT estimate at the start of every
//                                 ICP iteration, in place of BOTH the surf and the edge cloud (no pose prior, as so_register_undistort)
// Built by tests/undistort_edges_oracle.py with the oracle's flags.
#include "undistort_oracle.cpp"

extern "C" {

// Records of both clouds: x y z intensity (stride >= 4), time at float time_col.
int orc_register_undistort_edges(void* m, const float* scan_xyzi, size_t n, const float* edge_xyzi, size_t n_edge, size_t stride_floats,
                                 size_t time_col, const double pose_in[7], const double prev_pose[7], double dt, int rotation,
                                 const orc_opts* opt, orc_result* out) {
    using namespace orc;
    auto* M = static_cast<Map*>(m);
    std::memset(out, 0, sizeof(*out));
    double T[7], T0[7], last_T[7];
    std::memcpy(T, pose_in, sizeof(T)); std::memcpy(T0, pose_in, sizeof(T)); std::memcpy(last_T, pose_in, sizeof(T));
    std::memcpy(out->pose, T, sizeof(T)); std::memcpy(out->pose_opt, T, sizeof(T));
    out->scan_surf_num = int32_t(n); out->scan_edge_num = int32_t(n_edge);
    int32_t ijk[3];
    if (!opt->skip_map_checks) orc_map_shift(m, T, ijk);
    else for (int a = 0; a < 3; ++a) ijk[a] = block_coord(T[a] + kHalfBlock, M->origin[a]);
    out->pos_in_localmap[0] = ijk[0]; out->pos_in_localmap[1] = ijk[1]; out->pos_in_localmap[2] = ijk[2];
    out->map_surf_5x5 = orc_map_counts_5x5(m, ijk);
    out->map_edge_5x5 = orc_map_edge_counts_5x5(m, ijk);
    if (!(out->map_surf_5x5 > 50)) { out->status = 1; return 1; }
    const int max_iters = std::min<int>(opt->max_icp_iters, ORC_MAX_ICP_ITERS);
    std::vector<Corr> corr(n);
    std::vector<EdgeCorr> ecorr(n_edge);
    std::vector<float> pinit(n * 4), pinit_e(n_edge * 4);
    Evaluator E; { const double a = double(std::sqrt(3 * opt->plane_res)); E.a2 = a * a; const double al = double(std::sqrt(3 * opt->line_res)); E.a2_line = al * al; }
    bool have_cov = false;
    auto warp = [&](const orc_und::Delta& D, const float* src, size_t cnt, float* dst) {
        for (size_t i = 0; i < cnt; ++i) {
            const float* p = src + i * stride_floats;
            orc_und::point(D, dt, rotation, p, p[time_col], &dst[4 * i]);
            dst[4 * i + 3] = p[3];
        }
    };
    for (int it = 0; it < max_iters; ++it) {
        const orc_und::Delta D = orc_und::delta(prev_pose, T);                 // the estimate the previous iteration left
        warp(D, scan_xyzi, n, pinit.data());
        warp(D, edge_xyzi, n_edge, pinit_e.data());
        for (int k = 0; k < 7; ++k) out->hist_reject_line[k] = 0;
        E.edges.clear();
        for (size_t i = 0; i < n_edge; ++i) {
            line_correspondence(*M, &pinit_e[4 * i], T, opt->line_res, opt->knn_mode == 1 ? 1 : 0, ecorr[i]);
            out->hist_reject_line[ecorr[i].status]++;
            if (ecorr[i].status == SUCCESS) E.edges.push_back(&ecorr[i]);
        }
        correspond_all(*M, pinit.data(), n, 4, T, opt->plane_res, opt->max_surface_features, opt->knn_mode, opt->n_threads, corr.data(), out->hist_obs, out->hist_reject_plane);
        E.blocks.clear();
        for (size_t i = 0; i < n; ++i) if (corr[i].status == SUCCESS) E.blocks.push_back(&corr[i]);
        E.prior.on = false;
        double prev[7]; std::memcpy(prev, T, sizeof(T));
        double params[7]; std::memcpy(params, T, sizeof(T));
        SolveSummary S = ceres_solve(E, params, opt->lm_max_iterations);
        std::memcpy(T, params, sizeof(T));
        out->iter_n_surf[it] = int32_t(E.blocks.size()); out->iter_n_edge[it] = int32_t(E.edges.size());
        rel_motion(prev, T, &out->iter_dtrans[it], &out->iter_drot[it]);
        out->iter_lm_steps[it] = S.iterations; out->iter_lm_successful[it] = S.num_successful_steps; out->iter_lm_termination[it] = S.termination; out->iter_cost[it] = S.final_cost;
        out->n_iterations = it + 1;
        if (S.termination == 7) {                                 // SO_STATUS_INVALID_EVALUATION: no step, no covariance
            out->iter_lm_steps[it] = out->iter_lm_successful[it] = out->iter_lm_termination[it] = 0;
            out->status = 3;
            break;
        }
        if (S.num_successful_steps == 1 || it == max_iters - 1) {
            if (!E.blocks.empty() || !E.edges.empty()) { ceres_covariance(E, T, out->cov); have_cov = true; }
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
    } else if (out->n_iterations > 0 && out->iter_n_surf[out->n_iterations - 1] == 0 && out->iter_n_edge[out->n_iterations - 1] == 0) out->status = 2;
    std::memcpy(out->pose_opt, T, sizeof(T));
    manual_yaw_correction(last_T, T, double(opt->yaw_ratio));
    rel_motion(T0, T, &out->total_translation, &out->total_rotation);
    rel_motion(last_T, T, &out->translation_from_last, &out->rotation_from_last);
    std::memcpy(out->pose, T, sizeof(T));
    return out->status;
}

}  // extern "C"

// tools/integration_stub.cpp -- the reference-side binding of INTEGRATION.md as compilable C++ (C++14, like the reference).
// tests/test_abi.py compiles it (syntax + types only) against include/cerberus_b200.h, the header shims of oracle/shim that stand in
// for Eigen / Ceres / ROS / OpenCV, and the reference's interface it reads: tests/seam declares those members (pinned to the
// reference's feature_manager.h, imu_leg_integration_base.h, marginalization_factor.h and parameters.h by tests/golden/seam_v1.json);
// with a Cerberus checkout the reference's own headers can be used instead:
//     g++ -std=c++14 -fsyntax-only -Iinclude -Ioracle/shim -I$CERBERUS_SRC tools/integration_stub.cpp
// `EstimatorSeam` lists the members of class Estimator (src/estimator/estimator.h:134-241) that optimization() touches at the seam;
// estimator.h itself drags in the ROS node, the feature tracker and OpenCV.
#include <cstring>
#include <vector>
#include "cerberus_b200.h"
#include "utils/parameters.h"
#include "featureTracker/feature_manager.h"
#include "factor/imu_leg_integration_base.h"
#include "factor/marginalization_factor.h"

struct EstimatorSeam {
    double para_Pose[WINDOW_SIZE + 1][SIZE_POSE];                 // estimator.h:189-196
    double para_SpeedBias[WINDOW_SIZE + 1][SIZE_SPEEDBIAS];
    double para_LegBias[WINDOW_SIZE + 1][SIZE_LEG_BIAS];
    double para_Feature[NUM_OF_F][SIZE_FEATURE];
    double para_Ex_Pose[2][SIZE_POSE];
    double para_Td[1][1];
    FeatureManager *f_manager;                                    // estimator.h: FeatureManager f_manager
    IMULegIntegrationBase *il_pre_integrations[WINDOW_SIZE + 1];
    MarginalizationInfo *last_marginalization_info;
    std::vector<double *> last_marginalization_parameter_blocks;
    Eigen::Vector3d Vs[WINDOW_SIZE + 1];
    int frame_count;
    bool openExEstimation;
    // added by the binding
    CerbHandle *gpu_backend;
    std::vector<CerbFeature> gpu_features; std::vector<CerbObservation> gpu_obs;
    CerbIMULegPreint gpu_preint[WINDOW_SIZE];
};

// setParameter(): one handle for the life of the estimator (replaces building a ceres::Problem every frame, estimator.cpp:1059-1113)
int cerb_binding_create(EstimatorSeam &e) {
    CerbSolverConfig cfg; cerb_default_config(&cfg);
    cfg.max_batch = 1; cfg.max_features = NUM_OF_F; cfg.max_obs = NUM_OF_F * (WINDOW_SIZE + 1);
    cfg.max_num_iterations = NUM_ITERATIONS; cfg.optimize_leg_bias = OPTIMIZE_LEG_BIAS;
    cfg.g[0] = G.x(); cfg.g[1] = G.y(); cfg.g[2] = G.z(); cfg.visual_sqrt_info = FOCAL_LENGTH / 1.5;
    return cerb_create(&cfg, &e.gpu_backend);                     // != CERB_OK: no device -- there is no CPU fallback by design
}

// which para_* array a kept parameter block of the prior points into (the reference identifies blocks by address, estimator.cpp:1357-1372)
static bool classify(const EstimatorSeam &e, const double *addr, int32_t *kind, int32_t *index) {
    for (int i = 0; i <= WINDOW_SIZE; i++) {
        if (addr == e.para_Pose[i]) { *kind = CERB_BLOCK_POSE; *index = i; return true; }
        if (addr == e.para_SpeedBias[i]) { *kind = CERB_BLOCK_SPEEDBIAS; *index = i; return true; }
        if (addr == e.para_LegBias[i]) { *kind = CERB_BLOCK_LEGBIAS; *index = i; return true; }
    }
    for (int c = 0; c < 2; c++) if (addr == e.para_Ex_Pose[c]) { *kind = CERB_BLOCK_EX_POSE; *index = c; return true; }
    if (addr == e.para_Td[0]) { *kind = CERB_BLOCK_TD; *index = 0; return true; }
    return false;
}

// the body of Estimator::optimization() between vector2double() (estimator.cpp:1057) and double2vector() (:1241)
int cerb_binding_optimization(EstimatorSeam &e, CerbSolveReport *rep) {
    CerbWindowDesc d; std::memset(&d, 0, sizeof(d));
    // (a) features: the same walk as estimator.cpp:1173-1216
    e.gpu_features.clear(); e.gpu_obs.clear();
    for (auto &it_per_id : e.f_manager->feature) {
        it_per_id.used_num = it_per_id.feature_per_frame.size();
        if (it_per_id.used_num < 4) continue;
        CerbFeature f; f.start_frame = it_per_id.start_frame; f.n_obs = (int)it_per_id.feature_per_frame.size(); f.obs_offset = (int)e.gpu_obs.size(); f.reserved = 0;
        for (auto &o : it_per_id.feature_per_frame) {
            CerbObservation q; std::memset(&q, 0, sizeof(q));
            q.point[0] = o.point.x(); q.point[1] = o.point.y(); q.velocity[0] = o.velocity.x(); q.velocity[1] = o.velocity.y();
            q.pointRight[0] = o.pointRight.x(); q.pointRight[1] = o.pointRight.y(); q.velocityRight[0] = o.velocityRight.x(); q.velocityRight[1] = o.velocityRight.y();
            q.cur_td = o.cur_td; q.is_stereo = o.is_stereo ? 1 : 0;
            e.gpu_obs.push_back(q);
        }
        e.gpu_features.push_back(f);
    }
    // (b) preintegration: the public members of il_pre_integrations[i + 1] (imu_leg_integration_base.h:73-85); Eigen storage is column-major, as the ABI expects
    for (int i = 0; i < WINDOW_SIZE; i++) {
        IMULegIntegrationBase *p = e.il_pre_integrations[i + 1]; CerbIMULegPreint &q = e.gpu_preint[i];
        q.sum_dt = p->sum_dt;
        for (int k = 0; k < 3; k++) { q.delta_p[k] = p->delta_p(k); q.delta_v[k] = p->delta_v(k); q.linearized_ba[k] = p->linearized_ba(k); q.linearized_bg[k] = p->linearized_bg(k); }
        q.delta_q[0] = p->delta_q.x(); q.delta_q[1] = p->delta_q.y(); q.delta_q[2] = p->delta_q.z(); q.delta_q[3] = p->delta_q.w();
        for (int l = 0; l < NUM_OF_LEG; l++) for (int k = 0; k < 3; k++) q.delta_epsilon[3 * l + k] = p->delta_epsilon[l](k);
        for (int l = 0; l < NUM_OF_LEG; l++) q.linearized_rho[l] = p->linearized_rho(l);
        std::memcpy(q.jacobian, p->jacobian.data(), sizeof(q.jacobian));
        std::memcpy(q.covariance, p->covariance.data(), sizeof(q.covariance));
    }
    // (c) prior: what MarginalizationFactor::Evaluate reads (marginalization_factor.cpp:347-395)
    if (e.last_marginalization_info && e.last_marginalization_info->valid) {
        MarginalizationInfo *mi = e.last_marginalization_info; CerbPrior &pr = d.prior;
        pr.valid = 1; pr.n = mi->n; pr.num_blocks = (int32_t)mi->keep_block_size.size();
        for (int b = 0; b < pr.num_blocks; b++) {
            if (!classify(e, e.last_marginalization_parameter_blocks[b], &pr.block_kind[b], &pr.block_index[b])) return CERB_ERR_BAD_ARGUMENT;
            pr.block_col[b] = mi->keep_block_idx[b] - mi->m;
            std::memcpy(pr.block_x0[b], mi->keep_block_data[b], sizeof(double) * mi->keep_block_size[b]);
        }
        pr.linearized_jacobians = mi->linearized_jacobians.data(); pr.linearized_residuals = mi->linearized_residuals.data();
    }
    d.n_features = (int32_t)e.gpu_features.size(); d.n_obs = (int32_t)e.gpu_obs.size(); d.features = e.gpu_features.data(); d.obs = e.gpu_obs.data();
    d.preint = e.gpu_preint;
    if (ESTIMATE_EXTRINSIC && e.frame_count == WINDOW_SIZE && e.Vs[0].norm() > 0.2) e.openExEstimation = true;      // estimator.cpp:1091-1100
    d.extrinsic_open = (ESTIMATE_EXTRINSIC && e.openExEstimation) ? 1 : 0;
    d.td_open = (ESTIMATE_TD && e.Vs[0].norm() >= 0.2) ? 1 : 0;                                                       // estimator.cpp:1104
    // (d) the para_* arrays are laid out like CerbWindowState's (estimator.h:189-196): five memcpys in, five out
    CerbWindowState s; std::memset(&s, 0, sizeof(s));
    std::memcpy(s.para_Pose, e.para_Pose, sizeof(s.para_Pose)); std::memcpy(s.para_SpeedBias, e.para_SpeedBias, sizeof(s.para_SpeedBias));
    std::memcpy(s.para_LegBias, e.para_LegBias, sizeof(s.para_LegBias)); std::memcpy(s.para_Ex_Pose, e.para_Ex_Pose, sizeof(s.para_Ex_Pose));
    s.para_Td[0] = e.para_Td[0][0]; s.para_Feature = &e.para_Feature[0][0];
    const int rc = cerb_solve_window(e.gpu_backend, &d, &s, rep);
    if (rc != CERB_OK && rc != CERB_ERR_NON_FINITE) return rc;                                                         // cerb_last_error() has the text
    std::memcpy(e.para_Pose, s.para_Pose, sizeof(s.para_Pose)); std::memcpy(e.para_SpeedBias, s.para_SpeedBias, sizeof(s.para_SpeedBias));
    std::memcpy(e.para_LegBias, s.para_LegBias, sizeof(s.para_LegBias)); std::memcpy(e.para_Ex_Pose, s.para_Ex_Pose, sizeof(s.para_Ex_Pose));
    e.para_Td[0][0] = s.para_Td[0];
    return rc;
}

// the marginalization half (estimator.cpp:1247-1456) on the window that was just solved: call after double2vector() + vector2double()
// (the states the reference re-packs at :1251 / :1384); the result is the prior of the NEXT window (block indices already shifted).
int cerb_binding_marginalize(EstimatorSeam &e, int marginalization_flag /* MARGIN_OLD = 0, MARGIN_SECOND_NEW = 1 */, CerbPrior *next_prior /* matrix / vector storage set by the caller */) {
    CerbWindowState s; std::memset(&s, 0, sizeof(s));
    std::memcpy(s.para_Pose, e.para_Pose, sizeof(s.para_Pose)); std::memcpy(s.para_SpeedBias, e.para_SpeedBias, sizeof(s.para_SpeedBias));
    std::memcpy(s.para_LegBias, e.para_LegBias, sizeof(s.para_LegBias)); std::memcpy(s.para_Ex_Pose, e.para_Ex_Pose, sizeof(s.para_Ex_Pose));
    s.para_Td[0] = e.para_Td[0][0]; s.para_Feature = &e.para_Feature[0][0];
    const int32_t flag = marginalization_flag;
    return cerb_batch_marginalize(e.gpu_backend, &flag, &s, next_prior, nullptr);
}

// ---- resident variant: the window stays on the device across frames (cerb_resident_*), the estimator sends each frame's edits ---------------
// Set up once after cerb_binding_create with cerb_resident_start(e.gpu_backend, 1, 1).  The binding then mirrors what FeatureManager does to
// feature_per_frame: a cerb_resident_put_observations record per push_back in addFeatureCheckParallax (feature_manager.cpp:93-113), a
// cerb_resident_edit_tracks record per erase in removeBackShiftDepth / removeBack / removeFront (:450-529), and preintegrates the new
// interval into the slot of the one slideWindow dropped (cerb_resident_preintegrate).  `slot_of[k]` is the track slot the binding gave the k-th
// entry of f_manager.feature; `pre_slots[i]` is the slot of il_pre_integrations[i + 1].
int cerb_binding_optimization_resident(EstimatorSeam &e, const std::vector<int> &slot_of, const int32_t pre_slots[WINDOW_SIZE], CerbSolveReport *rep) {
    CerbWindowDesc d; std::memset(&d, 0, sizeof(d));
    e.gpu_features.clear();
    size_t k = 0;
    for (auto &it_per_id : e.f_manager->feature) {                    // the walk of estimator.cpp:1173-1216: only the track list travels
        const size_t at = k++;
        it_per_id.used_num = it_per_id.feature_per_frame.size();
        if (it_per_id.used_num < 4) continue;
        if (at >= slot_of.size() || slot_of[at] < 0) return CERB_ERR_BAD_ARGUMENT;
        const int slot = slot_of[at];
        CerbFeature f; f.start_frame = it_per_id.start_frame; f.n_obs = (int)it_per_id.feature_per_frame.size(); f.obs_offset = slot * CERB_NUM_FRAMES; f.reserved = 0;
        e.gpu_features.push_back(f);
    }
    d.n_features = (int32_t)e.gpu_features.size(); d.features = e.gpu_features.data();
    if (ESTIMATE_EXTRINSIC && e.frame_count == WINDOW_SIZE && e.Vs[0].norm() > 0.2) e.openExEstimation = true;
    d.extrinsic_open = (ESTIMATE_EXTRINSIC && e.openExEstimation) ? 1 : 0;
    d.td_open = (ESTIMATE_TD && e.Vs[0].norm() >= 0.2) ? 1 : 0;
    CerbWindowState s; std::memset(&s, 0, sizeof(s));
    std::memcpy(s.para_Pose, e.para_Pose, sizeof(s.para_Pose)); std::memcpy(s.para_SpeedBias, e.para_SpeedBias, sizeof(s.para_SpeedBias));
    std::memcpy(s.para_LegBias, e.para_LegBias, sizeof(s.para_LegBias)); std::memcpy(s.para_Ex_Pose, e.para_Ex_Pose, sizeof(s.para_Ex_Pose));
    s.para_Td[0] = e.para_Td[0][0]; s.para_Feature = &e.para_Feature[0][0];
    int rc = cerb_resident_upload(e.gpu_backend, 1, &d, &s, pre_slots); if (rc != CERB_OK) return rc;
    rc = cerb_batch_solve_resident(e.gpu_backend); if (rc != CERB_OK) return rc;
    rc = cerb_batch_download(e.gpu_backend, &s, rep);
    if (rc != CERB_OK && rc != CERB_ERR_NON_FINITE) return rc;
    std::memcpy(e.para_Pose, s.para_Pose, sizeof(s.para_Pose)); std::memcpy(e.para_SpeedBias, s.para_SpeedBias, sizeof(s.para_SpeedBias));
    std::memcpy(e.para_LegBias, s.para_LegBias, sizeof(s.para_LegBias)); std::memcpy(e.para_Ex_Pose, s.para_Ex_Pose, sizeof(s.para_Ex_Pose));
    e.para_Td[0][0] = s.para_Td[0];
    return rc;
}

// cerb_binding_marginalize with the new prior left on the device as the prior of the next cerb_resident_upload: nothing but *prior_valid returns
int cerb_binding_marginalize_resident(EstimatorSeam &e, int marginalization_flag, int32_t *prior_valid) {
    CerbWindowState s; std::memset(&s, 0, sizeof(s));
    std::memcpy(s.para_Pose, e.para_Pose, sizeof(s.para_Pose)); std::memcpy(s.para_SpeedBias, e.para_SpeedBias, sizeof(s.para_SpeedBias));
    std::memcpy(s.para_LegBias, e.para_LegBias, sizeof(s.para_LegBias)); std::memcpy(s.para_Ex_Pose, e.para_Ex_Pose, sizeof(s.para_Ex_Pose));
    s.para_Td[0] = e.para_Td[0][0]; s.para_Feature = &e.para_Feature[0][0];
    const int32_t flag = marginalization_flag;
    return cerb_resident_marginalize(e.gpu_backend, &flag, &s, prior_valid);
}

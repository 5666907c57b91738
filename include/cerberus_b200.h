/*
 * cerberus_b200.h -- C ABI of the B200-native sliding-window VILO backend.
 *
 * This is the drop-in boundary for ONE path of ShuoYangRobotics/Cerberus: the body of
 * Estimator::optimization() between vector2double() and double2vector()
 * (reference src/estimator/estimator.cpp:1057-1241), i.e. "build the Ceres problem over the
 * 11-frame window and run <= NUM_ITERATIONS DENSE_SCHUR/DOGLEG iterations", plus the factor
 * families it evaluates (the files of src/factor) and the leg-contact preintegration that feeds it
 * (src/factor/imu_leg_integration_base.cpp, src/legKinematics/A1Kinematics.cpp).
 *
 * The reference has no FFI for this path (everything is one C++ process linking Ceres), so the
 * seam is cut here.  Every struct mirrors, field by field, the data the reference holds at that
 * seam; the citation next to each field is the reference member it binds to.  Plain pointers and
 * sizes only; no C++ / torch types.  All floating point is fp64 like the reference.
 *
 * Conventions fixed by the reference (kept bit-for-bit in layout):
 *   pose block        = [px,py,pz,qx,qy,qz,qw]                 estimator.cpp:852-859
 *   speed-bias block  = [v(3), ba(3), bg(3)]                   estimator.cpp:863-873
 *   leg-bias block    = [rho1..rho4]                           estimator.cpp:877-880
 *   feature           = inverse depth of the anchor observation feature_manager.cpp:189
 *   Eigen dense matrices handed over as-is are COLUMN-major (Eigen default).
 *   Jacobians returned by the cerb_eval_* entry points are ROW-major rows x global_size with the
 *   7th column of every pose block zero, exactly like ceres::CostFunction::Evaluate.
 *
 * Error model: every entry point returns an int status (CERB_OK == 0); nothing throws across the
 * ABI.  cerb_last_error() returns a thread-local human readable string for the last failure.
 * Threading: one CerbHandle per calling thread (the reference calls optimization() from a single
 * thread, processThread, under mProcess: estimator.cpp:497-498).
 */
#ifndef CERBERUS_B200_H
#define CERBERUS_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- compile-time sizes (reference src/utils/parameters.h:22-24,93-102) ------------------- */
#define CERB_WINDOW_SIZE 10        /* WINDOW_SIZE */
#define CERB_NUM_FRAMES 11         /* WINDOW_SIZE + 1 states */
#define CERB_NUM_OF_F 1000         /* NUM_OF_F: para_Feature capacity of the reference */
#define CERB_MAX_FEATURES 2048     /* capacity limit of this library: the synthetic stress configuration (BASELINE.json configs[4]: 2000
                                      features per window) deliberately exceeds the reference's static limit (parameters.h:24) */
#define CERB_SIZE_POSE 7
#define CERB_SIZE_SPEEDBIAS 9
#define CERB_SIZE_LEG_BIAS 4
#define CERB_NUM_LEG 4
#define CERB_NUM_DOF 12
#define CERB_IL_RES 31             /* RESIDUAL_STATE_SIZE */
#define CERB_IL_NOISE 46           /* NOISE_SIZE */
#define CERB_MAX_PRIOR_BLOCKS 16   /* pose0..9, speedbias0, legbias0, ex0, ex1, td = 15 */
#define CERB_MAX_PRIOR_DIM 96      /* n <= 60+9+4+12+1 = 86 */

/* ---- status codes ------------------------------------------------------------------------- */
enum {
    CERB_OK = 0,
    CERB_ERR_BAD_ARGUMENT = 1,   /* null pointer, size over capacity, malformed descriptor */
    CERB_ERR_NO_DEVICE = 2,      /* CUDA device / driver missing: the product has NO CPU fallback */
    CERB_ERR_CUDA = 3,           /* a CUDA runtime call failed */
    CERB_ERR_NON_FINITE = 4      /* a window produced a non-finite cost (reported per window too) */
};

/* CerbSolveReport.termination: what ceres::Solver::Summary::termination_type would say. */
enum {
    CERB_TERM_CONVERGENCE = 0,   /* gradient / parameter / function tolerance reached */
    CERB_TERM_NO_CONVERGENCE = 1,/* max_num_iterations reached */
    CERB_TERM_FAILURE = 2        /* too many consecutive invalid steps / non-finite */
};

/* Kinds of parameter block a marginalization prior can keep (estimator.cpp:1253-1348). */
enum {
    CERB_BLOCK_POSE = 0,        /* para_Pose[index]       size 7 (local 6) */
    CERB_BLOCK_SPEEDBIAS = 1,   /* para_SpeedBias[index]  size 9 */
    CERB_BLOCK_LEGBIAS = 2,     /* para_LegBias[index]    size 4 */
    CERB_BLOCK_EX_POSE = 3,     /* para_Ex_Pose[index]    size 7 (local 6) */
    CERB_BLOCK_TD = 4           /* para_Td[0]             size 1 */
};

/* Projection factor families (src/factor/projection*Factor.h). */
enum {
    CERB_PROJ_TWO_FRAME_ONE_CAM = 0, /* ProjectionTwoFrameOneCamFactor <2,7,7,7,1,1>   */
    CERB_PROJ_TWO_FRAME_TWO_CAM = 1, /* ProjectionTwoFrameTwoCamFactor <2,7,7,7,7,1,1> */
    CERB_PROJ_ONE_FRAME_TWO_CAM = 2  /* ProjectionOneFrameTwoCamFactor <2,7,7,1,1>     */
};

/* ---- solver configuration ------------------------------------------------------------------
 * Globals of the reference that parameterise optimization() (src/utils/parameters.h:27-89,
 * values from config/a1_config/hardware_a1_vilo_config.yaml) + the Ceres 1.14 options the
 * reference leaves at their defaults (estimator.cpp:1221-1236). */
typedef struct CerbSolverConfig {
    int32_t device;               /* CUDA device ordinal */
    int32_t max_batch;            /* capacity: windows per batch call */
    int32_t max_features;         /* capacity: features per window (<= CERB_MAX_FEATURES; the reference stops at CERB_NUM_OF_F) */
    int32_t max_obs;              /* capacity: observations per window (sum of track lengths) */
    int32_t max_num_iterations;   /* NUM_ITERATIONS (yaml max_num_iterations, 12) */
    int32_t optimize_leg_bias;    /* OPTIMIZE_LEG_BIAS; 0 => para_LegBias constant (estimator.cpp:1074) */
    double g[3];                  /* G = (0,0,g_norm)  parameters.cpp:21,130 */
    double visual_sqrt_info;      /* FOCAL_LENGTH/1.5 = 460/1.5, sqrt_info = this * I2 (estimator.cpp:124) */
    double huber_delta;           /* ceres::HuberLoss(1.0) (estimator.cpp:1062) */
    /* ceres::Solver::Options defaults of Ceres 1.14.0 (not overridden by the reference) */
    double initial_trust_region_radius; /* 1e4  */
    double max_trust_region_radius;     /* 1e16 */
    double min_trust_region_radius;     /* 1e-32 */
    double min_relative_decrease;       /* 1e-3 */
    double function_tolerance;          /* 1e-6 */
    double gradient_tolerance;          /* 1e-10 */
    double parameter_tolerance;         /* 1e-8 */
} CerbSolverConfig;

/* ---- leg-contact preintegration result: IMULegIntegrationBase public members
 * (src/factor/imu_leg_integration_base.h:73-85) consumed by IMULegFactor::Evaluate. */
typedef struct CerbIMULegPreint {
    double sum_dt;                 /* sum_dt; factor skipped if > 10.0 (estimator.cpp:1119) */
    double delta_p[3];             /* delta_p  (alpha) */
    double delta_q[4];             /* delta_q  (gamma), Eigen coeffs order x,y,z,w */
    double delta_v[3];             /* delta_v  (beta)  */
    double delta_epsilon[12];      /* delta_epsilon[leg][3] */
    double linearized_ba[3];
    double linearized_bg[3];
    double linearized_rho[4];
    double jacobian[CERB_IL_RES * CERB_IL_RES];   /* jacobian,   31x31 column-major */
    double covariance[CERB_IL_RES * CERB_IL_RES]; /* covariance, 31x31 column-major (symmetric) */
} CerbIMULegPreint;

/* ---- plain IMU preintegration result: IntegrationBase public members (src/factor/integration_base.h:200-213)
 * consumed by IMUFactor::Evaluate (src/factor/imu_factor.h:28-188); used when USE_LEG == 0 (estimator.cpp:1160-1171).
 * Error-state order O_P 0, O_R 3, O_V 6, O_BA 9, O_BG 12 (parameters.h:119-126). */
typedef struct CerbIMUPreint {
    double sum_dt;
    double delta_p[3];
    double delta_q[4];             /* x,y,z,w */
    double delta_v[3];
    double linearized_ba[3];
    double linearized_bg[3];
    double jacobian[15 * 15];      /* column-major */
    double covariance[15 * 15];    /* column-major (symmetric) */
} CerbIMUPreint;

/* ---- one observation of a feature: FeaturePerFrame (src/featureTracker/feature_manager.h:28-59) */
typedef struct CerbObservation {
    double point[2];        /* point.x, point.y      (z == 1) */
    double velocity[2];     /* velocity              */
    double pointRight[2];   /* pointRight.x, .y      (valid iff is_stereo) */
    double velocityRight[2];
    double cur_td;          /* cur_td */
    int32_t is_stereo;      /* is_stereo */
    int32_t reserved;
} CerbObservation;

/* ---- one tracked feature: FeaturePerId (feature_manager.h:61-81), only those with
 * used_num >= 4 are passed (estimator.cpp:1178); index in the array == feature_index. */
typedef struct CerbFeature {
    int32_t start_frame;    /* start_frame = anchor frame imu_i */
    int32_t n_obs;          /* feature_per_frame.size(); frames start_frame .. start_frame+n_obs-1 */
    int32_t obs_offset;     /* first CerbObservation of this feature in CerbWindowDesc.obs */
    int32_t reserved;
} CerbFeature;

/* ---- marginalization prior: MarginalizationInfo members read by MarginalizationFactor::Evaluate
 * (src/factor/marginalization_factor.cpp:347-395) + last_marginalization_parameter_blocks. */
typedef struct CerbPrior {
    int32_t valid;                                /* last_marginalization_info && ->valid */
    int32_t n;                                    /* MarginalizationInfo::n */
    int32_t num_blocks;                           /* keep_block_size.size() */
    int32_t reserved;
    int32_t block_kind[CERB_MAX_PRIOR_BLOCKS];    /* which para_* array the kept block address maps to */
    int32_t block_index[CERB_MAX_PRIOR_BLOCKS];   /* index into that array */
    int32_t block_col[CERB_MAX_PRIOR_BLOCKS];     /* keep_block_idx[i] - m */
    double block_x0[CERB_MAX_PRIOR_BLOCKS][9];    /* keep_block_data[i] (global size <= 9, unused tail 0) */
    const double *linearized_jacobians;           /* n x n, column-major (Eigen::MatrixXd) */
    const double *linearized_residuals;           /* n */
} CerbPrior;

/* ---- everything optimization() reads besides the para_* arrays */
typedef struct CerbWindowDesc {
    int32_t n_features;
    int32_t n_obs;
    const CerbFeature *features;          /* [n_features] */
    const CerbObservation *obs;           /* [n_obs] */
    const CerbIMULegPreint *preint;       /* [CERB_WINDOW_SIZE]; preint[i] = il_pre_integrations[i+1] (frames i -> i+1); USE_LEG == 1 */
    const CerbIMUPreint *imu_preint;      /* [CERB_WINDOW_SIZE]; pre_integrations[i+1]; used iff preint == NULL (USE_LEG == 0:
                                             IMUFactor instead of IMULegFactor, no leg-bias blocks, estimator.cpp:1160-1171) */
    CerbPrior prior;
    int32_t extrinsic_open;               /* 1 => para_Ex_Pose free (openExEstimation latch, estimator.cpp:1091-1100) */
    int32_t td_open;                      /* 1 => para_Td free (ESTIMATE_TD && |Vs[0]| >= 0.2, estimator.cpp:1104) */
} CerbWindowDesc;

/* ---- the para_* arrays exactly as laid out in estimator.h:189-196; in/out */
typedef struct CerbWindowState {
    double para_Pose[CERB_NUM_FRAMES][CERB_SIZE_POSE];
    double para_SpeedBias[CERB_NUM_FRAMES][CERB_SIZE_SPEEDBIAS];
    double para_LegBias[CERB_NUM_FRAMES][CERB_SIZE_LEG_BIAS];
    double para_Ex_Pose[2][CERB_SIZE_POSE];
    double para_Td[1];
    double reserved;
    double *para_Feature;                 /* [n_features] */
} CerbWindowState;

/* ---- what ceres::Solver::Summary would have said (ignored by the reference, estimator.cpp:1235) */
typedef struct CerbSolveReport {
    int32_t iterations;            /* trust-region iterations performed (successful + unsuccessful) */
    int32_t num_successful_steps;
    int32_t termination;           /* CERB_TERM_* */
    int32_t status;                /* CERB_OK or CERB_ERR_NON_FINITE for this window */
    double initial_cost;
    double final_cost;
} CerbSolveReport;

/* ---- raw IMU + leg sample stream of one inter-frame interval, as pushed through
 * IMULegIntegrationBase::push_back (imu_leg_integration_base.cpp:49-59). */
typedef struct CerbIMULegSample {
    double dt;
    double acc[3];
    double gyr[3];
    double phi[CERB_NUM_DOF];    /* joint angles */
    double dphi[CERB_NUM_DOF];   /* joint velocities */
    double c[CERB_NUM_LEG];      /* contact flags (sensor type 0/1) or foot force (type 2) */
} CerbIMULegSample;

/* Noise / kinematics globals read by IMULegIntegrationBase (parameters.h:59-75, estimator.cpp:140-171). */
typedef struct CerbPreintConfig {
    double acc_n, acc_n_z, gyr_n, acc_w, gyr_w;      /* ACC_N, ACC_N_Z, GYR_N, ACC_W, GYR_W */
    double phi_n, dphi_n;                            /* PHI_N (joint_angle_n), DPHI_N */
    double rho_c_n, rho_nc_n;                        /* RHO_C_N, RHO_NC_N */
    double v_n_min_xy, v_n_min_z, v_n_min, v_n_max;  /* V_N_* */
    double v_n_force_thres_ratio, v_n_term1_steep, v_n_term2_var_rescale, v_n_term3_distance_rescale;
    int32_t contact_sensor_type;                     /* CONTACT_SENSOR_TYPE */
    int32_t reserved;
    double rho_fix[CERB_NUM_LEG][4];                 /* rho_fix_list[leg] = [ox, oy, d, lt] */
    double p_br[3];                                  /* p_br */
    double R_br[9];                                  /* R_br, row-major 3x3 */
} CerbPreintConfig;

/* One interval to preintegrate: constructor arguments (imu_leg_integration_base.cpp:7-47) + samples. */
typedef struct CerbPreintJob {
    double acc_0[3], gyr_0[3];
    double phi_0[CERB_NUM_DOF], dphi_0[CERB_NUM_DOF], c_0[CERB_NUM_LEG];
    double linearized_ba[3], linearized_bg[3], linearized_rho[4];
    int32_t n_samples;
    int32_t reserved;
    const CerbIMULegSample *samples;   /* [n_samples] */
} CerbPreintJob;

typedef struct CerbHandle CerbHandle;

/* ---- lifecycle ---------------------------------------------------------------------------- */
void cerb_default_config(CerbSolverConfig *cfg);            /* A1 yaml + Ceres 1.14 defaults */
void cerb_default_preint_config(CerbPreintConfig *cfg);     /* A1 yaml + A1 geometry */
int cerb_create(const CerbSolverConfig *cfg, CerbHandle **out);
void cerb_destroy(CerbHandle *h);
const char *cerb_last_error(void);
const char *cerb_version(void);

/* ---- the hot path: replaces estimator.cpp:1059-1236 ------------------------------------------
 * Host buffers in, host buffers out (the call a drop-in Estimator::optimization() makes).
 * H2D pack, solve, D2H happen inside; blocking. */
int cerb_solve_window(CerbHandle *h, const CerbWindowDesc *desc, CerbWindowState *state,
                      CerbSolveReport *report);
int cerb_solve_batch(CerbHandle *h, int32_t n, const CerbWindowDesc *descs,
                     CerbWindowState *states, CerbSolveReport *reports);

/* Device-resident variant used for batched replay / benchmarking: upload once, solve many times.
 * cerb_batch_upload packs and copies descriptors + initial states to HBM and keeps a pristine
 * device copy of the initial states; cerb_batch_solve_resident restores the states from that copy
 * and launches the solve on the handle's stream (asynchronous; *kernel_ms, if non-null, receives
 * the CUDA-event time of the previous completed resident solve); cerb_batch_download syncs and
 * copies states/reports back. */
int cerb_batch_upload(CerbHandle *h, int32_t n, const CerbWindowDesc *descs,
                      const CerbWindowState *states);
int cerb_batch_solve_resident(CerbHandle *h);
int cerb_batch_download(CerbHandle *h, CerbWindowState *states, CerbSolveReport *reports);
int cerb_sync(CerbHandle *h);
/* Zero-copy uploads.  The descriptors travel to the device as they are (the AoS -> HBM-layout transpose runs on the device); when a
 * source array lies in memory registered here, cerb_solve_batch / cerb_batch_upload DMA straight out of it (per array ONE 2-D copy per
 * pipeline chunk if the per-window arrays are uniformly strided, like members of one allocation), otherwise it is first copied into the
 * handle's pinned staging by a few host threads.  Register the long-lived buffers of the estimator once (page-locks them:
 * cudaHostRegister); unregister before freeing them.  Registration is an optimisation only: results are identical either way. */
int cerb_register_host_buffer(CerbHandle *h, void *ptr, size_t bytes);
int cerb_unregister_host_buffer(CerbHandle *h, void *ptr);
/* Diagnostics of the last cerb_solve_batch / cerb_batch_upload: DMA operations issued, bytes that went through staging memcpy. */
int cerb_last_upload_stats(CerbHandle *h, int32_t *dma_ops, int64_t *staged_bytes);
/* CUDA-event milliseconds of the last completed solve launch sequence on the handle's stream and
 * the number of kernels it launched. */
int cerb_last_solve_stats(CerbHandle *h, double *kernel_ms, int32_t *kernel_launches);
/* Debug/parity probe: linearisation of window `w` of the resident batch at its CURRENT state (the solved states after a solve, else
 * the uploaded initial ones), exactly what a first solver iteration there sees; read-only with respect to the batch and its reports: cost, gradient (tangent space, order
 * [pose0..10 (66) | ex0, ex1 (12) | speedbias0..10 (99) | legbias0..10 (44) | td (1) | features]),
 * the Schur-reduced 221x221 system is not exposed, only the gradient and diag(J^T J). */
int cerb_debug_linearize(CerbHandle *h, int32_t w, double *cost, double *gradient, double *jtj_diag,
                         int32_t n_alloc);

/* ---- one kernel per factor family: batched Evaluate (replaces the virtual
 * ceres::CostFunction::Evaluate calls; also what marginalization / outlier rejection need).
 * All arrays are host pointers, n factors, tightly packed. Outputs may be NULL to skip. ------- */

/* Projection factors (projectionTwoFrameOneCamFactor.cpp:43-150, ...TwoCam...:43-166,
 * projectionOneFrameTwoCamFactor.cpp:42-134).
 *   kind        CERB_PROJ_*
 *   pose_i/j    [n][7] (ignored for ONE_FRAME_TWO_CAM), ex0/ex1 [n][7] (ex1 ignored for ONE_CAM)
 *   inv_dep, td [n]
 *   pts_i,pts_j [n][3]; vel_i, vel_j [n][2]; td_i, td_j [n]
 *   residuals   [n][2]
 *   jacobians   [n][J] row-major blocks concatenated in the reference's parameter-block order:
 *               ONE_CAM: 2x7,2x7,2x7,2x1,2x1 (J=46); TWO_CAM: 2x7 x4,2x1,2x1 (J=60);
 *               ONE_FRAME: 2x7,2x7,2x1,2x1 (J=32). */
int cerb_eval_projection(CerbHandle *h, int32_t kind, int32_t n, const double *pose_i,
                         const double *pose_j, const double *ex0, const double *ex1,
                         const double *inv_dep, const double *td, const double *pts_i,
                         const double *pts_j, const double *vel_i, const double *vel_j,
                         const double *td_i, const double *td_j, double *residuals,
                         double *jacobians);

/* IMULegFactor::Evaluate (imu_leg_factor.cpp:173-386), <31,7,9,4,7,9,4>.
 *   params [n][40] = pose_i(7) speedbias_i(9) legbias_i(4) pose_j(7) speedbias_j(9) legbias_j(4)
 *   residuals [n][31]; jacobians [n][31*40] row-major blocks 31x7,31x9,31x4,31x7,31x9,31x4;
 *   sqrt_info [n][31*31] row-major (the upper-triangular LLT(cov^-1).matrixL().transpose()). */
int cerb_eval_imu_leg(CerbHandle *h, int32_t n, const CerbIMULegPreint *preint,
                      const double *params, double *residuals, double *jacobians,
                      double *sqrt_info);

/* IMUFactor::Evaluate (imu_factor.h:28-188), <15,7,9,7,9>.
 *   params [n][32] = pose_i(7) speedbias_i(9) pose_j(7) speedbias_j(9); residuals [n][15];
 *   jacobians [n][15*32] row-major blocks 15x7,15x9,15x7,15x9; sqrt_info [n][15*15] row-major. */
int cerb_eval_imu(CerbHandle *h, int32_t n, const CerbIMUPreint *preint, const double *params, double *residuals,
                  double *jacobians, double *sqrt_info);

/* MarginalizationFactor::Evaluate (marginalization_factor.cpp:347-395) for one prior at one state:
 * residuals [n]; jacobians: for each kept block b, n x global_size(b) row-major, concatenated. */
int cerb_eval_prior(CerbHandle *h, const CerbPrior *prior, const CerbWindowState *state,
                    double *residuals, double *jacobians);

/* ---- leg-contact preintegration on device (IMULegIntegrationBase::push_back loop,
 * imu_leg_integration_base.cpp:49-59,88-470): n independent intervals. */
int cerb_preintegrate_batch(CerbHandle *h, const CerbPreintConfig *cfg, int32_t n,
                            const CerbPreintJob *jobs, CerbIMULegPreint *out);

/* Plain IMU preintegration on device (IntegrationBase::push_back loop, integration_base.h:40-170): the jobs use the
 * acc/gyr fields of the samples only; noise = acc_n on all three axes (integration_base.h:31-37). */
int cerb_preintegrate_imu_batch(CerbHandle *h, const CerbPreintConfig *cfg, int32_t n, const CerbPreintJob *jobs,
                                CerbIMUPreint *out);

/* Jobs of several configurations in one launch: job j uses cfgs[cfg_of[j]] (0 <= cfg_of[j] < n_cfg); IMULegIntegrationBase into out[j]
 * where use_leg[cfg_of[j]], IntegrationBase into out_imu[j] otherwise (the other array's entry j is not touched; an array no job writes
 * may be NULL).  Each job's result is the one the single-configuration call above would give it.  cerb_preintegrate_batch and
 * cerb_preintegrate_imu_batch are this call with a one-entry table. */
int cerb_preintegrate_mixed(CerbHandle *h, int32_t n_cfg, const CerbPreintConfig *cfgs, const int32_t *use_leg, int32_t n,
                            const CerbPreintJob *jobs, const int32_t *cfg_of, CerbIMULegPreint *out, CerbIMUPreint *out_imu);

/* A1 leg kinematics (src/legKinematics/A1Kinematics.cpp:7-40), n legs:
 *   q [n][3], rho_opt [n] (lc), rho_fix [n][4];
 *   fk [n][3]; jac [n][9] column-major; dfk_drho [n][3]; dJ_dq [n][27] col-major 9x3; dJ_drho [n][9].
 * Any output may be NULL. */
int cerb_a1_kinematics(CerbHandle *h, int32_t n, const double *q, const double *rho_opt,
                       const double *rho_fix, double *fk, double *jac, double *dfk_drho,
                       double *dJ_dq, double *dJ_drho);

/* ---- per-feature steps either side of the solve, on the RESIDENT batch at its current device state
 * (after cerb_solve_batch / cerb_batch_solve_resident the device holds the solved para_* arrays).
 * Outputs are [n][max_features] in the caller's feature order; entries >= n_features of a window are left untouched. */

/* Estimator::outliersRejection + reprojectionError (estimator.cpp:1729-1798): mean reprojection error of every feature
 * over its observations (camera 0 of the other frames, camera 1 of every stereo observation), depth = 1 / para_Feature.
 * remove (may be NULL) receives the reference's decision ave_err * focal_length > 3 (FOCAL_LENGTH = 460). */
int cerb_batch_outlier_errors(CerbHandle *h, double focal_length, double *ave_err, int32_t *remove);

/* FeatureManager::triangulate + triangulatePoint (feature_manager.cpp:198-212,302-385): estimated_depth of every feature
 * whose para_Feature <= 0 (not triangulated yet): two-view SVD triangulation from the left/right cameras of the anchor
 * frame if that observation is stereo, else from camera 0 of the anchor frame and the next frame; a non-positive result
 * becomes init_depth (INIT_DEPTH = 5.0, parameters.cpp:250).  Features that already have a depth return 1 / para_Feature. */
int cerb_batch_triangulate(CerbHandle *h, double init_depth, double *depth);

/* FeatureManager::removeBackShiftDepth as called by Estimator::slideWindowOld (feature_manager.cpp:450-488, estimator.cpp:1660-1677)
 * when the oldest frame is marginalized: for every feature of the resident batch at its current state, the start_frame after the
 * slide, the estimated_depth after the slide (tracks anchored at frame 0 are re-anchored at the old frame 1; a non-positive depth
 * becomes init_depth) and keep = 0 for the tracks the reference erases (anchored at frame 0 with fewer than 2 remaining observations). */
int cerb_batch_shift_depth(CerbHandle *h, double init_depth, int32_t *new_start_frame, double *depth, int32_t *keep);

/* Replace the states of the RESIDENT batch (n = its size; same windows, same tracks, same order -- only para_* change): what the estimator
 * does between optimization() and outliersRejection() (double2vector() moves the window, estimator.cpp:1241 / :815) without shipping the tracks,
 * preintegrations and priors again.  The per-feature passes and cerb_batch_solve_resident then start from these states. */
int cerb_batch_update_states(CerbHandle *h, int32_t n, const CerbWindowState *states);

/* The dense tail of MarginalizationInfo::marginalize() (marginalization_factor.cpp:281-305), batched: for every window the
 * (m + n) x (m + n) Hessian A = sum J^T J (row-major, the m dropped coordinates first -- the reference's idx order) and b = sum J^T r
 * as ThreadsConstructA (:150-181) leaves them; out: linearized_jacobians [n_windows][n * n] column-major (CerbPrior layout) and
 * linearized_residuals [n_windows][n].  Amm is symmetrised, eigen-decomposed and pseudo-inverted with eigenvalues <= eps dropped
 * (eps = 1e-8 in the reference), the Schur complement is eigen-decomposed from its lower triangle, S / S_inv clamped the same way.
 * sweeps (optional, [n_windows][2]): Jacobi sweeps of the two eigen-decompositions, a convergence diagnostic.
 * 1 <= m <= 19 + CERB_MAX_FEATURES, 1 <= n <= CERB_MAX_PRIOR_DIM. */
int cerb_marginalize_schur(CerbHandle *h, int32_t n_windows, int32_t m, int32_t n, const double *A, const double *b, double eps,
                           double *linearized_jacobians, double *linearized_residuals, int32_t *sweeps);

/* The marginalization half of Estimator::optimization() (estimator.cpp:1247-1456; MarginalizationInfo::{addResidualBlockInfo, preMarginalize,
 * marginalize}, marginalization_factor.cpp:98-333) for every window of the RESIDENT batch (the descriptors of the last cerb_solve_batch /
 * cerb_batch_upload: tracks, preintegrations, old prior), entirely on the device: the factors that touch the dropped blocks are linearised
 * by the solver's own passes (same Huber corrector as ResidualBlockInfo::Evaluate), A = sum J^T J, b = sum J^T r assembled in the
 * reference's [dropped | kept] order and reduced by the eps = 1e-8 clamped eigen Schur complement (see cerb_marginalize_schur).
 *   flags  [n]  0: MARGIN_OLD (drop para_Pose[0], para_SpeedBias[0], para_LegBias[0] and the features anchored at frame 0),
 *               1: MARGIN_SECOND_NEW (drop para_Pose[WINDOW_SIZE - 1] from the old prior; without it the prior is carried over)
 *   states [n]  the para_* arrays to linearise at -- what vector2double() writes after double2vector() (estimator.cpp:1251 / :1384),
 *               para_Feature in the caller's feature order; NULL: the solved states as they sit on the device
 *   priors [n]  out.  On entry linearized_jacobians / linearized_residuals must point at storage for CERB_MAX_PRIOR_DIM^2 / CERB_MAX_PRIOR_DIM
 *               doubles (written: n x n column-major, n); valid / n / blocks / block_x0 are filled with the block indices already shifted
 *               to the next window (addr_shift, estimator.cpp:1357-1372 / :1413-1447), ready to be passed as CerbWindowDesc.prior.
 *   sweeps (optional) [n][2]  Jacobi sweeps of the two eigen-decompositions.
 * Kept-block order: poses ascending, speed bias, leg bias, ex0, ex1, td (the reference's order is that of an unordered_map keyed by pointer). */
int cerb_batch_marginalize(CerbHandle *h, const int32_t *flags, const CerbWindowState *states, CerbPrior *priors, int32_t *sweeps);

/* ---- resident sliding window: the tracks, the preintegrations and the prior of n windows stay in HBM across frames; the host sends edits ------
 * A second way to feed the resident batch, next to cerb_batch_upload.  Between two frames of one robot almost nothing of a window changes
 * (Estimator::processImage -> slideWindow, estimator.cpp:655-846, 1460-1677): one frame of observations arrives, one interval is
 * preintegrated, the prior is replaced by the one the marginalization has just computed.  The host keeps the bookkeeping (feature ids,
 * start_frame, list order, depths, the keyframe test, double2vector); the device keeps the data:
 *   track store     the raw observation array of a window used as max_obs / CERB_NUM_FRAMES fixed slots of CERB_NUM_FRAMES observations;
 *                   a track lives left-aligned in one slot and CerbFeature.obs_offset = slot * CERB_NUM_FRAMES addresses it.  Which slots
 *                   are free is the caller's knowledge.
 *   preintegrations CERB_WINDOW_SIZE slots per window; the resident upload names the slot of every interval i -> i + 1, so a slide is a
 *                   rotation of that table, not a copy
 *   prior           written by cerb_resident_marginalize (or cerb_resident_set_prior) and read by the next cerb_resident_upload
 * Every call validates its arguments before anything is launched (CERB_ERR_BAD_ARGUMENT leaves the store as it was).  cerb_batch_upload and
 * cerb_solve_batch overwrite the store: they end the resident mode of the handle. */
typedef struct CerbTrackPut {          /* FeaturePerId::feature_per_frame.push_back (feature_manager.cpp:93-113) */
    int32_t window, slot, position, reserved;      /* observation `position` (0 = the anchor frame's) of the track in `slot` */
    CerbObservation obs;
} CerbTrackPut;
typedef struct CerbTrackEdit {         /* feature_per_frame.erase(begin() + position): position 0 for removeBackShiftDepth / removeBack
                                          (feature_manager.cpp:450-506), WINDOW_SIZE - 1 - start_frame for removeFront (:508-529) */
    int32_t window, slot, n_obs, position;         /* n_obs: observations the track holds before the edit */
} CerbTrackEdit;
/* Start n resident windows with empty stores, identity slot tables and no prior.  use_leg: the record kind of every window, 1 =
 * CerbIMULegPreint records (USE_LEG == 1), 0 = CerbIMUPreint records. */
int cerb_resident_start(CerbHandle *h, int32_t n, int32_t use_leg);
/* Change the record kind of one window (windows of both kinds may share a batch: a VINS window has no leg-bias block).  Accepted only on an
 * empty window: no observation put since cerb_resident_start (or since the window's extent was reset) and no valid prior.  The window's
 * preintegration slots are zeroed, so no record of the other kind survives. */
int cerb_resident_set_window_kind(CerbHandle *h, int32_t window, int32_t use_leg);
/* Scatter observations into the track stores / apply one erase per listed track (a track may be listed once per call). */
int cerb_resident_put_observations(CerbHandle *h, int32_t count, const CerbTrackPut *puts);
int cerb_resident_edit_tracks(CerbHandle *h, int32_t count, const CerbTrackEdit *edits);
/* cerb_preintegrate_batch / cerb_preintegrate_imu_batch (by the record kind of window windows[j]) with the result of job j left in
 * preintegration slot slots[j] of window windows[j], in the layout an upload of the record would have produced; only sum_dt (optional,
 * [n]) returns to the host.  slideWindowNew's merge of two intervals (estimator.cpp:1576-1616) is one job over both sample buffers. */
int cerb_resident_preintegrate(CerbHandle *h, const CerbPreintConfig *cfg, int32_t n, const CerbPreintJob *jobs, const int32_t *windows,
                               const int32_t *slots, double *sum_dt);
/* cerb_resident_preintegrate with job j under cfgs[cfg_of[j]] (0 <= cfg_of[j] < n_cfg): one launch for jobs of several configurations; the
 * record kind is that of window windows[j].  cerb_resident_preintegrate is this call with a one-entry table. */
int cerb_resident_preintegrate_mixed(CerbHandle *h, int32_t n_cfg, const CerbPreintConfig *cfgs, int32_t n, const CerbPreintJob *jobs,
                                     const int32_t *cfg_of, const int32_t *windows, const int32_t *slots, double *sum_dt);
/* cerb_batch_upload against the resident data: of descs[w] only n_features, features (obs_offset = slot * CERB_NUM_FRAMES), extrinsic_open
 * and td_open are read; states as in cerb_batch_upload; pre_slots [n][CERB_WINDOW_SIZE]: slot of interval i -> i + 1, a permutation of
 * 0 .. CERB_WINDOW_SIZE - 1 per window.  n must be the n of cerb_resident_start.  Afterwards the resident batch is used as after
 * cerb_batch_upload (cerb_batch_solve_resident, cerb_batch_download, the per-feature steps, cerb_batch_update_states). */
int cerb_resident_upload(CerbHandle *h, int32_t n, const CerbWindowDesc *descs, const CerbWindowState *states, const int32_t *pre_slots);
/* cerb_resident_upload of a compact batch of 1 <= n <= (n of cerb_resident_start) rows: row i is resident window windows[i] (no window listed
 * twice), descs / states / pre_slots are in list order.  The batch calls that follow (cerb_batch_solve_resident, cerb_batch_download,
 * cerb_batch_update_states, the per-feature steps, cerb_resident_marginalize) work on the n rows; the marginalization leaves each new prior in
 * window windows[i].  The windows not listed are not touched.  cerb_resident_upload is this call with windows = 0 .. n - 1. */
int cerb_resident_upload_windows(CerbHandle *h, int32_t n, const int32_t *windows, const CerbWindowDesc *descs, const CerbWindowState *states,
                                 const int32_t *pre_slots);
/* cerb_batch_marginalize with the new prior kept on the device as the prior of the same window at the next cerb_resident_upload (block
 * indices already shifted to the next window).  valid [n]: whether window w has a prior afterwards (MARGIN_SECOND_NEW without an old prior
 * keeps none, MARGIN_OLD with nothing dropped invalidates, as MarginalizationInfo::valid does). */
int cerb_resident_marginalize(CerbHandle *h, const int32_t *flags, const CerbWindowState *states, int32_t *valid);
/* Seed or replace the prior of one window from the host (prior->valid == 0 removes it). */
int cerb_resident_set_prior(CerbHandle *h, int32_t window, const CerbPrior *prior);
/* Read one window's store back as ordinary CerbWindowDesc content (tests, debugging): obs [max_obs] slot by slot; preint or imu_preint
 * [CERB_WINDOW_SIZE] by preintegration slot, the members an upload carries filled in and the others zero (pass the one that matches the
 * window's record kind, NULL for the other); prior with linearized_jacobians / linearized_residuals pointing at storage for CERB_MAX_PRIOR_DIM^2 / CERB_MAX_PRIOR_DIM
 * doubles.  Any output may be NULL. */
int cerb_resident_read_window(CerbHandle *h, int32_t window, CerbObservation *obs, CerbIMULegPreint *preint, CerbIMUPreint *imu_preint,
                              CerbPrior *prior);
/* Bytes the handle has been asked to move between host and device since cerb_create, and the number of copy operations issued, summed where
 * the copies are issued: every host-to-device copy, and the device-to-host copies of the entry points a replay uses (download, the per-feature
 * steps, marginalization, preintegration, the resident group).  The factor-family evaluators' and debug probes' read-backs and copies within
 * the device are not counted. */
int cerb_traffic(CerbHandle *h, int64_t *h2d_bytes, int64_t *d2h_bytes, int64_t *dma_ops);

/* ---- sequence replay: the reference's steady-state frame loop for B robots in lock step, host side in C++ inside this library -----------------
 * (csrc/replay_host.inl mirrors Estimator::processIMULeg / processImage (NON_LINEAR) / optimization / slideWindow and FeatureManager,
 * estimator.cpp:590-846,1054-1677, feature_manager.cpp; every numerical step is one of the batched entry points above).  The reference's
 * initialisation (estimator.cpp:700-797) is out of scope: the window is seeded frame by frame at given states. */
typedef struct CerbReplay CerbReplay;
/* one camera frame of one robot as the feature tracker delivers it (main.cpp:200-233): per feature the 7-vector x, y, z = 1, u, v, vx, vy of
 * camera 0 and, where has1, of camera 1 */
typedef struct CerbImage {
    int32_t n;
    int32_t reserved;
    const int64_t *ids;        /* [n] feature ids */
    const double *pts0;        /* [n][7] */
    const uint8_t *has1;       /* [n] */
    const double *pts1;        /* [n][7] */
} CerbImage;
/* h must have max_batch >= n_robots and max_features >= 2 * max_features of the replay (the triangulation batch holds every track).
 * pcfg, estimate_extrinsic and estimate_td are every robot's configuration until cerb_replay_configure_robot changes it; every robot starts
 * with use_leg = 1. */
int cerb_replay_create(CerbHandle *h, const CerbPreintConfig *pcfg, int32_t n_robots, int32_t max_features, int32_t estimate_extrinsic,
                       int32_t estimate_td, CerbReplay **out);
void cerb_replay_destroy(CerbReplay *r);
/* The configuration of one robot, as setParameter() would load it from its yaml: use_leg = USE_LEG (0: processIMU, IntegrationBase,
 * IMUFactor, no leg-bias blocks, estimator.cpp:554-588, :1160-1171; slideWindow's USE_IMU-only branches move no Rho and double2vector
 * leaves Rho alone, so the rho columns of its path rows keep their seeded value), pcfg = its noise / kinematics globals (a use_leg = 0 robot
 * reads acc_n, gyr_n, acc_w, gyr_w only), estimate_extrinsic, estimate_td.  The leg fields (phi, dphi, c) of a use_leg = 0 robot's
 * CerbIMULegSamples are ignored.  Robots of both kinds step together, their intervals in one preintegration launch.  The robot must not be
 * seeded (just created, or reset); cerb_replay_reset_robot keeps the configuration.  Works before or after cerb_replay_set_resident.  A
 * rejected call changes nothing. */
int cerb_replay_configure_robot(CerbReplay *r, int32_t robot, int32_t use_leg, const CerbPreintConfig *pcfg, int32_t estimate_extrinsic,
                                int32_t estimate_td);
int cerb_replay_set_extrinsics(CerbReplay *r, int32_t robot, const double *tic /* [2][3] */, const double *ric /* [2][9] row-major */);
/* Seed frame k = 0 .. WINDOW_SIZE of a robot: states P, R (row-major), V; `first` = the IMU / leg sample at the previous frame instant (at
 * frame 0: at frame 0), `samples` = the interval k-1 -> k (ignored for k = 0); image = the tracked features of frame k (NULL for k = WINDOW_SIZE:
 * that frame's image arrives with the first cerb_replay_step, whose interval is then empty). */
int cerb_replay_seed_frame(CerbReplay *r, int32_t robot, int32_t k, const double *P, const double *R, const double *V, const CerbIMULegSample *first,
                           const CerbIMULegSample *samples, int32_t n_samples, const CerbImage *image, double header);
/* processMeasurements for one camera frame of every robot: images [n_robots], firsts [n_robots] (sample at the previous frame instant),
 * samples [n_robots] pointers / n_samples [n_robots] (the new interval), header = the frame's stamp; reports (optional) [n_robots]. */
int cerb_replay_step(CerbReplay *r, const CerbImage *images, const CerbIMULegSample *firsts, const CerbIMULegSample *const *samples,
                     const int32_t *n_samples, double header, CerbSolveReport *reports);
/* processMeasurements for one camera frame of the n_active robots robots[0 .. n_active - 1] only, each at its own stamp: every array is in
 * list order (images, firsts, samples, n_samples, headers [n_active]; reports, optional, [n_active]).  The robots not listed are not touched,
 * and the order of the list changes no result.  A robot must be listed at most once and be seeded (frames 0 .. WINDOW_SIZE since its
 * creation or its last cerb_replay_reset_robot).  A call that is rejected changes nothing and moves nothing.  cerb_replay_step is this call
 * with every robot, in order, at one stamp. */
int cerb_replay_step_robots(CerbReplay *r, int32_t n_active, const int32_t *robots, const CerbImage *images, const CerbIMULegSample *firsts,
                            const CerbIMULegSample *const *samples, const int32_t *n_samples, const double *headers, CerbSolveReport *reports);
/* Estimator::clearState for one robot (the reference's restart, main.cpp:236-251): its features, intervals, prior, extrinsic latch and frame
 * count are gone, extrinsics back at the values of cerb_replay_set_extrinsics; in resident mode its track slots are free again, its device
 * prior is invalid and its preintegration slot table is the identity.  Its path rows and flag history stay.  It is seeded again with
 * cerb_replay_seed_frame (frames 0 .. WINDOW_SIZE) before it is stepped; the other robots may step meanwhile. */
int cerb_replay_reset_robot(CerbReplay *r, int32_t robot);
/* Published states of the newest frame after every processed image: rows of 20 doubles = header, P(3), R(9, row-major), V(3), rho(4). */
int cerb_replay_path(CerbReplay *r, int32_t robot, int32_t *n_rows, double *out, int32_t max_rows);
int cerb_replay_feature_ids(CerbReplay *r, int32_t robot, int32_t *n, int32_t *ids, int32_t max_ids);
/* marginalization_flag (0 MARGIN_OLD, 1 MARGIN_SECOND_NEW) the keyframe test chose at every processed image */
int cerb_replay_flags(CerbReplay *r, int32_t robot, int32_t *n, int32_t *flags, int32_t max_flags);
/* seconds spent in: preintegrate, triangulate, solve, marginalize, outliers, shift (device + ABI) and in host bookkeeping */
int cerb_replay_timing(CerbReplay *r, double *device6, double *host);
/* resident = 1: the replay keeps every robot's window on the device (cerb_resident_*) and cerb_replay_step sends the frame's edits instead
 * of three full uploads; the trajectories are bit-identical to the default mode.  To be called before the first cerb_replay_seed_frame; the
 * handle needs max_obs >= 2 * max_features of the replay * CERB_NUM_FRAMES (one slot per live track).  The replay's long-lived host arrays
 * are registered with the handle (cerb_register_host_buffer) until cerb_replay_destroy. */
int cerb_replay_set_resident(CerbReplay *r, int32_t resident);
/* what cerb_replay_step has asked the library to move so far (see cerb_traffic) and the bytes of it that went through staging memcpy */
int cerb_replay_traffic(CerbReplay *r, int64_t *h2d_bytes, int64_t *d2h_bytes, int64_t *dma_ops, int64_t *staged_bytes);
/* The window of one robot as the replay would upload it for a per-feature step (every track, in list order), for tests and debugging.
 * desc points into the replay's own arrays (valid until the next call on r): in the default mode tracks, observations, the preintegration
 * records and the prior; in resident mode the tracks only (obs_offset = slot * CERB_NUM_FRAMES) and prior.valid.  ids [<= max_ids] feature
 * ids; the records are desc->imu_preint (desc->preint NULL) for a use_leg = 0 robot; preint_current [CERB_WINDOW_SIZE]: 1 where the record of interval i -> i + 1 is up to date (0: samples were added since);
 * pre_slots [CERB_WINDOW_SIZE]: resident mode's slot of that interval. */
int cerb_replay_window(CerbReplay *r, int32_t robot, CerbWindowDesc *desc, int32_t *ids, int32_t max_ids, int32_t *preint_current,
                       int32_t *pre_slots);
/* Snapshots of one robot: everything the robot carries that later steps read (its states, extrinsics, td, stamps, counters, the feature list
 * in list order with every observation, the intervals with their samples and linearisation points, the marginalization prior and the robot's
 * configuration), and nothing of where it lives on the device.  A robot saved after frame k and loaded into any robot of any replay, in
 * either mode and on any handle, continues bit for bit as the saved robot does.  The path rows and the flag history are outputs and do not
 * travel: a loaded robot starts both empty.  The buffer starts with a magic number, a format version, CERB_WINDOW_SIZE, the number of
 * features and the prior dimension; it is meant for the same build of this library, not as a file format.
 * save: the robot must be seeded.  *size = the snapshot's size in bytes; buf = NULL: nothing else, else the snapshot into buf [cap]
 * (CERB_ERR_BAD_ARGUMENT if cap is smaller, *size still set: a caller can offer a buffer first and grow it once).  In resident mode the
 * prior is read off the device. */
int cerb_replay_save_robot(CerbReplay *r, int32_t robot, void *buf, size_t cap, size_t *size);
/* Overwrite `robot` with a snapshot; it counts as seeded and is stepped as usual.  The snapshot is checked before anything changes (magic
 * number, version, sizes against `size`, tracks against the replay's capacity: 2 x max_features tracks, max_features of them with four or
 * more observations; observation counts against CERB_NUM_FRAMES, feature ids unique, the keyframe flag 0 or 1, the prior dimension against
 * CERB_MAX_PRIOR_DIM and its blocks, no leg-bias block for a use_leg = 0 robot, the intervals against frame_count): a rejected snapshot returns CERB_ERR_BAD_ARGUMENT, moves nothing and leaves the robot as it was.  In
 * resident mode the window is emptied and takes the snapshot's record kind, the observations are put into fresh track slots, the intervals
 * whose records were up to date are preintegrated again (cerb_resident_preintegrate_mixed: the same bits) and the prior is set. */
int cerb_replay_load_robot(CerbReplay *r, int32_t robot, const void *buf, size_t size);
/* Make robots dsts[0 .. n - 1] of the same replay copies of robot src: one save and n loads, done in place.  Resident mode: one put stream
 * and one preintegration launch for all of them, and the prior is copied from window to window on the device.  dsts must be distinct and not
 * contain src; a rejected call changes nothing. */
int cerb_replay_clone_robot(CerbReplay *r, int32_t src, int32_t n, const int32_t *dsts);

/* ---- host-side helpers that stay on the CPU in the reference too ---------------------------- */
/* Gauge re-anchoring of Estimator::double2vector (estimator.cpp:903-957): rotates the solved
 * window by the yaw difference of frame 0 and re-anchors its position.  before/after are the
 * para_* arrays at vector2double() time and after the solve; writes Ps[11][3], Rs[11][9]
 * (row-major), Vs[11][3]. */
void cerb_double2vector(const CerbWindowState *before, const CerbWindowState *after, double *Ps,
                        double *Rs, double *Vs);

#ifdef __cplusplus
}
#endif
#endif /* CERBERUS_B200_H */

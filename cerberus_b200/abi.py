"""ctypes mirror of include/cerberus_b200.h (the C ABI of the H100 VILO backend).

Pure declarations: struct layouts, enums and a `WindowBatch` container that owns contiguous numpy
storage for a batch of sliding windows and exposes it as arrays of CerbWindowDesc /
CerbWindowState for the C entry points.  No compute here.
"""
import ctypes as C
import numpy as np

WINDOW_SIZE = 10
NUM_FRAMES = 11
IL_RES = 31
MAX_PRIOR_BLOCKS = 16
MAX_PRIOR_DIM = 96
NUM_REDUCED = 222  # 66 pose + 12 extrinsic + 99 speed-bias + 44 leg-bias + 1 td tangent dims

OK, ERR_BAD_ARGUMENT, ERR_NO_DEVICE, ERR_CUDA, ERR_NON_FINITE = 0, 1, 2, 3, 4
TERM_CONVERGENCE, TERM_NO_CONVERGENCE, TERM_FAILURE = 0, 1, 2
BLOCK_POSE, BLOCK_SPEEDBIAS, BLOCK_LEGBIAS, BLOCK_EX_POSE, BLOCK_TD = 0, 1, 2, 3, 4
PROJ_TWO_FRAME_ONE_CAM, PROJ_TWO_FRAME_TWO_CAM, PROJ_ONE_FRAME_TWO_CAM = 0, 1, 2
PROJ_JAC_SIZE = {0: 46, 1: 60, 2: 32}

c_dp = C.POINTER(C.c_double)


class SolverConfig(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("max_batch", C.c_int32), ("max_features", C.c_int32), ("max_obs", C.c_int32),
        ("max_num_iterations", C.c_int32), ("optimize_leg_bias", C.c_int32),
        ("g", C.c_double * 3), ("visual_sqrt_info", C.c_double), ("huber_delta", C.c_double),
        ("initial_trust_region_radius", C.c_double), ("max_trust_region_radius", C.c_double),
        ("min_trust_region_radius", C.c_double), ("min_relative_decrease", C.c_double),
        ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double), ("parameter_tolerance", C.c_double),
    ]


class IMULegPreint(C.Structure):
    _fields_ = [
        ("sum_dt", C.c_double), ("delta_p", C.c_double * 3), ("delta_q", C.c_double * 4), ("delta_v", C.c_double * 3),
        ("delta_epsilon", C.c_double * 12), ("linearized_ba", C.c_double * 3), ("linearized_bg", C.c_double * 3),
        ("linearized_rho", C.c_double * 4), ("jacobian", C.c_double * 961), ("covariance", C.c_double * 961),
    ]


class IMUPreint(C.Structure):
    _fields_ = [
        ("sum_dt", C.c_double), ("delta_p", C.c_double * 3), ("delta_q", C.c_double * 4), ("delta_v", C.c_double * 3),
        ("linearized_ba", C.c_double * 3), ("linearized_bg", C.c_double * 3), ("jacobian", C.c_double * 225), ("covariance", C.c_double * 225),
    ]


class Observation(C.Structure):
    _fields_ = [
        ("point", C.c_double * 2), ("velocity", C.c_double * 2), ("pointRight", C.c_double * 2),
        ("velocityRight", C.c_double * 2), ("cur_td", C.c_double), ("is_stereo", C.c_int32), ("reserved", C.c_int32),
    ]


class Feature(C.Structure):
    _fields_ = [("start_frame", C.c_int32), ("n_obs", C.c_int32), ("obs_offset", C.c_int32), ("reserved", C.c_int32)]


class Prior(C.Structure):
    _fields_ = [
        ("valid", C.c_int32), ("n", C.c_int32), ("num_blocks", C.c_int32), ("reserved", C.c_int32),
        ("block_kind", C.c_int32 * MAX_PRIOR_BLOCKS), ("block_index", C.c_int32 * MAX_PRIOR_BLOCKS),
        ("block_col", C.c_int32 * MAX_PRIOR_BLOCKS), ("block_x0", (C.c_double * 9) * MAX_PRIOR_BLOCKS),
        ("linearized_jacobians", c_dp), ("linearized_residuals", c_dp),
    ]


class WindowDesc(C.Structure):
    _fields_ = [
        ("n_features", C.c_int32), ("n_obs", C.c_int32),
        ("features", C.POINTER(Feature)), ("obs", C.POINTER(Observation)), ("preint", C.POINTER(IMULegPreint)), ("imu_preint", C.POINTER(IMUPreint)),
        ("prior", Prior), ("extrinsic_open", C.c_int32), ("td_open", C.c_int32),
    ]


class WindowState(C.Structure):
    _fields_ = [
        ("para_Pose", (C.c_double * 7) * NUM_FRAMES), ("para_SpeedBias", (C.c_double * 9) * NUM_FRAMES),
        ("para_LegBias", (C.c_double * 4) * NUM_FRAMES), ("para_Ex_Pose", (C.c_double * 7) * 2),
        ("para_Td", C.c_double * 1), ("reserved", C.c_double), ("para_Feature", c_dp),
    ]


class SolveReport(C.Structure):
    _fields_ = [
        ("iterations", C.c_int32), ("num_successful_steps", C.c_int32), ("termination", C.c_int32), ("status", C.c_int32),
        ("initial_cost", C.c_double), ("final_cost", C.c_double),
    ]


class IMULegSample(C.Structure):
    _fields_ = [("dt", C.c_double), ("acc", C.c_double * 3), ("gyr", C.c_double * 3), ("phi", C.c_double * 12),
                ("dphi", C.c_double * 12), ("c", C.c_double * 4)]


class PreintConfig(C.Structure):
    _fields_ = [
        ("acc_n", C.c_double), ("acc_n_z", C.c_double), ("gyr_n", C.c_double), ("acc_w", C.c_double), ("gyr_w", C.c_double),
        ("phi_n", C.c_double), ("dphi_n", C.c_double), ("rho_c_n", C.c_double), ("rho_nc_n", C.c_double),
        ("v_n_min_xy", C.c_double), ("v_n_min_z", C.c_double), ("v_n_min", C.c_double), ("v_n_max", C.c_double),
        ("v_n_force_thres_ratio", C.c_double), ("v_n_term1_steep", C.c_double), ("v_n_term2_var_rescale", C.c_double),
        ("v_n_term3_distance_rescale", C.c_double), ("contact_sensor_type", C.c_int32), ("reserved", C.c_int32),
        ("rho_fix", (C.c_double * 4) * 4), ("p_br", C.c_double * 3), ("R_br", C.c_double * 9),
    ]


class PreintJob(C.Structure):
    _fields_ = [
        ("acc_0", C.c_double * 3), ("gyr_0", C.c_double * 3), ("phi_0", C.c_double * 12), ("dphi_0", C.c_double * 12),
        ("c_0", C.c_double * 4), ("linearized_ba", C.c_double * 3), ("linearized_bg", C.c_double * 3),
        ("linearized_rho", C.c_double * 4), ("n_samples", C.c_int32), ("reserved", C.c_int32),
        ("samples", C.POINTER(IMULegSample)),
    ]


class TrackPut(C.Structure):
    _fields_ = [("window", C.c_int32), ("slot", C.c_int32), ("position", C.c_int32), ("reserved", C.c_int32), ("obs", Observation)]


class TrackEdit(C.Structure):
    _fields_ = [("window", C.c_int32), ("slot", C.c_int32), ("n_obs", C.c_int32), ("position", C.c_int32)]


ABI_STRUCTS = [SolverConfig, IMULegPreint, Observation, Feature, Prior, WindowDesc, WindowState, SolveReport,
               IMULegSample, PreintConfig, PreintJob, IMUPreint]

feature_dtype = np.dtype(Feature)
obs_dtype = np.dtype(Observation)
preint_dtype = np.dtype(IMULegPreint)
imu_preint_dtype = np.dtype(IMUPreint)
sample_dtype = np.dtype(IMULegSample)
report_dtype = np.dtype(SolveReport)
track_put_dtype = np.dtype(TrackPut)
track_edit_dtype = np.dtype(TrackEdit)


def default_config():
    """A1 yaml (config/a1_config/hardware_a1_vilo_config.yaml) + Ceres 1.14 defaults; mirrors cerb_default_config."""
    c = SolverConfig()
    c.device = 0
    c.max_batch = 1024
    c.max_features = 160
    c.max_obs = 160 * NUM_FRAMES
    c.max_num_iterations = 12
    c.optimize_leg_bias = 1
    c.g[0], c.g[1], c.g[2] = 0.0, 0.0, 9.805
    c.visual_sqrt_info = 460.0 / 1.5
    c.huber_delta = 1.0
    c.initial_trust_region_radius = 1e4
    c.max_trust_region_radius = 1e16
    c.min_trust_region_radius = 1e-32
    c.min_relative_decrease = 1e-3
    c.function_tolerance = 1e-6
    c.gradient_tolerance = 1e-10
    c.parameter_tolerance = 1e-8
    return c


def default_preint_config():
    """Noise globals of the A1 yaml + A1 leg geometry (estimator.cpp:140-171); mirrors cerb_default_preint_config."""
    p = PreintConfig()
    p.acc_n, p.acc_n_z, p.gyr_n, p.acc_w, p.gyr_w = 0.9, 2.5, 0.05, 0.0004, 0.0002
    p.phi_n = p.dphi_n = 1e-5
    p.rho_c_n, p.rho_nc_n = 1e-8, 1e-11
    p.v_n_min_xy, p.v_n_min_z, p.v_n_min, p.v_n_max = 1e-3, 5e-3, 5e-3, 900.0
    p.v_n_force_thres_ratio, p.v_n_term1_steep = 0.8, 10.0
    p.v_n_term2_var_rescale, p.v_n_term3_distance_rescale = 1e-6, 1e-3
    p.contact_sensor_type = 0
    ox = [0.1805, 0.1805, -0.1805, -0.1805]
    oy = [0.047, -0.047, 0.047, -0.047]
    d = [0.0838, -0.0838, 0.0838, -0.0838]
    for leg in range(4):
        p.rho_fix[leg][0], p.rho_fix[leg][1], p.rho_fix[leg][2], p.rho_fix[leg][3] = ox[leg], oy[leg], d[leg], 0.21
    for k in range(3):
        p.p_br[k] = 0.0
    for k in range(9):
        p.R_br[k] = 1.0 if k in (0, 4, 8) else 0.0
    return p


def vins_preint_config():
    """The A1 VINS baseline (config/a1_config/hardware_a1_vins_config.yaml: no use_leg_odom, so USE_LEG == 0; acc_n 0.5, gyr_n 0.05,
    acc_w 0.0004, gyr_w 0.0002).  IntegrationBase reads acc_n (on all three axes), gyr_n, acc_w and gyr_w only; the other fields keep the
    A1 VILO values of default_preint_config."""
    p = default_preint_config()
    p.acc_n = 0.5
    return p


class WindowBatch:
    """Contiguous host storage for `n` sliding windows + the ctypes views the C ABI takes.

    Arrays (all C-contiguous numpy):
      features [n, max_features]  feature_dtype      obs    [n, max_obs]  obs_dtype
      preint   [n, 10]            preint_dtype       prior_J [n, 96*96], prior_r [n, 96]
      states   ctypes array of WindowState           para_Feature [n, max_features]
      descs    ctypes array of WindowDesc (pointers into the arrays above)
    Every descriptor starts with IMU-leg records (preint); set_kind switches one to IMUFactor records (imu_preint [n, 10], allocated with
    the first such window), so one batch may mix the two.
    """

    def __init__(self, n, max_features, max_obs=None):
        self.n = n
        self.max_features = max_features
        self.max_obs = max_obs if max_obs is not None else max_features * NUM_FRAMES
        self.features = np.zeros((n, self.max_features), dtype=feature_dtype)
        self.obs = np.zeros((n, self.max_obs), dtype=obs_dtype)
        self.preint = np.zeros((n, WINDOW_SIZE), dtype=preint_dtype)
        self.imu_preint = None                      # allocated by use_imu_only()
        self.prior_J = np.zeros((n, MAX_PRIOR_DIM * MAX_PRIOR_DIM))
        self.prior_r = np.zeros((n, MAX_PRIOR_DIM))
        self.para_Feature = np.zeros((n, self.max_features))
        self.states = (WindowState * n)()
        self.descs = (WindowDesc * n)()
        self.reports = (SolveReport * n)()
        for w in range(n):
            d = self.descs[w]
            d.features = self.features[w].ctypes.data_as(C.POINTER(Feature))
            d.obs = self.obs[w].ctypes.data_as(C.POINTER(Observation))
            d.preint = self.preint[w].ctypes.data_as(C.POINTER(IMULegPreint))
            d.prior.linearized_jacobians = self.prior_J[w].ctypes.data_as(c_dp)
            d.prior.linearized_residuals = self.prior_r[w].ctypes.data_as(c_dp)
            self.states[w].para_Feature = self.para_Feature[w].ctypes.data_as(c_dp)

    def set_kind(self, w, use_leg):
        """Descriptor w carries IMU-leg preintegrations (use_leg, USE_LEG == 1) or IMUFactor ones (USE_LEG == 0)."""
        d = self.descs[w]
        if use_leg:
            d.preint = self.preint[w].ctypes.data_as(C.POINTER(IMULegPreint)); d.imu_preint = None
            return
        if self.imu_preint is None:
            self.imu_preint = np.zeros((self.n, WINDOW_SIZE), dtype=imu_preint_dtype)
        d.preint = None
        d.imu_preint = self.imu_preint[w].ctypes.data_as(C.POINTER(IMUPreint))

    def use_imu_only(self):
        """Switch the batch to USE_LEG == 0: descriptors carry IMUFactor preintegrations instead of IMU-leg ones."""
        for w in range(self.n):
            self.set_kind(w, False)

    # numpy views of the state arrays (no copy): shape [n, ...]
    def state_array(self):
        """Structured view of the states (pointer field excluded from the named fields)."""
        dt = np.dtype({"names": ["para_Pose", "para_SpeedBias", "para_LegBias", "para_Ex_Pose", "para_Td"],
                       "formats": [(np.float64, (NUM_FRAMES, 7)), (np.float64, (NUM_FRAMES, 9)), (np.float64, (NUM_FRAMES, 4)),
                                   (np.float64, (2, 7)), (np.float64, (1,))],
                       "offsets": [WindowState.para_Pose.offset, WindowState.para_SpeedBias.offset, WindowState.para_LegBias.offset,
                                   WindowState.para_Ex_Pose.offset, WindowState.para_Td.offset],
                       "itemsize": C.sizeof(WindowState)})
        return np.frombuffer(self.states, dtype=dt, count=self.n)

    def report_array(self):
        return np.frombuffer(self.reports, dtype=report_dtype, count=self.n)

    def copy_states(self):
        """Deep copy of (states, para_Feature) as plain numpy (for restoring / comparing)."""
        return np.frombuffer(self.states, dtype=np.uint8).copy(), self.para_Feature.copy()

    def restore_states(self, saved):
        raw, feat = saved
        C.memmove(self.states, raw.ctypes.data, raw.nbytes)
        self.para_Feature[...] = feat
        for w in range(self.n):
            self.states[w].para_Feature = self.para_Feature[w].ctypes.data_as(c_dp)


class Image(C.Structure):
    """CerbImage: one camera frame of one robot (the feature tracker's output, main.cpp:200-233)."""
    _fields_ = [("n", C.c_int32), ("reserved", C.c_int32), ("ids", C.POINTER(C.c_int64)), ("pts0", c_dp), ("has1", C.POINTER(C.c_uint8)), ("pts1", c_dp)]

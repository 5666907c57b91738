"""Host-side mirror of the reference's Estimator / FeatureManager for the steady-state (NON_LINEAR) frame loop, and a lock-step
replay driver for B independent robots (SURVEY.md 8(f) n4, 7 step 7).

Mirrors, statement for statement where it matters for the numbers:
  FeatureManager                       src/featureTracker/feature_manager.{h,cpp}
  Estimator.processIMULeg              src/estimator/estimator.cpp:590-653 (buffers + midpoint propagation of the newest state);
                                       processIMU (:554-588) for a robot configured with use_leg = False (USE_LEG == 0: the VINS
                                       configurations), with IntegrationBase / IMUFactor, no leg-bias blocks and no Rho updates
  Estimator.processImage (NON_LINEAR)  :655-676, :798-846  triangulate -> optimization -> outliersRejection -> slideWindow -> removeFailures
  Estimator.vector2double/double2vector:848-1003
  Estimator.optimization               :1054-1456: the solve goes through the backend (cerb_solve_batch), the marginalization too
  Estimator.slideWindow{,Old,New}      :1460-1677

Everything numerical per window is a backend call over the C ABI (device: cerberus_b200.lib.Backend; tests drive the very same
class with the CPU oracle to get the reference arm of the comparison): preintegration, triangulation, the solve, marginalization,
outlier errors, depth shift.  What stays here is the bookkeeping the reference also does on the host in C++ (std::list / std::map walks).

The reference's initialisation (stereo PnP + gyroscope-bias alignment, estimator.cpp:700-797) needs OpenCV and is out of scope: a
replay is seeded with the first WINDOW_SIZE + 1 frames at given initial states and starts in NON_LINEAR at frame WINDOW_SIZE.
"""
import ctypes as C
import numpy as np
from . import abi

WINDOW_SIZE = abi.WINDOW_SIZE
FOCAL_LENGTH = 460.0          # parameters.h:22
MIN_PARALLAX = 10.0 / FOCAL_LENGTH   # yaml keyframe_parallax 10.0 / FOCAL_LENGTH (parameters.cpp:132)
INIT_DEPTH = 5.0              # parameters.cpp:250
MARGIN_OLD, MARGIN_SECOND_NEW = 0, 1


# ------------------------------------------------------------------------------------------------ small rotation helpers
def quat_to_R(q):
    """(x, y, z, w) -> 3x3, Eigen::Quaterniond::toRotationMatrix."""
    x, y, z, w = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1 - (txx + tyy)]])


def R_to_quat(m):
    """3x3 -> (x, y, z, w), Eigen's Quaternion(Matrix3) constructor (vector2double: Quaterniond q{Rs[i]}, estimator.cpp:855)."""
    t = m[0, 0] + m[1, 1] + m[2, 2]
    q = np.zeros(4)
    if t > 0:
        t = np.sqrt(t + 1.0); q[3] = 0.5 * t; t = 0.5 / t
        q[0], q[1], q[2] = (m[2, 1] - m[1, 2]) * t, (m[0, 2] - m[2, 0]) * t, (m[1, 0] - m[0, 1]) * t
    else:
        i = 0
        if m[1, 1] > m[0, 0]: i = 1
        if m[2, 2] > m[i, i]: i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0)
        q[i] = 0.5 * t; t = 0.5 / t
        q[3] = (m[k, j] - m[j, k]) * t; q[j] = (m[j, i] + m[i, j]) * t; q[k] = (m[k, i] + m[i, k]) * t
    return q


def delta_q_R(theta):
    """Utility::deltaQ(theta).toRotationMatrix() (utility.h:28-41): q = (1, theta / 2), NOT normalised (as in the reference)."""
    return quat_to_R(np.array([theta[0] / 2, theta[1] / 2, theta[2] / 2, 1.0]))


# ------------------------------------------------------------------------------------------------ FeatureManager
class FeaturePerFrame:
    __slots__ = ("point", "pointRight", "velocity", "velocityRight", "cur_td", "is_stereo")

    def __init__(self, p7, td):                       # feature_manager.h:31-43
        self.point = np.array(p7[0:3]); self.velocity = np.array(p7[5:7]); self.cur_td = td
        self.pointRight = np.zeros(3); self.velocityRight = np.zeros(2); self.is_stereo = False

    def rightObservation(self, p7):                   # :44-54
        self.pointRight = np.array(p7[0:3]); self.velocityRight = np.array(p7[5:7]); self.is_stereo = True


class FeaturePerId:
    __slots__ = ("feature_id", "start_frame", "feature_per_frame", "used_num", "estimated_depth", "solve_flag")

    def __init__(self, feature_id, start_frame):      # feature_manager.h:72-76
        self.feature_id, self.start_frame = feature_id, start_frame
        self.feature_per_frame = []; self.used_num = 0; self.estimated_depth = -1.0; self.solve_flag = 0

    def endFrame(self):
        return self.start_frame + len(self.feature_per_frame) - 1


class FeatureManager:
    """feature_manager.cpp; `feature` is the std::list<FeaturePerId> (insertion order = first-seen order)."""

    def __init__(self):
        self.feature = []
        self.last_track_num = 0; self.last_average_parallax = 0.0; self.new_feature_num = 0; self.long_track_num = 0

    def clearState(self):
        self.feature = []

    def getFeatureCount(self):                        # :37-49
        cnt = 0
        for it in self.feature:
            it.used_num = len(it.feature_per_frame)
            if it.used_num >= 4: cnt += 1
        return cnt

    def addFeatureCheckParallax(self, frame_count, image, td):     # :52-118; image = dict(ids, pts0, has1, pts1)
        parallax_sum, parallax_num = 0.0, 0
        self.last_track_num = 0; self.last_average_parallax = 0; self.new_feature_num = 0; self.long_track_num = 0
        index = {it.feature_id: it for it in self.feature}
        ids, pts0, has1, pts1 = image["ids"], image["pts0"], image["has1"], image["pts1"]
        for q in np.argsort(ids, kind="stable"):      # the reference iterates a std::map: ascending feature id
            f = FeaturePerFrame(pts0[q], td)
            if has1[q]: f.rightObservation(pts1[q])
            fid = int(ids[q])
            it = index.get(fid)
            if it is None:
                it = FeaturePerId(fid, frame_count); self.feature.append(it); index[fid] = it
                it.feature_per_frame.append(f); self.new_feature_num += 1
            else:
                it.feature_per_frame.append(f); self.last_track_num += 1
                if len(it.feature_per_frame) >= 4: self.long_track_num += 1
        if frame_count < 2 or self.last_track_num < 20 or self.long_track_num < 40 or self.new_feature_num > 0.5 * self.last_track_num:
            return True
        for it in self.feature:
            if it.start_frame <= frame_count - 2 and it.start_frame + len(it.feature_per_frame) - 1 >= frame_count - 1:
                parallax_sum += self.compensatedParallax2(it, frame_count); parallax_num += 1
        if parallax_num == 0:
            return True
        self.last_average_parallax = parallax_sum / parallax_num * FOCAL_LENGTH
        return parallax_sum / parallax_num >= MIN_PARALLAX

    @staticmethod
    def compensatedParallax2(it, frame_count):        # :531-565 (the compensation is commented out in the reference: p_i_comp = p_i)
        fi = it.feature_per_frame[frame_count - 2 - it.start_frame]; fj = it.feature_per_frame[frame_count - 1 - it.start_frame]
        u_j, v_j = fj.point[0], fj.point[1]
        dep_i = fi.point[2]
        du, dv = fi.point[0] / dep_i - u_j, fi.point[1] / dep_i - v_j
        return max(0.0, np.sqrt(min(du * du + dv * dv, du * du + dv * dv)))

    def setDepth(self, x):                            # :142-160
        k = -1
        for it in self.feature:
            it.used_num = len(it.feature_per_frame)
            if it.used_num < 4: continue
            k += 1
            it.estimated_depth = 1.0 / x[k]
            it.solve_flag = 2 if it.estimated_depth < 0 else 1

    def removeFailures(self):                         # :162-172
        self.feature = [it for it in self.feature if it.solve_flag != 2]

    def clearDepth(self):
        for it in self.feature: it.estimated_depth = -1

    def getDepthVector(self):                         # :180-196
        out = []
        for it in self.feature:
            it.used_num = len(it.feature_per_frame)
            if it.used_num < 4: continue
            out.append(1.0 / it.estimated_depth)
        return np.array(out)

    def removeOutlier(self, outlier_ids):             # :433-448
        self.feature = [it for it in self.feature if it.feature_id not in outlier_ids]

    def removeBackShiftDepth(self, new_depth):        # :450-488; new_depth: feature_id -> depth in the new anchor frame (backend.shift_depth)
        out = []
        for it in self.feature:
            if it.start_frame != 0:
                it.start_frame -= 1
            else:
                del it.feature_per_frame[0]
                if len(it.feature_per_frame) < 2: continue
                it.estimated_depth = new_depth[it.feature_id]
            out.append(it)
        self.feature = out

    def removeBack(self):                             # :490-506
        out = []
        for it in self.feature:
            if it.start_frame != 0: it.start_frame -= 1
            else:
                del it.feature_per_frame[0]
                if len(it.feature_per_frame) == 0: continue
            out.append(it)
        self.feature = out

    def removeFront(self, frame_count):               # :508-529
        out = []
        for it in self.feature:
            if it.start_frame == frame_count:
                it.start_frame -= 1
            else:
                j = WINDOW_SIZE - 1 - it.start_frame
                if it.endFrame() >= frame_count - 1:
                    del it.feature_per_frame[j]
                    if len(it.feature_per_frame) == 0: continue
            out.append(it)
        self.feature = out


# ------------------------------------------------------------------------------------------------ one robot
class Interval:
    """What an IMULegIntegrationBase holds besides its result: constructor arguments + the sample buffers (dt_buf, ... estimator.h:167-175)."""

    def __init__(self, first, ba, bg, rho):
        self.first = first.copy()                     # acc_0, gyr_0, phi_0, dphi_0, c_0 (sample_dtype record)
        self.ba, self.bg, self.rho = ba.copy(), bg.copy(), rho.copy()
        self.samples = np.zeros(0, dtype=abi.sample_dtype)
        self.result = None                            # abi.preint_dtype record, filled by the driver
        self.dirty = True


class Estimator:
    def __init__(self, cfg, estimate_extrinsic=1, estimate_td=0, use_leg=True, pcfg=None):
        """use_leg: USE_LEG of the robot's yaml; pcfg: its preintegration globals (abi.PreintConfig; None: abi.default_preint_config())."""
        self.cfg = cfg
        self.use_leg, self.pcfg = bool(use_leg), (pcfg if pcfg is not None else abi.default_preint_config())
        n = WINDOW_SIZE + 1
        self.Ps, self.Vs, self.Bas, self.Bgs = np.zeros((n, 3)), np.zeros((n, 3)), np.zeros((n, 3)), np.zeros((n, 3))
        self.Rs = np.tile(np.eye(3), (n, 1, 1)); self.Rho = np.full((n, 4), 0.21)
        self.tic, self.ric = np.zeros((2, 3)), np.tile(np.eye(3), (2, 1, 1))
        self.td = 0.0
        self.g = np.array([cfg.g[0], cfg.g[1], cfg.g[2]])
        self.f_manager = FeatureManager()
        self.frame_count = 0
        self.intervals = [None] * n                   # il_pre_integrations[i]: frames i-1 -> i
        self.last = None                              # acc_0 / gyr_0 / phi_0 / dphi_0 / c_0: the latest sample
        self.prior = None                             # dict(prior=abi.Prior, J, r): last_marginalization_info + parameter blocks
        self.marginalization_flag = MARGIN_OLD
        self.ESTIMATE_EXTRINSIC, self.ESTIMATE_TD = estimate_extrinsic, estimate_td
        self.openExEstimation = False
        self.back_R0, self.back_P0 = np.eye(3), np.zeros(3)
        self.Headers = np.zeros(n)
        self.path = []                                # published (header, P, R, V, rho) of the newest frame after every processed image

    # ---- processIMULeg, estimator.cpp:590-653: one whole inter-frame interval at a time (processIMU, :554-588, propagates the same way;
    # its IntegrationBase reads dt, acc and gyr of the buffered samples only)
    def process_interval(self, first_sample, samples):
        j = self.frame_count
        if self.last is None: self.last = first_sample.copy()
        if self.intervals[j] is None: self.intervals[j] = Interval(self.last, self.Bas[j], self.Bgs[j], self.Rho[j])
        if j == 0:
            self.last = samples[-1].copy() if len(samples) else self.last
            return
        iv = self.intervals[j]
        iv.samples = np.concatenate([iv.samples, samples]); iv.dirty = True
        acc_0, gyr_0 = np.array(self.last["acc"]), np.array(self.last["gyr"])
        R, P, V = self.Rs[j].copy(), self.Ps[j].copy(), self.Vs[j].copy()
        Ba, Bg, g = self.Bas[j], self.Bgs[j], self.g
        for s in samples:
            dt, acc, gyr = float(s["dt"]), np.array(s["acc"]), np.array(s["gyr"])
            un_acc_0 = R @ (acc_0 - Ba) - g
            un_gyr = 0.5 * (gyr_0 + gyr) - Bg
            R = R @ delta_q_R(un_gyr * dt)
            un_acc_1 = R @ (acc - Ba) - g
            un_acc = 0.5 * (un_acc_0 + un_acc_1)
            P = P + dt * V + 0.5 * dt * dt * un_acc
            V = V + dt * un_acc
            acc_0, gyr_0 = acc, gyr
        self.Rs[j], self.Ps[j], self.Vs[j] = R, P, V
        if len(samples): self.last = samples[-1].copy()

    # ---- vector2double, estimator.cpp:848-901
    def vector2double(self, st, para_feature=None):
        for i in range(WINDOW_SIZE + 1):
            st.para_Pose[i][0:3] = self.Ps[i]; st.para_Pose[i][3:7] = R_to_quat(self.Rs[i])
            st.para_SpeedBias[i][0:3] = self.Vs[i]; st.para_SpeedBias[i][3:6] = self.Bas[i]; st.para_SpeedBias[i][6:9] = self.Bgs[i]
            if self.use_leg: st.para_LegBias[i][0:4] = self.Rho[i]
        for c in range(2):
            st.para_Ex_Pose[c][0:3] = self.tic[c]; st.para_Ex_Pose[c][3:7] = R_to_quat(self.ric[c])
        st.para_Td[0] = self.td
        if para_feature is None: return 0
        dep = self.f_manager.getDepthVector()
        para_feature[:dep.size] = dep
        return dep.size

    # ---- the part of double2vector after the gauge fix (:936-1003); Ps / Rs / Vs come from backend.double2vector
    def double2vector_rest(self, st, para_feature, Ps, Rs, Vs):
        sb = np.array(st.para_SpeedBias); lb = np.array(st.para_LegBias); ex = np.array(st.para_Ex_Pose)
        self.Ps[:], self.Rs[:], self.Vs[:] = Ps, Rs, Vs
        self.Bas[:], self.Bgs[:] = sb[:, 3:6], sb[:, 6:9]
        for c in range(2):
            self.tic[c] = ex[c, 0:3]
            q = ex[c, 3:7]; self.ric[c] = quat_to_R(q / np.linalg.norm(q))
        if self.use_leg: self.Rho[:] = lb
        nf = self.f_manager.getFeatureCount()
        self.f_manager.setDepth(para_feature[:nf])
        self.td = st.para_Td[0]

    # ---- slideWindow, estimator.cpp:1460-1677 (frame_count == WINDOW_SIZE, USE_LEG && USE_IMU, or USE_IMU only: no Rho moves)
    def slide_window(self, new_depth):
        W = WINDOW_SIZE
        if self.marginalization_flag == MARGIN_OLD:
            self.back_R0, self.back_P0 = self.Rs[0].copy(), self.Ps[0].copy()
            for arr in (self.Headers, self.Rs, self.Ps, self.Vs, self.Bas, self.Bgs) + ((self.Rho,) if self.use_leg else ()):
                arr[0:W] = arr[1:W + 1].copy()        # the swaps of :1472-1497 followed by the copies of :1511-1524
            self.intervals = self.intervals[1:] + [None]
            self.intervals[W] = Interval(self.last, self.Bas[W], self.Bgs[W], self.Rho[W])       # :1529-1536
            self.f_manager.removeBackShiftDepth(new_depth)                                      # slideWindowOld, solver_flag == NON_LINEAR
        else:
            self.Headers[W - 1] = self.Headers[W]; self.Ps[W - 1] = self.Ps[W]; self.Rs[W - 1] = self.Rs[W]
            a, b = self.intervals[W - 1], self.intervals[W]
            a.samples = np.concatenate([a.samples, b.samples]); a.dirty = True                   # :1576-1596 push_back of the buffered samples
            self.Vs[W - 1], self.Bas[W - 1], self.Bgs[W - 1] = self.Vs[W], self.Bas[W], self.Bgs[W]
            if self.use_leg: self.Rho[W - 1] = self.Rho[W]
            self.intervals[W] = Interval(self.last, self.Bas[W], self.Bgs[W], self.Rho[W])       # :1609-1616
            self.f_manager.removeFront(self.frame_count)                                         # slideWindowNew


# ------------------------------------------------------------------------------------------------ window <-> ABI batch
def fill_window(batch, w, est, min_used=4, with_prior=True):
    """CerbWindowDesc / CerbWindowState of robot `est` in slot w: the factor enumeration of estimator.cpp:1114-1216 (features with
    used_num >= min_used in list order) and vector2double.  Returns the feature ids in para_Feature order."""
    ids = []
    fw, ow = batch.features[w], batch.obs[w]
    off = 0
    for it in est.f_manager.feature:
        it.used_num = len(it.feature_per_frame)
        if it.used_num < min_used: continue
        k = len(ids)
        if k >= batch.max_features or off + it.used_num > batch.max_obs:
            raise RuntimeError("window over the batch capacity")
        fw[k]["start_frame"], fw[k]["n_obs"], fw[k]["obs_offset"] = it.start_frame, it.used_num, off
        for f in it.feature_per_frame:
            o = ow[off]
            o["point"] = f.point[:2]; o["velocity"] = f.velocity; o["pointRight"] = f.pointRight[:2]; o["velocityRight"] = f.velocityRight
            o["cur_td"] = f.cur_td; o["is_stereo"] = 1 if f.is_stereo else 0
            off += 1
        ids.append(it.feature_id)
    d = batch.descs[w]
    d.n_features, d.n_obs = len(ids), off
    batch.set_kind(w, est.use_leg)                    # estimator.cpp:1114-1171: IMULegFactor or IMUFactor
    records = batch.preint if est.use_leg else batch.imu_preint
    for i in range(WINDOW_SIZE):
        records[w, i] = est.intervals[i + 1].result
    st = batch.states[w]
    est.vector2double(st, batch.para_Feature[w] if min_used >= 4 else None)
    # constant blocks, estimator.cpp:1091-1105 (the latch is evaluated where optimization() evaluates it: when the solve is set up)
    if with_prior and est.ESTIMATE_EXTRINSIC and est.frame_count == WINDOW_SIZE and np.linalg.norm(est.Vs[0]) > 0.2: est.openExEstimation = True
    d.extrinsic_open = 1 if (est.ESTIMATE_EXTRINSIC and est.openExEstimation) else 0
    d.td_open = 1 if (est.ESTIMATE_TD and np.linalg.norm(est.Vs[0]) >= 0.2) else 0
    pr = d.prior
    if with_prior and est.prior is not None and est.prior["prior"].valid:
        src = est.prior
        keepJ, keepr = pr.linearized_jacobians, pr.linearized_residuals
        C.memmove(C.byref(pr), C.byref(src["prior"]), C.sizeof(abi.Prior))
        n = pr.n
        batch.prior_J[w, :n * n] = src["J"][:n * n]; batch.prior_r[w, :n] = src["r"][:n]
        pr.linearized_jacobians, pr.linearized_residuals = keepJ, keepr
    else:
        pr.valid = 0
    return ids


def take_prior(batch, w):
    """Copy the prior the backend wrote into slot w (descriptor + matrices) into an owned dict."""
    pr = abi.Prior()
    C.memmove(C.byref(pr), C.byref(batch.descs[w].prior), C.sizeof(abi.Prior))
    n = pr.n                                          # read through the pointers: a carried-over prior aliases the source arrays
    J = np.zeros(abi.MAX_PRIOR_DIM * abi.MAX_PRIOR_DIM); r = np.zeros(abi.MAX_PRIOR_DIM)
    J[:n * n] = np.ctypeslib.as_array(pr.linearized_jacobians, shape=(n * n,)); r[:n] = np.ctypeslib.as_array(pr.linearized_residuals, shape=(n,))
    pr.linearized_jacobians = J.ctypes.data_as(abi.c_dp); pr.linearized_residuals = r.ctypes.data_as(abi.c_dp)
    return dict(prior=pr, J=J, r=r)


# ------------------------------------------------------------------------------------------------ lock-step replay of B robots
class ReplayDriver:
    """Runs B Estimators through a SynthSequence (or any source of per-frame images + per-interval samples) in lock step; every numerical
    step is one batched backend call.  `ops` is a backend adapter (DeviceOps / tests' OracleOps) with
        preintegrate(pcfg, jobs, n) / preintegrate_imu(pcfg, jobs, n) -> IMU-leg / IMU records;  triangulate(batch) -> depth [n, F];  solve(batch) -> reports;
        double2vector(before_state, after_state) -> (Ps, Rs, Vs);  marginalize(src, dst, flags);  outlier_errors(batch) -> [n, F];
        shift_depth(batch) -> (start, depth, keep)."""

    def __init__(self, ops, cfg, pcfg, n, max_features=160, estimate_td=0):
        self.ops, self.cfg, self.pcfg, self.n = ops, cfg, pcfg, n
        self.est = [Estimator(cfg, estimate_td=estimate_td, pcfg=pcfg) for _ in range(n)]
        self.F = max_features
        self.batch = abi.WindowBatch(n, max_features)
        self.batch_all = abi.WindowBatch(n, 2 * max_features)        # triangulation sees every track, also those with < 4 observations
        self.batch_next = abi.WindowBatch(n, 1, 1)                   # receives the priors of the next window
        self.reports = []
        self.flags = []                                              # marginalization flag of every robot at every processed frame
        self.timing = dict(preintegrate=0.0, triangulate=0.0, solve=0.0, marginalize=0.0, outliers=0.0, shift=0.0, host=0.0)

    def configure(self, w, use_leg, pcfg, estimate_extrinsic=1, estimate_td=0):
        """Robot w's configuration (NativeReplay.configure): use_leg = USE_LEG, pcfg its preintegration globals; before it is seeded."""
        if self.est[w].last is not None:
            raise RuntimeError("configure: the robot is seeded")
        self.est[w] = Estimator(self.cfg, estimate_extrinsic, estimate_td, use_leg=use_leg, pcfg=pcfg)

    def seed(self, seq):
        """First WINDOW_SIZE + 1 frames at the given initial states (stands in for the reference's initialisation)."""
        for w, e in enumerate(self.est):
            e.tic[:] = seq.tic_g[w]; e.ric[:] = seq.ric_g[w]
            for k in range(WINDOW_SIZE + 1):
                e.frame_count = k
                e.Ps[k], e.Rs[k], e.Vs[k] = seq.p_g[w, k], seq.R_g[w, k], seq.v_g[w, k]
                if k == 0: e.process_interval(seq.first[w, 0], seq.samples[w, 0][:0])
                else:
                    P, R, V = e.Ps[k].copy(), e.Rs[k].copy(), e.Vs[k].copy()
                    e.process_interval(seq.first[w, k - 1], seq.samples[w, k - 1])
                    e.Ps[k], e.Rs[k], e.Vs[k] = P, R, V                  # seeded states, not the IMU prediction
                e.Headers[k] = k
                if k < WINDOW_SIZE: e.f_manager.addFeatureCheckParallax(k, seq.images[k][w], e.td)
            e.frame_count = WINDOW_SIZE

    def _preintegrate_dirty(self):
        import time
        t0 = time.perf_counter()
        todo = [(e, i) for e in self.est for i in range(1, WINDOW_SIZE + 1) if e.intervals[i] is not None and e.intervals[i].dirty and len(e.intervals[i].samples)]
        groups = {}                                   # one backend call per configuration and record kind
        for q, (e, i) in enumerate(todo):
            groups.setdefault((bytes(e.pcfg), e.use_leg), []).append(q)
        for (_, use_leg), qs in groups.items():
            jobs = (abi.PreintJob * len(qs))()
            keep = []
            for j, q in zip(jobs, qs):
                iv = todo[q][0].intervals[todo[q][1]]
                j.acc_0[:] = iv.first["acc"]; j.gyr_0[:] = iv.first["gyr"]; j.phi_0[:] = iv.first["phi"]; j.dphi_0[:] = iv.first["dphi"]; j.c_0[:] = iv.first["c"]
                j.linearized_ba[:] = iv.ba; j.linearized_bg[:] = iv.bg; j.linearized_rho[:] = iv.rho
                s = np.ascontiguousarray(iv.samples); keep.append(s)
                j.n_samples = len(s); j.samples = s.ctypes.data_as(C.POINTER(abi.IMULegSample))
            pcfg = todo[qs[0]][0].pcfg
            out = self.ops.preintegrate(pcfg, jobs, len(qs)) if use_leg else self.ops.preintegrate_imu(pcfg, jobs, len(qs))
            for k, q in enumerate(qs):
                iv = todo[q][0].intervals[todo[q][1]]
                iv.result = out[k].copy(); iv.dirty = False
        self.timing["preintegrate"] += time.perf_counter() - t0

    def step(self, images, firsts, samples, header):
        """processMeasurements for one camera frame of every robot: images[w], firsts[w] (sample at the previous frame instant),
        samples[w] (the interval's IMU + leg samples)."""
        import time
        T = self.timing
        t_host = time.perf_counter()
        for w, e in enumerate(self.est):
            e.process_interval(firsts[w], samples[w])
            e.Headers[e.frame_count] = header
            e.marginalization_flag = MARGIN_OLD if e.f_manager.addFeatureCheckParallax(e.frame_count, images[w], e.td) else MARGIN_SECOND_NEW
        T["host"] += time.perf_counter() - t_host
        self._preintegrate_dirty()
        # ---- f_manager.triangulate (estimator.cpp:803)
        t0 = time.perf_counter()
        ids_all = [fill_window(self.batch_all, w, e, min_used=1, with_prior=False) for w, e in enumerate(self.est)]
        for w, e in enumerate(self.est):
            lam = self.batch_all.para_Feature[w]
            for k, it in enumerate(f for f in e.f_manager.feature if len(f.feature_per_frame) >= 1):
                lam[k] = 1.0 / it.estimated_depth if it.estimated_depth > 0 else -1.0
        T["host"] += time.perf_counter() - t0
        t0 = time.perf_counter()
        depth = self.ops.triangulate(self.batch_all)
        T["triangulate"] += time.perf_counter() - t0
        t0 = time.perf_counter()
        for w, e in enumerate(self.est):
            by_id = {fid: depth[w, k] for k, fid in enumerate(ids_all[w])}
            for it in e.f_manager.feature:
                if not (it.estimated_depth > 0): it.estimated_depth = float(by_id[it.feature_id])
        # ---- optimization(): solve
        ids = [fill_window(self.batch, w, e) for w, e in enumerate(self.est)]
        before = (abi.WindowState * self.n)()
        C.memmove(before, self.batch.states, C.sizeof(before))
        T["host"] += time.perf_counter() - t0
        t0 = time.perf_counter()
        rep = self.ops.solve(self.batch)
        T["solve"] += time.perf_counter() - t0
        self.reports.append(rep.copy())
        t0 = time.perf_counter()
        for w, e in enumerate(self.est):
            Ps, Rs, Vs = self.ops.double2vector(before[w], self.batch.states[w])
            e.double2vector_rest(self.batch.states[w], self.batch.para_Feature[w], Ps, Rs, Vs)
        # ---- optimization(): marginalization at the re-anchored states (vector2double again, estimator.cpp:1251 / :1384)
        for w, e in enumerate(self.est):
            e.vector2double(self.batch.states[w], self.batch.para_Feature[w])
        flags = np.array([e.marginalization_flag for e in self.est], dtype=np.int32)
        self.flags.append(flags.copy())
        T["host"] += time.perf_counter() - t0
        t0 = time.perf_counter()
        self.ops.marginalize(self.batch, self.batch_next, flags)
        T["marginalize"] += time.perf_counter() - t0
        for w, e in enumerate(self.est):
            e.prior = take_prior(self.batch_next, w) if self.batch_next.descs[w].prior.valid else (e.prior if flags[w] == MARGIN_SECOND_NEW else None)
        # ---- outliersRejection + removeOutlier (:812-814)
        t0 = time.perf_counter()
        err = self.ops.outlier_errors(self.batch)
        T["outliers"] += time.perf_counter() - t0
        t0 = time.perf_counter()
        for w, e in enumerate(self.est):
            bad = {fid for k, fid in enumerate(ids[w]) if err[w, k] * FOCAL_LENGTH > 3}
            if bad: e.f_manager.removeOutlier(bad)
        # ---- slideWindow (+ removeBackShiftDepth on the backend for the robots that marginalize the oldest frame)
        ids2 = [fill_window(self.batch_all, w, e, min_used=1, with_prior=False) for w, e in enumerate(self.est)]
        for w, e in enumerate(self.est):
            lam = self.batch_all.para_Feature[w]
            for k, it in enumerate(e.f_manager.feature): lam[k] = 1.0 / it.estimated_depth
        T["host"] += time.perf_counter() - t0
        t0 = time.perf_counter()
        _, sdepth, _ = self.ops.shift_depth(self.batch_all)
        T["shift"] += time.perf_counter() - t0
        t0 = time.perf_counter()
        for w, e in enumerate(self.est):
            e.slide_window({fid: float(sdepth[w, k]) for k, fid in enumerate(ids2[w])})
            e.f_manager.removeFailures()
            W = WINDOW_SIZE
            e.path.append((header, e.Ps[W].copy(), e.Rs[W].copy(), e.Vs[W].copy(), e.Rho[W].copy()))
        T["host"] += time.perf_counter() - t0
        return rep

    def run(self, seq, n_steps=None):
        self.seed(seq)
        last = seq.n_frames if n_steps is None else min(seq.n_frames, WINDOW_SIZE + n_steps)
        for k in range(WINDOW_SIZE, last):
            if k == WINDOW_SIZE:
                # the seeded frame WINDOW_SIZE: its interval is already buffered; only the image is new
                firsts = [seq.first[w, k - 1] for w in range(self.n)]; smp = [seq.samples[w, k - 1][:0] for w in range(self.n)]
            else:
                firsts = [seq.first[w, k - 1] for w in range(self.n)]; smp = [seq.samples[w, k - 1] for w in range(self.n)]
            self.step([seq.images[k][w] for w in range(self.n)], firsts, smp, float(k))
        return self

    def poses(self):
        """[n, steps, 3] published positions and [n, steps, 3, 3] rotations of the newest frame."""
        P = np.array([[p[1] for p in e.path] for e in self.est]); R = np.array([[p[2] for p in e.path] for e in self.est])
        return P, R


class DeviceOps:
    """Backend adapter of ReplayDriver over one CerbHandle (cerberus_b200.lib.Backend): every numerical step of the frame loop is a call
    through the C ABI.  The handle's feature capacity must cover the triangulation batch (2 x the solve batch)."""

    def __init__(self, backend, cfg):
        self.be, self.cfg = backend, cfg

    def preintegrate(self, pcfg, jobs, n): return self.be.preintegrate(pcfg, jobs, n)
    def preintegrate_imu(self, pcfg, jobs, n): return self.be.preintegrate_imu(pcfg, jobs, n)
    def solve(self, batch): return self.be.solve_batch(batch)
    def double2vector(self, before, after): return self.be.double2vector(before, after)

    def triangulate(self, batch):
        self.be.upload(batch)
        return self.be.triangulate(batch.n, INIT_DEPTH)[:, :batch.max_features]

    def outlier_errors(self, batch):
        self.be.upload(batch)                           # the states were re-anchored by double2vector after the solve
        return self.be.outlier_errors(batch.n, FOCAL_LENGTH)[0][:, :batch.max_features]

    def shift_depth(self, batch):
        self.be.upload(batch)
        a, b, c = self.be.shift_depth(batch.n, INIT_DEPTH)
        F = batch.max_features
        return a[:, :F], b[:, :F], c[:, :F]

    def marginalize(self, src, dst, flags):
        self.be.marginalize(self.cfg, src, dst, margin_old=(np.asarray(flags) == MARGIN_OLD))


class NativeReplay:
    """The replay with the host side in C++ inside the library (csrc/replay_host.inl, cerb_replay_*): one call per camera frame, for all robots
    in lock step (same inputs and outputs as ReplayDriver(DeviceOps(...)); tests/test_replay.py compares the two) or for any subset of them,
    each at its own stamp (step(robots=, headers=)); a robot restarts with reset() + seed_robot() while the others keep stepping."""

    def __init__(self, backend, pcfg, n, max_features=160, estimate_extrinsic=1, estimate_td=0, resident=False):
        """resident=True: every robot's window stays on the device across frames (cerb_resident_*) and a step sends the frame's edits
        instead of three full uploads; same trajectories bit for bit."""
        self.be, self.n = backend, n
        self.r = C.c_void_p()
        backend._check(backend.lib.cerb_replay_create(backend.h, C.byref(pcfg), n, max_features, estimate_extrinsic, estimate_td, C.byref(self.r)))
        if resident:
            backend._check(backend.lib.cerb_replay_set_resident(self.r, 1))
        self.reports = []
        self._snap_cap = 1 << 19                      # save()'s first buffer, grown to the largest snapshot

    def close(self):
        if self.r:
            # cerb_replay_destroy unregisters the replay's host buffers from its handle.  When the replay and its Backend are garbage of
            # one reference cycle, their finalizers run in any order: if the handle is already destroyed, the replay's host object is
            # left to the process exit instead of being freed through a dangling handle.
            if self.be.h:
                self.be.lib.cerb_replay_destroy(self.r)
            self.r = C.c_void_p()

    def __del__(self):
        try: self.close()
        except Exception: pass

    @staticmethod
    def _image(img, keep):
        ids = np.ascontiguousarray(img["ids"], dtype=np.int64); p0 = np.ascontiguousarray(img["pts0"], dtype=np.float64)
        h1 = np.ascontiguousarray(img["has1"], dtype=np.uint8); p1 = np.ascontiguousarray(img["pts1"], dtype=np.float64)
        keep.extend([ids, p0, h1, p1])
        im = abi.Image(); im.n = len(ids)
        im.ids = ids.ctypes.data_as(C.POINTER(C.c_int64)); im.pts0 = p0.ctypes.data_as(abi.c_dp); im.has1 = h1.ctypes.data_as(C.POINTER(C.c_uint8)); im.pts1 = p1.ctypes.data_as(abi.c_dp)
        return im

    def seed(self, seq):
        for w in range(self.n):
            self.seed_robot(w, seq, w)

    def seed_robot(self, robot, seq, w, k0=0):
        """Seed robot `robot` with frames k0 .. k0 + WINDOW_SIZE of robot w of seq (stamps k0 + k), at any time: a robot just created or reset
        while the others keep stepping.  Its first step then takes frame k0 + WINDOW_SIZE's image with an empty interval."""
        L, _p = self.be.lib, lambda a: np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(abi.c_dp)
        tic, ric = np.ascontiguousarray(seq.tic_g[w]), np.ascontiguousarray(seq.ric_g[w])
        self.be._check(L.cerb_replay_set_extrinsics(self.r, robot, _p(tic), _p(ric)))
        for k in range(WINDOW_SIZE + 1):
            keep, K = [], k0 + k
            first = np.ascontiguousarray(seq.first[w, K if k == 0 else K - 1: (K + 1 if k == 0 else K)])
            smp = np.ascontiguousarray(seq.samples[w][K - 1]) if k > 0 else first[:0]
            im = self._image(seq.images[K][w], keep) if k < WINDOW_SIZE else None
            P, R, V = np.ascontiguousarray(seq.p_g[w, K]), np.ascontiguousarray(seq.R_g[w, K]), np.ascontiguousarray(seq.v_g[w, K])
            self.be._check(L.cerb_replay_seed_frame(self.r, robot, k, _p(P), _p(R), _p(V), first.ctypes.data, smp.ctypes.data if len(smp) else None, len(smp),
                                                    C.byref(im) if im is not None else None, float(K)))

    def configure(self, robot, use_leg, pcfg, estimate_extrinsic=1, estimate_td=0):
        """cerb_replay_configure_robot: robot `robot` runs the configuration of its own yaml, e.g. the reference's VINS baseline (use_leg = False:
        processIMU, IntegrationBase / IMUFactor, no leg-bias blocks) with abi.vins_preint_config().  Only before the robot is seeded (just
        created, or reset: a reset keeps the configuration)."""
        self.be._check(self.be.lib.cerb_replay_configure_robot(self.r, robot, 1 if use_leg else 0, C.byref(pcfg), estimate_extrinsic, estimate_td))

    def reset(self, robot):
        """The reference's estimator restart (clearState) for one robot; it is seeded again (seed_robot) before it steps."""
        self.be._check(self.be.lib.cerb_replay_reset_robot(self.r, robot))

    def save(self, robot):
        """cerb_replay_save_robot: a snapshot of a seeded robot (its state, prior and configuration, no path or flag history) as bytes.  It can
        be loaded into any robot of any NativeReplay of this library build, in either mode and on any handle."""
        L, size = self.be.lib, C.c_size_t()
        while True:                                   # one call unless the snapshot outgrew the largest one so far
            buf = C.create_string_buffer(self._snap_cap)
            rc = L.cerb_replay_save_robot(self.r, robot, buf, self._snap_cap, C.byref(size))
            if rc == 0: return buf.raw[:size.value]
            if size.value <= self._snap_cap: self.be._check(rc)
            self._snap_cap = size.value

    def load(self, robot, blob):
        """cerb_replay_load_robot: robot `robot` becomes the saved robot and continues as it would have; a rejected snapshot (CerbError)
        changes nothing."""
        blob = bytes(blob)
        self.be._check(self.be.lib.cerb_replay_load_robot(self.r, robot, blob, len(blob)))

    def clone(self, src, dsts):
        """cerb_replay_clone_robot: robots `dsts` become copies of robot `src` (a save and a load each, in one batched call)."""
        d = np.ascontiguousarray(dsts, dtype=np.int32)
        self.be._check(self.be.lib.cerb_replay_clone_robot(self.r, src, len(d), d.ctypes.data_as(C.POINTER(C.c_int32))))

    def step(self, images, firsts, samples, header, robots=None, headers=None):
        """One camera frame of every robot at stamp `header`, or of the robots listed in `robots` (each at its own stamp headers[i] if given);
        images / firsts / samples are in the order of `robots`.  self.reports gets the step's solve reports in that order."""
        keep = []
        m = self.n if robots is None else len(robots)
        ims = (abi.Image * m)(*[self._image(images[i], keep) for i in range(m)])
        fr = np.ascontiguousarray(np.stack([np.asarray(firsts[i]).reshape(()) for i in range(m)]))
        smp = [np.ascontiguousarray(samples[i]) for i in range(m)]
        ptrs = (C.c_void_p * m)(*[s.ctypes.data if len(s) else None for s in smp])
        ns = (C.c_int32 * m)(*[len(s) for s in smp])
        rep = (abi.SolveReport * m)()
        if robots is None and headers is None:
            self.be._check(self.be.lib.cerb_replay_step(self.r, ims, fr.ctypes.data, ptrs, ns, float(header), rep))
        else:
            rob = np.ascontiguousarray(np.arange(self.n) if robots is None else robots, dtype=np.int32)
            hdr = np.ascontiguousarray(np.full(m, float(header)) if headers is None else headers, dtype=np.float64)
            self.be._check(self.be.lib.cerb_replay_step_robots(self.r, m, rob.ctypes.data_as(C.POINTER(C.c_int32)), ims, fr.ctypes.data, ptrs, ns,
                                                               hdr.ctypes.data_as(abi.c_dp), rep))
        self.reports.append(np.frombuffer(rep, dtype=abi.report_dtype, count=m).copy())

    def run(self, seq, n_steps=None):
        self.seed(seq)
        last = seq.n_frames if n_steps is None else min(seq.n_frames, WINDOW_SIZE + n_steps)
        for k in range(WINDOW_SIZE, last):
            firsts = [seq.first[w, k - 1] for w in range(self.n)]
            smp = [seq.samples[w][k - 1][:0] if k == WINDOW_SIZE else seq.samples[w][k - 1] for w in range(self.n)]
            self.step([seq.images[k][w] for w in range(self.n)], firsts, smp, float(k))
        return self

    def path(self, w):
        n = C.c_int32()
        self.be._check(self.be.lib.cerb_replay_path(self.r, w, C.byref(n), None, 0))
        out = np.zeros((n.value, 20))
        self.be._check(self.be.lib.cerb_replay_path(self.r, w, C.byref(n), out.ctypes.data_as(abi.c_dp), n.value))
        return out

    def poses(self):
        rows = np.stack([self.path(w) for w in range(self.n)])
        return rows[:, :, 1:4], rows[:, :, 4:13].reshape(self.n, -1, 3, 3)

    def feature_ids(self, w):
        n = C.c_int32(); ids = np.zeros(4096, dtype=np.int32)
        self.be._check(self.be.lib.cerb_replay_feature_ids(self.r, w, C.byref(n), ids.ctypes.data_as(C.POINTER(C.c_int32)), ids.size))
        return ids[:n.value].tolist()

    def flag_history(self, w):
        n = C.c_int32(); out = np.zeros(4096, dtype=np.int32)
        self.be._check(self.be.lib.cerb_replay_flags(self.r, w, C.byref(n), out.ctypes.data_as(C.POINTER(C.c_int32)), out.size))
        return out[:n.value]

    def timing(self):
        dev = np.zeros(6); host = C.c_double()
        self.be._check(self.be.lib.cerb_replay_timing(self.r, dev.ctypes.data_as(abi.c_dp), C.cast(C.byref(host), abi.c_dp)))
        return dict(zip(("preintegrate", "triangulate", "solve", "marginalize", "outliers", "shift"), dev.tolist()), host=host.value)

    def traffic(self):
        """What the steps so far asked the library to move: bytes host -> device and device -> host, copy operations, and the bytes of it
        that went through a staging memcpy on the host."""
        v = [C.c_int64() for _ in range(4)]
        self.be._check(self.be.lib.cerb_replay_traffic(self.r, *[C.byref(x) for x in v]))
        return dict(zip(("h2d_bytes", "d2h_bytes", "dma_ops", "staged_bytes"), [x.value for x in v]))

    def window(self, w):
        """cerb_replay_window: (features, ids, obs, preint [10] (IMU-leg or IMU records by the robot's kind), preint_current [10], pre_slots [10], Prior, prior_J [n, n], prior_r [n]) of
        robot w as the replay would upload it for a per-feature step; in resident mode obs / preint are empty and prior carries valid only."""
        d = abi.WindowDesc(); ids = np.zeros(4096, dtype=np.int32); cur = np.zeros(WINDOW_SIZE, dtype=np.int32); slots = np.zeros(WINDOW_SIZE, dtype=np.int32)
        i32p = C.POINTER(C.c_int32)
        self.be._check(self.be.lib.cerb_replay_window(self.r, w, C.byref(d), ids.ctypes.data_as(i32p), ids.size, cur.ctypes.data_as(i32p), slots.ctypes.data_as(i32p)))
        take = lambda ptr, n, dt: np.ctypeslib.as_array(ptr, shape=(n,)).view(dt).reshape(n).copy() if n else np.zeros(0, dtype=dt)
        feats = take(d.features, d.n_features, abi.feature_dtype); obs = take(d.obs, d.n_obs, abi.obs_dtype)
        pre = np.zeros(0, dtype=abi.preint_dtype)
        if d.n_obs:                                   # IMU records for a robot configured with use_leg = False
            pre = take(d.preint, WINDOW_SIZE, abi.preint_dtype) if d.preint else take(d.imu_preint, WINDOW_SIZE, abi.imu_preint_dtype)
        n = d.prior.n if (d.prior.valid and d.prior.linearized_jacobians) else 0
        J = np.ctypeslib.as_array(d.prior.linearized_jacobians, shape=(n * n,)).reshape(n, n).T.copy() if n else np.zeros((0, 0))
        r = np.ctypeslib.as_array(d.prior.linearized_residuals, shape=(n,)).copy() if n else np.zeros(0)
        return feats, ids[:d.n_features], obs, pre, cur, slots, d.prior, J, r


def write_csv(path, est, pcfg):
    """The result file of the reference's main loop (src/main.cpp:153-197): time [ns], robot-body position / velocity (IMU pose moved
    by R_br p_br), six Kalman-filter columns and three mocap columns (not produced here: 0), rho1..rho4 of the newest frame."""
    R_br = np.array([pcfg.R_br[k] for k in range(9)]).reshape(3, 3); p_br = np.array([pcfg.p_br[k] for k in range(3)])
    with open(path, "a") as f:
        for (t, P, R, V, rho) in est.path:
            p_wr = P + R @ R_br @ p_br
            f.write(f"{t * 1e9:.0f}," + ",".join(f"{v:.5f}" for v in list(p_wr) + list(V) + [0.0] * 9 + list(rho)) + ",\n")

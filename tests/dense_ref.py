"""Dense extended-precision reference of one window's solve -- TEST INFRASTRUCTURE.

What it restates, and from where:
  * The factor list of Estimator::optimization() (the reference's estimator.cpp:1107-1216): the marginalization prior; one IMU(-leg)
    factor i -> i+1 unless its preintegration spans sum_dt > 10 s; per track, K1 (ProjectionTwoFrameOneCamFactor) for every non-anchor
    observation, K2 (ProjectionTwoFrameTwoCamFactor) for every stereo non-anchor observation and K3 (ProjectionOneFrameTwoCamFactor)
    for a stereo anchor observation, all three under HuberLoss(huber_delta).  It is written here in numpy from the descriptors; the
    residuals and Jacobians of each factor come from the oracle's per-factor evaluators (eval_projection, eval_imu_leg / eval_imu,
    eval_prior), which tests/test_reference_pin.py pins against the reference's own sources.  The oracle's window assembly
    (oracle/ref_window.cpp) and its solver (oracle/ref_solver.cpp) are not used.
  * Ceres' ResidualBlock / Corrector (corrector.cc) for the loss, and PoseLocalParameterization (Plus, and a ComputeJacobian that keeps
    the first 6 of the 7 global columns).
  * Ceres 1.14's TrustRegionMinimizer with DoglegStrategy (TRADITIONAL_DOGLEG): Jacobi scaling fixed at iteration 0, the dogleg
    diagonal clamped to [1e-6, 1e32], the Cauchy point, the Gauss-Newton step of (Js^T Js + mu D^2) y = Js^T r, the three dogleg cases,
    the mu retry / update, the radius update, accept / reject with reuse of the step, and the parameter / function tolerances.
    Ceres itself is not built: this is a restatement of its documented algorithm, as the oracle is.

The linear algebra does not restate the Schur elimination of the inverse depths.  The full normal equations are assembled factor by
factor in np.longdouble (80-bit extended precision on x86-64, eps = 1.1e-19; require_extended_precision() fails loudly where it is plain
double), solved by LAPACK in fp64 and refined with residuals in longdouble until the correction is below 1e-3 of kappa * eps64 of the
solution, the rounding scale every tolerance derived from it is a multiple of.

Columns are in the order of cerb_debug_linearize: [pose0..10 (66) | ex0, ex1 (12) | speedbias0..10 (99) | legbias0..10 (44) | td |
inverse depths]; a constant block keeps its columns, which stay zero.

Every iteration of `solve` records the iterate, its cost, the step, the dogleg case, mu, the radius, kappa (2-norm condition number of
the scaled, regularised system on its coupled columns) and the decision margins with the rounding uncertainty of each.
"""
import ctypes as C
import numpy as np
import scipy.linalg
from cerberus_b200 import abi

LD = np.longdouble
EPS64 = float(np.finfo(np.float64).eps)
NR = abi.NUM_REDUCED
COST_REL_UNC = 1e-12        # relative rounding of an fp64 cost summed over ~1e4 factors (the linearisation tests hold it to 1e-12)


def require_extended_precision():
    assert np.finfo(LD).eps < 1e-18, f"np.longdouble is not extended precision here (eps = {np.finfo(LD).eps}); the dense reference needs it"


# ---------------------------------------------------------------------------------------------------------------- state
class State:
    """The parameter blocks of one window, as plain arrays."""

    def __init__(self, pose, sb, lb, ex, td, lam):
        self.pose, self.sb, self.lb, self.ex, self.td, self.lam = pose, sb, lb, ex, td, lam

    @staticmethod
    def from_batch(batch, w):
        st = batch.state_array()[w]
        nf = batch.descs[w].n_features
        return State(st["para_Pose"].copy(), st["para_SpeedBias"].copy(), st["para_LegBias"].copy(), st["para_Ex_Pose"].copy(),
                     st["para_Td"].copy(), batch.para_Feature[w][:nf].copy())

    def copy(self):
        return State(*(a.copy() for a in (self.pose, self.sb, self.lb, self.ex, self.td, self.lam)))

    def struct(self):
        """An abi.WindowState of this state (its para_Feature points into a copy kept alive by the returned object)."""
        s = abi.WindowState()
        for name, a in (("para_Pose", self.pose), ("para_SpeedBias", self.sb), ("para_LegBias", self.lb), ("para_Ex_Pose", self.ex)):
            C.memmove(C.byref(getattr(s, name)), np.ascontiguousarray(a).ctypes.data, a.nbytes)
        s.para_Td[0] = self.td[0]
        s._lam = np.ascontiguousarray(self.lam if self.lam.size else np.zeros(1))
        s.para_Feature = s._lam.ctypes.data_as(abi.c_dp)
        return s

    def global_vector(self, blocks):
        """The global (7-wide pose) coordinates of the active blocks, the vector Ceres' parameter tolerance measures."""
        parts = [self.pose.ravel(), self.sb.ravel()]
        if blocks["lb"]: parts.append(self.lb.ravel())
        if blocks["ex"]: parts.append(self.ex.ravel())
        if blocks["td"]: parts.append(self.td)
        parts.append(self.lam)
        return np.concatenate(parts)


def quat_mul(a, b):
    """Hamilton product of (x, y, z, w) quaternions, [..., 4]."""
    ax, ay, az, aw = np.moveaxis(a, -1, 0)
    bx, by, bz, bw = np.moveaxis(b, -1, 0)
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def pose_plus(x, d):
    """PoseLocalParameterization::Plus: p + dp, (q * [dtheta / 2, 1]).normalized(); x [..., 7], d [..., 6]."""
    dq = np.concatenate([0.5 * d[..., 3:6], np.ones(d.shape[:-1] + (1,))], axis=-1)
    q = quat_mul(x[..., 3:7], dq)
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    return np.concatenate([x[..., :3] + d[..., :3], q], axis=-1)


def plus(x, delta, blocks):
    """Evaluator::Plus over the ABI tangent vector `delta` (constant blocks are left alone, as Ceres leaves them)."""
    y = x.copy()
    y.pose = pose_plus(x.pose, delta[:66].reshape(11, 6))
    y.sb = x.sb + delta[78:177].reshape(11, 9)
    if blocks["lb"]: y.lb = x.lb + delta[177:221].reshape(11, 4)
    if blocks["ex"]: y.ex = pose_plus(x.ex, delta[66:78].reshape(2, 6))
    if blocks["td"]: y.td = x.td + delta[221:222]
    y.lam = x.lam + delta[NR:]
    return y


# ---------------------------------------------------------------------------------------------------------------- the window
def huber_corrector(delta, s):
    """ceres::HuberLoss(delta) and Corrector (corrector.cc) for squared norms s: (0.5 rho(s), sqrt(rho'), residual scaling, alpha / s)."""
    b = delta * delta
    rt = np.sqrt(s)
    out = s > b
    rho0 = np.where(out, 2.0 * delta * rt - b, s)
    with np.errstate(divide="ignore", invalid="ignore"):
        rho1 = np.where(out, np.maximum(np.finfo(np.float64).tiny, delta / np.where(out, rt, 1.0)), 1.0)
        rho2 = np.where(out, -rho1 / (2.0 * np.where(out, s, 1.0)), 0.0)
        sqrt_rho1 = np.sqrt(rho1)
        plain = (s == 0.0) | (rho2 <= 0.0)
        D = 1.0 + 2.0 * s * rho2 / rho1
        alpha = 1.0 - np.sqrt(np.where(plain, 1.0, D))
        scaling = np.where(plain, sqrt_rho1, sqrt_rho1 / (1.0 - alpha))
        alpha_sq_norm = np.where(plain, 0.0, alpha / np.where(plain, 1.0, s))
    return 0.5 * rho0, sqrt_rho1, scaling, alpha_sq_norm


class Factors:
    """One evaluated group of same-shaped factors: residuals r [n, m], local Jacobian J [n, m, c], ABI column of each local column
    [n, c] (-1: a constant block), and whether the rows are under the Huber loss."""

    def __init__(self, name, r, J, cols, huber):
        self.name, self.r, self.J, self.cols, self.huber = name, r, J, cols, huber


class DenseWindow:
    """Window w of `batch` under `cfg`, evaluated through the oracle's per-factor evaluators `ob` (an oracle_lib.OracleBackend)."""

    def __init__(self, batch, w, cfg, ob):
        require_extended_precision()
        self.cfg, self.ob = cfg, ob
        d = batch.descs[w]
        self.nf = d.n_features
        self.n = NR + self.nf
        self.use_leg = batch.imu_preint is None
        self.blocks = {"ex": bool(d.extrinsic_open), "td": bool(d.td_open), "lb": self.use_leg and bool(cfg.optimize_leg_bias)}
        self.x0 = State.from_batch(batch, w)
        self.g = tuple(cfg.g)
        # prior (estimator.cpp:1107-1113): the descriptor itself, with its matrices copied
        self.prior = None
        if d.prior.valid:
            pr = abi.Prior.from_buffer_copy(d.prior)
            self._prior_J = batch.prior_J[w].copy(); self._prior_r = batch.prior_r[w].copy()
            pr.linearized_jacobians = self._prior_J.ctypes.data_as(abi.c_dp); pr.linearized_residuals = self._prior_r.ctypes.data_as(abi.c_dp)
            self.prior = pr
        # IMU(-leg) factors i -> i + 1, skipped when sum_dt > 10 (estimator.cpp:1114-1171)
        pre = batch.preint[w] if self.use_leg else batch.imu_preint[w]
        self.imu = [i for i in range(abi.WINDOW_SIZE) if not pre[i]["sum_dt"] > 10.0]
        self.pre = np.ascontiguousarray(pre[self.imu])
        # visual factors (estimator.cpp:1173-1216)
        feats, obs = batch.features[w][:self.nf], batch.obs[w]
        k1, k2, k3 = [], [], []
        for f in range(self.nf):
            a, L, off = int(feats[f]["start_frame"]), int(feats[f]["n_obs"]), int(feats[f]["obs_offset"])
            for k in range(L):
                o = off + k
                if k > 0: k1.append((f, a, a + k, off, o))
                if obs[o]["is_stereo"]:
                    (k2 if k > 0 else k3).append((f, a, a + k, off, o))
        self.vis = []
        for kind, lst in ((abi.PROJ_TWO_FRAME_ONE_CAM, k1), (abi.PROJ_TWO_FRAME_TWO_CAM, k2), (abi.PROJ_ONE_FRAME_TWO_CAM, k3)):
            if not lst:
                continue
            t = np.array(lst, dtype=np.int64)
            o0, o = obs[t[:, 3]], obs[t[:, 4]]
            right = kind != abi.PROJ_TWO_FRAME_ONE_CAM
            pts_j = o["pointRight"] if right else o["point"]
            vel_j = o["velocityRight"] if right else o["velocity"]
            const = dict(pts_i=np.ascontiguousarray(np.c_[o0["point"], np.ones(len(t))]), pts_j=np.ascontiguousarray(np.c_[pts_j, np.ones(len(t))]),
                         vel_i=np.ascontiguousarray(o0["velocity"]), vel_j=np.ascontiguousarray(vel_j),
                         td_i=np.ascontiguousarray(o0["cur_td"]), td_j=np.ascontiguousarray(o["cur_td"]))
            self.vis.append((kind, t[:, 0], t[:, 1], t[:, 2], const))
        self.counts = {"K1": len(k1), "K2": len(k2), "K3": len(k3), "imu": len(self.imu), "prior": int(self.prior is not None)}

    # ---- columns -------------------------------------------------------------------------------------------------------
    def _pose_cols(self, i):
        return 6 * np.asarray(i)[..., None] + np.arange(6)

    def _ex_cols(self, k, n):
        return np.tile(66 + 6 * k + np.arange(6), (n, 1)) if self.blocks["ex"] else np.full((n, 6), -1)

    def _td_cols(self, n):
        return np.full((n, 1), 221 if self.blocks["td"] else -1)

    def active_columns(self):
        m = np.zeros(self.n, dtype=bool)
        m[:66] = True; m[78:177] = True; m[NR:] = True
        m[66:78] = self.blocks["ex"]; m[177:221] = self.blocks["lb"]; m[221] = self.blocks["td"]
        return m

    # ---- evaluation ----------------------------------------------------------------------------------------------------
    def evaluate(self, x):
        """All factors at state x, as a list of Factors (Jacobians already local and Huber-corrected, residuals corrected)."""
        out = []
        if self.prior is not None:
            pr = self.prior
            n = pr.n
            loc = {abi.BLOCK_POSE: (7, 6), abi.BLOCK_SPEEDBIAS: (9, 9), abi.BLOCK_LEGBIAS: (4, 4), abi.BLOCK_EX_POSE: (7, 6), abi.BLOCK_TD: (1, 1)}
            ncols = sum(loc[pr.block_kind[b]][0] for b in range(pr.num_blocks))
            r, jac = self.ob.eval_prior(pr, x.struct(), ncols)
            Js, cols, off = [], [], 0
            for b in range(pr.num_blocks):
                kind, idx = pr.block_kind[b], pr.block_index[b]
                gsz, lsz = loc[kind]
                Js.append(jac[off:off + n * gsz].reshape(n, gsz)[:, :lsz]); off += n * gsz
                base = {abi.BLOCK_POSE: 6 * idx, abi.BLOCK_SPEEDBIAS: 78 + 9 * idx, abi.BLOCK_LEGBIAS: 177 + 4 * idx, abi.BLOCK_EX_POSE: 66 + 6 * idx, abi.BLOCK_TD: 221}[kind]
                on = {abi.BLOCK_LEGBIAS: self.blocks["lb"], abi.BLOCK_EX_POSE: self.blocks["ex"], abi.BLOCK_TD: self.blocks["td"]}.get(kind, True)
                cols.append(base + np.arange(lsz) if on else np.full(lsz, -1))
            out.append(Factors("prior", r[None], np.concatenate(Js, axis=1)[None], np.concatenate(cols)[None], False))
        if self.imu:
            i = np.array(self.imu); j = i + 1; n = len(i)
            if self.use_leg:
                params = np.concatenate([x.pose[i], x.sb[i], x.lb[i], x.pose[j], x.sb[j], x.lb[j]], axis=1)
                r, jac, _ = self.ob.eval_imu_leg(self.pre, np.ascontiguousarray(params), g=self.g)
                jac = jac.reshape(n, 31 * 40)
                spans = [(0, 7, 6), (7, 9, 9), (16, 4, 4), (20, 7, 6), (27, 9, 9), (36, 4, 4)]
                lbc = lambda f: (177 + 4 * f[:, None] + np.arange(4)) if self.blocks["lb"] else np.full((n, 4), -1)
                cols = [self._pose_cols(i), 78 + 9 * i[:, None] + np.arange(9), lbc(i), self._pose_cols(j), 78 + 9 * j[:, None] + np.arange(9), lbc(j)]
                m = 31
            else:
                params = np.concatenate([x.pose[i], x.sb[i], x.pose[j], x.sb[j]], axis=1)
                r, jac, _ = self.ob.eval_imu(self.pre, np.ascontiguousarray(params), g=self.g)
                spans = [(0, 7, 6), (7, 9, 9), (16, 7, 6), (23, 9, 9)]
                cols = [self._pose_cols(i), 78 + 9 * i[:, None] + np.arange(9), self._pose_cols(j), 78 + 9 * j[:, None] + np.arange(9)]
                m = 15
            J = np.concatenate([jac[:, m * s0:m * (s0 + g)].reshape(n, m, g)[:, :, :l] for s0, g, l in spans], axis=2)
            out.append(Factors("imu", r, J, np.concatenate(cols, axis=1), False))
        for kind, f, a, jf, c in self.vis:
            n = len(f)
            lam, td = np.ascontiguousarray(x.lam[f]), np.full(n, x.td[0])
            ex0, ex1 = np.tile(x.ex[0], (n, 1)), np.tile(x.ex[1], (n, 1))
            r, jac = self.ob.eval_projection(kind, np.ascontiguousarray(x.pose[a]), np.ascontiguousarray(x.pose[jf]), ex0, ex1, lam, td,
                                             c["pts_i"], c["pts_j"], c["vel_i"], c["vel_j"], c["td_i"], c["td_j"], sqrt_info=self.cfg.visual_sqrt_info)
            lamc, tdc = (NR + f)[:, None], self._td_cols(n)
            if kind == abi.PROJ_TWO_FRAME_ONE_CAM:
                J = np.concatenate([jac[:, 0:14].reshape(n, 2, 7)[..., :6], jac[:, 14:28].reshape(n, 2, 7)[..., :6], jac[:, 28:42].reshape(n, 2, 7)[..., :6],
                                    jac[:, 42:44].reshape(n, 2, 1), jac[:, 44:46].reshape(n, 2, 1)], axis=2)
                cols = np.concatenate([self._pose_cols(a), self._pose_cols(jf), self._ex_cols(0, n), lamc, tdc], axis=1)
            elif kind == abi.PROJ_TWO_FRAME_TWO_CAM:
                J = np.concatenate([jac[:, 14 * k:14 * k + 14].reshape(n, 2, 7)[..., :6] for k in range(4)] +
                                   [jac[:, 56:58].reshape(n, 2, 1), jac[:, 58:60].reshape(n, 2, 1)], axis=2)
                cols = np.concatenate([self._pose_cols(a), self._pose_cols(jf), self._ex_cols(0, n), self._ex_cols(1, n), lamc, tdc], axis=1)
            else:
                J = np.concatenate([jac[:, 0:14].reshape(n, 2, 7)[..., :6], jac[:, 14:28].reshape(n, 2, 7)[..., :6],
                                    jac[:, 28:30].reshape(n, 2, 1), jac[:, 30:32].reshape(n, 2, 1)], axis=2)
                cols = np.concatenate([self._ex_cols(0, n), self._ex_cols(1, n), lamc, tdc], axis=1)
            out.append(Factors({0: "K1", 1: "K2", 2: "K3"}[kind], r, J, cols, True))
        for fa in out:
            fa.sq = (fa.r * fa.r).sum(axis=1)
            if fa.huber:
                fa.cost, sqrt_rho1, scaling, asn = huber_corrector(self.cfg.huber_delta, fa.sq)
                rtj = np.einsum("nm,nmc->nc", fa.r, fa.J)                               # Corrector::CorrectJacobian
                fa.J = sqrt_rho1[:, None, None] * (fa.J - asn[:, None, None] * fa.r[:, :, None] * rtj[:, None, :])
                fa.r = fa.r * scaling[:, None]                                          # Corrector::CorrectResiduals
            else:
                fa.cost = 0.5 * fa.sq
        return out

    def cost(self, x):
        return float(sum(np.sum(fa.cost.astype(LD)) for fa in self.evaluate(x)))

    def linearize(self, x):
        """(cost, gradient J^T r [n], normal matrix J^T J [n, n]) at x in ABI column order, accumulated in longdouble per factor."""
        n = self.n
        H = np.zeros((n + 1, n + 1), dtype=LD)         # row / column n collects the (dropped) constant-block columns
        g = np.zeros(n + 1, dtype=LD)
        cost = LD(0)
        for fa in self.evaluate(x):
            cost += np.sum(fa.cost.astype(LD))
            J, r = fa.J.astype(LD), fa.r.astype(LD)
            cols = np.where(fa.cols < 0, n, fa.cols)
            np.add.at(H, (cols[:, :, None], cols[:, None, :]), np.einsum("nmi,nmj->nij", J, J))
            np.add.at(g, cols, np.einsum("nmi,nm->ni", J, r))
        return float(cost), g[:n], H[:n, :n]

    def dense_jacobian(self, x):
        """(J [rows, n], r [rows]) in fp64: only for small windows (the least-squares and mpmath checks)."""
        Js, rs = [], []
        for fa in self.evaluate(x):
            m = fa.r.shape[1]
            for k in range(fa.r.shape[0]):
                Jk = np.zeros((m, self.n))
                for c in range(fa.cols.shape[1]):
                    if fa.cols[k, c] >= 0:
                        Jk[:, fa.cols[k, c]] += fa.J[k, :, c]
                Js.append(Jk); rs.append(fa.r[k])
        return np.concatenate(Js), np.concatenate(rs)

    # ---- the trust-region solve ----------------------------------------------------------------------------------------
    def solve(self, max_iterations=None, initial_radius=None, min_relative_decrease=None, initial_mu=None):
        """Ceres 1.14 TrustRegionMinimizer + DoglegStrategy (TRADITIONAL_DOGLEG) from x0.  Returns a Trace."""
        cfg = self.cfg
        K = cfg.max_num_iterations if max_iterations is None else max_iterations
        mrd = cfg.min_relative_decrease if min_relative_decrease is None else min_relative_decrease
        act = np.flatnonzero(self.active_columns())
        x = self.x0.copy()
        cost, g, H = self.linearize(x)
        Ha, ga = H[np.ix_(act, act)], g[act]
        scaling = (1.0 / (1.0 + np.sqrt(np.diagonal(Ha).astype(np.float64)))).astype(LD)      # Jacobi scaling, fixed at iteration 0
        tr = Trace(self, act, cost, g, H)
        radius = cfg.initial_trust_region_radius if initial_radius is None else initial_radius
        mu, min_mu, max_mu = (1e-8 if initial_mu is None else initial_mu), 1e-8, 1.0
        reuse, invalid, it, nsucc = False, 0, 0, 0
        x_norm = np.linalg.norm(x.global_vector(self.blocks))
        step_ok = False
        lin = None
        while True:
            if step_ok: nsucc += 1
            gmax = float(np.abs(ga).max()) if ga.size else 0.0
            if it >= K: tr.finish(it, nsucc, abi.TERM_NO_CONVERGENCE, cost); break
            tr.margin(it + 1, "gradient_tolerance", gmax - cfg.gradient_tolerance, EPS64 * gmax)
            if gmax <= cfg.gradient_tolerance: tr.finish(it, nsucc, abi.TERM_CONVERGENCE, cost); break
            if radius <= cfg.min_trust_region_radius: tr.finish(it, nsucc, abi.TERM_CONVERGENCE, cost); break
            it += 1
            step_ok = False
            rec = {"k": it, "radius": radius, "reuse": reuse}
            # ---- DoglegStrategy::ComputeStep
            if not reuse:
                reuse = True
                A = scaling[:, None] * Ha * scaling[None, :]                           # Js^T Js
                bs = scaling * ga                                                      # Js^T r
                D = np.sqrt(np.clip(np.diagonal(A).astype(np.float64), 1e-6, 1e32)).astype(LD)
                grad = bs / D
                v = grad / D
                alpha = float(np.dot(grad, grad) / np.dot(v, A @ v))                   # Cauchy point
                gn, solved = None, False
                while mu < max_mu:
                    Areg = A + np.diag(mu * D * D)
                    kappa = coupled_condition(Areg)
                    y = refined_solve(Areg, bs, 1e-3 * kappa * EPS64)
                    if y is not None:
                        solved = True
                        break
                    mu *= 10.0
                if not solved:
                    lin = None
                else:
                    gn = -D * y
                    lin = dict(A=A, bs=bs, D=D, grad=grad, alpha=alpha, gn=gn, mu=mu, kappa=kappa, y=y)
            if lin is None:
                rec.update(case="invalid"); tr.steps.append(rec)
                invalid += 1
                if invalid >= 5: tr.finish(it, nsucc, abi.TERM_FAILURE, cost); break
                mu *= 10.0; reuse = False
                continue
            step, case, step_norm_s = dogleg(lin, radius, tr, it)
            rec.update(case=case, mu=lin["mu"], kappa=lin["kappa"], alpha=lin["alpha"], gn_norm=float(np.sqrt(np.dot(lin["gn"], lin["gn"]))),
                       grad_norm=float(np.sqrt(np.dot(lin["grad"], lin["grad"]))))
            model = float(-(np.dot(step, lin["bs"]) + 0.5 * np.dot(step, lin["A"] @ step)))
            rec["model_cost_change"] = model
            tr.margin(it, "model_cost_change", model, COST_REL_UNC * cost)
            if not model > 0.0:
                rec.update(valid=False); tr.steps.append(rec)
                invalid += 1
                if invalid >= 5: tr.finish(it, nsucc, abi.TERM_FAILURE, cost); break
                mu *= 10.0; reuse = False
                continue
            invalid = 0
            delta = np.zeros(self.n)
            delta[act] = (step * scaling).astype(np.float64)
            rec["delta_norm"] = float(np.linalg.norm(delta))
            cand = plus(x, delta, self.blocks)
            ccost = self.cost(cand)
            xv, cv = x.global_vector(self.blocks), cand.global_vector(self.blocks)
            step_norm = float(np.linalg.norm(xv - cv))
            ptol = cfg.parameter_tolerance * (x_norm + cfg.parameter_tolerance)
            tr.margin(it, "parameter_tolerance", step_norm - ptol, lin["kappa"] * EPS64 * step_norm)
            rec.update(candidate_cost=ccost, x_cost=cost)
            if step_norm <= ptol:
                rec["outcome"] = "parameter_tolerance"; tr.steps.append(rec); tr.finish(it, nsucc, abi.TERM_CONVERGENCE, cost); break
            change = cost - ccost
            tr.margin(it, "function_tolerance", abs(change) - cfg.function_tolerance * cost, COST_REL_UNC * cost)
            if abs(change) <= cfg.function_tolerance * cost:
                rec["outcome"] = "function_tolerance"; tr.steps.append(rec); tr.finish(it, nsucc, abi.TERM_CONVERGENCE, cost); break
            q = change / model
            q_unc = COST_REL_UNC * cost / model + lin["kappa"] * EPS64
            rec["q"] = q
            tr.margin(it, "min_relative_decrease", q - mrd, q_unc)
            if q > mrd:
                tr.margin(it, "decrease_threshold", q - 0.25, q_unc)
                tr.margin(it, "increase_threshold", q - 0.75, q_unc)
                x, cost = cand, ccost
                x_norm = np.linalg.norm(x.global_vector(self.blocks))
                _, g, H = self.linearize(x)
                Ha, ga = H[np.ix_(act, act)], g[act]
                step_ok = True
                if q < 0.25: radius *= 0.5                                              # DoglegStrategy::StepAccepted
                if q > 0.75: radius = max(radius, 3.0 * step_norm_s)
                mu = max(min_mu, 2.0 * mu / 10.0)
                reuse = False
                rec["outcome"] = "accepted"
            else:
                radius *= 0.5                                                           # DoglegStrategy::StepRejected
                reuse = True
                rec["outcome"] = "rejected"
            rec["x"] = x.copy(); rec["cost"] = cost
            tr.steps.append(rec)
        tr.x_final = x
        return tr


def refined_solve(A, b, rtol, max_rounds=40):
    """Solve A y = b (A symmetric positive definite in longdouble): LAPACK Cholesky in fp64, then refinement with longdouble residuals
    until the correction is below rtol * |y| (the callers pass 1e-3 of the tolerance the step feeds, kappa * eps64).  None where the fp64
    factorisation fails (Ceres: LINEAR_SOLVER_FAILURE)."""
    try:
        cf = scipy.linalg.cho_factor(A.astype(np.float64), lower=True, check_finite=True)
    except (np.linalg.LinAlgError, ValueError):
        return None
    y = scipy.linalg.cho_solve(cf, b.astype(np.float64)).astype(LD)
    for _ in range(max_rounds):
        res = b - A @ y
        dy = scipy.linalg.cho_solve(cf, res.astype(np.float64))
        y = y + dy.astype(LD)
        if np.linalg.norm(dy) <= rtol * float(np.sqrt(np.dot(y, y))):
            return y
    raise AssertionError("iterative refinement did not converge: the system is too ill-conditioned for a longdouble residual")


def coupled_condition(A):
    """2-norm condition number of A on the columns that carry information (a column with no factor is decoupled: its row and column
    are zero but for the mu D^2 floor, and it cannot spread rounding into the others)."""
    A64 = A.astype(np.float64)
    off = np.abs(A64 - np.diag(np.diagonal(A64))).sum(axis=1)
    keep = off > 0
    if not keep.any():
        return 1.0
    ev = scipy.linalg.eigvalsh(A64[np.ix_(keep, keep)], check_finite=False)     # A is symmetric positive definite
    return float(ev[-1] / ev[0])


def dogleg(lin, radius, tr, k):
    """DoglegStrategy::ComputeTraditionalDoglegStep: (step in the Jacobi-scaled space, case, dogleg_step_norm)."""
    grad, gn, D, alpha = lin["grad"], lin["gn"], lin["D"], lin["alpha"]
    gnorm = float(np.sqrt(np.dot(grad, grad))); gn_norm = float(np.sqrt(np.dot(gn, gn)))
    unc = lin["kappa"] * EPS64
    tr.margin(k, "gauss_newton_in_radius", gn_norm - radius, unc * max(gn_norm, radius))
    if gn_norm <= radius:
        return gn / D, "gauss_newton", gn_norm
    tr.margin(k, "cauchy_outside_radius", alpha * gnorm - radius, unc * max(alpha * gnorm, radius))
    if gnorm * alpha >= radius:
        return -(LD(radius) / LD(gnorm)) * grad / D, "gradient", radius
    b_dot_a = -alpha * float(np.dot(grad, gn))
    a2 = (alpha * gnorm) ** 2
    bma2 = a2 - 2 * b_dot_a + gn_norm ** 2
    c = b_dot_a - a2
    d = np.sqrt(c * c + bma2 * (radius ** 2 - a2))
    beta = (d - c) / bma2 if c <= 0 else (radius * radius - a2) / (d + c)
    v = LD(-alpha * (1.0 - beta)) * grad + LD(beta) * gn
    return v / D, "interpolated", float(np.sqrt(np.dot(v, v)))


class Trace:
    """What one reference solve did: `steps` (one dict per iteration), `margins` [(iteration, name, margin, uncertainty)] and the
    summary (iterations, num_successful_steps, termination, final_cost) of every iteration limit k."""

    def __init__(self, win, act, cost, g, H):
        self.win, self.act, self.initial_cost, self.g0, self.H0 = win, act, cost, g, H
        self.steps, self.margins = [], []

    def margin(self, k, name, value, unc):
        self.margins.append((k, name, float(value), float(unc)))

    def finish(self, it, nsucc, term, cost):
        self.iterations, self.num_successful_steps, self.termination, self.final_cost = it, nsucc, term, cost

    def at(self, k):
        """(state, report) of the same solve stopped by max_num_iterations = k."""
        if k >= self.iterations:
            x = self.x_final
            return x, dict(iterations=self.iterations, num_successful_steps=self.num_successful_steps, termination=self.termination, final_cost=self.final_cost)
        steps = self.steps[:k]
        x = self.win.x0
        cost = self.initial_cost
        for s in steps:
            if "x" in s: x, cost = s["x"], s["cost"]
        n = sum(s.get("outcome") == "accepted" for s in steps)
        return x, dict(iterations=k, num_successful_steps=n, termination=abi.TERM_NO_CONVERGENCE, final_cost=cost)

    def step_scale(self, k):
        """sum over the accepted steps j <= k of kappa_j * ||delta_j||: rounding of step j moves every later iterate by ~eps of it."""
        return sum(s["kappa"] * s["delta_norm"] for s in self.steps[:k] if s.get("outcome") == "accepted")

    def closest_margin(self, k=None):
        """The decision (up to iteration k) whose margin is the smallest multiple of its rounding uncertainty."""
        ms = [m for m in self.margins if k is None or m[0] <= k]
        return min(ms, key=lambda m: abs(m[2]) / max(m[3], 1e-300)) if ms else None

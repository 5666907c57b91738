"""ctypes binding of libcerberus_b200.so (the C ABI of include/cerberus_b200.h).

The product library is the nvcc-built sm_90a one next to this file; it has no CPU fallback and
`Backend()` raises if it (or a CUDA device) is missing.  Tests that run without a GPU pass the path of
the CPU kernel *simulator* build (tests/cusim) explicitly -- that is test infrastructure, never a default.
"""
import ctypes as C
import os
import numpy as np
from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
PRODUCT_LIB = os.path.join(_HERE, "libcerberus_b200.so")


class CerbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"cerberus_b200 error {code}: {msg}")
        self.code = code


def _p(a):
    return None if a is None else a.ctypes.data_as(abi.c_dp)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class Backend:
    """One CerbHandle.  Implements the hot-path calls, the factor-family evaluators, device preintegration and
    the `backend` protocol of cerberus_b200.synth (preintegrate / marginalize)."""

    def __init__(self, cfg=None, lib_path=None):
        path = lib_path or PRODUCT_LIB
        if not os.path.exists(path):
            raise CerbError(abi.ERR_NO_DEVICE, f"{path} not built: run `python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)")
        self.lib = C.CDLL(path)
        L = self.lib
        L.cerb_last_error.restype = C.c_char_p
        L.cerb_version.restype = C.c_char_p
        L.cerb_create.argtypes = [C.POINTER(abi.SolverConfig), C.POINTER(C.c_void_p)]
        L.cerb_destroy.argtypes = [C.c_void_p]
        L.cerb_solve_batch.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.WindowDesc), C.POINTER(abi.WindowState), C.POINTER(abi.SolveReport)]
        L.cerb_solve_window.argtypes = [C.c_void_p, C.POINTER(abi.WindowDesc), C.POINTER(abi.WindowState), C.POINTER(abi.SolveReport)]
        L.cerb_batch_upload.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.WindowDesc), C.POINTER(abi.WindowState)]
        L.cerb_batch_update_states.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.WindowState)]
        L.cerb_batch_solve_resident.argtypes = [C.c_void_p]
        L.cerb_batch_download.argtypes = [C.c_void_p, C.POINTER(abi.WindowState), C.POINTER(abi.SolveReport)]
        L.cerb_sync.argtypes = [C.c_void_p]
        L.cerb_last_solve_stats.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int32)]
        L.cerb_debug_linearize.argtypes = [C.c_void_p, C.c_int32, abi.c_dp, abi.c_dp, abi.c_dp, C.c_int32]
        L.cerb_eval_projection.argtypes = [C.c_void_p, C.c_int32, C.c_int32] + [abi.c_dp] * 14
        L.cerb_eval_imu_leg.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.IMULegPreint), abi.c_dp, abi.c_dp, abi.c_dp, abi.c_dp]
        L.cerb_eval_imu.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.IMUPreint), abi.c_dp, abi.c_dp, abi.c_dp, abi.c_dp]
        L.cerb_preintegrate_imu_batch.argtypes = [C.c_void_p, C.POINTER(abi.PreintConfig), C.c_int32, C.POINTER(abi.PreintJob), C.POINTER(abi.IMUPreint)]
        L.cerb_eval_prior.argtypes = [C.c_void_p, C.POINTER(abi.Prior), C.POINTER(abi.WindowState), abi.c_dp, abi.c_dp]
        L.cerb_preintegrate_batch.argtypes = [C.c_void_p, C.POINTER(abi.PreintConfig), C.c_int32, C.POINTER(abi.PreintJob), C.POINTER(abi.IMULegPreint)]
        L.cerb_a1_kinematics.argtypes = [C.c_void_p, C.c_int32] + [abi.c_dp] * 8
        L.cerb_double2vector.argtypes = [C.POINTER(abi.WindowState), C.POINTER(abi.WindowState), abi.c_dp, abi.c_dp, abi.c_dp]
        L.cerb_batch_outlier_errors.argtypes = [C.c_void_p, C.c_double, abi.c_dp, C.POINTER(C.c_int32)]
        L.cerb_batch_triangulate.argtypes = [C.c_void_p, C.c_double, abi.c_dp]
        L.cerb_marginalize_schur.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, abi.c_dp, abi.c_dp, C.c_double, abi.c_dp, abi.c_dp, C.POINTER(C.c_int32)]
        L.cerb_batch_shift_depth.argtypes = [C.c_void_p, C.c_double, C.POINTER(C.c_int32), abi.c_dp, C.POINTER(C.c_int32)]
        L.cerb_register_host_buffer.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.cerb_unregister_host_buffer.argtypes = [C.c_void_p, C.c_void_p]
        L.cerb_last_upload_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
        L.cerb_batch_marginalize.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(abi.WindowState), C.POINTER(abi.Prior), C.POINTER(C.c_int32)]
        L.cerb_double2vector.restype = None
        self.cfg = cfg or abi.default_config()
        self.h = C.c_void_p()
        self._check(L.cerb_create(C.byref(self.cfg), C.byref(self.h)))

    def _check(self, rc, allow=()):
        if rc != 0 and rc not in allow:
            raise CerbError(rc, self.lib.cerb_last_error().decode())
        return rc

    def close(self):
        if self.h:
            self.lib.cerb_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def version(self):
        return self.lib.cerb_version().decode()

    # ---- the hot path ------------------------------------------------------------------------------
    def solve_batch(self, batch):
        """Host buffers in / out (the drop-in call): pack + H2D + solve + D2H.  Returns the report array."""
        self._check(self.lib.cerb_solve_batch(self.h, batch.n, batch.descs, batch.states, batch.reports), allow=(abi.ERR_NON_FINITE,))
        return batch.report_array().copy()

    def solve_window(self, batch, w):
        self._check(self.lib.cerb_solve_window(self.h, C.byref(batch.descs[w]), C.byref(batch.states[w]), C.byref(batch.reports[w])), allow=(abi.ERR_NON_FINITE,))

    def upload(self, batch):
        self._check(self.lib.cerb_batch_upload(self.h, batch.n, batch.descs, batch.states))

    def update_states(self, batch):
        """cerb_batch_update_states: new para_* of the resident windows (same tracks, same order), nothing else travels"""
        self._check(self.lib.cerb_batch_update_states(self.h, batch.n, batch.states))

    def solve_resident(self):
        self._check(self.lib.cerb_batch_solve_resident(self.h))

    def download(self, batch):
        self._check(self.lib.cerb_batch_download(self.h, batch.states, batch.reports), allow=(abi.ERR_NON_FINITE,))
        return batch.report_array().copy()

    def register_batch(self, batch):
        """cerb_register_host_buffer on every array of a WindowBatch: later solve_batch / upload calls DMA straight out of them."""
        bufs = [batch.features, batch.obs, batch.preint, batch.prior_J, batch.prior_r, batch.para_Feature]
        if batch.imu_preint is not None: bufs.append(batch.imu_preint)
        regs = [(a.ctypes.data, a.nbytes) for a in bufs] + [(C.addressof(batch.states), C.sizeof(batch.states)), (C.addressof(batch.descs), C.sizeof(batch.descs))]
        for ptr, nbytes in regs:
            self._check(self.lib.cerb_register_host_buffer(self.h, C.c_void_p(ptr), nbytes))
        return [p for p, _ in regs]

    def unregister(self, ptrs):
        for p in ptrs:
            self._check(self.lib.cerb_unregister_host_buffer(self.h, C.c_void_p(p)))

    def last_upload_stats(self):
        ops, staged = C.c_int32(), C.c_int64()
        self._check(self.lib.cerb_last_upload_stats(self.h, C.byref(ops), C.byref(staged)))
        return ops.value, staged.value

    def sync(self):
        self._check(self.lib.cerb_sync(self.h))

    def last_solve_stats(self):
        ms, nl = C.c_double(), C.c_int32()
        self._check(self.lib.cerb_last_solve_stats(self.h, C.byref(ms), C.byref(nl)))
        return ms.value, nl.value

    def debug_linearize(self, batch, w):
        """cost, gradient, diag(J^T J) of resident window w at its current state (solved states after a solve, else the uploaded ones; ABI tangent order)."""
        nf = batch.descs[w].n_features
        g, d = np.zeros(abi.NUM_REDUCED + nf), np.zeros(abi.NUM_REDUCED + nf)
        cost = C.c_double()
        self._check(self.lib.cerb_debug_linearize(self.h, w, C.cast(C.byref(cost), abi.c_dp), _p(g), _p(d), g.size))
        return cost.value, g, d

    # ---- factor families -----------------------------------------------------------------------------
    def eval_projection(self, kind, pose_i, pose_j, ex0, ex1, inv_dep, td, pts_i, pts_j, vel_i, vel_j, td_i, td_j, want_jac=True):
        n = inv_dep.shape[0]
        args = [None if a is None else _f64(a) for a in (pose_i, pose_j, ex0, ex1, inv_dep, td, pts_i, pts_j, vel_i, vel_j, td_i, td_j)]
        res = np.zeros((n, 2))
        jac = np.zeros((n, abi.PROJ_JAC_SIZE[kind])) if want_jac else None
        self._check(self.lib.cerb_eval_projection(self.h, kind, n, *[_p(a) for a in args], _p(res), _p(jac)))
        return res, jac

    def eval_imu_leg(self, preint, params, want_jac=True):
        n = params.shape[0]
        params = _f64(params)
        res, si = np.zeros((n, 31)), np.zeros((n, 961))
        jac = np.zeros((n, 31 * 40)) if want_jac else None
        self._check(self.lib.cerb_eval_imu_leg(self.h, n, preint.ctypes.data_as(C.POINTER(abi.IMULegPreint)), _p(params), _p(res), _p(jac), _p(si)))
        return res, jac, si

    def eval_imu(self, preint, params, want_jac=True):
        """IMUFactor::Evaluate (USE_LEG == 0): params [n, 32] = pose_i, speedbias_i, pose_j, speedbias_j."""
        n = params.shape[0]
        params = _f64(params)
        res, si = np.zeros((n, 15)), np.zeros((n, 225))
        jac = np.zeros((n, 15 * 32)) if want_jac else None
        self._check(self.lib.cerb_eval_imu(self.h, n, preint.ctypes.data_as(C.POINTER(abi.IMUPreint)), _p(params), _p(res), _p(jac), _p(si)))
        return res, jac, si

    def preintegrate_imu(self, pcfg, jobs, n):
        out = np.zeros(n, dtype=abi.imu_preint_dtype)
        self._check(self.lib.cerb_preintegrate_imu_batch(self.h, C.byref(pcfg), n, jobs, out.ctypes.data_as(C.POINTER(abi.IMUPreint))))
        return out

    def eval_prior(self, prior, state, n_cols):
        res, jac = np.zeros(prior.n), np.zeros(prior.n * n_cols)
        self._check(self.lib.cerb_eval_prior(self.h, C.byref(prior), C.byref(state), _p(res), _p(jac)))
        return res, jac

    def a1_kinematics(self, q, rho_opt, rho_fix):
        q, rho_opt, rho_fix = _f64(q), _f64(rho_opt), _f64(rho_fix)
        n = q.shape[0]
        fk, jac, dfk, djq, djr = np.zeros((n, 3)), np.zeros((n, 9)), np.zeros((n, 3)), np.zeros((n, 27)), np.zeros((n, 9))
        self._check(self.lib.cerb_a1_kinematics(self.h, n, _p(q), _p(rho_opt), _p(rho_fix), _p(fk), _p(jac), _p(dfk), _p(djq), _p(djr)))
        return fk, jac, dfk, djq, djr

    def double2vector(self, before_state, after_state):
        Ps, Rs, Vs = np.zeros((11, 3)), np.zeros((11, 3, 3)), np.zeros((11, 3))
        self.lib.cerb_double2vector(C.byref(before_state), C.byref(after_state), _p(Ps), _p(Rs), _p(Vs))
        return Ps, Rs, Vs

    # ---- per-feature steps on the resident batch (after upload / solve) -----------------------------------------------
    def outlier_errors(self, n, focal_length=460.0):
        """Estimator::outliersRejection on the resident batch: (ave_err [n][max_features], remove flags)."""
        F = self.cfg.max_features
        err = np.full((n, F), np.nan); rem = np.zeros((n, F), dtype=np.int32)
        self._check(self.lib.cerb_batch_outlier_errors(self.h, focal_length, _p(err), rem.ctypes.data_as(C.POINTER(C.c_int32))))
        return err, rem

    def shift_depth(self, n, init_depth=5.0):
        """FeatureManager::removeBackShiftDepth on the resident batch: (new start_frame, new depth, keep flag), each [n][max_features]."""
        F = self.cfg.max_features
        start = np.full((n, F), -1, dtype=np.int32); depth = np.full((n, F), np.nan); keep = np.full((n, F), -1, dtype=np.int32)
        self._check(self.lib.cerb_batch_shift_depth(self.h, init_depth, start.ctypes.data_as(C.POINTER(C.c_int32)), _p(depth), keep.ctypes.data_as(C.POINTER(C.c_int32))))
        return start, depth, keep

    def triangulate(self, n, init_depth=5.0):
        """FeatureManager::triangulate on the resident batch: estimated_depth [n][max_features]."""
        depth = np.full((n, self.cfg.max_features), np.nan)
        self._check(self.lib.cerb_batch_triangulate(self.h, init_depth, _p(depth)))
        return depth

    # ---- synth backend protocol -----------------------------------------------------------------------------
    def preintegrate(self, pcfg, jobs, n):
        out = np.zeros(n, dtype=abi.preint_dtype)
        self._check(self.lib.cerb_preintegrate_batch(self.h, C.byref(pcfg), n, jobs, out.ctypes.data_as(C.POINTER(abi.IMULegPreint))))
        return out

    def marginalize_schur(self, A, b, m, eps=1e-8, return_sweeps=False):
        """MarginalizationInfo::marginalize() after the A / b assembly (marginalization_factor.cpp:281-305) for a stack of windows:
        A [B, pos, pos], b [B, pos], dropped coordinates first -> (linearized_jacobians [B, n, n] row k = sqrt(S_k) v_k^T, linearized_residuals [B, n])."""
        A = np.ascontiguousarray(A, dtype=np.float64); b = np.ascontiguousarray(b, dtype=np.float64)
        B, pos = b.shape; n = pos - m
        J = np.zeros((B, n * n)); r = np.zeros((B, n)); sw = np.zeros((B, 2), dtype=np.int32)
        self._check(self.lib.cerb_marginalize_schur(self.h, B, m, n, _p(A), _p(b), eps, _p(J), _p(r), sw.ctypes.data_as(C.POINTER(C.c_int32))))
        J = J.reshape(B, n, n).transpose(0, 2, 1)          # column-major on the wire
        return (J, r, sw) if return_sweeps else (J, r)

    def batch_marginalize(self, flags, states, priors):
        """cerb_batch_marginalize on the resident batch: flags [n] int32 (0 MARGIN_OLD, 1 MARGIN_SECOND_NEW), states: ctypes array of WindowState
        (or None: the solved states on the device), priors: ctypes array of Prior with their matrix / vector pointers set.  Returns the Jacobi sweeps [n, 2]."""
        n = len(priors)
        sw = np.zeros((n, 2), dtype=np.int32)
        self._check(self.lib.cerb_batch_marginalize(self.h, flags.ctypes.data_as(C.POINTER(C.c_int32)), states, priors, sw.ctypes.data_as(C.POINTER(C.c_int32))))
        return sw

    def marginalize(self, cfg, src, dst, margin_old=True):
        from . import marginalization
        return marginalization.marginalize_batch(self, cfg, src, dst, margin_old)

"""ctypes binding of oracle/liboracle.so -- TEST INFRASTRUCTURE (the CPU restatement of the reference).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg import this.
"""
import ctypes as C
import os
import subprocess
import numpy as np
from cerberus_b200 import abi

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None


def build():
    subprocess.check_call(["make", "-s", "-C", os.path.join(_ROOT, "oracle")])


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_ROOT, "oracle", "liboracle.so")
        if not os.path.exists(path):
            build()
        _LIB = C.CDLL(path)
        sizes = (C.c_int * 16)()
        k = _LIB.oracle_abi_sizes(sizes, 16)
        got = [sizes[i] for i in range(k)]
        want = [C.sizeof(s) for s in abi.ABI_STRUCTS]
        assert got == want, f"ABI struct size mismatch oracle={got} python={want}"
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(abi.c_dp)


class OracleBackend:
    """Implements the synth `backend` protocol and the solve/eval entry points with the CPU oracle."""

    def __init__(self, cfg=None):
        self.cfg = cfg or abi.default_config()
        self.lib = lib()

    def preintegrate(self, pcfg, jobs, n):
        out = np.zeros(n, dtype=abi.preint_dtype)
        rc = self.lib.oracle_preintegrate(C.byref(pcfg), n, jobs, out.ctypes.data_as(C.POINTER(abi.IMULegPreint)))
        assert rc == 0
        return out

    def marginalize(self, cfg, src, dst, margin_old=True):
        """margin_old: one flag for the batch, or one per window (True / 1: MARGIN_OLD, False / 0: MARGIN_SECOND_NEW)."""
        flags = np.broadcast_to(np.asarray(margin_old, dtype=bool), (src.n,))
        for w in range(src.n):
            pr = dst.descs[w].prior
            J, r = dst.prior_J[w], dst.prior_r[w]
            rc = self.lib.oracle_marginalize(C.byref(cfg), C.byref(src.descs[w]), C.byref(src.states[w]), 1 if flags[w] else 0,
                                             C.byref(pr), _p(J), _p(r))
            assert rc == 0

    def set_eig_mode(self, mode):
        """0: tridiagonal QR (the reference's Eigen::SelfAdjointEigenSolver; default), 1: cyclic Jacobi."""
        self.lib.oracle_set_eig_mode(int(mode))

    def solve_batch(self, batch, nthreads=1, cfg=None):
        cfg = cfg or self.cfg
        rc = self.lib.oracle_solve_batch(C.byref(cfg), batch.n, batch.descs, batch.states, batch.reports, nthreads)
        assert rc == 0
        return batch.report_array().copy()

    def solve_window(self, batch, w, want_probe=False, cfg=None):
        cfg = cfg or self.cfg
        nf = batch.descs[w].n_features
        g = np.zeros(abi.NUM_REDUCED + nf)
        d = np.zeros(abi.NUM_REDUCED + nf)
        rc = self.lib.oracle_solve_window(C.byref(cfg), C.byref(batch.descs[w]), C.byref(batch.states[w]), C.byref(batch.reports[w]),
                                          _p(g) if want_probe else None, _p(d) if want_probe else None, g.size)
        assert rc == 0
        return (g, d) if want_probe else None

    def eval_projection(self, kind, pose_i, pose_j, ex0, ex1, inv_dep, td, pts_i, pts_j, vel_i, vel_j, td_i, td_j, sqrt_info=460.0 / 1.5, want_jac=True):
        n = inv_dep.shape[0]
        res = np.zeros((n, 2))
        jac = np.zeros((n, abi.PROJ_JAC_SIZE[kind])) if want_jac else None
        self.lib.oracle_eval_projection.argtypes = [C.c_int, C.c_int, C.c_double] + [abi.c_dp] * 14
        rc = self.lib.oracle_eval_projection(kind, n, sqrt_info, _p(pose_i), _p(pose_j), _p(ex0), _p(ex1), _p(inv_dep), _p(td), _p(pts_i), _p(pts_j),
                                             _p(vel_i), _p(vel_j), _p(td_i), _p(td_j), _p(res), _p(jac))
        assert rc == 0
        return res, jac

    def eval_imu_leg(self, preint, params, g=(0.0, 0.0, 9.805), want_jac=True):
        n = params.shape[0]
        res = np.zeros((n, 31))
        jac = np.zeros((n, 31 * 40)) if want_jac else None
        si = np.zeros((n, 961))
        garr = np.array(g, dtype=np.float64)
        rc = self.lib.oracle_eval_imu_leg(n, _p(garr), preint.ctypes.data_as(C.POINTER(abi.IMULegPreint)), _p(params), _p(res), _p(jac), _p(si))
        assert rc == 0
        return res, jac, si

    def eval_imu(self, preint, params, g=(0.0, 0.0, 9.805), want_jac=True):
        n = params.shape[0]
        res, si = np.zeros((n, 15)), np.zeros((n, 225))
        jac = np.zeros((n, 15 * 32)) if want_jac else None
        garr = np.array(g, dtype=np.float64)
        rc = self.lib.oracle_eval_imu(n, _p(garr), preint.ctypes.data_as(C.POINTER(abi.IMUPreint)), _p(np.ascontiguousarray(params)), _p(res), _p(jac), _p(si))
        assert rc == 0
        return res, jac, si

    def preintegrate_imu(self, pcfg, jobs, n):
        out = np.zeros(n, dtype=abi.imu_preint_dtype)
        rc = self.lib.oracle_preintegrate_imu(C.byref(pcfg), n, jobs, out.ctypes.data_as(C.POINTER(abi.IMUPreint)))
        assert rc == 0
        return out

    def eval_prior(self, prior, state, n_cols):
        res = np.zeros(prior.n)
        jac = np.zeros(prior.n * n_cols)
        rc = self.lib.oracle_eval_prior(C.byref(prior), C.byref(state), _p(res), _p(jac))
        assert rc == 0
        return res, jac

    def a1_kinematics(self, q, rho_opt, rho_fix):
        n = q.shape[0]
        fk, jac, dfk, djq, djr = np.zeros((n, 3)), np.zeros((n, 9)), np.zeros((n, 3)), np.zeros((n, 27)), np.zeros((n, 9))
        rc = self.lib.oracle_a1_kinematics(n, _p(q), _p(rho_opt), _p(rho_fix), _p(fk), _p(jac), _p(dfk), _p(djq), _p(djr))
        assert rc == 0
        return fk, jac, dfk, djq, djr

    def double2vector(self, before_state, after_state):
        Ps, Rs, Vs = np.zeros((11, 3)), np.zeros((11, 3, 3)), np.zeros((11, 3))
        self.lib.oracle_double2vector(C.byref(before_state), C.byref(after_state), _p(Ps), _p(Rs), _p(Vs))
        return Ps, Rs, Vs

    def outlier_errors(self, batch):
        out = np.full((batch.n, batch.max_features), np.nan)
        for w in range(batch.n):
            assert self.lib.oracle_outlier_errors(C.byref(batch.descs[w]), C.byref(batch.states[w]), _p(out[w])) == 0
        return out

    def marginalize_schur(self, A, b, m, eps=1e-8):
        A = np.ascontiguousarray(A, dtype=np.float64); b = np.ascontiguousarray(b, dtype=np.float64)
        B, pos = b.shape; n = pos - m
        J = np.zeros((B, n * n)); r = np.zeros((B, n))
        self.lib.oracle_marginalize_schur.argtypes = [C.c_int, C.c_int, abi.c_dp, abi.c_dp, C.c_double, abi.c_dp, abi.c_dp]
        for w in range(B):
            assert self.lib.oracle_marginalize_schur(m, n, _p(A[w]), _p(b[w]), eps, _p(J[w]), _p(r[w])) == 0
        return J.reshape(B, n, n).transpose(0, 2, 1), r

    def shift_depth(self, batch, init_depth=5.0):
        n, F = batch.n, batch.max_features
        start = np.full((n, F), -1, dtype=np.int32); depth = np.full((n, F), np.nan); keep = np.full((n, F), -1, dtype=np.int32)
        self.lib.oracle_shift_depth.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.POINTER(C.c_int32), abi.c_dp, C.POINTER(C.c_int32)]
        for w in range(n):
            assert self.lib.oracle_shift_depth(C.byref(batch.descs[w]), C.byref(batch.states[w]), init_depth, start[w].ctypes.data_as(C.POINTER(C.c_int32)),
                                               _p(depth[w]), keep[w].ctypes.data_as(C.POINTER(C.c_int32))) == 0
        return start, depth, keep

    def triangulate(self, batch, init_depth=5.0):
        out = np.full((batch.n, batch.max_features), np.nan)
        self.lib.oracle_triangulate.argtypes = [C.c_void_p, C.c_void_p, C.c_double, abi.c_dp]
        for w in range(batch.n):
            assert self.lib.oracle_triangulate(C.byref(batch.descs[w]), C.byref(batch.states[w]), init_depth, _p(out[w])) == 0
        return out


# ---------------------------------------------------------------------------------------------------------------
# The reference's OWN factor sources compiled against the header shims (oracle/shim) into oracle/_ref/libcerberus_ref.so by
# `make -C oracle ref REF=<Cerberus checkout>/src`.  The tests do not need that build: RefBackend replays the outputs the compiled
# sources gave for the same inputs, stored in tests/golden/ref_v1.npz by tests/golden/make_ref_golden.py.  Each stored call is
# found by a fingerprint of its inputs; a call that matches none (to ~1e-9 relative) fails, because the stored outputs are then stale.
GOLDEN_REF = os.path.join(_ROOT, "tests", "golden", "ref_v1.npz")
_REF = None


def ref_lib():
    """The compiled reference sources (oracle/_ref), or None where they were not built."""
    global _REF
    if _REF is None:
        path = os.path.join(_ROOT, "oracle", "_ref", "libcerberus_ref.so")
        if not os.path.exists(path):
            return None
        _REF = C.CDLL(path)
    return _REF


def _flat(x, out):
    """Append the numbers of x (numpy arrays, ctypes structures and arrays, window batches, scalars) to `out`; pointers are skipped."""
    if x is None:
        return
    if isinstance(x, abi.WindowBatch):
        for a in (x.state_array(), x.para_Feature, x.features, x.obs, x.preint, x.imu_preint, x.prior_J, x.prior_r):
            _flat(a, out)
        for w in range(x.n):
            _flat(x.descs[w], out)
    elif isinstance(x, np.ndarray):
        if x.dtype.names:
            for name in x.dtype.names:
                _flat(x[name], out)
        else:
            out.append(np.asarray(x, dtype=np.float64).ravel())
    elif isinstance(x, C.Structure):
        for name, t in x._fields_:
            if not issubclass(t, (C._Pointer, C.c_void_p)):
                _flat(getattr(x, name), out)
    elif isinstance(x, (C.Array, tuple, list)):
        for v in x:
            _flat(v, out)
    else:
        out.append(np.array([float(x)]))


def _fingerprint(*xs):
    """[size, sum |v|, sum v cos(k), 64 evenly spaced entries] of the inputs flattened into one vector v."""
    out = []
    for x in xs:
        _flat(x, out)
    v = np.nan_to_num(np.concatenate(out), nan=0.0, posinf=1e300, neginf=-1e300)
    idx = np.unique(np.linspace(0, v.size - 1, 64).astype(np.int64))
    return np.concatenate([[v.size, np.abs(v).sum(), (v * np.cos(np.arange(v.size))).sum()], v[idx]])


def _same_inputs(a, b):
    if a.shape != b.shape or a[0] != b[0]:
        return False
    scale = max(abs(b[1]), 1e-300)
    return abs(a[1] - b[1]) <= 1e-9 * scale and abs(a[2] - b[2]) <= 1e-9 * scale and (np.abs(a[3:] - b[3:]) <= 1e-9 * np.maximum(np.abs(b[3:]), 1.0)).all()


class _Golden:
    """The stored calls: method name -> [(input fingerprint, outputs, outputs-is-a-tuple)]."""

    def __init__(self):
        self.calls = None

    def load(self):
        if self.calls is None:
            self.calls = {}
            if os.path.exists(GOLDEN_REF) and not RefBackend.record:
                z = np.load(GOLDEN_REF, allow_pickle=False)
                for key in sorted(k for k in z.files if k.endswith(".fp")):
                    stem = key[:-3]
                    outs = [z[f"{stem}.out{i}"] for i in range(int(z[f"{stem}.nout"]))]
                    self.calls.setdefault(stem.split(".")[0], []).append((z[key], outs, bool(z[f"{stem}.tuple"])))
        return self.calls

    def find(self, name, fp):
        for rfp, outs, is_tuple in self.load().get(name, []):
            if _same_inputs(fp, rfp):
                outs = [o.copy() for o in outs]
                return tuple(outs) if is_tuple else outs[0]
        raise LookupError(f"RefBackend.{name}: no stored output of the reference sources for these inputs in {GOLDEN_REF}; "
                          "regenerate it with tests/golden/make_ref_golden.py")

    def add(self, name, fp, out):
        recs = self.load().setdefault(name, [])
        if not any(_same_inputs(fp, r[0]) for r in recs):
            is_tuple = isinstance(out, (tuple, list))
            recs.append((fp, [np.array(o) for o in (out if is_tuple else [out])], is_tuple))

    def save(self, path=GOLDEN_REF):
        arrays = {}
        for name, recs in sorted(self.load().items()):
            for i, (fp, outs, is_tuple) in enumerate(recs):
                stem = f"{name}.{i:03d}"
                arrays[f"{stem}.fp"], arrays[f"{stem}.nout"], arrays[f"{stem}.tuple"] = fp, np.int64(len(outs)), np.int64(is_tuple)
                for k, o in enumerate(outs):
                    arrays[f"{stem}.out{k}"] = o
        np.savez_compressed(path, **arrays)


GOLDEN = _Golden()


class RefBackend:
    """Factor evaluators / preintegration / kinematics / marginalization / FeatureManager steps of the reference's own sources (no
    solver: Ceres is a third-party library).  Replays tests/golden/ref_v1.npz; with live=True (or RefBackend.record, set by
    tests/golden/make_ref_golden.py, which also stores every call) it calls the compiled sources in oracle/_ref instead."""
    record = False

    def __init__(self, pcfg=None, g=(0.0, 0.0, 9.805), visual_sqrt_info=460.0 / 1.5, live=None):
        self.live = RefBackend.record if live is None else live
        self.lib = ref_lib() if self.live else None
        if self.live and self.lib is None:
            raise RuntimeError("oracle/_ref/libcerberus_ref.so is not built (make -C oracle ref REF=<Cerberus checkout>/src)")
        self.set_globals(pcfg or abi.default_preint_config(), g, visual_sqrt_info)

    def set_globals(self, pcfg, g=(0.0, 0.0, 9.805), visual_sqrt_info=460.0 / 1.5):
        garr = (C.c_double * 3)(*g)
        self.globals = (abi.PreintConfig.from_buffer_copy(pcfg), np.array(g, dtype=np.float64), visual_sqrt_info)
        if self.live:
            self.lib.ref_set_globals.argtypes = [C.POINTER(abi.PreintConfig), C.POINTER(C.c_double), C.c_double]
            self.lib.ref_set_globals(C.byref(pcfg), garr, visual_sqrt_info)

    def _call(self, name, inputs, live):
        fp = _fingerprint(self.globals, *inputs)
        if not self.live:
            return GOLDEN.find(name, fp)
        out = live()
        if RefBackend.record:
            GOLDEN.add(name, fp, out)
        return out

    def eval_projection(self, kind, pose_i, pose_j, ex0, ex1, inv_dep, td, pts_i, pts_j, vel_i, vel_j, td_i, td_j, want_jac=True):
        args = (pose_i, pose_j, ex0, ex1, inv_dep, td, pts_i, pts_j, vel_i, vel_j, td_i, td_j)

        def live():
            n = inv_dep.shape[0]
            res = np.zeros((n, 2))
            jac = np.zeros((n, abi.PROJ_JAC_SIZE[kind]))
            self.lib.ref_eval_projection(kind, n, *[_p(a) for a in args], _p(res), _p(jac))
            return res, jac
        res, jac = self._call("eval_projection", (kind,) + args, live)
        return res, (jac if want_jac else None)

    def eval_imu_leg(self, preint, params, want_jac=True):
        def live():
            n = params.shape[0]
            res, si, jac = np.zeros((n, 31)), np.zeros((n, 961)), np.zeros((n, 31 * 40))
            self.lib.ref_eval_imu_leg(n, preint.ctypes.data_as(C.POINTER(abi.IMULegPreint)), _p(params), _p(res), _p(jac), _p(si))
            return res, jac, si
        res, jac, si = self._call("eval_imu_leg", (preint, params), live)
        return res, (jac if want_jac else None), si

    def preintegrate(self, pcfg, jobs, n):
        saved = self.globals                # the preintegration config holds for this call only
        self.set_globals(pcfg, *saved[1:])

        def live():
            out = np.zeros(n, dtype=abi.preint_dtype)
            self.lib.ref_preintegrate(n, jobs, out.ctypes.data_as(C.POINTER(abi.IMULegPreint)))
            return out
        try:
            return self._call("preintegrate", (_jobs_inputs(jobs, n),), live)
        finally:
            self.set_globals(*saved)

    def a1_kinematics(self, q, rho_opt, rho_fix):
        def live():
            n = q.shape[0]
            fk, jac, dfk, djq, djr = np.zeros((n, 3)), np.zeros((n, 9)), np.zeros((n, 3)), np.zeros((n, 27)), np.zeros((n, 9))
            self.lib.ref_a1_kinematics(n, _p(q), _p(rho_opt), _p(rho_fix), _p(fk), _p(jac), _p(dfk), _p(djq), _p(djr))
            return fk, jac, dfk, djq, djr
        return self._call("a1_kinematics", (q, rho_opt, rho_fix), live)

    def pose_plus(self, x, delta):
        def live():
            out = np.zeros(7)
            self.lib.ref_pose_plus(_p(np.ascontiguousarray(x)), _p(np.ascontiguousarray(delta)), _p(out))
            return out
        return self._call("pose_plus", (x, delta), live)

    def eval_prior(self, prior, state, n_cols, rows):
        """Residual rows `rows` of MarginalizationFactor::Evaluate and their Jacobian rows ([len(rows), n_cols])."""
        rows = np.asarray(rows)

        def live():
            res, jac = np.zeros(prior.n), np.zeros(prior.n * n_cols)
            self.lib.ref_eval_prior(C.byref(prior), C.byref(state), _p(res), _p(jac))
            return res[rows], jac.reshape(prior.n, n_cols)[rows]
        n = prior.n
        J = np.ctypeslib.as_array(prior.linearized_jacobians, shape=(n * n,)) if n else None
        r = np.ctypeslib.as_array(prior.linearized_residuals, shape=(n,)) if n else None
        return self._call("eval_prior", (prior, J, r, state, n_cols, rows), live)

    def marginal_priors(self, cfg, src, margin_old=True):
        """The reference's own MarginalizationInfo / ResidualBlockInfo classes on every window of src: per window the new prior as
        helpers.prior_canonical gives it, (A = J^T J, b = J^T r, {(block kind, index): x0}).  The stored A is the float32 upper
        triangle: the tests compare priors to 1e-5 of max |A|, float32 rounds to 6e-8 of each entry."""
        flags = np.broadcast_to(np.asarray(margin_old, dtype=bool), (src.n,))

        def live():
            from cerberus_b200 import synth
            from helpers import prior_canonical
            dst, outs = synth.tile_batch(src, src.n), []
            for w in range(src.n):
                rc = self.lib.ref_marginalize(C.byref(src.descs[w]), C.byref(src.states[w]), 1 if flags[w] else 0, C.byref(dst.descs[w].prior), _p(dst.prior_J[w]), _p(dst.prior_r[w]))
                assert rc == 0
                A, b, x0 = prior_canonical(dst, w)
                keys = sorted(x0)
                outs += [A[np.triu_indices(A.shape[0])].astype(np.float32), b, np.array(keys, dtype=np.int64).reshape(-1, 2), np.array([x0[k] for k in keys])]
            return outs
        outs, priors = self._call("marginal_priors", (cfg, src, flags), live), []
        for w in range(src.n):
            Au, b, keys, vals = outs[4 * w:4 * w + 4]
            A = np.zeros((b.size, b.size)); A[np.triu_indices(b.size)] = Au
            A = A + np.triu(A, 1).T
            priors.append((A, b, {(int(k), int(i)): v for (k, i), v in zip(keys, vals)}))
        return priors

    def marginalize(self, cfg, src, dst, margin_old=True):
        """The new priors written into dst, by the compiled sources only (live=True: tools/eig_study.py)."""
        flags = np.broadcast_to(np.asarray(margin_old, dtype=bool), (src.n,))
        for w in range(src.n):
            assert self.lib.ref_marginalize(C.byref(src.descs[w]), C.byref(src.states[w]), 1 if flags[w] else 0, C.byref(dst.descs[w].prior), _p(dst.prior_J[w]), _p(dst.prior_r[w])) == 0

    def double2vector(self, before_state, after_state):
        def live():
            Ps, Rs, Vs = np.zeros((11, 3)), np.zeros((11, 3, 3)), np.zeros((11, 3))
            self.lib.ref_double2vector(C.byref(before_state), C.byref(after_state), _p(Ps), _p(Rs), _p(Vs))
            return Ps, Rs, Vs
        return self._call("double2vector", (before_state, after_state), live)

    def triangulate(self, batch, init_depth=5.0):
        def live():
            out = np.full((batch.n, batch.max_features), np.nan)
            self.lib.ref_triangulate.argtypes = [C.c_void_p, C.c_void_p, C.c_double, abi.c_dp]
            for w in range(batch.n):
                assert self.lib.ref_triangulate(C.byref(batch.descs[w]), C.byref(batch.states[w]), init_depth, _p(out[w])) == 0
            return out
        return self._call("triangulate", (batch, init_depth), live)

    def outlier_errors(self, batch):
        def live():
            out = np.full((batch.n, batch.max_features), np.nan)
            for w in range(batch.n):
                assert self.lib.ref_outlier_errors(C.byref(batch.descs[w]), C.byref(batch.states[w]), _p(out[w])) == 0
            return out
        return self._call("outlier_errors", (batch,), live)

    def shift_depth(self, batch, init_depth=5.0):
        def live():
            n, F = batch.n, batch.max_features
            start = np.full((n, F), -1, dtype=np.int32); depth = np.full((n, F), np.nan); keep = np.full((n, F), -1, dtype=np.int32)
            self.lib.ref_shift_depth.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.POINTER(C.c_int32), abi.c_dp, C.POINTER(C.c_int32)]
            for w in range(n):
                assert self.lib.ref_shift_depth(C.byref(batch.descs[w]), C.byref(batch.states[w]), init_depth, start[w].ctypes.data_as(C.POINTER(C.c_int32)),
                                                _p(depth[w]), keep[w].ctypes.data_as(C.POINTER(C.c_int32))) == 0
            return start, depth, keep
        return self._call("shift_depth", (batch, init_depth), live)

    def eval_imu(self, preint, params, want_jac=True):
        def live():
            n = params.shape[0]
            res, si, jac = np.zeros((n, 15)), np.zeros((n, 225)), np.zeros((n, 15 * 32))
            self.lib.ref_eval_imu(n, preint.ctypes.data_as(C.POINTER(abi.IMUPreint)), _p(np.ascontiguousarray(params)), _p(res), _p(jac), _p(si))
            return res, jac, si
        res, jac, si = self._call("eval_imu", (preint, params), live)
        return res, (jac if want_jac else None), si

    def preintegrate_imu(self, pcfg, jobs, n):
        saved = self.globals                # the preintegration config holds for this call only
        self.set_globals(pcfg, *saved[1:])

        def live():
            out = np.zeros(n, dtype=abi.imu_preint_dtype)
            self.lib.ref_preintegrate_imu(n, jobs, out.ctypes.data_as(C.POINTER(abi.IMUPreint)))
            return out
        try:
            return self._call("preintegrate_imu", (_jobs_inputs(jobs, n),), live)
        finally:
            self.set_globals(*saved)


def ref_rows(n, k):
    """The k rows (of n) on which a test compares with the reference sources: their stored outputs are kept small."""
    return np.unique(np.linspace(0, n - 1, k).round().astype(np.int64))


def sub_jobs(jobs, rows):
    """The preintegration jobs `rows` of a job array (their samples stay where the original jobs point)."""
    out = (abi.PreintJob * len(rows))(*[jobs[int(i)] for i in rows])
    out._keepalive = jobs
    return out


def _jobs_inputs(jobs, n):
    """The numbers of n preintegration jobs, including the IMU / leg samples they point to."""
    per = C.sizeof(abi.IMULegSample) // 8
    return [jobs[k] for k in range(n)] + [np.ctypeslib.as_array(C.cast(jobs[k].samples, C.POINTER(C.c_double)), shape=(jobs[k].n_samples * per,)) for k in range(n)]


class OracleOps:
    """Backend adapter of cerberus_b200.estimator.ReplayDriver on the CPU oracle (the reference arm of the replay comparison)."""

    def __init__(self, cfg, nthreads=8, eig_mode=0, marg=None, feat=None):
        self.o, self.cfg, self.nthreads, self.eig_mode = OracleBackend(cfg), cfg, nthreads, eig_mode
        self.marg = marg          # optional RefBackend: the reference's own MarginalizationInfo classes for the marginalization step
        self.feat = feat          # optional RefBackend: the reference's own FeatureManager for triangulation / depth shift / outlier errors

    def preintegrate(self, pcfg, jobs, n): return self.o.preintegrate(pcfg, jobs, n)
    def solve(self, batch): return self.o.solve_batch(batch, nthreads=self.nthreads)
    def double2vector(self, before, after): return self.o.double2vector(before, after)
    def triangulate(self, batch): return (self.feat or self.o).triangulate(batch)
    def outlier_errors(self, batch): return (self.feat or self.o).outlier_errors(batch)
    def shift_depth(self, batch): return (self.feat or self.o).shift_depth(batch)

    def marginalize(self, src, dst, flags):
        if self.marg is not None:
            self.marg.lib.ref_set_eigen_mode(int(self.eig_mode))
            self.marg.marginalize(self.cfg, src, dst, margin_old=(np.asarray(flags) == 0))
        else:
            self.o.set_eig_mode(self.eig_mode)
            self.o.marginalize(self.cfg, src, dst, margin_old=(np.asarray(flags) == 0))

"""Every trust-region iterate of the solve kernel (and of the oracle) against the dense extended-precision reference of tests/dense_ref.py,
on track layouts at the edges of the kernel's visual passes (chunks of <= 64 tracks per anchor, two frames per pass, 15 chunks cached in
shared memory, 32-feature staging of the inverse-depth Schur complement).

Tolerance.  The kernel and the oracle run fp64; the reference is exact to far below that.  A backward-stable fp64 solve of step j is off
by ~kappa_j * eps * ||delta_j|| (kappa_j: condition number of the Jacobi-scaled, regularised system of step j on its coupled columns,
delta_j: the tangent step), and that error carries into every later iterate.  So iterate k of an arm must satisfy

    max |x_k - x_k^ref|  <=  C_X * eps * sum_{accepted j <= k} kappa_j ||delta_j||,        C_X = 2.5

C_X is set from the measured ratios max |x_k - x_k^ref| / (eps * sum kappa_j ||delta_j||) (printed per case by `pytest -s`): on the
CPU simulator (K = 2) 2.5e-3 .. 3.8e-2 over the layouts below; on an H100 80GB HBM3 (K = 12, every layout under every mode)
9.8e-5 .. 0.24, worst all_mono with the leg biases held constant; the oracle 6.3e-4 .. 8.8e-2.  C_X = 2.5 is 10x the worst of them.
Iteration counts, successful steps and termination must be equal, and the arm's final cost must be the reference cost of the arm's
own iterate to 1e-11 relative (1.1e-12 measured on the H100, whose summation order differs; the cost of x_k^ref itself differs by the gradient times the rounding of x_k, up to ~1e-8 relative
after a first step that moves the inverse depths by O(10)).

Decisions are never near ties: every branch of the loop (dogleg case, accept / reject, radius update, tolerance tests) is recorded with
its margin and its rounding uncertainty; a margin below 100x its uncertainty errors with a request to pick another seed, so that a
discrete flip never decides whether these tests pass.
"""
import ctypes as C
import numpy as np
import pytest
import scipy.linalg
from cerberus_b200 import abi, synth, lib
from oracle_lib import OracleBackend
from helpers import sim_backend, small_cfg
import dense_ref as dr

C_X = 2.5
MARGIN_FACTOR = 100.0
RATIOS = {}                 # (arm, case) -> max ratio, reported by the summary test under `pytest -s`

MODES = ("prior", "no_prior", "td_open", "ex_closed", "leg_bias_fixed", "imu_only", "skipped_imu")
LAYOUTS = ("chunk_split", "full_tile", "uncached_chunks", "sparse_anchors", "all_mono", "unseen_frame", "schur_staging", "abi_short_tracks", "huber_band")


# ---------------------------------------------------------------------------------------------------------------- layouts
def _cut(batch, w, f, anchor, n_obs, stereo=True):
    """Track f of a uniform window (anchor 0, 11 observations at obs_offset + k) cut to frames anchor .. anchor + n_obs - 1."""
    fe = batch.features[w]
    off = int(fe["obs_offset"][f]) + anchor
    fe["start_frame"][f], fe["n_obs"][f], fe["obs_offset"][f] = anchor, n_obs, off
    if not stereo:
        batch.obs[w]["is_stereo"][off:off + n_obs] = 0
    batch.para_Feature[w][f] = -1.0                   # re-triangulated below


def _retriangulate(batch, ob):
    """FeatureManager::triangulate for the tracks that were cut (para_Feature <= 0), as the estimator initialises them."""
    depth = ob.triangulate(batch)
    for w in range(batch.n):
        nf = batch.descs[w].n_features
        cut = batch.para_Feature[w][:nf] <= 0
        batch.para_Feature[w][:nf][cut] = 1.0 / depth[w][:nf][cut]


def layout_features(name):
    return {"chunk_split": 130, "full_tile": 64, "uncached_chunks": 521, "sparse_anchors": 8, "all_mono": 24, "unseen_frame": 40,
            "schur_staging": 65, "abi_short_tracks": 24, "huber_band": 30}[name]


def make_layout(name, mode, ob, cfg, window0=0, staging=(31, 32, 33, 65)):
    """A WindowBatch of layout `name` under window mode `mode` (1 window; schur_staging: one window per feature count in `staging`)."""
    F = layout_features(name)
    n = len(staging) if name == "schur_staging" else 1
    b = synth.generate_batch(n, F, ob, cfg=cfg, window0=window0 + 7 * LAYOUTS.index(name), prior_features=8, realistic=(name == "schur_staging"),
                             with_prior=mode != "no_prior", use_leg=mode != "imu_only")
    if name == "chunk_split":
        for f in range(65, 130): _cut(b, 0, f, 7, 4)
    elif name == "full_tile":
        for f in range(64): _cut(b, 0, f, 3, 8)
    elif name == "uncached_chunks":
        for f in range(520): _cut(b, 0, f, f // 65, 11 - f // 65)
        _cut(b, 0, 520, 8, 3)                          # chunk 17, anchor 8: read from the global chunk table
    elif name == "sparse_anchors":
        for f in range(8): _cut(b, 0, f, f, 4, stereo=f % 2 == 0)
    elif name == "all_mono":
        for f in range(F): _cut(b, 0, f, f % 8, min(4 + f % 3, 11 - f % 8), stereo=False)
    elif name == "unseen_frame":
        for f in range(F): _cut(b, 0, f, 0 if f % 2 == 0 else 6, 5)
    elif name == "schur_staging":
        for w, nf in enumerate(staging): b.descs[w].n_features = nf
    elif name == "abi_short_tracks":
        for f in range(F):
            a, L, st = [(8, 3, True), (9, 2, True), (10, 1, True), (2, 1, True), (5, 2, False), (0, 11, True)][f % 6]
            _cut(b, 0, f, a, L, stereo=st)
    elif name == "huber_band":
        o, fe = b.obs[0], b.features[0]
        for f in range(F):
            if f % 3 == 0: continue
            shift = (1.0 if f % 3 == 1 else 25.0) / cfg.visual_sqrt_info      # whitened |r| ~ 1 (the Huber knee) or ~ 25 (far outside)
            off = int(fe["obs_offset"][f])
            for k in range(1, 11):
                o["point"][off + k] += shift * np.array([np.cos(k + f), np.sin(k + f)])
                o["pointRight"][off + k] += shift * np.array([np.sin(k + f), -np.cos(k + f)])
    _retriangulate(b, ob)
    for w in range(b.n):
        if mode == "td_open":
            b.descs[w].td_open = 1; b.states[w].para_Td[0] = 0.004
        elif mode == "ex_closed":
            b.descs[w].extrinsic_open = 0
        elif mode == "skipped_imu":
            (b.preint if b.imu_preint is None else b.imu_preint)[w][3]["sum_dt"] = 10.5
    return b


def mode_cfg(mode, max_features, iters, max_batch=4):
    cfg = small_cfg(max_batch=max_batch, max_features=max_features, iters=iters)
    if mode == "leg_bias_fixed":
        cfg.optimize_leg_bias = 0
    return cfg


def with_iterations(cfg, k, **kw):
    c = abi.SolverConfig.from_buffer_copy(cfg)
    c.max_num_iterations = k
    for name, v in kw.items():
        setattr(c, name, v)
    return c


# ---------------------------------------------------------------------------------------------------------------- comparisons
def check_no_near_ties(tr, K, label, min_k=None):
    """Error when a decision up to iteration K is within MARGIN_FACTOR x its rounding uncertainty.  With min_k, the comparison is
    instead cut before the first such decision (tr.k_safe), and only an earlier one than min_k errors: late iterations of a
    converging window are ill-conditioned (kappa up to 1e16 along the gauge of a prior-less window), and past a near tie the
    reference cannot say which branch an fp64 arm should take."""
    if min_k is not None:
        ties = [m[0] for m in tr.margins if m[0] <= K and abs(m[2]) < MARGIN_FACTOR * m[3]]
        tr.k_safe = min(ties) - 1 if ties else K
        if tr.k_safe >= min_k:
            return
        K = min_k
    m = tr.closest_margin(K)
    if m is not None and abs(m[2]) < MARGIN_FACTOR * m[3]:
        raise RuntimeError(f"{label}: decision '{m[1]}' at iteration {m[0]} has margin {m[2]:.3e}, only {abs(m[2]) / m[3]:.1f}x its rounding "
                           f"uncertainty {m[3]:.3e}: the arms may legitimately branch differently here -- pick another seed (window0)")


def state_error(batch, w, x_ref, x0, blocks):
    """max |x - x_ref| over the active blocks; the constant blocks must not have moved at all."""
    got = dr.State.from_batch(batch, w)
    err = 0.0
    for name in ("pose", "sb", "lb", "ex", "td", "lam"):
        a, r = getattr(got, name), getattr(x_ref, name)
        if name in blocks and not blocks[name]:
            assert (a == getattr(x0, name)).all(), f"constant block {name} moved"
            continue
        err = max(err, float(np.abs(a - r).max()) if a.size else 0.0)
    return err


def compare_arm(arm_name, make_solver, batch, cfg, traces, ks, label, **cfg_kw):
    """Solve `batch` from its current states with max_num_iterations = k for every k in ks; compare with iterate k of each trace."""
    saved = batch.copy_states()
    worst = 0.0
    try:
        for k in ks:
            batch.restore_states(saved)
            solve = make_solver(with_iterations(cfg, k, **cfg_kw))
            rep = solve(batch)
            for w, tr in enumerate(traces):
                if k > getattr(tr, "k_safe", k):
                    continue
                x_ref, rr = tr.at(k)
                where = f"{label} window {w} [{arm_name}, k={k}]"
                assert rep["iterations"][w] == rr["iterations"], (where, rep[w], rr)
                assert rep["num_successful_steps"][w] == rr["num_successful_steps"], (where, rep[w], rr)
                assert rep["termination"][w] == rr["termination"], (where, rep[w], rr)
                err = state_error(batch, w, x_ref, tr.win.x0, tr.win.blocks)
                # the arm's cost is that of its own iterate (which differs from x_k^ref by the rounding bounded below)
                own = tr.win.cost(dr.State.from_batch(batch, w))
                assert abs(rep["final_cost"][w] - own) <= 1e-11 * own, (where, rep["final_cost"][w], own, rr["final_cost"])
                scale = dr.EPS64 * tr.step_scale(k)
                ratio = err / scale if scale > 0 else (0.0 if err == 0 else np.inf)
                worst = max(worst, ratio)
                assert ratio <= C_X, f"{where}: max |x_k - x_k^ref| = {err:.3e} is {ratio:.3g} x eps * sum kappa_j |delta_j| ({scale:.3e}); C_X = {C_X}"
    finally:
        batch.restore_states(saved)
    RATIOS[(arm_name, label)] = max(RATIOS.get((arm_name, label), 0.0), worst)
    return worst


def sim_solver(cfg):
    be = sim_backend(cfg)
    return lambda batch: be.solve_batch(batch)


def oracle_solver(cfg):
    o = OracleBackend(cfg)
    return lambda batch: o.solve_batch(batch, nthreads=4)


def references(batch, cfg, ob, K, **solve_kw):
    trs = [dr.DenseWindow(batch, w, cfg, ob).solve(max_iterations=K, **solve_kw) for w in range(batch.n)]
    return trs


ob = OracleBackend()


# ---------------------------------------------------------------------------------------------------------------- the reference itself
@pytest.fixture(scope="module")
def small():
    cfg = mode_cfg("prior", 8, 2)
    b = make_layout("sparse_anchors", "prior", ob, cfg)
    return b, cfg, dr.DenseWindow(b, 0, cfg, ob)


def test_reference_cost_and_gradient_equal_the_oracle_probe(small):
    b, cfg, win = small
    saved = b.copy_states()
    g0, d0 = OracleBackend(with_iterations(cfg, 0)).solve_window(b, 0, want_probe=True)
    b.restore_states(saved)
    cost, g, H = win.linearize(win.x0)
    g, dg = g.astype(np.float64), np.diagonal(H).astype(np.float64)
    assert abs(cost - b.reports[0].initial_cost) <= 1e-12 * cost
    assert np.abs(g - g0).max() <= 1e-12 * np.abs(g0).max() * 1e2 and (np.abs(g - g0) <= 1e-12 * np.abs(g0) + 1e-13 * np.abs(g0).max()).all()
    assert (np.abs(dg - d0) <= 1e-12 * np.abs(d0)).all()
    assert win.counts["K3"] > 0 and win.counts["K2"] > 0 and win.counts["prior"] == 1


def test_reference_gradient_matches_central_differences_of_the_cost(small):
    """Columns of J^T r against (cost(x [+] h e_c) - cost(x [+] -h e_c)) / 2h through Plus: a position, a rotation, an extrinsic rotation,
    a velocity, a gyroscope bias, a leg bias, and inverse depths of a mono and a stereo track."""
    b, cfg, win = small
    _, g, _ = win.linearize(win.x0)
    g = g.astype(np.float64)
    for c in (6 * 4 + 1, 6 * 7 + 4, 66 + 5, 78 + 9 * 3, 78 + 9 * 5 + 7, 177 + 4 * 2 + 1, dr.NR + 1, dr.NR + 4):
        h = 1e-6 * max(1.0, abs(win.x0.lam[c - dr.NR]) if c >= dr.NR else 1.0)
        e = np.zeros(win.n); e[c] = h
        fd = (win.cost(dr.plus(win.x0, e, win.blocks)) - win.cost(dr.plus(win.x0, -e, win.blocks))) / (2 * h)
        assert abs(fd - g[c]) <= 1e-5 * np.abs(g).max() + 1e-6 * abs(g[c]), (c, fd, g[c])


def test_reference_step_matches_qr_least_squares_and_mpmath(small):
    """The refined Gauss-Newton solve of the first step against (i) scipy lstsq (QR, no normal equations) of [Js; sqrt(mu) D] y = [r; 0]
    within 10 kappa eps, (ii) the residual of the same longdouble system evaluated by mpmath at 30 digits."""
    import mpmath
    b, cfg, win = small
    tr = win.solve(max_iterations=1)
    act = tr.act
    J, r = win.dense_jacobian(win.x0)
    J = J[:, act]
    H = tr.H0[np.ix_(act, act)]
    s = 1.0 / (1.0 + np.sqrt(np.diagonal(H).astype(np.float64)))
    Js = J * s
    A = (s[:, None] * H.astype(np.float64) * s[None, :])
    D = np.sqrt(np.clip(np.diagonal(A), 1e-6, 1e32))
    mu = tr.steps[0]["mu"]
    aug = np.vstack([Js, np.sqrt(mu) * np.diag(D)])
    y_qr = scipy.linalg.lstsq(aug, np.concatenate([r, np.zeros(len(act))]), lapack_driver="gelsd")[0]
    Areg = (s[:, None] * H * s[None, :]).astype(dr.LD) + np.diag((mu * D * D).astype(dr.LD))
    bs = (s * tr.g0[act]).astype(dr.LD)
    kappa = tr.steps[0]["kappa"]
    y = dr.refined_solve(Areg, bs, 1e-3 * kappa * dr.EPS64)
    ny = float(np.sqrt(np.dot(y, y)))
    assert np.abs(y.astype(np.float64) - y_qr).max() <= 10 * kappa * dr.EPS64 * ny
    mpmath.mp.dps = 30
    n = len(act)
    def mp(v):                                            # a longdouble as the exact sum of two doubles
        hi = np.float64(v)
        return mpmath.mpf(float(hi)) + mpmath.mpf(float(np.float64(v - dr.LD(hi))))
    Am = mpmath.matrix([[mp(Areg[i, j]) if Areg[i, j] != 0 else 0 for j in range(n)] for i in range(n)])
    ym = mpmath.matrix([mp(v) for v in y])
    bm = mpmath.matrix([mp(v) for v in bs])
    res = bm - Am * ym
    res64 = np.array([float(v) for v in res])
    corr = scipy.linalg.cho_solve(scipy.linalg.cho_factor(Areg.astype(np.float64), lower=True), res64)
    assert np.linalg.norm(corr) <= 2e-3 * kappa * dr.EPS64 * ny          # the refined solution is the 30-digit one to far below kappa * eps64


# ---------------------------------------------------------------------------------------------------------------- linearisation
LIN_CASES = [("chunk_split", "prior"), ("full_tile", "td_open"), ("uncached_chunks", "prior"), ("sparse_anchors", "no_prior"),
             ("all_mono", "prior"), ("unseen_frame", "skipped_imu"), ("schur_staging", "leg_bias_fixed"), ("abi_short_tracks", "td_open"),
             ("huber_band", "ex_closed"), ("abi_short_tracks", "imu_only")]


@pytest.mark.parametrize("layout,mode", LIN_CASES)
def test_linearisation_matches_dense_reference_sim(layout, mode):
    """cerb_debug_linearize at x0: cost to 1e-12 relative, gradient and diag(J^T J) elementwise to 1e-10 of their max."""
    F = layout_features(layout)
    cfg = mode_cfg(mode, F, 1)
    b = make_layout(layout, mode, ob, cfg)
    s = sim_backend(cfg)
    s.upload(b)
    for w in range(b.n):
        win = dr.DenseWindow(b, w, cfg, ob)
        cost, g, H = win.linearize(win.x0)
        g, dg = g.astype(np.float64), np.diagonal(H).astype(np.float64)
        c1, g1, d1 = s.debug_linearize(b, w)
        assert abs(c1 - cost) <= 1e-12 * cost, (layout, mode, w, c1, cost)
        assert np.abs(g1 - g).max() <= 1e-10 * np.abs(g).max(), (layout, mode, w, int(np.abs(g1 - g).argmax()))
        assert np.abs(d1 - dg).max() <= 1e-10 * np.abs(dg).max(), (layout, mode, w, int(np.abs(d1 - dg).argmax()))
    if layout == "huber_band":
        sq = np.concatenate([fa.sq for fa in win.evaluate(win.x0) if fa.huber])
        assert ((sq > 0.5) & (sq < 2.0)).sum() >= 5 and (sq > 100.0).sum() >= 100 and (sq <= 1.0).sum() >= 5     # both Huber branches, and the knee
    if layout == "all_mono":
        assert win.counts["K2"] == 0 and win.counts["K3"] == 0
    if layout == "abi_short_tracks":
        k3_only = [f for f in range(win.nf) if b.features[0]["n_obs"][f] == 1]
        assert k3_only and (np.abs(g[dr.NR + np.array(k3_only)]) > 0).all()


# ---------------------------------------------------------------------------------------------------------------- every iterate
ITER_CASES_SIM = [("chunk_split", "prior"), ("full_tile", "no_prior"), ("sparse_anchors", "td_open"), ("all_mono", "prior"),
                  ("unseen_frame", "skipped_imu"), ("schur_staging", "prior"), ("abi_short_tracks", "ex_closed"), ("huber_band", "leg_bias_fixed"),
                  ("sparse_anchors", "imu_only")]


@pytest.mark.parametrize("layout,mode", ITER_CASES_SIM)
def test_every_iterate_matches_dense_reference_sim(layout, mode):
    K = 2
    cfg = mode_cfg(mode, layout_features(layout), K)
    b = make_layout(layout, mode, ob, cfg, staging=(31, 32, 33))          # (the GPU tier adds the 65-feature window)
    trs = references(b, cfg, ob, K)
    for w, tr in enumerate(trs):
        check_no_near_ties(tr, K, f"{layout}/{mode} window {w}")
    compare_arm("oracle", oracle_solver, b, cfg, trs, range(1, K + 1), f"{layout}/{mode}")
    compare_arm("sim", sim_solver, b, cfg, trs, range(1, K + 1), f"{layout}/{mode}")


# ---------------------------------------------------------------------------------------------------------------- dogleg branches
def _branch_case(make_solver, arm_name, K):
    cfg = mode_cfg("prior", 30, K)
    b = make_layout("huber_band", "prior", ob, cfg, window0=3)
    win = dr.DenseWindow(b, 0, cfg, ob)
    first = win.solve(max_iterations=1).steps[0]
    gn, cauchy = first["gn_norm"], first["alpha"] * first["grad_norm"]
    assert cauchy < 0.5 * gn, "the window has no room between the Cauchy point and the Gauss-Newton step"
    for case, radius in (("gauss_newton", 4.0 * gn), ("gradient", 0.25 * cauchy), ("interpolated", np.sqrt(gn * cauchy))):
        tr = win.solve(max_iterations=K, initial_radius=radius)
        assert tr.steps[0]["case"] == case, (case, tr.steps[0]["case"])
        check_no_near_ties(tr, K, f"dogleg {case}")
        compare_arm(arm_name, make_solver, b, cfg, [tr], range(1, K + 1), f"dogleg_{case}", initial_trust_region_radius=radius)


def _rejected_case(make_solver, arm_name, K):
    """min_relative_decrease raised to 0.97 on a perturbed window: a step is rejected, the next one reuses the Gauss-Newton step and the
    gradient of the same linearisation with half the radius (and the kernel discards its speculative linearisation of the candidate)."""
    cfg = mode_cfg("prior", 12, K)
    b = synth.generate_batch(1, 12, ob, cfg=cfg, window0=900, prior_features=6)
    st, rng = b.state_array(), np.random.default_rng(3)
    st["para_Pose"][0, :, :3] += rng.normal(0, 0.3, (11, 3))
    b.para_Feature[0] *= np.exp(rng.normal(0, 0.5, b.para_Feature.shape[1]))
    tr = dr.DenseWindow(b, 0, cfg, ob).solve(max_iterations=K, min_relative_decrease=0.97)
    rej = [s["k"] for s in tr.steps if s.get("outcome") == "rejected"]
    assert rej and any(s["reuse"] for s in tr.steps), [s.get("outcome") for s in tr.steps]
    check_no_near_ties(tr, K, "rejected step")
    ks = sorted({rej[0] - 1, rej[0], min(rej[0] + 1, K), K})
    compare_arm(arm_name, make_solver, b, cfg, [tr], ks, "rejected_step", min_relative_decrease=0.97)


def test_dogleg_branches_match_dense_reference_sim():
    _branch_case(sim_solver, "sim", 1)
    _branch_case(oracle_solver, "oracle", 1)


def test_rejected_step_matches_dense_reference_sim():
    _rejected_case(sim_solver, "sim", 5)
    _rejected_case(oracle_solver, "oracle", 5)


def test_mu_update_after_accepted_step_sim(monkeypatch):
    """Started at mu = 1e-3 (CERB_TEST_INITIAL_MU, read by both arms), an accepted step lowers mu to 2e-4 and the second Gauss-Newton
    step is damped by that: the second iterate pins DoglegStrategy::StepAccepted's mu update."""
    monkeypatch.setenv("CERB_TEST_INITIAL_MU", "1e-3")
    cfg = mode_cfg("prior", 30, 2)
    b = make_layout("huber_band", "prior", ob, cfg, window0=9)
    tr = dr.DenseWindow(b, 0, cfg, ob).solve(max_iterations=2, initial_mu=1e-3)
    assert [s["mu"] for s in tr.steps] == [1e-3, 2e-4] and all(s["outcome"] == "accepted" for s in tr.steps)
    check_no_near_ties(tr, 2, "mu update")
    compare_arm("oracle", oracle_solver, b, cfg, [tr], (1, 2), "mu_update")
    compare_arm("sim", sim_solver, b, cfg, [tr], (1, 2), "mu_update")


# ---------------------------------------------------------------------------------------------------------------- GPU tier
def gpu_solver(cfg):
    def solve(batch):
        be = lib.Backend(cfg)
        try:
            return be.solve_batch(batch)
        finally:
            be.close()
    return solve


_GPU_REFS = {}


def gpu_case(layout, mode, K=12):
    """(batch, cfg, references) of one layout under one mode, built once per process for the two GPU tests below."""
    if (layout, mode) not in _GPU_REFS:
        cfg = mode_cfg(mode, layout_features(layout), K)
        b = make_layout(layout, mode, ob, cfg, window0=100)
        trs = references(b, cfg, ob, K)
        for w, tr in enumerate(trs):
            check_no_near_ties(tr, K, f"{layout}/{mode} window {w}", min_k=2)
        _GPU_REFS[(layout, mode)] = (b, cfg, trs)
    return _GPU_REFS[(layout, mode)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_every_iterate_matches_dense_reference_gpu(mode):
    """Every layout under this window mode on the H100: the kernel against the reference at every k = 1..12, the oracle at k = 1, 2, 12
    (each window up to its last iteration before a near-tie decision, at least 2)."""
    K = 12
    for layout in LAYOUTS:
        b, cfg, trs = gpu_case(layout, mode, K)
        compare_arm("gpu", gpu_solver, b, cfg, trs, range(1, K + 1), f"{layout}/{mode}")
        compare_arm("oracle", oracle_solver, b, cfg, trs, (1, 2, K), f"{layout}/{mode}")


def merge_batches(batches):
    """One WindowBatch holding the windows of `batches` (same preintegration kind)."""
    n = sum(b.n for b in batches)
    F = max(b.max_features for b in batches)
    O = max(b.max_obs for b in batches)
    out = abi.WindowBatch(n, F, O)
    if batches[0].imu_preint is not None:
        out.use_imu_only()
    w = 0
    for b in batches:
        for v in range(b.n):
            out.features[w][:b.max_features] = b.features[v]; out.obs[w][:b.max_obs] = b.obs[v]
            out.prior_J[w] = b.prior_J[v]; out.prior_r[w] = b.prior_r[v]; out.para_Feature[w][:b.max_features] = b.para_Feature[v]
            if b.imu_preint is None: out.preint[w] = b.preint[v]
            else: out.imu_preint[w] = b.imu_preint[v]
            C.memmove(C.byref(out.states[w]), C.byref(b.states[v]), C.sizeof(abi.WindowState))
            out.states[w].para_Feature = out.para_Feature[w].ctypes.data_as(abi.c_dp)
            d, sd = out.descs[w], b.descs[v]
            d.n_features, d.n_obs, d.extrinsic_open, d.td_open = sd.n_features, sd.n_obs, sd.extrinsic_open, sd.td_open
            C.memmove(C.byref(d.prior), C.byref(sd.prior), C.sizeof(abi.Prior))
            d.prior.linearized_jacobians = out.prior_J[w].ctypes.data_as(abi.c_dp)
            d.prior.linearized_residuals = out.prior_r[w].ctypes.data_as(abi.c_dp)
            w += 1
    return out


@pytest.mark.gpu
def test_batch_scale_every_window_matches_dense_reference_gpu():
    """All layouts under the window modes of the default config, tiled to 264 windows (two waves of the persistent grid on 132 SMs),
    so that chunks of different layouts share CTAs; every window against its reference at k = 1, 2, 6 and 12."""
    K = 12
    cfg = mode_cfg("prior", 521, K, max_batch=264)
    parts, trs = [], []
    for mode in ("prior", "no_prior", "td_open", "ex_closed", "skipped_imu"):
        for layout in LAYOUTS:
            b, _, t = gpu_case(layout, mode, K)
            parts.append(b)
            trs += t
    base = merge_batches(parts)
    big = synth.tile_batch(base, 264)
    tiled = [trs[w % base.n] for w in range(264)]
    compare_arm("gpu", gpu_solver, big, cfg, tiled, (1, 2, 6, 12), "batch_264")


@pytest.mark.gpu
def test_dogleg_branches_and_rejected_step_gpu():
    _branch_case(gpu_solver, "gpu", 3)
    _rejected_case(gpu_solver, "gpu", 8)


def test_report_ratios():
    """Prints the measured ratios max |x_k - x_k^ref| / (eps sum kappa_j |delta_j|) of the tests that ran in this process, and how
    many iterations each GPU case compared (pytest -s)."""
    for (arm, label), r in sorted(RATIOS.items()):
        print(f"ratio {arm:7s} {label:32s} {r:.3e}")
    for (layout, mode), (_, _, trs) in sorted(_GPU_REFS.items()):
        print(f"compared iterations {layout}/{mode}: {[getattr(t, 'k_safe', None) for t in trs]}")

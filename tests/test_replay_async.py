"""Asynchronous fleet replay (cerb_replay_step_robots, cerb_replay_reset_robot): each step takes whichever robots have a frame, each at its
own stamp; robots start late, stop when their sequence ends and restart (the reference's clearState) while the others keep running.  Checked
on one schedule with every such event:
  * resident mode == default mode (paths, flags, feature ids, reports, the device store after every step),
  * every robot in the fleet == the same robot replayed alone with the same seeds and reset,
  * every robot listed, in any order, at one stamp == cerb_replay_step,
  * after a reset + re-seed at k0 a robot continues exactly as a fresh replay seeded at k0,
  * rejected calls change nothing and move nothing,
  * a step of a subset moves what a replay holding only that subset moves,
  * each robot against the oracle arm (ReplayDriver(OracleOps)) on its own slice of the sequence.
CPU tier on the kernel simulator, GPU tier under -m gpu."""
import ctypes as C
import numpy as np
import pytest
from cerberus_b200 import abi, synth, estimator, lib
from cerberus_b200.lib import CerbError
from helpers import sim_backend
from oracle_lib import OracleOps
from test_resident import _assert_store_matches

W = abi.WINDOW_SIZE


def _cfg(n, F, iters):
    cfg = abi.default_config(); cfg.max_batch = n; cfg.max_features = 2 * F; cfg.max_obs = 2 * F * abi.NUM_FRAMES; cfg.max_num_iterations = iters
    return cfg


class Fleet:
    """A schedule over robots 0 .. n - 1; robot r replays robot src[r] of seq, frames [0, lengths[r]).  events: ("seed", r, k0),
    ("reset", r), ("step", [(r, frame, first_after_seed), ...]) with the rows of a step in list order."""

    def __init__(self, n, lengths, src=None, late=None, late_tick=3, reset=None, reset_after=2, reset_k0=2, p_step=0.6, seed=11):
        self.n, self.lengths = n, list(lengths)
        self.src = list(range(n)) if src is None else list(src)
        self.phase = [0.0371 * r for r in range(n)]
        rng = np.random.default_rng(seed)
        ev, nxt, first, done = [], {}, {}, {r: 0 for r in range(n)}
        for r in range(n):
            if r != late: ev.append(("seed", r, 0)); nxt[r] = first[r] = W
        pending, tick = None, 0
        while True:
            if late is not None and tick == late_tick: ev.append(("seed", late, 0)); nxt[late] = first[late] = W
            if pending is not None: ev.append(("seed", pending, reset_k0)); nxt[pending] = first[pending] = reset_k0 + W; pending = None
            ready = [r for r in nxt if nxt[r] < self.lengths[r]]
            if not ready:
                if late is not None and late not in nxt: tick += 1; continue
                break
            pick = [r for r in ready if rng.uniform() < p_step] or [ready[int(rng.integers(len(ready)))]]
            rng.shuffle(pick)
            ev.append(("step", [(r, nxt[r], nxt[r] == first[r]) for r in pick]))
            for r in pick: nxt[r] += 1; done[r] += 1
            if reset is not None and reset in pick and done[reset] == reset_after:
                ev.append(("reset", reset)); del nxt[reset]; pending = reset     # the others step once before it is seeded again
            tick += 1
        self.events = ev

    def header(self, r, k):
        return 0.1 * k + self.phase[r]

    def segments(self, r):
        """(k0, k_end) of every stretch robot r was stepped through after a seed"""
        out = []
        for e in self.events:
            if e[0] == "seed" and e[1] == r: out.append([e[2], e[2] + W])
            if e[0] == "step":
                for (q, k, _) in e[1]:
                    if q == r: out[-1][1] = k + 1
        return [tuple(s) for s in out]

    def step_args(self, seq, rows):
        imgs = [seq.images[k][self.src[r]] for (r, k, _) in rows]
        firsts = [seq.first[self.src[r], k - 1] for (r, k, _) in rows]
        smp = [seq.samples[self.src[r]][k - 1][:0] if fst else seq.samples[self.src[r]][k - 1] for (r, k, fst) in rows]
        return imgs, firsts, smp, [self.header(r, k) for (r, k, _) in rows]

    def apply(self, rep, seq, e):
        if e[0] == "seed": rep.seed_robot(e[1], seq, self.src[e[1]], e[2])
        elif e[0] == "reset": rep.reset(e[1])
        else:
            imgs, firsts, smp, hdr = self.step_args(seq, e[1])
            rep.step(imgs, firsts, smp, 0.0, robots=[r for (r, _, _) in e[1]], headers=hdr)

    def run_alone(self, rep, seq, r):
        """robot r's events only, on robot 0 of a one-robot replay, with cerb_replay_step"""
        for e in self.events:
            if e[0] == "seed" and e[1] == r: rep.seed_robot(0, seq, self.src[r], e[2])
            elif e[0] == "reset" and e[1] == r: rep.reset(0)
            elif e[0] == "step":
                rows = [x for x in e[1] if x[0] == r]
                if rows:
                    imgs, firsts, smp, hdr = self.step_args(seq, rows)
                    rep.step(imgs, firsts, smp, hdr[0])
        return rep

    def reports_of(self, rep, r):
        out = []
        for e, got in zip([e for e in self.events if e[0] == "step"], rep.reports):
            out += [got[i] for i, x in enumerate(e[1]) if x[0] == r]
        return out


def _same(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _assert_robot_equal(ra, wa, rb, wb, reports_a, reports_b):
    assert _same(ra.path(wa), rb.path(wb)), f"robot {wa} / {wb}: published states differ"
    assert (ra.flag_history(wa) == rb.flag_history(wb)).all()
    assert ra.feature_ids(wa) == rb.feature_ids(wb)
    assert len(reports_a) == len(reports_b) and all(x.tobytes() == y.tobytes() for x, y in zip(reports_a, reports_b))


def _setup(n, F, frames, tracked, iters, src_n=None):
    cfg, pcfg = _cfg(n, F, iters), abi.default_preint_config()
    seq = synth.generate_sequence(src_n or n, frames, tracked=tracked, max_len=12, min_len=3)
    return cfg, pcfg, seq


def _small_fleet():
    # robot 0 restarts after one step from frame 1, robot 2 joins after one tick, the lengths differ
    return Fleet(3, [13, 12, 12], late=2, late_tick=1, reset=0, reset_after=1, reset_k0=1)


# the kernel simulator takes ~3 s per robot and step at this size
SIM = dict(F=24, frames=13, tracked=14, iters=2)


# ---- the checks, on any backend ----------------------------------------------------------------------------------------------------------

def _check_modes_and_alone(make_backend, fleet, cfg, pcfg, seq, F, alone=None, store_every_step=True):
    """(1) resident == default under the schedule, with (store_every_step) every robot's store after every step and reset; (2) each robot in the
    fleet == alone"""
    be_r = make_backend(cfg)
    dflt = estimator.NativeReplay(make_backend(cfg), pcfg, fleet.n, max_features=F)
    res = estimator.NativeReplay(be_r, pcfg, fleet.n, max_features=F, resident=True)
    for e in fleet.events:
        fleet.apply(dflt, seq, e); fleet.apply(res, seq, e)
        if store_every_step and e[0] != "seed":        # every robot's store, listed or not: a step leaves the others' windows alone
            for r in range(fleet.n): _assert_store_matches(be_r, dflt, res, r)
    for r in range(fleet.n):
        _assert_robot_equal(dflt, r, res, r, fleet.reports_of(dflt, r), fleet.reports_of(res, r))
        assert dflt.path(r).shape[0] == sum(k1 - k0 - W for (k0, k1) in fleet.segments(r))
    for r in (range(fleet.n) if alone is None else alone):
        one = fleet.run_alone(estimator.NativeReplay(make_backend(_cfg(1, F, cfg.max_num_iterations)), pcfg, 1, max_features=F, resident=True), seq, r)
        _assert_robot_equal(res, r, one, 0, fleet.reports_of(res, r), [x[0] for x in one.reports])
    return dflt, res


def _check_all_listed_equals_step(make_backend, cfg, pcfg, seq, F, n_steps, resident):
    """(3) every robot listed, shuffled, at one stamp == cerb_replay_step"""
    n = seq.n
    a = estimator.NativeReplay(make_backend(cfg), pcfg, n, max_features=F, resident=resident).run(seq, n_steps)
    b = estimator.NativeReplay(make_backend(cfg), pcfg, n, max_features=F, resident=resident)
    b.seed(seq)
    rng = np.random.default_rng(3)
    for k in range(W, W + n_steps):
        order = rng.permutation(n)
        smp = [seq.samples[w][k - 1][:0] if k == W else seq.samples[w][k - 1] for w in order]
        b.step([seq.images[k][w] for w in order], [seq.first[w, k - 1] for w in order], smp, float(k), robots=order.tolist())
        back = np.argsort(order)
        b.reports[-1] = b.reports[-1][back]
    for w in range(n):
        _assert_robot_equal(a, w, b, w, [x[w] for x in a.reports], [x[w] for x in b.reports])


def _check_reset(make_backend, cfg, pcfg, seq, F, modes=(False, True), k0=1):
    """(4) reset + seed_robot(k0) continues exactly as a fresh replay seeded at k0; in resident mode the reset empties the window"""
    for resident in modes:
        be = make_backend(cfg)
        rep = estimator.NativeReplay(be, pcfg, 2, max_features=F, resident=resident).run(seq, 1)
        rows_before = rep.path(0).shape[0]
        rep.reset(0)
        feats, ids, _, _, cur, slots, prior, _, _ = rep.window(0)
        assert len(feats) == 0 and len(ids) == 0 and not prior.valid and slots.tolist() == list(range(W))
        if resident:
            assert not be.resident_read_window(0)[2].valid
        assert rep.path(0).shape[0] == rows_before == rep.flag_history(0).shape[0]
        # robot 1 steps while robot 0 waits for its seed
        rep.step([seq.images[W + 1][1]], [seq.first[1, W]], [seq.samples[1][W]], float(W + 1), robots=[1])
        rep.seed_robot(0, seq, 0, k0)
        fresh = estimator.NativeReplay(make_backend(_cfg(1, F, cfg.max_num_iterations)), pcfg, 1, max_features=F, resident=resident)
        fresh.seed_robot(0, seq, 0, k0)
        for k in range(k0 + W, seq.n_frames):
            smp = seq.samples[0][k - 1][:0] if k == k0 + W else seq.samples[0][k - 1]
            rep.step([seq.images[k][0]], [seq.first[0, k - 1]], [smp], float(k), robots=[0])
            fresh.step([seq.images[k][0]], [seq.first[0, k - 1]], [smp], float(k))
            fa, fb = rep.window(0)[0], fresh.window(0)[0]
            assert fa.tobytes() == fb.tobytes()                # same tracks in the same slots: the reset returned every slot, in order
        assert _same(rep.path(0)[rows_before:], fresh.path(0))
        assert (rep.flag_history(0)[rows_before:] == fresh.flag_history(0)).all() and rep.feature_ids(0) == fresh.feature_ids(0)


def _check_rejections(make_backend, cfg, pcfg, seq, F):
    """(5) every malformed step leaves paths, flags, the store and the traffic counters as they were"""
    be = make_backend(cfg)
    rep = estimator.NativeReplay(be, pcfg, 3, max_features=F, resident=True)
    for w in range(2): rep.seed_robot(w, seq, w)
    k = W
    rep.step([seq.images[k][w] for w in range(2)], [seq.first[w, k - 1] for w in range(2)], [seq.samples[w][k - 1][:0] for w in range(2)], 0.0, robots=[0, 1])
    rep.reset(1)                                                        # robot 1: reset, not seeded again
    L = be.lib
    # robot 2 is half seeded: frames 0 .. 4 only
    _p = lambda a: np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(abi.c_dp)
    for kk in range(5):
        first = np.ascontiguousarray(seq.first[2, max(kk - 1, 0): max(kk - 1, 0) + 1]); smp = np.ascontiguousarray(seq.samples[2][kk - 1]) if kk else first[:0]
        keep = []; im = rep._image(seq.images[kk][2], keep)
        be._check(L.cerb_replay_seed_frame(rep.r, 2, kk, _p(seq.p_g[2, kk]), _p(seq.R_g[2, kk]), _p(seq.v_g[2, kk]), first.ctypes.data,
                                           smp.ctypes.data if len(smp) else None, len(smp), C.byref(im), float(kk)))
    snap = lambda: ([rep.path(w).tobytes() for w in range(3)], [rep.flag_history(w).tobytes() for w in range(3)],
                    [[a.tobytes() if isinstance(a, np.ndarray) else bytes(a)[:C.sizeof(abi.Prior) - 16] for a in be.resident_read_window(w)] for w in range(3)],
                    rep.traffic(), len(rep.reports))
    before = snap(); moved = be.traffic()                            # (reading the store back is counted too)
    k = W + 1
    data = lambda rs: [min(max(r, 0), 2) for r in rs]                          # the inputs of a robot in range
    args = lambda rs: ([seq.images[k][r] for r in data(rs)], [seq.first[r, k - 1] for r in data(rs)], [seq.samples[r][k - 1] for r in data(rs)], 0.0)

    def rejected(call):
        with pytest.raises(CerbError) as e: call()
        assert e.value.code == abi.ERR_BAD_ARGUMENT

    rejected(lambda: rep.step(*args([0, 3]), robots=[0, 3]))                  # out of range
    rejected(lambda: rep.step(*args([0, -1]), robots=[0, -1]))
    rejected(lambda: rep.step(*args([0, 0]), robots=[0, 0]))                  # listed twice
    rejected(lambda: rep.step(*args([0, 1]), robots=[0, 1]))                  # reset, not seeded again
    rejected(lambda: rep.step(*args([2, 0]), robots=[2, 0]))                  # half seeded
    keep = []
    ims = (abi.Image * 1)(rep._image(seq.images[k][0], keep))
    fr = np.ascontiguousarray(np.stack([seq.first[0, k - 1]])); smp = np.ascontiguousarray(seq.samples[0][k - 1])
    ptrs = (C.c_void_p * 1)(smp.ctypes.data); ns = (C.c_int32 * 1)(len(smp)); hdr = np.zeros(1); rob = np.zeros(1, dtype=np.int32)
    i32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
    good = [rep.r, 1, i32(rob), ims, fr.ctypes.data, ptrs, ns, hdr.ctypes.data_as(abi.c_dp), None]
    rejected(lambda: be._check(L.cerb_replay_step_robots(*([rep.r, 0] + good[2:]))))      # n_active < 1
    for q in (2, 3, 4, 5, 6, 7):                                                # each array null in turn
        bad = list(good); bad[q] = None
        rejected(lambda: be._check(L.cerb_replay_step_robots(*bad)))
    # the resident layer's compact upload: repeats and windows out of range
    batch = synth.generate_batch(2, 6, make_backend(cfg), prior_features=0)      # (a backend of its own: it uploads)
    for w in range(2):
        for f in range(batch.descs[w].n_features): batch.features[w][f]["obs_offset"] = f * abi.NUM_FRAMES
    rejected(lambda: be.resident_upload_windows([1, 1], batch))
    rejected(lambda: be.resident_upload_windows([0, 3], batch))
    assert be.traffic() == moved and snap() == before
    be._check(L.cerb_replay_step_robots(*good))                                 # the accepted form of the same call
    assert rep.path(0).shape[0] == 2


def _check_subset_traffic(make_backend, cfg, pcfg, seq, F, n_steps):
    """(6) a step of subset S in a 3-robot resident replay moves what the same step moves in a replay that holds only S; robot 1 of the big
    replay steps on its own in between and changes nothing for S.  The first step after the seed also sends the seeded frames' observations,
    in as many copies as the replay's edit buffer (sized by its number of robots) needs: there the bytes are compared, later the copies too."""
    S = [2, 0]
    big = estimator.NativeReplay(make_backend(cfg), pcfg, 3, max_features=F, resident=True)
    small = estimator.NativeReplay(make_backend(_cfg(2, F, cfg.max_num_iterations)), pcfg, 2, max_features=F, resident=True)
    for w in range(3): big.seed_robot(w, seq, w)
    for i, w in enumerate(S): small.seed_robot(i, seq, w)
    for k in range(W, W + n_steps):
        smp = lambda w: seq.samples[w][k - 1][:0] if k == W else seq.samples[w][k - 1]
        big.step([seq.images[k][1]], [seq.first[1, k - 1]], [smp(1)], float(k), robots=[1])
        t0, s0 = big.traffic(), small.traffic()
        big.step([seq.images[k][w] for w in S], [seq.first[w, k - 1] for w in S], [smp(w) for w in S], float(k), robots=S)
        small.step([seq.images[k][w] for w in S], [seq.first[w, k - 1] for w in S], [smp(w) for w in S], float(k))
        t1, s1 = big.traffic(), small.traffic()
        for key in ("h2d_bytes", "d2h_bytes", "staged_bytes") + (("dma_ops",) if k > W else ()):
            assert t1[key] - t0[key] == s1[key] - s0[key], (k, key, t1[key] - t0[key], s1[key] - s0[key])
    for i, w in enumerate(S):
        assert _same(big.path(w), small.path(i))


class _Slice:
    """frames [k0, k1) of robot w of a sequence, as a one-robot sequence"""

    def __init__(self, seq, w, k0, k1):
        self.n, self.n_frames = 1, k1 - k0
        self.tic_g, self.ric_g = seq.tic_g[w: w + 1], seq.ric_g[w: w + 1]
        for name in ("p_g", "R_g", "v_g", "first", "p"):
            setattr(self, name, getattr(seq, name)[w: w + 1, k0: k1])
        self.samples = seq.samples[w: w + 1, k0: k1 - 1]
        self.images = [[seq.images[k][w]] for k in range(k0, k1)]


def _check_oracle(fleet, res, cfg, pcfg, seq, F, robots, tol_first=1e-6, tol=1e-6):
    """(7) each robot of the async run against the oracle arm on its slice: the first three frames of a stretch within tol_first, all within
    tol (the tolerances of test_replay_matches_oracle_sim on the simulator, of test_replay_50_frames_gpu on the H100, where 12 iterations and
    long chains let the eps-clamped marginalization amplify rounding differences)"""
    for r in robots:
        path, reps, row = res.path(r), fleet.reports_of(res, r), 0
        for (k0, k1) in fleet.segments(r):
            ora = estimator.ReplayDriver(OracleOps(cfg, eig_mode=1), cfg, pcfg, 1, max_features=F).run(_Slice(seq, fleet.src[r], k0, k1))
            Po, Ro = ora.poses(); m = Po.shape[1]
            P, R = path[row: row + m, 1:4], path[row: row + m, 4:13].reshape(m, 3, 3)
            dP, dR = np.abs(P - Po[0]).max(axis=1), np.abs(R - Ro[0]).max(axis=(1, 2))
            assert dP[:3].max() < tol_first and dR[:3].max() < tol_first and dP.max() < tol and dR.max() < tol, (r, k0, dP, dR)
            for a, b in zip(reps[row: row + m], ora.reports):
                assert a["iterations"] == b["iterations"][0]
            row += m
        assert row == path.shape[0]


# ---- CPU tier ---------------------------------------------------------------------------------------------------------------------------

def test_fleet_modes_and_alone_sim():
    fleet = _small_fleet()
    cfg, pcfg, seq = _setup(3, SIM["F"], SIM["frames"], SIM["tracked"], SIM["iters"])
    kinds = [e[0] for e in fleet.events]
    assert "reset" in kinds and len(set(fleet.lengths)) > 1
    assert any(len(e[1]) < fleet.n for e in fleet.events if e[0] == "step")
    _, res = _check_modes_and_alone(sim_backend, fleet, cfg, pcfg, seq, SIM["F"], alone=[0])
    _check_oracle(fleet, res, cfg, pcfg, seq, SIM["F"], [0])


def test_all_listed_equals_step_sim():
    cfg, pcfg, seq = _setup(2, SIM["F"], 12, SIM["tracked"], SIM["iters"])
    _check_all_listed_equals_step(sim_backend, cfg, pcfg, seq, SIM["F"], 2, True)


def test_reset_equals_fresh_replay_sim():
    cfg, pcfg, seq = _setup(2, SIM["F"], 13, SIM["tracked"], SIM["iters"])
    _check_reset(sim_backend, cfg, pcfg, seq, SIM["F"], modes=(True,))


def test_rejected_steps_change_nothing_sim():
    cfg, pcfg, seq = _setup(3, SIM["F"], 12, SIM["tracked"], 1)
    _check_rejections(sim_backend, cfg, pcfg, seq, SIM["F"])


def test_subset_traffic_sim():
    cfg, pcfg, seq = _setup(3, SIM["F"], 12, SIM["tracked"], 1)
    _check_subset_traffic(sim_backend, cfg, pcfg, seq, SIM["F"], 2)


# ---- GPU tier ---------------------------------------------------------------------------------------------------------------------------

def _gpu_backend(cfg):
    return lib.Backend(cfg)


@pytest.mark.gpu
def test_fleet_64_robots_gpu():
    """64 robots x up to 40 frames at F = 160: every check; the oracle arm on four robots (one of them restarted)"""
    n, F = 64, 160
    rng = np.random.default_rng(5)
    lengths = [40 - int(rng.integers(0, 12)) for _ in range(n)]
    fleet = Fleet(n, lengths, late=5, reset=0, reset_after=6, reset_k0=4, p_step=0.5)
    cfg, pcfg, seq = _setup(n, F, 40, 90, 12)
    _, res = _check_modes_and_alone(_gpu_backend, fleet, cfg, pcfg, seq, F, store_every_step=False)
    _check_oracle(fleet, res, cfg, pcfg, seq, F, [0, 1, 5, 17], tol_first=1e-5, tol=2e-3)
    cfg4, _, seq4 = _setup(4, F, 18, 90, 12)
    _check_all_listed_equals_step(_gpu_backend, cfg4, pcfg, seq4, F, 6, True)
    _check_all_listed_equals_step(_gpu_backend, cfg4, pcfg, seq4, F, 6, False)
    _check_reset(_gpu_backend, _cfg(2, F, 12), pcfg, seq4, F)
    _check_rejections(_gpu_backend, _cfg(3, F, 12), pcfg, seq4, F)
    _check_subset_traffic(_gpu_backend, _cfg(3, F, 12), pcfg, seq4, F, 4)


@pytest.mark.gpu
def test_fleet_256_robots_gpu():
    """256 robots, about a quarter stepping per tick, both modes equal; robots on the same source slice stay identical to each other"""
    n, F = 256, 160
    cfg, pcfg, seq = _setup(n, F, 24, 90, 12, src_n=16)
    fleet = Fleet(n, [24 - (r % 5) for r in range(n)], src=[r % 16 for r in range(n)], late=7, reset=3, reset_after=3, reset_k0=2, p_step=0.25)
    _check_modes_and_alone(_gpu_backend, fleet, cfg, pcfg, seq, F, alone=[0, 3, 7, 200], store_every_step=False)

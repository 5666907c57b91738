"""Resident sliding window (cerb_resident_*, cerb_replay_set_resident): the tracks, the preintegration records and the prior of every window
stay on the device across frames and the host sends each frame's edits.  The kernels and their inputs are the same as in the default mode, so
everything here is compared with `==`:
  * the device's store after every step against the window the default mode would have uploaded,
  * trajectories, keyframe decisions, feature lists and solve reports of the two modes,
  * a rejected call leaves the store as it was and issues no copy,
  * the bytes a step asks the library to move (a count, so it holds on the CPU simulator too).
CPU tier on the kernel simulator, GPU tier under -m gpu."""
import ctypes as C
import numpy as np
import pytest
from cerberus_b200 import abi, synth, estimator, lib
from cerberus_b200.lib import CerbError
from helpers import sim_backend

W = abi.WINDOW_SIZE
NFRM = abi.NUM_FRAMES
TRAVELLED = ("sum_dt", "delta_p", "delta_q", "delta_v", "delta_epsilon", "linearized_ba", "linearized_bg", "linearized_rho", "covariance")


def _cfg(n, F, iters=None):
    cfg = abi.default_config(); cfg.max_batch = n; cfg.max_features = 2 * F; cfg.max_obs = 2 * F * NFRM
    if iters is not None: cfg.max_num_iterations = iters
    return cfg


def _steps(rep, seq):
    """rep.run(seq), yielding after every step"""
    rep.seed(seq)
    for k in range(W, seq.n_frames):
        firsts = [seq.first[w, k - 1] for w in range(rep.n)]
        smp = [seq.samples[w][k - 1][:0] if k == W else seq.samples[w][k - 1] for w in range(rep.n)]
        rep.step([seq.images[k][w] for w in range(rep.n)], firsts, smp, float(k))
        yield k


def _pair(make_backend, cfg, pcfg, n, F, **kw):
    be_d, be_r = make_backend(cfg), make_backend(cfg)
    return (be_d, estimator.NativeReplay(be_d, pcfg, n, max_features=F, **kw)), (be_r, estimator.NativeReplay(be_r, pcfg, n, max_features=F, resident=True, **kw))


def _same_bits(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _assert_same_replay(dflt, res, n):
    for w in range(n):
        assert _same_bits(dflt.path(w), res.path(w)), f"robot {w}: published states differ"
        assert (dflt.flag_history(w) == res.flag_history(w)).all()
        assert dflt.feature_ids(w) == res.feature_ids(w)
    assert len(dflt.reports) == len(res.reports)
    for a, b in zip(dflt.reports, res.reports):
        assert a.tobytes() == b.tobytes()


def _assert_store_matches(be_r, dflt, res, w):
    """the store of window w on the device == the window the default mode holds on the host"""
    f_d, ids_d, obs_d, pre_d, cur_d, _, prior_d, J_d, r_d = dflt.window(w)
    f_r, ids_r, _, _, cur_r, slots, prior_r, _, _ = res.window(w)
    store_obs, store_pre, prior_s, J_s, r_s = be_r.resident_read_window(w)
    assert (ids_d == ids_r).all() and (f_d["start_frame"] == f_r["start_frame"]).all() and (f_d["n_obs"] == f_r["n_obs"]).all()
    assert len(set(f_r["obs_offset"].tolist())) == len(f_r) and (f_r["obs_offset"] % NFRM == 0).all()       # every live track has a slot of its own
    for k in range(len(f_d)):
        a = obs_d[f_d["obs_offset"][k]: f_d["obs_offset"][k] + f_d["n_obs"][k]]
        b = store_obs[f_r["obs_offset"][k]: f_r["obs_offset"][k] + f_r["n_obs"][k]]
        assert a.tobytes() == b.tobytes(), f"window {w} track {ids_d[k]}"
    assert (cur_d == cur_r).all() and sorted(slots.tolist()) == list(range(W))
    for i in range(W):
        if not cur_d[i]: continue                      # samples were added since: both modes preintegrate it again before it is used
        a, b = pre_d[i], store_pre[slots[i]]
        for name in TRAVELLED:
            assert _same_bits(a[name], b[name]), (w, i, name)
        assert _same_bits(a["jacobian"][21 * 31:], b["jacobian"][21 * 31:]), (w, i, "jacobian")
    assert bool(prior_d.valid) == bool(prior_s.valid) == bool(prior_r.valid)
    if prior_d.valid:
        nb = prior_d.num_blocks
        assert prior_d.n == prior_s.n and nb == prior_s.num_blocks
        for name in ("block_kind", "block_index", "block_col"):
            assert list(getattr(prior_d, name))[:nb] == list(getattr(prior_s, name))[:nb]
        assert [list(prior_d.block_x0[b]) for b in range(nb)] == [list(prior_s.block_x0[b]) for b in range(nb)]
        assert _same_bits(J_d, J_s) and _same_bits(r_d, r_s)


def _slow_sequence(n, n_frames, tracked):
    """robots that hardly move: the keyframe test says MARGIN_SECOND_NEW on most frames"""
    return synth.generate_sequence(n, n_frames, tracked=tracked, max_len=30, min_len=6, speed=0.01, yaw_rate=0.01, seed0=7100)


def _flag_counts(rep, n):
    fl = np.concatenate([rep.flag_history(w) for w in range(n)])
    return int((fl == 0).sum()), int((fl == 1).sum())


# ---- CPU tier ---------------------------------------------------------------------------------------------------------------------------

def test_store_equals_default_window_sim():
    """(1) after every step of a resident replay the store is what the default mode would have uploaded, with both marginalization modes."""
    n, F = 1, 64
    cfg, pcfg = _cfg(n, F, 2), abi.default_preint_config()
    seq = _slow_sequence(n, 15, 48)
    (be_d, dflt), (be_r, res) = _pair(sim_backend, cfg, pcfg, n, F)
    for _ in zip(_steps(dflt, seq), _steps(res, seq)):
        for w in range(n):
            _assert_store_matches(be_r, dflt, res, w)
    old, second_new = _flag_counts(res, n)
    assert old >= 1 and second_new >= 1, (old, second_new)
    _assert_same_replay(dflt, res, n)


@pytest.mark.parametrize("estimate_td", [0, 1])
def test_bit_identical_replay_sim(estimate_td):
    """(2) resident vs default mode: published states, keyframe decisions, feature lists and solve reports are equal bit for bit."""
    n, F = 2, 24
    cfg, pcfg = _cfg(n, F, 2), abi.default_preint_config()
    seq = synth.generate_sequence(n, 14, tracked=14, max_len=12, min_len=3)
    (be_d, dflt), (be_r, res) = _pair(sim_backend, cfg, pcfg, n, F, estimate_td=estimate_td)
    dflt.run(seq); res.run(seq)
    assert dflt.path(0).shape == (4, 20)
    _assert_same_replay(dflt, res, n)
    for w in range(n):
        _assert_store_matches(be_r, dflt, res, w)
    assert res.traffic()["staged_bytes"] == 0 and dflt.traffic()["staged_bytes"] > 0


def _put(window, slot, position, x=0.0):
    p = np.zeros(1, dtype=abi.track_put_dtype)
    p["window"], p["slot"], p["position"] = window, slot, position
    p["obs"]["point"] = (x, -x); p["obs"]["cur_td"] = 0.5 * x
    return p


def test_edit_records_match_the_c_layout():
    assert C.sizeof(abi.TrackPut) == 96 and C.sizeof(abi.TrackEdit) == 16 and abi.TrackPut.obs.offset == 16


def _check_rejections(be, F):
    """(3) every malformed call returns CERB_ERR_BAD_ARGUMENT, leaves the store as it was and issues no copy (so no kernel either: a kernel of
    these entry points always follows a copy of its arguments)"""
    pcfg = abi.default_preint_config()
    batch = synth.generate_batch(2, 6, be, prior_features=0)
    for w in range(2):
        for f in range(batch.descs[w].n_features): batch.features[w][f]["obs_offset"] = f * NFRM
    ident = np.tile(np.arange(W, dtype=np.int32), (2, 1))

    def rejected(call):
        with pytest.raises(CerbError) as e: call()
        assert e.value.code == abi.ERR_BAD_ARGUMENT

    rejected(lambda: be.resident_upload(batch, ident))                            # before any window was started
    rejected(lambda: be.resident_put(_put(0, 0, 0)))
    be.resident_start(2)
    be.resident_put(np.concatenate([_put(w, s, p, 1.0 + w + 0.1 * s + 0.01 * p) for w in range(2) for s in range(3) for p in range(4)]))
    snap = lambda: [[a.tobytes() if isinstance(a, np.ndarray) else bytes(a)[:C.sizeof(abi.Prior) - 16] for a in be.resident_read_window(w)] for w in range(2)]
    before = snap(); ops = be.traffic()["dma_ops"]
    slots = be.cfg.max_obs // NFRM
    edit = lambda w, s, n, p: np.array([(w, s, n, p)], dtype=abi.track_edit_dtype)
    rejected(lambda: be.resident_put(_put(0, slots, 0)))                          # slot out of range
    rejected(lambda: be.resident_put(_put(0, 0, NFRM)))                           # position out of range
    rejected(lambda: be.resident_put(_put(2, 0, 0)))                              # window out of range
    rejected(lambda: be.resident_put(np.concatenate([_put(1, 2, 1), _put(1, 2, 1)])))
    rejected(lambda: be.resident_edit(edit(0, -1, 4, 0)))
    rejected(lambda: be.resident_edit(edit(0, 0, 4, 4)))                          # position past the track
    rejected(lambda: be.resident_edit(edit(0, 0, NFRM + 1, 0)))
    rejected(lambda: be.resident_edit(np.concatenate([edit(0, 1, 4, 0), edit(0, 1, 4, 2)])))
    twice = ident.copy(); twice[1, 3] = twice[1, 4]
    rejected(lambda: be.resident_upload(batch, twice))                            # slot table not a permutation
    far = ident.copy(); far[0, 0] = W
    rejected(lambda: be.resident_upload(batch, far))
    batch.descs[0].n_features = be.cfg.max_features + 1
    rejected(lambda: be.resident_upload(batch, ident))                            # more tracks than max_features
    batch.descs[0].n_features = 6
    batch.features[1][2]["obs_offset"] = 5                                        # not a slot
    rejected(lambda: be.resident_upload(batch, ident))
    batch.features[1][2]["obs_offset"] = slots * NFRM                             # past the store
    rejected(lambda: be.resident_upload(batch, ident))
    batch.features[1][2]["obs_offset"] = 2 * NFRM
    smp = np.zeros((2, 3), dtype=abi.sample_dtype); smp["dt"] = 0.005; smp["acc"][..., 2] = 9.8
    jobs = (abi.PreintJob * 2)()
    for j in range(2): jobs[j].n_samples = 3; jobs[j].samples = smp[j].ctypes.data_as(C.POINTER(abi.IMULegSample))
    rejected(lambda: be.resident_preintegrate(pcfg, jobs, 2, [0, 0], [W, 1]))       # slot out of range
    rejected(lambda: be.resident_preintegrate(pcfg, jobs, 2, [1, 1], [2, 2]))       # two jobs, one slot
    bad = abi.Prior(); bad.valid = 1; bad.n = abi.MAX_PRIOR_DIM + 1
    rejected(lambda: be.resident_set_prior(0, bad))
    assert be.traffic()["dma_ops"] == ops
    assert snap() == before
    # and the accepted forms of the same calls do what they say
    be.resident_edit(edit(1, 2, 4, 1))
    obs = be.resident_read_window(1)[0]
    assert obs["point"][2 * NFRM: 2 * NFRM + 3, 0].tolist() == [1.0 + 1 + 0.2 + 0.01 * p for p in (0, 2, 3)]
    assert be.resident_preintegrate(pcfg, jobs, 2, [0, 1], [W - 1, 0]).tolist() == pytest.approx([0.015, 0.015])
    be.resident_upload(batch, ident)


def test_rejected_calls_leave_the_store_alone_sim():
    _check_rejections(sim_backend(_cfg(2, 8)), 8)


@pytest.mark.parametrize("use_leg", [True, False])
def test_preintegration_into_slots_equals_the_host_result_sim(use_leg):
    """a result left in a slot is the record cerb_preintegrate_batch / cerb_preintegrate_imu_batch returns (the members an upload carries)"""
    be, pcfg = sim_backend(_cfg(2, 8)), abi.default_preint_config()
    rng = np.random.default_rng(5)
    smp = np.zeros((2, 6), dtype=abi.sample_dtype); smp["dt"] = 0.004
    smp["acc"] = rng.normal(0, 1, (2, 6, 3)) + (0, 0, 9.8); smp["gyr"] = rng.normal(0, 0.3, (2, 6, 3))
    smp["phi"] = rng.normal(0, 0.5, (2, 6, 12)) + np.tile((0.0, 0.8, -1.6), 4); smp["dphi"] = rng.normal(0, 0.5, (2, 6, 12)); smp["c"] = 1.0
    jobs = (abi.PreintJob * 2)()
    for j in range(2):
        jobs[j].n_samples = 6; jobs[j].samples = smp[j].ctypes.data_as(C.POINTER(abi.IMULegSample))
        for k in range(4): jobs[j].linearized_rho[k] = 0.21
        for k in range(12): jobs[j].phi_0[k] = smp["phi"][j, 0, k]
    want = be.preintegrate(pcfg, jobs, 2) if use_leg else be.preintegrate_imu(pcfg, jobs, 2)
    be.resident_start(2, use_leg=use_leg)
    sum_dt = be.resident_preintegrate(pcfg, jobs, 2, [0, 1], [3, 7])
    for j, slot in ((0, 3), (1, 7)):
        got = be.resident_read_window(j, use_leg=use_leg)[1][slot]
        assert sum_dt[j] == want[j]["sum_dt"] == got["sum_dt"]
        if use_leg:
            for name in TRAVELLED: assert _same_bits(got[name], want[j][name]), name
            assert _same_bits(got["jacobian"][21 * 31:], want[j]["jacobian"][21 * 31:]) and not got["jacobian"][:21 * 31].any()
        else:
            assert got.tobytes() == want[j].tobytes()


def _traffic_per_robot_frame(rep, n, steps):
    t = rep.traffic()
    return (t["h2d_bytes"] + t["d2h_bytes"]) / (n * steps), t


def test_counted_traffic_sim():
    """(4) bytes per robot and frame a step asks the library to move, on the 90-tracked-feature sequence: resident <= 1/5 of the default mode's,
    none of it through a staging copy."""
    n, F, steps = 1, 160, 2
    cfg, pcfg = _cfg(n, F, 1), abi.default_preint_config()
    seq = synth.generate_sequence(n, W + steps, tracked=90, max_len=14, min_len=3)
    (be_d, dflt), (be_r, res) = _pair(sim_backend, cfg, pcfg, n, F)
    dflt.run(seq); res.run(seq)
    _assert_same_replay(dflt, res, n)
    # the first step also sends the eleven seeded frames; a steady-state frame is the difference of two steps
    per_d, t_d = _traffic_per_robot_frame(dflt, n, steps)
    per_r, t_r = _traffic_per_robot_frame(res, n, steps)
    print(f"bytes moved per robot and frame over the first {steps} frames (seeding included): default {per_d:.0f}, resident {per_r:.0f}")
    assert t_r["staged_bytes"] == 0
    assert per_r <= per_d / 5, (per_r, per_d)


# ---- GPU tier ---------------------------------------------------------------------------------------------------------------------------

def _gpu_backend(cfg):
    return lib.Backend(cfg)


@pytest.mark.gpu
def test_bit_identical_replay_gpu():
    """(2) on the H100: 4 robots x 52 frames at F = 160; the slow 2 x 40 sequence (>= 10 MARGIN_SECOND_NEW frames) with the store checked
    after every step; (4) the traffic counts of the 4 x 52 replay."""
    n, F = 4, 160
    cfg, pcfg = _cfg(n, F), abi.default_preint_config()
    seq = synth.generate_sequence(n, 62, tracked=90, max_len=14, min_len=3)
    (be_d, dflt), (be_r, res) = _pair(_gpu_backend, cfg, pcfg, n, F)
    dflt.run(seq); res.run(seq)
    assert dflt.path(0).shape == (52, 20)
    _assert_same_replay(dflt, res, n)
    per_d, _ = _traffic_per_robot_frame(dflt, n, 52); per_r, t_r = _traffic_per_robot_frame(res, n, 52)
    print(f"bytes moved per robot and frame, 4 robots x 52 frames, 90 tracked features: default {per_d:.0f}, resident {per_r:.0f}")
    assert t_r["staged_bytes"] == 0 and per_r <= per_d / 5, (per_r, per_d, t_r)
    slow = _slow_sequence(2, 40, 90)
    (be_d, dflt), (be_r, res) = _pair(_gpu_backend, cfg, pcfg, 2, F)
    for _ in zip(_steps(dflt, slow), _steps(res, slow)):
        for w in range(2):
            _assert_store_matches(be_r, dflt, res, w)
    old, second_new = _flag_counts(res, 2)
    assert second_new >= 10 and old >= 2, (old, second_new)
    _assert_same_replay(dflt, res, 2)


@pytest.mark.gpu
def test_bit_identical_replay_256_robots_gpu():
    """(2) 256 robots x 30 frames replaying 8 distinct sequences: equal to the default mode, and identical robots stay identical."""
    nb, fb, F = 256, 30, 160
    cfg, pcfg = _cfg(nb, F), abi.default_preint_config()
    seq8 = synth.generate_sequence(8, fb, tracked=90, max_len=14, min_len=3)
    class Tiled: pass
    big = Tiled(); big.n, big.n_frames = nb, fb
    idx = np.arange(nb) % 8
    for name in ("tic_g", "ric_g", "p_g", "R_g", "v_g", "first", "samples"):
        setattr(big, name, getattr(seq8, name)[idx])
    big.images = [[seq8.images[k][w % 8] for w in range(nb)] for k in range(fb)]
    (be_d, dflt), (be_r, res) = _pair(_gpu_backend, cfg, pcfg, nb, F)
    dflt.run(big); res.run(big)
    _assert_same_replay(dflt, res, nb)
    P, _ = res.poses()
    assert P.shape[1] == fb - W
    for k in range(1, nb // 8):
        assert P[8 * k: 8 * k + 8].tobytes() == P[0:8].tobytes()


@pytest.mark.gpu
def test_rejected_calls_leave_the_store_alone_gpu():
    _check_rejections(_gpu_backend(_cfg(2, 8)), 8)

"""Robot snapshots (cerb_replay_save_robot / _load_robot / _clone_robot; NativeReplay.save / load / clone): a robot saved after frame k and
restored anywhere continues exactly as the saved robot does.  Every comparison is `==` on bytes:
  (1) resume: robot 0 of replay A saved at frame k and loaded into robot 1 of a fresh replay B on a handle of its own; stepped on, B's path
      rows, flags, feature ids, solve reports and its next snapshot are A's.  A VILO and a VINS robot on slow sequences, each with its prior
      and a MARGIN_SECOND_NEW frame after k, and an estimate_td = 1 robot on a fast one, whose td, extrinsics and openEx latch have moved by k,
  (2) across modes: snapshots of a default-mode replay loaded into resident replays and the reverse; both modes save the same bytes,
  (3) right after a resident load the device store is the window the default mode holds for the same robot,
  (4) clone robot 0 (VINS) into robots 3 (a VILO robot that was running), 5 and 1: all continue as the robot that was never cloned,
  (5) ... except robot 1, fed a sample whose dt differs by 1e-9: the copies share no state,
  (6) rejected snapshots (truncated, wrong magic or version, oversized prior, duplicate feature id, bad keyframe flag, a leg-bias prior block
      in a use_leg = 0 robot, too many tracks) change nothing and move nothing, and the robot steps on as if the calls had not been made,
  (7) a snapshot taken on one GPU and loaded on another (skipped with one device).
CPU tier on the kernel simulator, GPU tier under -m gpu."""
import ctypes as C
import numpy as np
import pytest
from cerberus_b200 import abi, synth, estimator, lib
from cerberus_b200.lib import CerbError
from helpers import sim_backend
from test_replay_configs import _assert_store_matches

W = abi.WINDOW_SIZE
SNAP_PRIOR_N = 16                      # byte offset of the prior dimension in the snapshot's head (magic, version, window size, features)


class _Layout:
    """byte offsets of the snapshot fields the checks read or edit, in the order snapshot() in replay_host.inl writes them (one build's format)"""
    P = C.sizeof(abi.PreintConfig)
    use_leg = 48                                       # after the head (24) and g (24)
    cfg_tic = 60 + P                                   # after use_leg, pcfg, estimate_extrinsic, estimate_td
    tic = 252 + P + 8 * abi.NUM_FRAMES * (4 * 3 + 9 + 4)     # after the configuration's ric and Ps, Vs, Bas, Bgs, Rs, Rho
    td = tic + 8 * (6 + 18)
    frame_count = td + 8 + 8 * abi.NUM_FRAMES          # after td and Headers; then marginalization_flag, openEx and four more int32
    flag, openEx = frame_count + 4, frame_count + 8
    features = frame_count + 28 + C.sizeof(abi.IMULegSample)        # each: 5 int32, a double, n_obs x (11 doubles + int32)

    @staticmethod
    def i32(blob, off):
        return int(np.frombuffer(blob, dtype=np.int32, count=1, offset=off)[0])

    @classmethod
    def second_feature_id(cls, blob):
        return cls.features + 28 + 92 * cls.i32(blob, cls.features + 8)


def _cfg(n, F, iters, device=0):
    cfg = abi.default_config(); cfg.max_batch = n; cfg.max_features = 2 * F; cfg.max_obs = 2 * F * abi.NUM_FRAMES
    cfg.max_num_iterations = iters; cfg.device = device
    return cfg


def _replay(make_backend, n, F, iters, kind, resident, robots=None, device=0):
    """n robots; `robots` (default: all) configured as kind: "vilo", "vins" (use_leg = 0, the VINS preintegration globals) or "td" (estimate_td = 1)"""
    rep = estimator.NativeReplay(make_backend(_cfg(n, F, iters, device)), abi.default_preint_config(), n, max_features=F, resident=resident)
    for w in (range(n) if robots is None else robots):
        if kind == "vins": rep.configure(w, False, abi.vins_preint_config())
        elif kind == "td": rep.configure(w, True, abi.default_preint_config(), 1, 1)
    return rep


def _sequence(n, frames, tracked, fast=False):
    """slow robots: the keyframe test says MARGIN_SECOND_NEW on some frames; fast ones (0.5 m/s) open td and the extrinsics from the first step"""
    if fast:
        return synth.generate_sequence(n, frames, tracked=tracked, max_len=14, min_len=3)
    return synth.generate_sequence(n, frames, tracked=tracked, max_len=30, min_len=6, speed=0.01, yaw_rate=0.01, seed0=7100)


def _inputs(seq, src, k, perturb=False):
    smp = seq.samples[src][k - 1][:0] if k == W else seq.samples[src][k - 1]
    if perturb:
        smp = smp.copy(); smp["dt"][0] += 1e-9
    return seq.images[k][src], seq.first[src, k - 1], smp


def _step(rep, robots, seq, k, src=0, perturbed=()):
    """frame k of robot src of seq for each listed robot (perturbed ones get one dt changed by 1e-9)"""
    rows = [_inputs(seq, src, k, r in perturbed) for r in robots]
    rep.step([x[0] for x in rows], [x[1] for x in rows], [x[2] for x in rows], float(k), robots=list(robots))


def _seed_and_step(rep, robots, seq, srcs, k_end):
    """seed robots[i] with robot srcs[i] of seq and step them together up to frame k_end (excluded)"""
    for r, s in zip(robots, srcs): rep.seed_robot(r, seq, s)
    for k in range(W, k_end):
        rows = [_inputs(seq, s, k) for s in srcs]
        rep.step([x[0] for x in rows], [x[1] for x in rows], [x[2] for x in rows], float(k), robots=list(robots))


def _same(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _reports(rep, i):
    return [r[i].tobytes() for r in rep.reports]


def _assert_continues(a, wa, rows, n_reports, b, wb, b_reports):
    """robot wb of b == robot wa of a from a's path row `rows` and a's step `n_reports` on; b_reports: robot wb's report of each step of b"""
    assert _same(b.path(wb), a.path(wa)[rows:]), f"robot {wb}: published states differ"
    assert (b.flag_history(wb) == a.flag_history(wa)[rows:]).all()
    assert b.feature_ids(wb) == a.feature_ids(wa)
    assert b_reports == _reports(a, 0)[n_reports:]


# ---- the checks, on any backend ----------------------------------------------------------------------------------------------------------

def _check_resume(make_backend, seq, F, iters, kind, k_save, pairs):
    """(1), (2), (3): robot 0 of a default and of a resident replay A run to frame k_save and save; each (source mode, destination mode) of
    `pairs` loads the source's snapshot into robot 1 of a fresh two-robot replay; all are stepped to the end of seq"""
    src = {m: _replay(make_backend, 1, F, iters, kind, m) for m in (False, True)}
    for a in src.values(): _seed_and_step(a, [0], seq, [0], k_save)
    rows = src[False].path(0).shape[0]
    blobs = {m: a.save(0) for m, a in src.items()}
    assert blobs[False] == blobs[True], "the two modes save different snapshots of the same robot"
    assert src[False].window(0)[6].valid, "no prior to carry"
    blob = blobs[False]
    assert _Layout.i32(blob, _Layout.frame_count) == W
    if kind == "td":                                  # what only an estimate_td robot on the move carries
        td = np.frombuffer(blob, dtype=np.float64, count=1, offset=_Layout.td)[0]
        tic, cfg_tic = (np.frombuffer(blob, dtype=np.float64, count=6, offset=o) for o in (_Layout.tic, _Layout.cfg_tic))
        assert td != 0 and _Layout.i32(blob, _Layout.openEx) == 1 and not (tic == cfg_tic).all(), (td, tic, cfg_tic)
    dst = {}
    for pair in pairs:
        b = _replay(make_backend, 2, F, iters, "vilo", pair[1])
        b.load(1, blobs[pair[0]])
        assert b.save(1) == blobs[pair[0]]
        if pair[1]:
            class Source:                     # robot 0 of the default-mode source, seen as robot 1
                window = staticmethod(lambda _w: src[False].window(0))
            _assert_store_matches(b.be, Source, b, 1, kind != "vins")
        dst[pair] = b
    for k in range(k_save, seq.n_frames):
        for a in src.values(): _step(a, [0], seq, k)
        for b in dst.values(): _step(b, [1], seq, k)
    if kind != "td":
        assert 1 in src[False].flag_history(0)[rows:].tolist(), "no MARGIN_SECOND_NEW frame after the save"
    assert _same(src[False].path(0), src[True].path(0))
    for b in dst.values():
        _assert_continues(src[False], 0, rows, k_save - W, b, 1, _reports(b, 0))
        assert b.save(1) == src[False].save(0)


def _check_clone(make_backend, seq, F, iters, k_clone, resident):
    """(4), (5): robot 0 (VINS) and robot 3 (VILO, another sequence) step to k_clone; robot 0 is cloned into 3, 5 and 1; then robots 0, 3 and
    5 take robot 0's frames and robot 1 the same frames with one dt changed.  Reference: robot 0 alone in a replay where no clone happened."""
    ref = _replay(make_backend, 1, F, iters, "vins", False)
    ref.seed_robot(0, seq, 0)
    for k in range(W, seq.n_frames): _step(ref, [0], seq, k)
    rep = _replay(make_backend, 6, F, iters, "vins", resident, robots=[0])
    _seed_and_step(rep, [0, 3], seq, [0, 1], k_clone)
    rows = rep.path(0).shape[0]
    rep.clone(0, [3, 5, 1])
    for w in (3, 5, 1):
        assert rep.path(w).shape[0] == 0 and rep.flag_history(w).shape[0] == 0
    for k in range(k_clone, seq.n_frames): _step(rep, [0, 3, 5, 1], seq, k, perturbed=(1,))
    assert _same(rep.path(0), ref.path(0)) and (rep.flag_history(0) == ref.flag_history(0)).all()
    for w in (3, 5):
        assert _same(rep.path(w), ref.path(0)[rows:]), f"clone {w} differs"
        assert (rep.flag_history(w) == ref.flag_history(0)[rows:]).all() and rep.feature_ids(w) == ref.feature_ids(0)
    assert rep.path(1).shape == rep.path(3).shape and not _same(rep.path(1), rep.path(3)), "the perturbed copy did not depart"
    with pytest.raises(CerbError):
        rep.clone(0, [3, 3])
    with pytest.raises(CerbError):
        rep.clone(0, [2, 0])
    with pytest.raises(CerbError):
        rep.clone(2, [4])                                        # robot 2 was never seeded


def _check_rejections(make_backend, seq, F, iters, k_save):
    """(6): bad snapshots into a stepping resident robot and into a replay too small for the snapshot: CerbError, no copy, no change"""
    a = _replay(make_backend, 1, F, iters, "vilo", False)
    b = _replay(make_backend, 1, F, iters, "vilo", True)
    for rep in (a, b): _seed_and_step(rep, [0], seq, [0], k_save)
    blob = a.save(0)
    small_F = 4
    small = _replay(make_backend, 1, small_F, iters, "vilo", False)
    assert len(a.feature_ids(0)) > 2 * small_F
    head = np.frombuffer(blob[:24], dtype=np.int32)
    assert head[2] == W and head[3] == len(a.feature_ids(0)) and head[4] > 0
    prior_too_big = bytearray(blob); prior_too_big[SNAP_PRIOR_N: SNAP_PRIOR_N + 4] = np.int32(abi.MAX_PRIOR_DIM + 1).tobytes()
    bad_magic = bytearray(blob); bad_magic[0] ^= 0xFF
    bad_version = bytearray(blob); bad_version[4: 8] = np.int32(2).tobytes()
    assert _Layout.i32(blob, _Layout.frame_count) == W and _Layout.i32(blob, _Layout.use_leg) == 1
    first_id, second = _Layout.i32(blob, _Layout.features), _Layout.second_feature_id(blob)
    assert a.feature_ids(0)[:2] == [first_id, _Layout.i32(blob, second)]
    twice = bytearray(blob); twice[second: second + 4] = np.int32(first_id).tobytes()
    bad_flag = bytearray(blob); bad_flag[_Layout.flag: _Layout.flag + 4] = np.int32(2).tobytes()
    prior = a.window(0)[6]
    assert abi.BLOCK_LEGBIAS in list(prior.block_kind)[:prior.num_blocks]
    leg_prior_vins = bytearray(blob); leg_prior_vins[_Layout.use_leg: _Layout.use_leg + 4] = np.int32(0).tobytes()
    state = lambda: (b.path(0).tobytes(), b.flag_history(0).tobytes(), b.feature_ids(0), b.save(0), b.traffic(), small.window(0)[0].tobytes())
    before = state()
    moved = (b.be.traffic(), small.be.traffic())
    for rep, bad in ((b, blob[:-8]), (b, blob[:20]), (b, b""), (b, bytes(bad_magic)), (b, bytes(bad_version)), (b, bytes(prior_too_big)),
                     (b, blob + b"\0"), (b, bytes(twice)), (b, bytes(bad_flag)), (b, bytes(leg_prior_vins)), (small, blob)):
        with pytest.raises(CerbError) as e:
            rep.load(0, bad)
        assert e.value.code == abi.ERR_BAD_ARGUMENT
    assert (b.be.traffic(), small.be.traffic()) == moved
    assert state() == before
    for k in range(k_save, seq.n_frames):
        for rep in (a, b): _step(rep, [0], seq, k)
    assert _same(a.path(0), b.path(0)) and a.feature_ids(0) == b.feature_ids(0) and _reports(a, 0) == _reports(b, 0)


# ---- CPU tier ---------------------------------------------------------------------------------------------------------------------------

# the kernel simulator takes about 3 s per robot and step at this size; 48 tracked slow features give MARGIN_SECOND_NEW frames
SIM = dict(F=64, frames=16, tracked=48, iters=1, k=W + 2)
ALL_PAIRS = ((False, False), (False, True), (True, False), (True, True))


@pytest.mark.parametrize("kind,pairs", [("vilo", ALL_PAIRS), ("vins", ((False, True), (True, False))), ("td", ((False, True), (True, False)))])
def test_resume_equals_uninterrupted_sim(kind, pairs):
    seq = _sequence(1, SIM["frames"], SIM["tracked"], fast=kind == "td")
    _check_resume(sim_backend, seq, SIM["F"], SIM["iters"], kind, SIM["k"], pairs)


def test_clone_and_fork_sim():
    seq = _sequence(2, 14, SIM["tracked"])
    _check_clone(sim_backend, seq, SIM["F"], SIM["iters"], W + 2, True)


def test_rejected_loads_change_nothing_sim():
    seq = _sequence(1, 13, SIM["tracked"])
    _check_rejections(sim_backend, seq, SIM["F"], SIM["iters"], W + 2)


# ---- GPU tier ---------------------------------------------------------------------------------------------------------------------------

def _gpu_backend(cfg):
    return lib.Backend(cfg)


GPU = dict(F=160, frames=34, tracked=90, iters=12, k=W + 12)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["vilo", "vins", "td"])
def test_resume_equals_uninterrupted_gpu(kind):
    seq = _sequence(1, GPU["frames"], GPU["tracked"], fast=kind == "td")
    _check_resume(_gpu_backend, seq, GPU["F"], GPU["iters"], kind, GPU["k"], ALL_PAIRS)


@pytest.mark.gpu
@pytest.mark.parametrize("resident", [False, True])
def test_clone_and_fork_gpu(resident):
    seq = _sequence(2, 30, GPU["tracked"])
    _check_clone(_gpu_backend, seq, GPU["F"], GPU["iters"], W + 8, resident)


@pytest.mark.gpu
def test_rejected_loads_change_nothing_gpu():
    seq = _sequence(1, 24, GPU["tracked"])
    _check_rejections(_gpu_backend, seq, GPU["F"], GPU["iters"], W + 8)


@pytest.mark.gpu
def test_second_gpu_gpu():
    """(7) save on a handle on device 0, load on a handle on device 1, both resident"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device visible")
    seq = _sequence(1, GPU["frames"], GPU["tracked"])
    F, iters = GPU["F"], GPU["iters"]
    a = _replay(_gpu_backend, 1, F, iters, "vilo", True, device=0)
    _seed_and_step(a, [0], seq, [0], GPU["k"])
    rows, blob = a.path(0).shape[0], a.save(0)
    b = _replay(_gpu_backend, 2, F, iters, "vilo", True, device=1)
    b.load(1, blob)
    for k in range(GPU["k"], seq.n_frames):
        _step(a, [0], seq, k); _step(b, [1], seq, k)
    _assert_continues(a, 0, rows, GPU["k"] - W, b, 1, _reports(b, 0))

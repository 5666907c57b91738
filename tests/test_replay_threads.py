"""The native replay's host bookkeeping on host threads (cerb_replay_step_robots fans the per-robot work out from 16 listed robots on): a
step of 16 robots of a 17-robot replay, listed in shuffled order, each at its own stamp, equals the same step of replays of 4 robots, which
run on the calling thread alone.  Paths, flag histories, feature lists and solve reports are compared byte for byte, in default and
resident mode.  CPU tier on the kernel simulator (one step, one iteration: about three minutes per mode); the GPU tier of test_replay.py,
test_replay_async.py and test_resident.py runs 64 to 256 robots."""
import numpy as np
import pytest
from cerberus_b200 import abi, synth, estimator
from helpers import sim_backend
from test_replay_async import _cfg, _assert_robot_equal

W = abi.WINDOW_SIZE
F, TRACKED, SOURCES = 16, 10, 4


def _step(rep, seq, robots, src):
    """frame W (the first after the seed) of the listed robots, robot r replaying robot src[r] of seq at stamp W + 0.01 src[r]"""
    k = W
    rep.step([seq.images[k][src[r]] for r in robots], [seq.first[src[r], k - 1] for r in robots], [seq.samples[src[r]][k - 1][:0] for r in robots],
             0.0, robots=list(robots), headers=[k + 0.01 * src[r] for r in robots])


@pytest.mark.parametrize("resident", [False, True], ids=["default", "resident"])
def test_threaded_step_equals_small_replays_sim(resident):
    n = 17
    src = [r % SOURCES for r in range(n)]
    seq = synth.generate_sequence(SOURCES, W + 1, tracked=TRACKED, max_len=12, min_len=3)
    pcfg = abi.default_preint_config()
    rng = np.random.default_rng(7)
    idle = 6                                                            # not listed: its window stays as seeded
    listed = [int(r) for r in rng.permutation([r for r in range(n) if r != idle])]
    big = estimator.NativeReplay(sim_backend(_cfg(n, F, 1)), pcfg, n, max_features=F, resident=resident)
    for r in range(n): big.seed_robot(r, seq, src[r])
    _step(big, seq, listed, src)
    # the same step, each source once, in replays small enough to stay on the calling thread
    small = estimator.NativeReplay(sim_backend(_cfg(SOURCES, F, 1)), pcfg, SOURCES, max_features=F, resident=resident)
    small.seed(seq)
    order = [int(s) for s in rng.permutation(SOURCES)]
    _step(small, seq, order, list(range(SOURCES)))
    for i, r in enumerate(listed):
        s = src[r]
        _assert_robot_equal(big, r, small, s, [big.reports[0][i]], [small.reports[0][order.index(s)]])
    assert big.path(idle).shape[0] == 0 and big.flag_history(idle).shape[0] == 0
    assert big.path(listed[0]).shape[0] == 1

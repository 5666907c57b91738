"""Robot snapshots on the GPU (NativeReplay.save / load / clone, cerb_replay_save_robot / _load_robot / _clone_robot): the time to save one
robot, to load one robot and to clone one robot into all the others, and the bytes of a snapshot, in a resident replay of 256 robots
(8 distinct synthetic sequences, 90 tracked features) that has stepped past its first priors.  Each operation runs once as a warm-up, then
three times; the medians are printed with the minimum and maximum.  The card's name, power limit and maximum SM clock are read in the same
run.  After the timed clones every robot takes one more frame, and the copies must publish the source's states bit for bit.

    python tools/replay_snapshot.py [--robots 256] [--frames 20] [--reps 3] [--out replay_snapshot.txt]"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from cerberus_b200 import abi, synth, estimator, lib  # noqa: E402
from replay_resident import tiled  # noqa: E402


def timed(fn, reps):
    fn()                                           # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    return np.array(ts) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--robots", type=int, default=256); ap.add_argument("--frames", type=int, default=20); ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, F, W = a.robots, 160, abi.WINDOW_SIZE
    cfg = abi.default_config(); cfg.max_batch = n; cfg.max_features = 2 * F; cfg.max_obs = 2 * F * abi.NUM_FRAMES
    pcfg = abi.default_preint_config()
    be = lib.Backend(cfg)                          # fails here without the library or a device
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True, check=True).stdout.strip()
    seq = tiled(synth.generate_sequence(8, a.frames + 1, tracked=90, max_len=14, min_len=3), n)
    rep = estimator.NativeReplay(be, pcfg, n, max_features=F, resident=True)
    rep.seed(seq)

    def step(k, src):                              # frame k of robot src[w] of seq for robot w
        smp = [seq.samples[s][k - 1][:0] if k == W else seq.samples[s][k - 1] for s in src]
        rep.step([seq.images[k][s] for s in src], [seq.first[s, k - 1] for s in src], smp, float(k))
    t0 = time.perf_counter()
    for k in range(W, a.frames): step(k, range(n))
    t_step = (time.perf_counter() - t0) / (a.frames - W) * 1e3

    blob = rep.save(0)
    t_save = timed(lambda: rep.save(0), a.reps)
    t_load = timed(lambda: rep.load(1, blob), a.reps)
    t_clone = timed(lambda: rep.clone(0, list(range(1, n))), a.reps)
    step(a.frames, [0] * n)
    rows = np.stack([rep.path(w)[-1] for w in range(n)])
    same = all(rows[w].tobytes() == rows[0].tobytes() for w in range(1, n))
    nf = len(rep.feature_ids(0)); prior_n = int(np.frombuffer(blob[16:20], dtype=np.int32)[0])
    fmt = lambda v: f"{np.median(v):.2f} ms (min {v.min():.2f}, max {v.max():.2f})"
    lines = [smi.replace("\n", " | "),
             f"resident replay of {n} robots, F = {F}, 90 tracked features, after {a.frames - W} frames ({t_step:.1f} ms per frame of all robots); "
             f"{a.reps} repetitions after a warm-up, medians; wall = Python glue + library",
             f"snapshot of robot 0: {len(blob)} bytes ({nf} tracks, prior dimension {prior_n}; an IMU / leg sample is {C.sizeof(abi.IMULegSample)} bytes)",
             f"save one robot:           {fmt(t_save)}",
             f"load one robot:           {fmt(t_load)}",
             f"clone one into {n - 1} others: {fmt(t_clone)} ({np.median(t_clone) / (n - 1) * 1e3:.1f} us per copy)",
             f"after one more frame every copy publishes robot 0's states bit for bit: {same}"]
    print("\n".join(lines))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")
    if not same: sys.exit(1)


if __name__ == "__main__":
    main()

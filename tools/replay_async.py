"""Asynchronous fleet replay (cerb_replay_step_robots) against the lock-step replay of tools/replay_resident.py, on the GPU, in both modes
(default and resident).  Every robot has its own camera clock: robot r has a frame ready on the ticks t with t = phase[r] (mod --period),
so about 1 / period of the fleet steps per tick; every third robot's sequence is --short frames shorter and it drops out early.  Each tick
steps the robots that have a frame ready, each at its own stamp.  Reported per mode: robot-frames per second, the distribution of batch
sizes, the cerb_replay_timing split and the counted traffic, next to the lock-step replay of the same robots over their full sequences.
Configurations alternate (lock-step, async; default, resident), --reps repetitions each after a warm-up run of each; min / median / max.
The card's name, power limit and maximum SM clock are read in the same run.  There is no fallback: without the sm_90a library and a CUDA
device lib.Backend raises.

    python tools/replay_async.py [--robots 256] [--frames 30] [--period 4] [--short 6] [--reps 3] [--out replay_async.txt]"""
import argparse
import os
import subprocess
import sys
import time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from cerberus_b200 import abi, synth, estimator, lib  # noqa: E402
from replay_resident import PHASES, tiled, one_replay  # noqa: E402

W = abi.WINDOW_SIZE


def schedule(n, frames, period, short):
    """per tick the robots (ascending) that have a frame ready and the frame each of them takes"""
    phase = np.arange(n) * 7 % period
    length = np.where(np.arange(n) % 3 == 0, frames - short, frames)
    nxt, ticks, t = np.full(n, W), [], 0
    while (nxt < length).any():
        ready = [r for r in range(n) if nxt[r] < length[r] and (t - phase[r]) % period == 0]
        if ready:
            ticks.append([(r, int(nxt[r])) for r in ready])
            for r in ready: nxt[r] += 1
        t += 1
    return phase, length, ticks


def async_replay(cfg, pcfg, seq, n, F, resident, period, phase, ticks):
    """seeding is outside the timed window; the steps end in synchronising downloads"""
    rep = estimator.NativeReplay(lib.Backend(cfg), pcfg, n, max_features=F, resident=resident)
    rep.seed(seq)
    t0 = time.perf_counter()
    for rows in ticks:
        rob = [r for (r, _) in rows]
        smp = [seq.samples[r][k - 1][:0] if k == W else seq.samples[r][k - 1] for (r, k) in rows]
        rep.step([seq.images[k][r] for (r, k) in rows], [seq.first[r, k - 1] for (r, k) in rows], smp, 0.0, robots=rob,
                 headers=[float(k) + phase[r] / period for (r, k) in rows])
    wall = time.perf_counter() - t0
    out = dict(wall=wall, timing=rep.timing(), traffic=rep.traffic(), path=[rep.path(w) for w in range(n)])
    rep.close(); rep.be.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--robots", type=int, default=256); ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--period", type=int, default=4); ap.add_argument("--short", type=int, default=6); ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, F = a.robots, 160
    cfg = abi.default_config(); cfg.max_batch = n; cfg.max_features = 2 * F; cfg.max_obs = 2 * F * abi.NUM_FRAMES
    pcfg = abi.default_preint_config()
    lib.Backend(cfg).close()                       # fails here without the library or a device
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True, check=True).stdout.strip()
    seq = tiled(synth.generate_sequence(8, a.frames, tracked=90, max_len=14, min_len=3), n)
    phase, length, ticks = schedule(n, a.frames, a.period, a.short)
    rf_async, rf_lock = sum(len(t) for t in ticks), n * (a.frames - W)
    sizes = np.array([len(t) for t in ticks])
    configs = [(mode, resident) for resident in (False, True) for mode in ("lock-step", "async")]

    def run(mode, resident):
        return one_replay(cfg, pcfg, seq, n, F, resident) if mode == "lock-step" else async_replay(cfg, pcfg, seq, n, F, resident, a.period, phase, ticks)

    for c in configs: run(*c)                      # warm-up: module load, arena growth, page locking
    runs = {c: [] for c in configs}
    for _ in range(a.reps):
        for c in configs: runs[c].append(run(*c))
    lines = [smi.replace("\n", " | "),
             f"{n} robots, F = {F}, 90 tracked features, frame phases mod {a.period}, every third robot {a.short} frames shorter; {a.reps} repetitions per "
             f"configuration after a warm-up, configurations alternating; wall = Python glue + library",
             f"async: {len(ticks)} steps, {rf_async} robot-frames; robots per step min {sizes.min()}, median {np.median(sizes):.0f}, max {sizes.max()} "
             f"(quartiles {np.percentile(sizes, 25):.0f} / {np.percentile(sizes, 75):.0f}); lock-step: {a.frames - W} steps of {n} robots, {rf_lock} robot-frames"]
    for c in configs:
        rs, rf = runs[c], (rf_lock if c[0] == "lock-step" else rf_async)
        steps = (a.frames - W) if c[0] == "lock-step" else len(ticks)
        rate = np.array([rf / r["wall"] for r in rs])
        tr = rs[0]["traffic"]
        lines.append(f"{c[0]:9s} {'resident' if c[1] else 'default '}: {np.median(rate):.0f} robot-frames/s (min {rate.min():.0f}, max {rate.max():.0f}); "
                     f"{np.median([r['wall'] for r in rs]) / steps * 1e3:.1f} ms per step; moved per robot-frame {(tr['h2d_bytes'] + tr['d2h_bytes']) / rf / 1e3:.1f} kB, "
                     f"staged {tr['staged_bytes'] / rf / 1e3:.1f} kB")
        for ph in PHASES:
            v = np.array([r["timing"][ph] for r in rs]) / rf * 1e3
            lines.append(f"    {ph:13s} {np.median(v):8.3f} ms per robot-frame (min {v.min():.3f}, max {v.max():.3f})")
    paths = lambda c: b"".join(p.tobytes() for p in runs[c][0]["path"])
    same = all(b"".join(p.tobytes() for p in r["path"]) == paths(("async", False)) for c in configs if c[0] == "async" for r in runs[c])
    lines.append(f"published states of all async runs, both modes, bit-identical: {same}")
    print("\n".join(lines))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")
    if not same: sys.exit(1)


if __name__ == "__main__":
    main()

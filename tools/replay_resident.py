"""Batched replay, default mode against resident mode (cerb_replay_set_resident), on the GPU: robot-frames per second, the
cerb_replay_timing split and the counted traffic of 256 robots x 30 frames (8 distinct synthetic sequences, 90 tracked features), the two
modes alternating, three repetitions each after a warm-up replay of each.  The card's name, power limit and maximum SM clock are read in
the same run.  There is no fallback: without the sm_90a library and a CUDA device lib.Backend raises.

    python tools/replay_resident.py [--robots 256] [--frames 30] [--reps 3] [--out replay_resident.txt]"""
import argparse
import os
import subprocess
import sys
import time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cerberus_b200 import abi, synth, estimator, lib  # noqa: E402

PHASES = ("preintegrate", "triangulate", "solve", "marginalize", "outliers", "shift", "host")


def tiled(seq, n):
    class Tiled: pass
    big = Tiled(); big.n, big.n_frames = n, seq.n_frames
    idx = np.arange(n) % seq.n
    for name in ("tic_g", "ric_g", "p_g", "R_g", "v_g", "first", "samples"):
        setattr(big, name, getattr(seq, name)[idx])
    big.images = [[seq.images[k][w % seq.n] for w in range(n)] for k in range(seq.n_frames)]
    return big


def one_replay(cfg, pcfg, seq, n, F, resident):
    """seeding is outside the timed window; the steps end in synchronising downloads"""
    rep = estimator.NativeReplay(lib.Backend(cfg), pcfg, n, max_features=F, resident=resident)
    rep.seed(seq)
    t0 = time.perf_counter()
    for k in range(abi.WINDOW_SIZE, seq.n_frames):
        firsts = [seq.first[w, k - 1] for w in range(n)]
        smp = [seq.samples[w][k - 1][:0] if k == abi.WINDOW_SIZE else seq.samples[w][k - 1] for w in range(n)]
        rep.step([seq.images[k][w] for w in range(n)], firsts, smp, float(k))
    wall = time.perf_counter() - t0
    out = dict(wall=wall, timing=rep.timing(), traffic=rep.traffic(), path=np.stack([rep.path(w) for w in range(n)]))
    rep.close(); rep.be.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--robots", type=int, default=256); ap.add_argument("--frames", type=int, default=30); ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, F = a.robots, 160
    steps = a.frames - abi.WINDOW_SIZE
    cfg = abi.default_config(); cfg.max_batch = n; cfg.max_features = 2 * F; cfg.max_obs = 2 * F * abi.NUM_FRAMES
    pcfg = abi.default_preint_config()
    lib.Backend(cfg).close()                       # fails here without the library or a device
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True, check=True).stdout.strip()
    seq = tiled(synth.generate_sequence(8, a.frames, tracked=90, max_len=14, min_len=3), n)
    runs = {False: [], True: []}
    for resident in (False, True): one_replay(cfg, pcfg, seq, n, F, resident)          # warm-up: module load, arena growth, page locking
    for _ in range(a.reps):
        for resident in (False, True): runs[resident].append(one_replay(cfg, pcfg, seq, n, F, resident))
    lines = [smi.replace("\n", " | "), f"{n} robots x {steps} frames, F = {F}, 90 tracked features, {a.reps} repetitions per mode, modes alternating; wall = Python glue + library"]
    for resident in (False, True):
        rs = runs[resident]
        rate = np.array([n * steps / r["wall"] for r in rs])
        tr = rs[0]["traffic"]; per = (tr["h2d_bytes"] + tr["d2h_bytes"]) / (n * steps)
        lines.append(f"{'resident' if resident else 'default '}: {np.median(rate):.0f} robot-frames/s (min {rate.min():.0f}, max {rate.max():.0f}); "
                     f"moved per robot-frame {per / 1e3:.1f} kB (h2d {tr['h2d_bytes'] / (n * steps) / 1e3:.1f}, d2h {tr['d2h_bytes'] / (n * steps) / 1e3:.1f}), "
                     f"{tr['dma_ops'] / steps:.0f} copies per frame, staged {tr['staged_bytes'] / (n * steps) / 1e3:.1f} kB")
        for ph in PHASES:
            v = np.array([r["timing"][ph] for r in rs]) / steps * 1e3
            lines.append(f"    {ph:13s} {np.median(v):8.2f} ms per frame (min {v.min():.2f}, max {v.max():.2f})")
        glue = np.array([r["wall"] - sum(r["timing"].values()) for r in rs]) / steps * 1e3
        lines.append(f"    {'python glue':13s} {np.median(glue):8.2f} ms per frame (min {glue.min():.2f}, max {glue.max():.2f})")
    same = all(r["path"].tobytes() == runs[False][0]["path"].tobytes() for rs in runs.values() for r in rs)
    lines.append(f"published states of all runs bit-identical: {same}")
    print("\n".join(lines))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")
    if not same: sys.exit(1)


if __name__ == "__main__":
    main()

"""VILO and VINS robots in one resident replay (cerb_replay_configure_robot) against the two configurations as two replays, on the GPU.

The fleet is 2N robots: N synthetic sequences (90 tracked features), each replayed once as A1 VILO (abi.default_preint_config, USE_LEG = 1)
and once as A1 VINS (abi.vins_preint_config, USE_LEG = 0).  "mixed" steps all 2N robots in one replay; "split" steps an N-robot VILO replay
and an N-robot VINS replay one after the other every frame, each on its own handle.  The two arrangements alternate: a warm-up run of each,
then --reps repetitions each.  Reported: robot-frames/s, the cerb_replay_timing split (summed over both replays for "split"), the
preintegration launches per step (kernel launches counted by torch.profiler in a separate run), the distance of the published positions
from the truth per configuration, whether the mixed trajectories are bit-identical to the split ones, and the card's name and power limit,
read in the same run.  There is no fallback: without the sm_90a library and a CUDA device lib.Backend raises.

    python tools/replay_configs.py [--sequences 128] [--frames 30] [--reps 3] [--out replay_configs.txt]"""
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
F = 160
W = abi.WINDOW_SIZE


def tiled(seq, src):
    class Tiled: pass
    big = Tiled(); big.n, big.n_frames = len(src), seq.n_frames
    for name in ("tic_g", "ric_g", "p_g", "R_g", "v_g", "first", "samples", "p"):
        setattr(big, name, getattr(seq, name)[src])
    big.images = [[seq.images[k][w] for w in src] for k in range(seq.n_frames)]
    return big


def make(seq, kinds):
    """a resident replay of seq, robot w VILO (kinds[w]) or VINS, seeded"""
    n = seq.n
    cfg = abi.default_config(); cfg.max_batch = n; cfg.max_features = 2 * F; cfg.max_obs = 2 * F * abi.NUM_FRAMES
    rep = estimator.NativeReplay(lib.Backend(cfg), abi.default_preint_config(), n, max_features=F, resident=True)
    for w, leg in enumerate(kinds):
        if not leg: rep.configure(w, False, abi.vins_preint_config())
    rep.seed(seq)
    return rep


def step(rep, seq, k):
    n = seq.n
    smp = [seq.samples[w][k - 1][:0] if k == W else seq.samples[w][k - 1] for w in range(n)]
    rep.step([seq.images[k][w] for w in range(n)], [seq.first[w, k - 1] for w in range(n)], smp, float(k))


def run(arrangement, seqs):
    """seeding is outside the timed window; every step ends in synchronising downloads"""
    reps = [make(s, kinds) for s, kinds in seqs]
    t0 = time.perf_counter()
    for k in range(W, seqs[0][0].n_frames):
        for rep, (s, _) in zip(reps, seqs): step(rep, s, k)
    wall = time.perf_counter() - t0
    timing = {ph: sum(r.timing()[ph] for r in reps) for ph in PHASES}
    paths = np.concatenate([np.stack([r.path(w) for w in range(r.n)]) for r in reps])
    for r in reps: r.close(); r.be.close()
    return dict(wall=wall, timing=timing, path=paths)


def launches_per_step(seqs, frames):
    """preintegrate_kernel / preint_store_kernel launches per step, counted by torch.profiler over `frames` steps (None: not measured)"""
    try:
        import torch
        from torch.profiler import profile, ProfilerActivity
        reps = [make(s, kinds) for s, kinds in seqs]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(W, W + frames):
                for rep, (s, _) in zip(reps, seqs): step(rep, s, k)
            torch.cuda.synchronize()
        for r in reps: r.close(); r.be.close()
        names = [e.name for e in prof.events()]
        return tuple(sum(1 for x in names if kname in x) / frames for kname in ("preintegrate_kernel", "preint_store_kernel"))
    except Exception as e:            # a profiler that cannot attach leaves the count unmeasured, not guessed
        print(f"launch count not measured: {e}", file=sys.stderr)
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sequences", type=int, default=128); ap.add_argument("--frames", type=int, default=30); ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    N, steps = a.sequences, a.frames - W
    lib.Backend(abi.default_config()).close()                       # fails here without the library or a device
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True, check=True).stdout.strip()
    seq = synth.generate_sequence(N, a.frames, tracked=90, max_len=14, min_len=3)
    fleet = tiled(seq, np.concatenate([np.arange(N), np.arange(N)]))
    arrangements = {"mixed": [(fleet, [True] * N + [False] * N)], "split": [(seq, [True] * N), (seq, [False] * N)]}
    runs = {name: [] for name in arrangements}
    for name, seqs in arrangements.items(): run(name, seqs)         # warm-up: module load, arena growth, page locking
    for _ in range(a.reps):
        for name, seqs in arrangements.items(): runs[name].append(run(name, seqs))
    lines = [smi.replace("\n", " | "),
             f"{2 * N} robots ({N} sequences x {{A1 VILO, A1 VINS}}) x {steps} frames, F = {F}, 90 tracked features, resident mode, "
             f"{a.reps} repetitions per arrangement, arrangements alternating; wall = Python glue + library"]
    m = min(N, 8)                                                   # the count does not depend on the fleet's size
    small = {"mixed": [(tiled(seq, np.concatenate([np.arange(m), np.arange(m)])), [True] * m + [False] * m)],
             "split": [(tiled(seq, np.arange(m)), [True] * m), (tiled(seq, np.arange(m)), [False] * m)]}
    counts = {name: launches_per_step(seqs, 3) for name, seqs in small.items()}
    for name in arrangements:
        rs = runs[name]
        rate = np.array([2 * N * steps / r["wall"] for r in rs])
        c = counts[name]
        lines.append(f"{name:6s}: {np.median(rate):.0f} robot-frames/s (min {rate.min():.0f}, max {rate.max():.0f}); preintegration launches per step: "
                     + (f"{c[0]:.0f} preintegrate_kernel + {c[1]:.0f} preint_store_kernel" if c else "not measured"))
        for ph in PHASES:
            v = np.array([r["timing"][ph] for r in rs]) / steps * 1e3
            lines.append(f"    {ph:13s} {np.median(v):8.2f} ms per frame (min {v.min():.2f}, max {v.max():.2f})")
        glue = np.array([r["wall"] - sum(r["timing"].values()) for r in rs]) / steps * 1e3
        lines.append(f"    {'python glue':13s} {np.median(glue):8.2f} ms per frame (min {glue.min():.2f}, max {glue.max():.2f})")
    P = runs["mixed"][0]["path"][:, :, 1:4]
    truth = seq.p[:, W:W + P.shape[1]]
    for label, half in (("A1 VILO", slice(0, N)), ("A1 VINS", slice(N, 2 * N))):
        err = np.linalg.norm(P[half] - truth, axis=-1)
        lines.append(f"{label}: distance of the published positions from the truth: mean {err.mean():.4f} m, median {np.median(err):.4f} m, "
                     f"max {err.max():.4f} m, at the last frame mean {err[:, -1].mean():.4f} m")
    ref = runs["split"][0]["path"].tobytes()
    same = all(r["path"].tobytes() == ref for rs in runs.values() for r in rs)
    lines.append(f"mixed trajectories bit-identical to the single-configuration ones (every run): {same}")
    print("\n".join(lines))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")
    if not same: sys.exit(1)


if __name__ == "__main__":
    main()

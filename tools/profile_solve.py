"""Driver for ncu: upload NW synthetic windows and run the resident solve REP times."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from cerberus_b200 import abi, synth, lib
NW = int(sys.argv[1]) if len(sys.argv) > 1 else 132
F = int(sys.argv[2]) if len(sys.argv) > 2 else 150
REP = int(sys.argv[3]) if len(sys.argv) > 3 else 2
cfg = abi.default_config(); cfg.max_batch = NW; cfg.max_features = 160; cfg.max_obs = 160 * 11
gb = lib.Backend(cfg)
batch = synth.generate_batch(min(NW, 8), F, gb, prior_features=24)
big = synth.tile_batch(batch, NW)
gb.upload(big)
for _ in range(REP):
    gb.solve_resident(); gb.sync()
    print("ms", gb.last_solve_stats())

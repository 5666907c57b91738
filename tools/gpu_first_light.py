"""First-light check on a real H100: parity of the GPU solve vs the CPU oracle + a first timing."""
import sys, time, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from cerberus_b200 import abi, synth, lib
from oracle_lib import OracleBackend

NW = int(sys.argv[1]) if len(sys.argv) > 1 else 16
F = int(sys.argv[2]) if len(sys.argv) > 2 else 150
cfg = abi.default_config(); cfg.max_batch = max(NW, 1024); cfg.max_features = 160; cfg.max_obs = 160 * 11
t0 = time.time(); gb = lib.Backend(cfg); print("create", time.time() - t0, gb.version(), flush=True)
ob = OracleBackend(cfg)
t0 = time.time(); batch = synth.generate_batch(NW, F, gb, prior_features=24); print("synth (gpu backend)", time.time() - t0, flush=True)
st = batch.state_array()
saved = batch.copy_states()
t0 = time.time(); rep_o = ob.solve_batch(batch, nthreads=os.cpu_count()); t_or = time.time() - t0
so_ = st.copy(); fo = batch.para_Feature.copy()
print("oracle: %.3f s for %d windows on %d threads -> %.1f solves/s" % (t_or, NW, os.cpu_count(), NW / t_or), flush=True)
batch.restore_states(saved)
t0 = time.time(); rep_g = gb.solve_batch(batch); t_g = time.time() - t0
print("gpu e2e first call: %.4f s" % t_g, "kernel ms", gb.last_solve_stats())
st2 = batch.state_array()
print("iters oracle", rep_o["iterations"][:16], "gpu", rep_g["iterations"][:16])
print("final cost rel diff max", np.abs(rep_o["final_cost"] - rep_g["final_cost"]).max() / np.abs(rep_o["final_cost"]).max())
for name in ["para_Pose", "para_SpeedBias", "para_LegBias", "para_Ex_Pose"]:
    print(name, "max abs diff", np.abs(st2[name] - so_[name]).max())
print("feat diff", np.abs(batch.para_Feature - fo).max())
worst = np.abs(st2["para_Pose"][:, :, :3] - so_["para_Pose"][:, :, :3]).reshape(NW, -1).max(axis=1)
print("per-window worst position diff: max %.3e  median %.3e" % (worst.max(), np.median(worst)))
# timing: replicate to 1024 windows resident
big = abi.WindowBatch(1024, batch.max_features)
for arr in ("features", "obs", "preint", "prior_J", "prior_r", "para_Feature"):
    getattr(big, arr)[:] = np.tile(getattr(batch, arr), (1024 // NW + 1,) + (1,) * (getattr(batch, arr).ndim - 1))[:1024]
batch.restore_states(saved)
import ctypes as C
for w in range(1024):
    s = w % NW
    C.memmove(C.byref(big.states[w]), C.byref(batch.states[s]), C.sizeof(abi.WindowState))
    big.states[w].para_Feature = big.para_Feature[w].ctypes.data_as(abi.c_dp)
    d, sd = big.descs[w], batch.descs[s]
    d.n_features, d.n_obs, d.extrinsic_open, d.td_open = sd.n_features, sd.n_obs, sd.extrinsic_open, sd.td_open
    pj, prr = d.prior.linearized_jacobians, d.prior.linearized_residuals
    C.memmove(C.byref(d.prior), C.byref(sd.prior), C.sizeof(abi.Prior))
    d.prior.linearized_jacobians, d.prior.linearized_residuals = big.prior_J[w].ctypes.data_as(abi.c_dp), big.prior_r[w].ctypes.data_as(abi.c_dp)
t0 = time.time(); gb.upload(big); gb.sync(); print("upload 1024: %.3f s" % (time.time() - t0))
for it in range(4):
    t0 = time.time(); gb.solve_resident(); gb.sync(); wall = time.time() - t0
    ms, nl = gb.last_solve_stats()
    print("resident solve 1024 windows: wall %.2f ms, cuda-event %.2f ms -> %.0f solves/s" % (wall * 1e3, ms, 1024 / (ms * 1e-3)), flush=True)
t0 = time.time(); rep = gb.solve_batch(big); t = time.time() - t0
print("e2e 1024 (host buffers): %.2f ms -> %.0f solves/s; mean iters %.2f" % (t * 1e3, 1024 / t, rep["iterations"].mean()))

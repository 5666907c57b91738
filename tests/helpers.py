"""Shared helpers of the test-suite."""
import os
import subprocess
import numpy as np
from cerberus_b200 import abi, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM_LIB = os.path.join(ROOT, "tests", "cusim", "libcerberus_b200_sim.so")


def sim_backend(cfg=None):
    """The CUDA kernels compiled for CPU threads (tests/cusim): exercises the real kernel sources without a GPU.
    TEST ONLY -- the product never loads this library."""
    if not os.path.exists(SIM_LIB):
        subprocess.check_call(["make", "-s", "-C", ROOT, "sim"])
    return lib.Backend(cfg, lib_path=SIM_LIB)


def small_cfg(max_batch=4, max_features=32, iters=12):
    cfg = abi.default_config()
    cfg.max_batch, cfg.max_features, cfg.max_obs, cfg.max_num_iterations = max_batch, max_features, max_features * abi.NUM_FRAMES, iters
    return cfg


def state_diffs(a, b):
    return {k: float(np.abs(a[k] - b[k]).max()) for k in ("para_Pose", "para_SpeedBias", "para_LegBias", "para_Ex_Pose")}


def prior_canonical(batch, w):
    """(A = J^T J, b = J^T r, x0 dict) of window w's prior with blocks in canonical order (independent of block order)."""
    pr = batch.descs[w].prior
    n = pr.n
    J = batch.prior_J[w][:n * n].reshape(n, n).T
    r = batch.prior_r[w][:n]
    A, b = J.T @ J, J.T @ r
    loc = {0: 6, 1: 9, 2: 4, 3: 6, 4: 1}
    keys = sorted((pr.block_kind[i], pr.block_index[i], pr.block_col[i]) for i in range(pr.num_blocks))
    perm = [c + t for (k, i, c) in keys for t in range(loc[k])]
    x0 = {(pr.block_kind[i], pr.block_index[i]): np.array(pr.block_x0[i][:]) for i in range(pr.num_blocks)}
    return A[np.ix_(perm, perm)], b[perm], x0


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "kat_v1.npz"), allow_pickle=False)


def golden_window(g):
    """Rebuild the WindowBatch of the golden window from the arrays frozen in kat_v1.npz."""
    import ctypes as C
    nf, no = g["win_features"].shape[0], g["win_obs"].shape[0]
    b = abi.WindowBatch(1, max(nf, g["win_para_Feature"].shape[0]), max(no, 1))
    b.features[0][:nf] = g["win_features"]; b.obs[0][:no] = g["win_obs"]; b.preint[0] = g["win_preint"]
    b.prior_J[0] = g["win_prior_J"]; b.prior_r[0] = g["win_prior_r"]; b.para_Feature[0][:g["win_para_Feature"].shape[0]] = g["win_para_Feature"]
    d = b.descs[0]
    prior_raw, state_raw = np.ascontiguousarray(g["win_prior_raw"]), np.ascontiguousarray(g["win_state_raw"])   # keep alive across memmove
    C.memmove(C.byref(d.prior), prior_raw.ctypes.data, C.sizeof(abi.Prior))
    d.prior.linearized_jacobians = b.prior_J[0].ctypes.data_as(abi.c_dp)
    d.prior.linearized_residuals = b.prior_r[0].ctypes.data_as(abi.c_dp)
    C.memmove(C.byref(b.states[0]), state_raw.ctypes.data, C.sizeof(abi.WindowState))
    b.states[0].para_Feature = b.para_Feature[0].ctypes.data_as(abi.c_dp)
    d.n_features, d.n_obs, d.extrinsic_open, d.td_open = nf, no, 1, 0
    return b


def check_against_golden(backend, g, tol_scale=1.0, solve=True):
    """Factor evaluators, kinematics and (optionally) the full solve of `backend` against the frozen KATs."""
    names = ("fk", "jac", "dfk_drho", "dJ_dq", "dJ_drho")
    for n, a in zip(names, backend.a1_kinematics(g["kin_q"], g["kin_lc"], g["kin_fix"])):
        assert np.abs(a - g["kin_" + n]).max() < 1e-14 * tol_scale, n
    for kind in range(3):
        args = [g[f"proj{kind}_in{i}"] for i in range(12)]
        r, j = backend.eval_projection(kind, *args)
        assert np.abs(r - g[f"proj{kind}_res"]).max() < 1e-9 * tol_scale * max(1.0, np.abs(g[f"proj{kind}_res"]).max())
        assert np.abs(j - g[f"proj{kind}_jac"]).max() < 1e-10 * tol_scale * np.abs(g[f"proj{kind}_jac"]).max()
    pre = np.ascontiguousarray(g["imu_pre"])
    out = backend.eval_imu_leg(pre, g["imu_params"])
    for got, key in zip(out, ("imu_res", "imu_jac", "imu_sqrt_info")):
        assert np.abs(got - g[key]).max() < 1e-9 * tol_scale * np.abs(g[key]).max(), key
    if solve:
        b = golden_window(g)
        rep = backend.solve_batch(b)
        st = b.state_array()
        assert rep["iterations"][0] == g["win_report"]["iterations"][0]
        assert abs(rep["final_cost"][0] - g["win_report"]["final_cost"][0]) < 1e-7 * g["win_report"]["final_cost"][0]
        assert np.abs(st["para_Pose"][0] - g["win_solved_pose"]).max() < 1e-7       # << the 1e-4 m bar of BASELINE.json
        assert np.abs(st["para_SpeedBias"][0] - g["win_solved_sb"]).max() < 1e-6
        assert np.abs(st["para_Ex_Pose"][0] - g["win_solved_ex"]).max() < 1e-7
        nf = g["win_solved_feature"].shape[0]
        assert np.abs(b.para_Feature[0][:nf] - g["win_solved_feature"]).max() < 1e-7


SEAM = os.path.join(ROOT, "tests", "seam")


def seam_probe(include_dir, workdir):
    """The JSON printed by tests/seam/probe.cpp built against `include_dir` (tests/seam or the reference's src directory)."""
    import json
    exe = os.path.join(workdir, "seam_probe")
    subprocess.run(["g++", "-std=c++14", "-w", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "oracle", "shim"), "-I" + include_dir,
                    os.path.join(SEAM, "probe.cpp"), "-o", exe], check=True, capture_output=True, text=True)
    return json.loads(subprocess.run([exe], check=True, capture_output=True, text=True).stdout)

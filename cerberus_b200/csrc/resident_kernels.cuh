// resident_kernels.cuh -- device side of the resident sliding window (cerb_resident_*, include/cerberus_b200.h): the raw arrays an upload
// fills (robs, rpre, the prior in rdesc / prior_J / prior_r) stay in HBM across frames and are edited in place; pack_kernel then reads them
// exactly as it reads an uploaded window.
//   * track store: robs of a window as slots of CERB_NUM_FRAMES observations, a track left-aligned in its slot
//       track_put_kernel   FeaturePerId::feature_per_frame.push_back   (feature_manager.cpp:93-113)
//       track_edit_kernel  feature_per_frame.erase(begin() + k)        (removeBackShiftDepth / removeBack / removeFront, :450-529)
//   * preint_store_kernel: a result of preintegrate_kernel into a slot of rpre, in the raw row layout of an uploaded record
//   * prior_handover_kernel: the result of marg_assemble_kernel + marg_schur_kernel becomes the window's CerbPrior
// Every index these kernels use has been validated by the host (cabi.cu); they check nothing.
#pragma once
#include "pack_kernels.cuh"

namespace cerb {

CERB_GLOBAL void track_put_kernel(int count, const CerbTrackPut *puts, CerbObservation *robs, int maxObs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const CerbTrackPut &p = puts[i];
    robs[(size_t)p.window * maxObs + p.slot * CERB_NUM_FRAMES + p.position] = p.obs;
}

// one thread per track: at most ten 80-byte records move one place to the left
CERB_GLOBAL void track_edit_kernel(int count, const CerbTrackEdit *edits, CerbObservation *robs, int maxObs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const CerbTrackEdit e = edits[i];
    CerbObservation *t = robs + (size_t)e.window * maxObs + e.slot * CERB_NUM_FRAMES;
    for (int k = e.position; k + 1 < e.n_obs; k++) t[k] = t[k + 1];
}

// Job j of a preintegrate_kernel launch (packed: [n][PRE_STRIDE], full: [n][1922] = jacobian | covariance, row-major 31 x 31) into slot
// where[3 j + 1] of window where[3 j]; where[3 j + 2] is the record kind of that window.  leg (0): head (33 doubles in struct order) |
// jacobian columns 21..30 | covariance, column-major; imu only (1): the CerbIMUPreint struct (467 doubles), rows / columns P, R, V, BA, BG
// gathered from their ILStateOrder places.
CERB_GLOBAL void preint_store_kernel(int n, const int *where, const double *packed, const double *full, double *rpre, double *sum_dt) {
    const int j = blockIdx.x;
    if (j >= n) return;
    const double *o = packed + (size_t)j * PRE_STRIDE, *f = full + (size_t)j * 1922;
    double *raw = rpre + ((size_t)where[3 * j] * CERB_WINDOW_SIZE + where[3 * j + 1]) * RAW_PRE_STRIDE;
    const int imu_only = where[3 * j + 2];
    if (threadIdx.x == 0) sum_dt[j] = o[PRE_SUM_DT];
    if (!imu_only) {
        for (int k = threadIdx.x; k < RAW_PRE_STRIDE; k += blockDim.x) {
            double v;
            if (k < RAW_PRE_HEAD) v = o[k];                        // PRE_SUM_DT .. PRE_RHO are the struct's order
            else if (k < RAW_PRE_HEAD + 310) { const int e = k - RAW_PRE_HEAD, c = RAW_PRE_JCOL0 + e / 31, r = e % 31; v = f[r * 31 + c]; }
            else { const int e = k - RAW_PRE_HEAD - 310, c = e / 31, r = e % 31; v = f[961 + r * 31 + c]; }
            raw[k] = v;
        }
        return;
    }
    for (int k = threadIdx.x; k < 467; k += blockDim.x) {
        double v;
        if (k == 0) v = o[PRE_SUM_DT];
        else if (k < 4) v = o[PRE_DP + k - 1];
        else if (k < 8) v = o[PRE_DQ + k - 4];
        else if (k < 11) v = o[PRE_DV + k - 8];
        else if (k < 14) v = o[PRE_BA + k - 11];
        else if (k < 17) v = o[PRE_BG + k - 14];
        else {
            const int e = (k - 17) % 225, c = e / 15, r = e % 15, r31 = r < 9 ? r : r + 12, c31 = c < 9 ? c : c + 12;      // inverse of imu15_slot
            v = f[(k < 242 ? 0 : 961) + r31 * 31 + c31];
        }
        raw[k] = v;
    }
}

// After marg_schur_kernel has finished: window w's new prior (dims / blocks of marg_assemble_kernel, x0 from the states it linearised at,
// J / r from the Schur kernel's output) replaces the old one, which was an input of those kernels.  status 2 (carried over) leaves it alone,
// status 0 (MARGIN_OLD with nothing dropped) invalidates it.  window [n] (a compact batch): row w's prior goes to store window window[w];
// null: to window w.
CERB_GLOBAL void prior_handover_kernel(int n, const int *window, const int *dims, const int *blocks, const double *state, const double *J, long j_stride, const double *r,
                                       long r_stride, CerbWindowDesc *rdesc, double *prior_J, double *prior_r) {
    for (int w = blockIdx.x; w < n; w += gridDim.x) {
        const int status = dims[4 * w + 2], nn = dims[4 * w + 1], nb = dims[4 * w + 3];
        const int sw = window ? window[w] : w;
        if (status == 2) continue;
        CerbPrior &pr = rdesc[sw].prior;
        if (status == 0) { if (threadIdx.x == 0) pr.valid = 0; continue; }
        if (threadIdx.x == 0) { pr.valid = 1; pr.n = nn; pr.num_blocks = nb; pr.reserved = 0; }
        if (threadIdx.x < CERB_MAX_PRIOR_BLOCKS) {
            const int b = threadIdx.x, *q = blocks + (size_t)w * 64 + 4 * b;
            const bool on = b < nb;
            pr.block_kind[b] = on ? q[0] : 0; pr.block_index[b] = on ? q[1] : 0; pr.block_col[b] = on ? q[2] : 0;
            const int size = on ? prior_block_size(q[0]) : 0;
            const double *x = state + (size_t)w * ST_STRIDE + (on ? prior_block_state_offset(q[0], q[3]) : 0);
            for (int k = 0; k < 9; k++) pr.block_x0[b][k] = k < size ? x[k] : 0.0;
        }
        const double *Js = J + (size_t)w * j_stride, *rs = r + (size_t)w * r_stride;
        double *Jd = prior_J + (size_t)sw * PRIOR_LD * PRIOR_LD, *rd = prior_r + (size_t)sw * PRIOR_LD;
        for (int e = threadIdx.x; e < nn * nn; e += blockDim.x) Jd[e] = Js[e];
        for (int e = threadIdx.x; e < nn; e += blockDim.x) rd[e] = rs[e];
    }
}

// A compact batch of resident windows: the prior matrix and residuals of store window window[w] into row w of a per-step area.  The solve,
// prior_prepare_kernel and marg_assemble_kernel index the prior by batch row; pointed at this area they read each row's own prior without
// a change, and the store keeps one prior per window (prior_handover_kernel writes the next one there).
CERB_GLOBAL void prior_gather_kernel(int n, const int *window, const CerbWindowDesc *rdesc, const double *prior_J, const double *prior_r, double *step_J, double *step_r) {
    for (int w = blockIdx.x; w < n; w += gridDim.x) {
        const int sw = window[w];
        const CerbPrior &pr = rdesc[sw].prior;
        if (!pr.valid) continue;
        const int nn = pr.n;
        const double *Js = prior_J + (size_t)sw * PRIOR_LD * PRIOR_LD, *rs = prior_r + (size_t)sw * PRIOR_LD;
        double *Jd = step_J + (size_t)w * PRIOR_LD * PRIOR_LD, *rd = step_r + (size_t)w * PRIOR_LD;
        for (int e = threadIdx.x; e < nn * nn; e += blockDim.x) Jd[e] = Js[e];
        for (int e = threadIdx.x; e < nn; e += blockDim.x) rd[e] = rs[e];
    }
}

}  // namespace cerb

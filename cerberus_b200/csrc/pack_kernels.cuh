// pack_kernels.cuh -- the reference-shaped host descriptors (AoS, Eigen column-major; include/cerberus_b200.h) are shipped to the
// device AS THEY ARE (plain DMA out of the caller's buffers) and turned into the solver's HBM layout here, one CTA per window:
//   * tracks sorted by anchor frame (stable counting sort; the solver's feature chunks share one anchor), para_Feature permuted along
//   * observations AoS (FeaturePerFrame records, 80 B) -> 9 planes + stereo flags
//   * IMULegIntegrationBase / IntegrationBase results -> the compact 1096-double record (33 nominal + 93 bias-Jacobian entries +
//     31 x 31 covariance, row-major)
//   * prior block list -> meta / x0 arrays (the n x n matrix and residual vector are DMA'd in place)
//   * para_* arrays -> state vector (same order, contiguous)
// and back (unpack_kernel): inverse depths into the caller's feature order, reports as CerbSolveReport records.
// The host side of a solve is then validation + a handful of cudaMemcpy(2D)Async calls; no per-field scatter on CPU threads.
#pragma once
#include "solve_kernel.cuh"

namespace cerb {

enum { RAW_PRE_STRIDE = 1304, RAW_PRE_HEAD = 33, RAW_PRE_JCOL0 = 21, PACK_THREADS = 256 };
// raw leg record: [0,33) the scalar / vector members in struct order; [33, 343) jacobian columns 21..30 (column-major: the d/d(ba, bg, rho)
// columns, the only ones IMULegFactor::Evaluate reads, imu_leg_factor.cpp:204-219); [343, 1304) covariance (column-major).
// raw imu-only record: the CerbIMUPreint struct as is (467 doubles).

struct PackParams {
    int n, maxF, maxObs;
    const CerbWindowDesc *rdesc; const CerbFeature *rfeat; const CerbObservation *robs; const double *rpre; const CerbWindowState *rstate; const double *rlam;
    int *n_features, *feat_start, *feat_nobs, *feat_off, *flags, *obs_stereo, *prior_meta, *perm;
    double *obs, *pre, *prior_x0, *state0, *lam0;
    const int *pre_slot = nullptr;       // [n][CERB_WINDOW_SIZE] row of rpre that holds interval i -> i + 1 (resident sliding window); null: row i
    // [n] store window of batch row w (a compact batch of resident windows): robs, rpre and the prior inside rdesc are read at window[w],
    // everything else (the descriptor's head and tail, rfeat, rstate, rlam and every output) at w; null: window w
    const int *window = nullptr;
};

CERB_HD double pack_pre_leg(const double *raw, int k) {
    if (k < RAW_PRE_HEAD) return raw[k];
    if (k >= PRE_INFO) { const int e = k - PRE_INFO; if (e >= 961) return 0.0; const int r = e / 31, c = e % 31; return raw[343 + c * 31 + r]; }
    if (k >= PRE_IMU_ONLY) return 0.0;
    auto J = [&](int r, int c) { return raw[RAW_PRE_HEAD + (c - RAW_PRE_JCOL0) * 31 + r]; };
    if (k < PRE_DEP_DBG) {                      // five 3 x 3 blocks
        const int blk = (k - PRE_DP_DBA) / 9, e = (k - PRE_DP_DBA) % 9, a = e / 3, b = e % 3;
        switch (blk) {
            case 0: return J(ILO_P + a, ILO_BA + b);
            case 1: return J(ILO_P + a, ILO_BG + b);
            case 2: return J(ILO_R + a, ILO_BG + b);
            case 3: return J(ILO_V + a, ILO_BA + b);
            default: return J(ILO_V + a, ILO_BG + b);
        }
    }
    if (k < PRE_DEP_DRHO) { const int e = k - PRE_DEP_DBG, leg = e / 9, a = (e % 9) / 3, b = e % 3; return J(ILO_EPS1 + 3 * leg + a, ILO_BG + b); }
    { const int e = k - PRE_DEP_DRHO, leg = e / 3, a = e % 3; return J(ILO_EPS1 + 3 * leg + a, ILO_RHO1 + leg); }
}
// IntegrationBase result embedded in the 31-row layout (see the note at pack_imu_preint's former place in DESIGN.md 1): rows / columns
// P, R, V, BA, BG go to their ILStateOrder slots, the EPS / RHO diagonal of the covariance is the identity
CERB_HD int imu15_slot(int r31) { return r31 < 9 ? r31 : (r31 >= 21 && r31 < 27 ? r31 - 12 : -1); }
CERB_HD double pack_pre_imu(const double *raw, int k) {
    // CerbIMUPreint: sum_dt 0, delta_p 1, delta_q 4, delta_v 8, linearized_ba 11, linearized_bg 14, jacobian 17 (15 x 15 col-major), covariance 242
    if (k == PRE_SUM_DT) return raw[0];
    if (k == PRE_IMU_ONLY) return 1.0;
    if (k >= PRE_DP && k < PRE_DP + 3) return raw[1 + k - PRE_DP];
    if (k >= PRE_DQ && k < PRE_DQ + 4) return raw[4 + k - PRE_DQ];
    if (k >= PRE_DV && k < PRE_DV + 3) return raw[8 + k - PRE_DV];
    if (k >= PRE_BA && k < PRE_BA + 3) return raw[11 + k - PRE_BA];
    if (k >= PRE_BG && k < PRE_BG + 3) return raw[14 + k - PRE_BG];
    if (k >= PRE_INFO) {
        const int e = k - PRE_INFO; if (e >= 961) return 0.0;
        const int r = e / 31, c = e % 31, r15 = imu15_slot(r), c15 = imu15_slot(c);
        if (r15 >= 0 && c15 >= 0) return raw[242 + c15 * 15 + r15];
        return r == c ? 1.0 : 0.0;
    }
    if (k >= PRE_DP_DBA && k < PRE_DEP_DBG) {
        auto J = [&](int r, int c) { return raw[17 + c * 15 + r]; };
        const int blk = (k - PRE_DP_DBA) / 9, e = (k - PRE_DP_DBA) % 9, a = e / 3, b = e % 3;
        switch (blk) {
            case 0: return J(0 + a, 9 + b);
            case 1: return J(0 + a, 12 + b);
            case 2: return J(3 + a, 12 + b);
            case 3: return J(6 + a, 9 + b);
            default: return J(6 + a, 12 + b);
        }
    }
    return 0.0;
}

CERB_GLOBAL void __launch_bounds__(PACK_THREADS) pack_kernel(CERB_GRID_CONSTANT PackParams P) {
    __shared__ int s_start[2048], s_cnt[16], s_perm[2048];
    const int tid = threadIdx.x;
    for (int w = blockIdx.x; w < P.n; w += gridDim.x) {
        const CerbWindowDesc &d = P.rdesc[w];
        const int sw = P.window ? P.window[w] : w;                   // the window of the store this row reads
        const int F = P.maxF, O = P.maxObs, nF = d.n_features, nO = d.n_obs;
        const bool leg = d.preint != nullptr;                        // host pointer value: only its null-ness is used
        const CerbFeature *ft = P.rfeat + (size_t)w * F;
        // ---- tracks: stable counting sort by anchor frame ----------------------------------------------------------
        if (tid < 16) s_cnt[tid] = 0;
        for (int f = tid; f < nF; f += PACK_THREADS) s_start[f] = ft[f].start_frame;
        __syncthreads();
        if (tid == 0) {
            int c[CERB_NUM_FRAMES + 1] = {0};
            for (int f = 0; f < nF; f++) c[s_start[f] + 1]++;
            for (int a = 0; a < CERB_NUM_FRAMES; a++) { c[a + 1] += c[a]; s_cnt[a] = c[a]; }
        }
        __syncthreads();
        if (tid < CERB_NUM_FRAMES) { int pos = s_cnt[tid]; for (int f = 0; f < nF; f++) if (s_start[f] == tid) s_perm[pos++] = f; }
        __syncthreads();
        for (int k = tid; k < nF; k += PACK_THREADS) {
            const int f = s_perm[k];
            const size_t o = (size_t)w * F + k;
            P.feat_start[o] = ft[f].start_frame; P.feat_nobs[o] = ft[f].n_obs; P.feat_off[o] = ft[f].obs_offset;
            P.lam0[o] = P.rlam[(size_t)w * F + f]; P.perm[o] = f;
        }
        if (tid == 0) { P.n_features[w] = nF; P.flags[w] = (d.extrinsic_open ? 1 : 0) | (d.td_open ? 2 : 0) | (leg ? 0 : 4); }
        // ---- observations: AoS -> planes ----------------------------------------------------------------------------
        {
            const CerbObservation *ob = P.robs + (size_t)sw * O;
            double *op = P.obs + (size_t)w * NOBS_PLANES * O;
            int *so = P.obs_stereo + (size_t)w * O;
            for (int o = tid; o < nO; o += PACK_THREADS) {
                const CerbObservation q = ob[o];
                op[0 * O + o] = q.point[0]; op[1 * O + o] = q.point[1]; op[2 * O + o] = q.velocity[0]; op[3 * O + o] = q.velocity[1];
                op[4 * O + o] = q.pointRight[0]; op[5 * O + o] = q.pointRight[1]; op[6 * O + o] = q.velocityRight[0]; op[7 * O + o] = q.velocityRight[1];
                op[8 * O + o] = q.cur_td; so[o] = q.is_stereo;
            }
        }
        // ---- preintegration records ----------------------------------------------------------------------------------
        for (int e = tid; e < CERB_WINDOW_SIZE * PRE_STRIDE; e += PACK_THREADS) {
            const int i = e / PRE_STRIDE, k = e % PRE_STRIDE;
            const double *raw = P.rpre + ((size_t)sw * CERB_WINDOW_SIZE + (P.pre_slot ? P.pre_slot[w * CERB_WINDOW_SIZE + i] : i)) * RAW_PRE_STRIDE;
            P.pre[((size_t)w * CERB_WINDOW_SIZE + i) * PRE_STRIDE + k] = leg ? pack_pre_leg(raw, k) : pack_pre_imu(raw, k);
        }
        // ---- prior block list -----------------------------------------------------------------------------------------
        {
            int *meta = P.prior_meta + (size_t)w * PRIOR_META_STRIDE;
            const CerbPrior &pr = P.rdesc[sw].prior;
            for (int k = tid; k < PRIOR_META_STRIDE; k += PACK_THREADS) {
                int v = 0;
                if (pr.valid) {
                    if (k == 0) v = 1; else if (k == 1) v = pr.n; else if (k == 2) v = pr.num_blocks;
                    else if (k >= 4 && k < 4 + 3 * pr.num_blocks) { const int b = (k - 4) / 3, q = (k - 4) % 3; v = q == 0 ? pr.block_kind[b] : (q == 1 ? pr.block_index[b] : pr.block_col[b]); }
                }
                meta[k] = v;
            }
            if (pr.valid) for (int k = tid; k < 9 * pr.num_blocks; k += PACK_THREADS) P.prior_x0[(size_t)w * 16 * 9 + k] = pr.block_x0[k / 9][k % 9];
        }
        // ---- para_* arrays (same order as the state vector: pose 0, speed-bias 77, leg-bias 176, extrinsics 220, td 234) ---------------
        {
            const double *rs = reinterpret_cast<const double *>(P.rstate + w);
            for (int k = tid; k < ST_STRIDE; k += PACK_THREADS) P.state0[(size_t)w * ST_STRIDE + k] = k < ST_SIZE ? rs[k] : 0.0;
        }
        __syncthreads();
    }
}

// after a solve: inverse depths back into the caller's feature order, reports as CerbSolveReport records, states in CerbWindowState layout
struct UnpackParams {
    int n, maxF;
    const int *n_features, *perm, *rep_i; const double *rep_d, *lam, *state;
    double *olam; CerbSolveReport *orep; double *ostate;           // ostate: [n][ST_STRIDE] (first 235 doubles = the para_* arrays)
};
CERB_GLOBAL void __launch_bounds__(PACK_THREADS) unpack_kernel(CERB_GRID_CONSTANT UnpackParams P) {
    const int tid = threadIdx.x;
    for (int w = blockIdx.x; w < P.n; w += gridDim.x) {
        const int nF = P.n_features[w], F = P.maxF;
        for (int k = tid; k < nF; k += PACK_THREADS) P.olam[(size_t)w * F + P.perm[(size_t)w * F + k]] = P.lam[(size_t)w * F + k];
        for (int k = tid; k < ST_STRIDE; k += PACK_THREADS) P.ostate[(size_t)w * ST_STRIDE + k] = P.state[(size_t)w * ST_STRIDE + k];
        if (tid == 0) {
            CerbSolveReport r;
            r.iterations = P.rep_i[4 * w]; r.num_successful_steps = P.rep_i[4 * w + 1]; r.termination = P.rep_i[4 * w + 2]; r.status = P.rep_i[4 * w + 3];
            r.initial_cost = P.rep_d[2 * w]; r.final_cost = P.rep_d[2 * w + 1];
            P.orep[w] = r;
        }
    }
}

// per-feature outputs of the resident-batch passes: device slot order -> the caller's feature order
CERB_GLOBAL void unpermute_kernel(int n, int F, int narr, const int *n_features, const int *perm, const double *in, double *out) {
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long)n * F) return;
    const int w = (int)(idx / F), k = (int)(idx % F);
    if (k >= n_features[w]) return;
    const int f = perm[idx];
    for (int a = 0; a < narr; a++) out[(size_t)a * n * F + (size_t)w * F + f] = in[(size_t)a * n * F + idx];
}

}  // namespace cerb

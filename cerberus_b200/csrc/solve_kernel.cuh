// solve_kernel.cuh -- the fused sliding-window solve: everything Estimator::optimization() does between
// vector2double() and double2vector() (reference src/estimator/estimator.cpp:1059-1236), one window per
// CTA, the whole trust-region loop device resident.
//
// Unknowns of a window (tangent space): x = [pose0..10 (66) | ex0, ex1 (12) | td (1)] = 79 "camera" dims,
// y_f = [speedbias_f (9) | legbias_f (4)] = 13 dims per frame (143), lambda = one inverse depth per
// feature.  Structure exploited (SURVEY.md appendix B):
//   * visual factors touch only x and lambda  -> lambda is Schur-eliminated with rank-1 updates
//     S = Hxx - W diag(1/h) W^T   (W = 78 x F, the per-landmark 1x1 blocks)
//   * IMU-leg factors couple (pose_f, y_f, pose_f+1, y_f+1) only -> Hyy is block tridiagonal (13x13
//     blocks) and is eliminated by a block-bidiagonal Cholesky:  S' = S - (L^-1 Hyx)^T (L^-1 Hyx)
//   * the 78 x 78 remainder is factored densely in shared memory.
// The solver semantics restated on top of that are those of Ceres 1.14: TRUST_REGION + TRADITIONAL
// DOGLEG (mu-regularised Gauss-Newton, Cauchy point), Jacobi scaling from iteration 0, HuberLoss
// corrector, the accept / reject / tolerance logic of TrustRegionMinimizer.  Constant parameter blocks
// are masked (scale 0): leg bias if !optimize_leg_bias, extrinsics until extrinsic_open, td unless td_open.
#pragma once
#include "eval_kernels.cuh"

namespace cerb {

// Optional per-phase cycle counters (tools/phase_profile.py builds a separate library with -DCERB_PHASE_TIMING; the
// product build compiles these macros to nothing).
#if defined(CERB_PHASE_TIMING) && !defined(CERB_CUSIM)
__device__ unsigned long long g_phase_cycles[48];
#define PH_DECL() long long ph_t = clock64()
#define PH_MARK_T(id, t) do { if ((threadIdx.x & 31) == 0) { const long long ph_n = clock64(); if (threadIdx.x == (t)) atomicAdd(&g_phase_cycles[id], (unsigned long long)(ph_n - ph_t)); ph_t = ph_n; } __syncwarp(); } while (0)
#define PH_MARK(id) PH_MARK_T(id, 0)
#define PH_ARG , long long &ph_t          // the phase functions of the solve kernel share the kernel's clock
#define PH_FWD , ph_t
#else
#define PH_DECL()
#define PH_MARK_T(id, t)
#define PH_MARK(id)
#define PH_ARG
#define PH_FWD
#endif

enum { CERB_WINDOW = 10, NX = 79, NYB = 13, NFR = 11, NY = 143, NR = 222, NRP = 224, HXX_SZ = 79 * 79, HXY_SZ = 79 * 143, X_TD = 78, SOLVE_THREADS = 256, FT = 64, TILE_LD = 33, NOBS_PLANES = 9 };
// block-tridiagonal Hyy: Ad = the NFR diagonal 13 x 13 blocks, Bo = the NFR - 1 blocks above the diagonal (row-major each)
enum { HBLK = NYB * NYB, AD_SZ = NFR * HBLK, BO_SZ = (NFR - 1) * HBLK };
#ifndef CERB_SOLVE_MIN_BLOCKS
#define CERB_SOLVE_MIN_BLOCKS 1
#endif
// prior Hessian image in global memory: [Hxx (6241) | pad (1) | Hxy | Ad | Bo]: both parts start on 16-byte boundaries and have sizes that are
// multiples of 16 bytes, so that each is ONE bulk copy (TMA 1-D, cp.async.bulk); shared memory has the same pad after Hxx (+ two mbarriers)
enum { PIMG_HXY = HXX_SZ + 1, PIMG_REST = HXY_SZ + AD_SZ + BO_SZ, PIMG_SZ = PIMG_HXY + PIMG_REST, SMEM_HXX_PAD = 3 };
static_assert((PIMG_HXY * 8) % 16 == 0 && (PIMG_REST * 8) % 16 == 0 && ((HXX_SZ + SMEM_HXX_PAD) * 8) % 16 == 0, "bulk-copy alignment of the prior image");

struct SolveParams {
    int n_windows, maxF, maxObs, max_iters, optimize_leg_bias;
    double G[3], sqrt_info, huber;
    double radius0, max_radius, min_radius, min_rel_dec, ftol, gtol, ptol;
    // batch (device pointers)
    const int *n_features, *feat_start, *feat_nobs, *feat_off, *flags;      // flags bit0 ex_open, bit1 td_open, bit2 no leg-bias blocks (USE_LEG == 0)
    const double *obs; const int *obs_stereo;                               // obs [B][9][maxObs] planar
    const double *pre;                                                      // [B][10][PRE_STRIDE] compact preintegration results
    const double *sinfo;                                                    // [B][10][961] sqrt_info (imu_leg_prepare_kernel)
    const double *prior_J, *prior_r, *prior_x0, *prior_Hp; const int *prior_meta;
    double *state, *lam;                                                    // [B][ST_STRIDE], [B][maxF]  in/out
    int *rep_i; double *rep_d;                                              // [B][4], [B][2]
    double *ws;                                                             // [grid][ws_stride] per-CTA workspace
    long ws_stride;
    double *dbg; int dbg_window;                                            // optional probe (cost, gradient, diag)
    double test_initial_mu;                                                 // parity tests only (env CERB_TEST_INITIAL_MU): DoglegStrategy::mu_ at the start (0: Ceres' 1e-8)
    int no_bulk_copy;                                                       // diagnostics (env CERB_NO_TMA): prior image by per-element cp.async instead of TMA bulk copies
    int test_fail_factorizations;                                           // parity tests only (env CERB_TEST_FAIL_FACTORIZATIONS): report the first k
                                                                            // Gauss-Newton solves of every window as failed (LINEAR_SOLVER_FAILURE path)
};

// per-CTA global workspace layout (doubles); F = maxF
CERB_HD long ws_vecs(int F) { return (long)NX * F; }                        // 9 vectors of F: hh, gl, sl, Dl, ghl, gnl, stl, lamc, sinv (windows with > 1024 features)
CERB_HD long ws_prior(int F) { return (long)NX * F + 9L * F; }              // image of the prior Hessian in the layout of Hxx | Hxy | Ad | Bo
CERB_HD long ws_chunks(int F) { return ws_prior(F) + PIMG_SZ; }                          // feature chunk table (ints)
CERB_HD long ws_imuplan(int F) { return (ws_chunks(F) + (F + 4) / 2 + 8 + 1) & ~1L; }                  // scatter plan of the IMU-leg Gram matrix (ints)
CERB_HD long ws_size(int F) { return ws_imuplan(F) + 15 * 2 * 32 * 4 / 2 + 8; }                            // even: the plan is read as int4
// this CTA's slice of the workspace
struct CtaWs {
    double *W, *hh, *gl, *sl, *Dl, *ghl, *gnl, *stl, *lamc, *sinv;     // sinv: 1 / sqrt(h + mu D^2) of windows with > 1024 features
    int *chunks;                                                        // [0] n, [1..n] chunk starts, [n + 1] end of the last chunk
    int *imu_plan;                                                      // scatter plan of the IMU-leg Gram matrix (build_imu_plan)
    double *pimg;                                                       // prior Hessian image, built once per window
    int F;                                                              // max_features: length of the vectors, leading dimension of W
};
CERB_D CtaWs ws_carve(const SolveParams &P) {
    double *ws = P.ws + (size_t)blockIdx.x * P.ws_stride;
    const int F = P.maxF;
    CtaWs v;
    v.W = ws;                                                           // [NX][F]
    v.hh = ws + ws_vecs(F); v.gl = v.hh + F; v.sl = v.gl + F; v.Dl = v.sl + F; v.ghl = v.Dl + F; v.gnl = v.ghl + F; v.stl = v.gnl + F; v.lamc = v.stl + F; v.sinv = v.lamc + F;
    v.chunks = reinterpret_cast<int *>(ws + ws_chunks(F)); v.imu_plan = reinterpret_cast<int *>(ws + ws_imuplan(F));
    v.pimg = ws + ws_prior(F); v.F = F;
    return v;
}

struct Smem {
    double *Hxx, *Hxy, *Ad, *Bo;            // 78x78, 78x143, 11x13x13, 10x13x13
    double *g, *sc, *D, *gh, *gn, *stp, *yv; // NRP each: gradient, jacobi scale, dogleg diag, g/D, GN step (z space), step (scaled), work
    double *xs, *xc;                        // current / candidate state (ST_STRIDE)
    double *Rw, *Rex;                       // rotation matrices: 11x9, 2x9 (of the state being evaluated)
    double *Ju;                             // 31 x 39
    double *lin;                            // 10 x 96 (IMULegLin)
    double *pdx, *pr;                       // prior dx, residual (96 each)
    double *red;                            // 8 x 256 reduction scratch
    double *wj;                             // 128 x 8 per-thread exchange
    double *sca;                            // 32 scalars (S_*)
    double *chain_col;                      // 2 x 16: double-buffered column line of the Hyy chain factorisation
    double *idg;                            // 143 (+pad): 1 / diag(L) of the block-bidiagonal factor of Hyy
    double *idx;                            // 79 (+pad): 1 / diag(L) of the dense factor of the reduced camera system
    int *ti;                                // TI_INTS ints (TI_*)
    unsigned long long *mbar;               // two mbarriers (bulk copies of the prior image: [0] Hxx part, [1] Hxy | Ad | Bo part)
    double *tile;                           // alias of Hxy (+ Ad, Bo): 256 x TILE_LD tile + 8 x 640 partial Gram tiles
};
// scalar slots of s.sca
enum { S_RADIUS = 0, S_MU, S_REUSE, S_XCOST, S_CCOST, S_ALPHA, S_GNORM2, S_GNNORM2, S_GDOTGN, S_MODEL, S_STEPNORM, S_XNORM, S_DLNORM,
       S_OK, S_DONE, S_TERM, S_ITER, S_NSUCC, S_INVALID, S_GMAX, S_INIT_COST, S_P, S_Q, S_VHV, S_LCOST, S_LNORM, S_LGMAX, S_COUNT };
static_assert(S_COUNT <= 32, "scalar slots overlap the chain's column line");
// int slots of s.ti: the prior's column -> destination map from 0 (build_prior_image), the feature chunk count, the first
// TI_CACHED_CHUNKS chunks as (start, count << 8 | anchor) pairs (build_chunks), the number of Hyy blocks the chain factorisation has
// published, the IMU-leg factor mask (0: all factors, 1: only factor 0, 2: none)
enum { TI_PRIOR_MAP = 0, TI_NCHUNKS = 96, TI_CHUNK_CACHE = 97, TI_CACHED_CHUNKS = 15, TI_CHAIN_DONE = 130, TI_IMU_MASK = 131, TI_INTS = 132 };
static_assert(TI_PRIOR_MAP + CERB_MAX_PRIOR_DIM <= TI_NCHUNKS && TI_CHUNK_CACHE + 2 * TI_CACHED_CHUNKS <= TI_CHAIN_DONE && TI_IMU_MASK < TI_INTS && TI_INTS % 2 == 0,
              "s.ti slots overlap");
enum { SMEM_DOUBLES = HXX_SZ + SMEM_HXX_PAD + HXY_SZ + AD_SZ + BO_SZ + 7 * NRP + 2 * ST_STRIDE + 99 + 18 + 3 + 31 * 39 + 960 + 192 + 8 * 256 + 128 * 8 + 32 + 32 + TI_INTS / 2 + 144 + 80 };

CERB_D void smem_carve(double *base, Smem &s) {
    double *p = base;
    s.Hxx = p; p += HXX_SZ; s.mbar = reinterpret_cast<unsigned long long *>(p + 1); p += SMEM_HXX_PAD; s.Hxy = p; p += HXY_SZ; s.Ad = p; p += AD_SZ; s.Bo = p; p += BO_SZ;
    s.g = p; p += NRP; s.sc = p; p += NRP; s.D = p; p += NRP; s.gh = p; p += NRP; s.gn = p; p += NRP; s.stp = p; p += NRP; s.yv = p; p += NRP;
    s.xs = p; p += ST_STRIDE; s.xc = p; p += ST_STRIDE;
    s.Rw = p; p += 99; s.Rex = p; p += 18; p += 3;
    s.Ju = p; p += 31 * 39; s.red = p; p += 8 * 256; s.wj = p; p += 128 * 8;      // contiguous scratch (4281 doubles): IMU_SCRATCH, Schur tile
    s.lin = p; p += 960; s.pdx = p; p += 96; s.pr = p; p += 96; s.sca = p; p += 32; s.chain_col = p; p += 32;
    s.ti = reinterpret_cast<int *>(p); p += TI_INTS / 2;
    s.idg = p; p += 144;
    s.idx = p; p += 80;
    s.tile = s.Hxy;
}

// deterministic block-wide sums of up to 8 values per thread; result broadcast in out[0..nv)
template <int NV>
CERB_D void block_sum(const double *v, double *red, double *out, int tid) {
    for (int k = 0; k < NV; k++) red[k * 256 + tid] = v[k];
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (tid < s) for (int k = 0; k < NV; k++) red[k * 256 + tid] += red[k * 256 + tid + s];
        __syncthreads();
    }
    for (int k = 0; k < NV; k++) out[k] = red[k * 256];
    __syncthreads();
}

// global -> shared copy with the loads of 8 strides issued before the first store (a plain copy loop is compiled as
// load, store, load, ... because the compiler cannot prove that the two pointers do not alias: one L2 round trip per element)
CERB_D void copy_g2s(double *dst, const double *src, int n, int tid) {
    for (int k0 = tid; k0 < n; k0 += 8 * SOLVE_THREADS) {
        double b[8];
        _Pragma("unroll")
        for (int u = 0; u < 8; u++) { const int k = k0 + u * SOLVE_THREADS; b[u] = (k < n) ? src[k] : 0.0; }
        _Pragma("unroll")
        for (int u = 0; u < 8; u++) { const int k = k0 + u * SOLVE_THREADS; if (k < n) dst[k] = b[u]; }
    }
}
// the same copy, asynchronous (no registers, no stall): completed by CERB_CP_ASYNC_WAIT() + a barrier
CERB_D void copy_g2s_async(double *dst, const double *src, int n, int tid) {
    for (int k = tid; k < n; k += SOLVE_THREADS) CERB_CP_ASYNC8(dst + k, src + k);
}
CERB_D void load_geometry(const double *x, Smem &s, int tid) {
    if (tid < 11) { const m33 R = qtoR(ldq(x + ST_POSE + 7 * tid + 3)); for (int k = 0; k < 9; k++) s.Rw[9 * tid + k] = R.m[k]; }
    else if (tid < 13) { const int e = tid - 11; const m33 R = qtoR(ldq(x + ST_EX + 7 * e + 3)); for (int k = 0; k < 9; k++) s.Rex[9 * e + k] = R.m[k]; }
    __syncthreads();
}

struct ObsCtx { int start, nobs, off; double lam, pix, piy, vix, viy, tdi; };

struct ObsVals { double px, py, vx, vy, td; int stereo; };
CERB_D void obs_fetch(const double *obs, const int *stereo, int mo, int o, int cam, ObsVals &v) {
    v.px = obs[(cam ? 4 : 0) * mo + o]; v.py = obs[(cam ? 5 : 1) * mo + o]; v.vx = obs[(cam ? 6 : 2) * mo + o]; v.vy = obs[(cam ? 7 : 3) * mo + o];
    v.td = obs[8 * mo + o]; v.stereo = stereo[o];
}

// ---- visual part: cost only (candidate evaluation) -------------------------------------------------------
CERB_NOINLINE double vision_cost(const SolveParams &P, int w, const double *x, const double *lam, int tid) {
    CERB_DYN_SMEM(double, smem_base);
    Smem s; smem_carve(smem_base, s);
    // One (feature, camera, track half) per thread and round.  The pass is bound by the L2 latency of the observation loads,
    // so all loads of an item are issued before its first factor is evaluated.
    const int nF = P.n_features[w], mo = P.maxObs;
    const double *obs = P.obs + (size_t)w * NOBS_PLANES * P.maxObs;
    const int *stereo = P.obs_stereo + (size_t)w * P.maxObs;
    double cost = 0.0;
    for (int idx = tid; idx < 4 * nF; idx += SOLVE_THREADS) {
        const int f = idx >> 2, cam = idx & 1, part = (idx >> 1) & 1;
        ObsCtx c;
        c.start = P.feat_start[(size_t)w * P.maxF + f]; c.nobs = P.feat_nobs[(size_t)w * P.maxF + f]; c.off = P.feat_off[(size_t)w * P.maxF + f];
        c.lam = lam[f];
        c.pix = obs[0 * mo + c.off]; c.piy = obs[1 * mo + c.off]; c.vix = obs[2 * mo + c.off]; c.viy = obs[3 * mo + c.off];
        c.tdi = obs[8 * mo + c.off];
        const int k0 = part ? 6 : 0, k1 = part ? c.nobs : (c.nobs < 6 ? c.nobs : 6);      // observations [k0, k1) of the track
        const double inv_l = 1.0 / c.lam;
        const int i = c.start;
        const d3 tic = ld3(x + ST_EX);
        const double tdv = x[ST_TD];
        const d3 pts_i_td = mk3(c.pix, c.piy, 1.0) - (tdv - c.tdi) * mk3(c.vix, c.viy, 0.0);
        const d3 p_bi = mv33(ldm33(s.Rex), inv_l * pts_i_td) + tic;                          // anchor-frame body point: shared by all factors
        const d3 p_w = mv33(ldm33(s.Rw + 9 * i), p_bi) + ld3(x + ST_POSE + 7 * i);
        const double *Rcp = cam ? s.Rex + 9 : s.Rex;
        const d3 tc = cam ? ld3(x + ST_EX + 7) : tic;
        ObsVals cur, nxt;
        cur.px = cur.py = cur.vx = cur.vy = cur.td = 0.0; cur.stereo = 0;
        if (k0 < k1) obs_fetch(obs, stereo, mo, c.off + k0, cam, cur);
        _Pragma("unroll 1")
        for (int k = k0; k < k1; k++) {                                   // compact loop body (instruction cache), next observation in flight
            nxt = cur;
            if (k + 1 < k1) obs_fetch(obs, stereo, mo, c.off + k + 1, cam, nxt);
            const bool k3 = (k == 0);
            const bool on = k3 ? (cam == 1 && cur.stereo) : (cam == 0 || cur.stereo);
            if (on) {
                const int j = c.start + k;
                const d3 p_bj = k3 ? p_bi : mTv33(ldm33(s.Rw + 9 * j), p_w - ld3(x + ST_POSE + 7 * j));
                const d3 p_cj = mTv33(ldm33(Rcp), p_bj - tc);
                const double iz = 1.0 / p_cj.z;
                const double r0 = P.sqrt_info * (p_cj.x * iz - (cur.px - (tdv - cur.td) * cur.vx));
                const double r1 = P.sqrt_info * (p_cj.y * iz - (cur.py - (tdv - cur.td) * cur.vy));
                double cf; huber_weight(P.huber, r0 * r0 + r1 * r1, &cf);
                cost += cf;
            }
            cur = nxt;
        }
    }
    return cost;
}

// ---- visual part: linearisation.  Accumulates the upper triangle of Hxx, g_x, writes W, hh, gl (global) ----
// Features are processed in chunks of <= 64 consecutive tracks that share one anchor frame a (the host sorts the tracks by
// anchor; `chunks` = [n, c0_0, c0_1, ..., nF] is built once per window).  A pass covers two frames: thread (jj, cam, fl)
// evaluates the factor of feature c0 + fl in frame j0 + jj seen by camera `cam` (K1 / K2, or K3 for the anchor frame) and
// writes its two Huber-corrected Jacobian rows into a column-major tile T[26][VT_LD]:
//     physical columns  0..5 pose_a | 6 td | 7 residual | 8..13 pose_j | 14..19 ex0 | 20..25 ex1
// The Gram matrix of the tile is a dense contraction and runs on the fp64 tensor cores: warp (jj, cam, feature half) contracts
// its 64 rows over the four 8-wide column groups g0 = [pose_a, td, r], g1 = [pose_j, 0, 0], g2 = [ex0, 0, 0], g3 = [ex1, 0, 0].
// Blocks that do not involve g1 have a destination that is independent of the frame and are accumulated per warp in shared
// memory over all passes of the chunk; the four g1 blocks are reduced over the warps of a frame and scattered after every
// pass.  Blocks that are structurally zero are skipped: g3 for camera 0 (K1 has no ex1 columns), g1 for the anchor frame (K3).
// prescale: write W, hh, gl already multiplied by the Jacobi scales (s.sc for x, sl for the inverse depths), which are
// fixed after iteration 0 -- saves a read-modify-write pass over W per linearisation.
enum { VT_LD = 516, VT_COLS = 26, VT_SZ = VT_COLS * VT_LD, VP_SZ = 6 * 64, VJ_SZ = 4 * 64 };
// destination of local column c (0..7) of group g in the x numbering; -1: padding, -2: the residual column (gradient)
CERB_D int vis_col_dest(int g, int c, int a, int j) {
    if (g == 0) return c < 6 ? 6 * a + c : (c == 6 ? X_TD : -2);
    if (c >= 6) return -1;
    return g == 1 ? 6 * j + c : (g == 2 ? 66 + c : 72 + c);
}
CERB_D void vis_scatter(Smem &s, int ga, int gb, int ra, int rb, int a, int j, double v) {
    if (ga == gb && ra > rb) return;
    const int da = vis_col_dest(ga, ra, a, j), db = vis_col_dest(gb, rb, a, j);
    if (da == -1 || db == -1) return;                                  // padding columns
    if (da == -2) { if (db >= 0) s.g[db] += v; return; }               // (r, c): gradient of c; (r, r) is the cost, summed elsewhere
    if (db == -2) { s.g[da] += v; return; }
    if (da <= db) s.Hxx[da * NX + db] += v; else s.Hxx[db * NX + da] += v;
}
// Destination of entry el = (blk, ra, rb) of the frame-dependent blocks (g0,g1), (g1,g1), (g1,g2), (g1,g3) as an affine function of the
// anchor a and the frame j: offset = base + ca * a + cj * j doubles from the start of shared memory (base < 0: no destination).
CERB_D void vis_jplan(const Smem &s, const double *smem_base, int el, int *base, int *ca, int *cj) {
    const int blk = el >> 6, ra = (el >> 3) & 7, rb = el & 7;
    const int hxx = (int)(s.Hxx - smem_base), g = (int)(s.g - smem_base);
    *base = -1; *ca = 0; *cj = 0;
    if (rb >= 6) return;                                                // padding columns of g1 / g2 / g3
    if (blk == 0) {                                                     // rows: pose_a (0..5), td (6), residual (7); columns: pose_j
        if (ra < 6) { *base = hxx + ra * NX + rb; *ca = 6 * NX; *cj = 6; }
        else if (ra == 6) { *base = hxx + rb * NX + X_TD; *cj = 6 * NX; }          // H(pose_j, td), stored in the upper triangle
        else { *base = g + rb; *cj = 6; }                                           // gradient of pose_j
    } else {
        if (ra >= 6 || (blk == 1 && ra > rb)) return;
        *base = hxx + ra * NX + (blk == 1 ? rb : (blk == 2 ? 66 + rb : 72 + rb)); *cj = 6 * NX + (blk == 1 ? 6 : 0);
    }
}
CERB_NOINLINE double vision_linearize(const SolveParams &P, int w, const double *x, const double *lam, double *W, double *hh, double *gl,
                                      const double *sl, bool prescale, const int *chunks, int tid) {
    CERB_DYN_SMEM(double, smem_base);
    Smem s; smem_carve(smem_base, s);
    const int nF = P.n_features[w], F = P.maxF, mo = P.maxObs;
    const double *obs = P.obs + (size_t)w * NOBS_PLANES * P.maxObs;
    const int *stereo = P.obs_stereo + (size_t)w * P.maxObs;
    double cost = 0.0;
    PH_DECL();
    for (int i = tid; i < NX * nF; i += SOLVE_THREADS) W[(i / nF) * F + (i % nF)] = 0.0;
    __syncthreads();                                                    // the passes below overwrite / add to rows of W
    const int wid = tid >> 5, lane = tid & 31;
    const int cam = tid >> 7, jj = (tid >> 6) & 1, fl = tid & 63;      // tile rows: tid (first residual row) and 256 + tid (second)
    double *T = s.tile;
    double *jp = s.Ju;                                                  // [8 warps][4 blocks][64]  frame-dependent partial blocks
    double *pp = (wid < 5) ? s.Ju + 8 * VJ_SZ + VP_SZ * wid : s.tile + VT_SZ + VP_SZ * (wid - 5);     // [6 blocks][64] of this warp
    // fragment sources of this lane: group g, local column lane / 4 -> physical column (or none)
    const int c8 = lane >> 2;
    const double *tq[4];
    bool tv[4];
    for (int g = 0; g < 4; g++) { const int pc = g == 0 ? c8 : 8 + 6 * (g - 1) + c8; tv[g] = (g == 0) || c8 < 6; tq[g] = T + (tv[g] ? pc : 0) * VT_LD + (lane & 3); }
    int jbase, jca, jcj;                                                // scatter plan of this thread's entry of the frame-dependent blocks
    vis_jplan(s, smem_base, tid, &jbase, &jca, &jcj);
    const int nchunks = s.ti[TI_NCHUNKS];
    for (int ch = 0; ch < nchunks; ch++) {
        int c0, nc, a;                                                  // chunk table: shared-memory cache (no dependent L2 round trips), else global
        if (ch < TI_CACHED_CHUNKS) { const int *cc = s.ti + TI_CHUNK_CACHE + 2 * ch; c0 = cc[0]; nc = cc[1] >> 8; a = cc[1] & 255; }
        else { c0 = chunks[1 + ch]; nc = chunks[2 + ch] - c0; a = P.feat_start[(size_t)w * F + c0]; }
        const int f = c0 + fl;
        const bool ev = fl < nc;
        int nobs = 0, off = 0;
        double lamf = 1.0, pix = 0.0, piy = 0.0, vix = 0.0, viy = 0.0, tdi = 0.0;
        const double slf = (prescale && ev) ? sl[f] : 1.0;
        if (ev) {
            nobs = P.feat_nobs[(size_t)w * F + f]; off = P.feat_off[(size_t)w * F + f];
            lamf = 1.0 / lam[f];                                          // inverse of the inverse depth, used by every factor of the track
            pix = obs[0 * mo + off]; piy = obs[1 * mo + off]; vix = obs[2 * mo + off]; viy = obs[3 * mo + off]; tdi = obs[8 * mo + off];
        }
        // first observation of this thread, issued with the loads above (the shared-memory stores below would otherwise order it after them)
        ObsVals ov; ov.px = ov.py = ov.vx = ov.vy = ov.td = 0.0; ov.stereo = 0;
        { const int j = a + jj; if (ev && j < a + nobs) obs_fetch(obs, stereo, mo, off + (j - a), cam, ov); }
        for (int k = lane; k < VP_SZ; k += 32) pp[k] = 0.0;
        // rotation products shared by all factors of (anchor a, frame j, camera c): A = Rc^T Rj^T, A Ri, T = A Ri ric (27 doubles per
        // (j, c) in s.lin, which is idle until the inertial pass); slot 20: T3 = ric2^T ric of the anchor-frame stereo factor (K3)
        if (tid < 2 * (NFR - 1 - a)) {
            const int jq = a + 1 + (tid >> 1), cq = tid & 1;
            const m33 Rc = ldm33(cq ? s.Rex + 9 : s.Rex);
            const m33 A = mulT33(Rc, tr33(ldm33(s.Rw + 9 * jq)));
            const m33 ARi = mul33(A, ldm33(s.Rw + 9 * a));
            const m33 Tm = mul33(ARi, ldm33(s.Rex));
            double *C = s.lin + 27 * tid;
            for (int k = 0; k < 9; k++) { C[k] = A.m[k]; C[9 + k] = ARi.m[k]; C[18 + k] = Tm.m[k]; }
        } else if (tid == 32) {
            const m33 T3 = mul33(tr33(ldm33(s.Rex + 9)), ldm33(s.Rex));
            for (int k = 0; k < 9; k++) s.lin[540 + k] = T3.m[k];
        }
        __syncthreads();
        double h = 0.0, gq = 0.0, wT = 0.0, wI[6], wE0[6], wE1[6];
        for (int k = 0; k < 6; k++) { wI[k] = 0.0; wE0[k] = 0.0; wE1[k] = 0.0; }
        PH_MARK(20);
        for (int j0 = a; j0 < NFR; j0 += 2) {
            const int j = j0 + jj;
            // --- evaluate this thread's factor into the tile -----------------------------------------------------------
            bool valid = ev && j < a + nobs;
            int kind = PROJ_K1;
            if (valid) {
                if (j == a) { if (cam == 0 || !ov.stereo) valid = false; kind = PROJ_K3; }
                else if (cam == 1) { if (!ov.stereo) valid = false; kind = PROJ_K2; }
            }
            double wjv[6] = {0, 0, 0, 0, 0, 0};
            double *t0 = T + tid, *t1 = T + 256 + tid;
            if (valid) {
                // Streamed evaluation (same algebra as proj_eval / the reference, regrouped): with e0, e1 the two Huber-scaled rows
                // of d(pixel)/d(p_cj) and u_M = [e0; e1] M, every rotation block is a cross product, e.g.
                // d r / d theta_i = [e0; e1] (-A Ri [p_bi]x) = p_bi x u_ARi.  Blocks go straight to the tile.
                const d3 tic = ld3(x + ST_EX), tc = kind == PROJ_K1 ? tic : ld3(x + ST_EX + 7);
                const double *Rcp = kind == PROJ_K1 ? s.Rex : s.Rex + 9;
                const double tdv = x[ST_TD];
                const d3 pts_i = mk3(pix, piy, 1.0), vel_i = mk3(vix, viy, 0.0);
                const d3 pts_i_td = pts_i - (tdv - tdi) * vel_i;
                const double pjx_td = ov.px - (tdv - ov.td) * ov.vx, pjy_td = ov.py - (tdv - ov.td) * ov.vy;
                const double inv_l = lamf;
                const d3 p_ci = inv_l * pts_i_td;
                const d3 p_bi = mv33(ldm33(s.Rex), p_ci) + tic;
                d3 p_bj = p_bi;
                if (kind != PROJ_K3) p_bj = mTv33(ldm33(s.Rw + 9 * j), (mv33(ldm33(s.Rw + 9 * a), p_bi) + ld3(x + ST_POSE + 7 * a)) - ld3(x + ST_POSE + 7 * j));
                const d3 p_cj = mTv33(ldm33(Rcp), p_bj - tc);
                const double iz = 1.0 / p_cj.z;
                double r0 = P.sqrt_info * (p_cj.x * iz - pjx_td), r1 = P.sqrt_info * (p_cj.y * iz - pjy_td);
                double cf; const double hw = huber_weight(P.huber, r0 * r0 + r1 * r1, &cf);
                cost += cf;
                r0 *= hw; r1 *= hw;
                const double q = hw * P.sqrt_info * iz, c0 = -q * p_cj.x * iz, c1 = -q * p_cj.y * iz;
                const d3 e0 = mk3(q, 0.0, c0), e1 = mk3(0.0, q, c1);
#define VIS_U(M, u0, u1) const d3 u0 = mk3(q * (M)[0] + c0 * (M)[6], q * (M)[1] + c0 * (M)[7], q * (M)[2] + c0 * (M)[8]), u1 = mk3(q * (M)[3] + c1 * (M)[6], q * (M)[4] + c1 * (M)[7], q * (M)[5] + c1 * (M)[8])
#define VIS_PUT(col, a0, a1) do { t0[(col) * VT_LD] = (a0); t1[(col) * VT_LD] = (a1); } while (0)
#define VIS_PUT3(col, v0_, v1_) do { VIS_PUT(col, (v0_).x, (v1_).x); VIS_PUT((col) + 1, (v0_).y, (v1_).y); VIS_PUT((col) + 2, (v0_).z, (v1_).z); } while (0)
                const double *Tm = kind == PROJ_K3 ? s.lin + 540 : s.lin + 27 * (2 * (j - a - 1) + cam) + 18;
                VIS_U(Tm, uT0, uT1);
                const d3 ptl = kind == PROJ_K3 ? pts_i : pts_i_td;              // reference quirk: K3 uses pts_i (projectionOneFrameTwoCamFactor.cpp:119)
                const double l0 = -inv_l * inv_l * dot3(uT0, ptl), l1 = -inv_l * inv_l * dot3(uT1, ptl);
                const double d0 = -inv_l * dot3(uT0, vel_i) + hw * P.sqrt_info * ov.vx, d1 = -inv_l * dot3(uT1, vel_i) + hw * P.sqrt_info * ov.vy;
                h += l0 * l0 + l1 * l1; gq += l0 * r0 + l1 * r1; wT += d0 * l0 + d1 * l1;
                VIS_PUT(6, d0, d1); VIS_PUT(7, r0, r1);
                // u_{Rc^T}: rows of Rc^T are the columns of Rc
                const d3 uC0 = mk3(q * Rcp[0] + c0 * Rcp[2], q * Rcp[3] + c0 * Rcp[5], q * Rcp[6] + c0 * Rcp[8]);
                const d3 uC1 = mk3(q * Rcp[1] + c1 * Rcp[2], q * Rcp[4] + c1 * Rcp[5], q * Rcp[7] + c1 * Rcp[8]);
                const d3 er0 = cross3(e0, p_cj), er1 = cross3(e1, p_cj);        // [e0; e1] [p_cj]x
                const d3 et0 = cross3(p_ci, uT0), et1 = cross3(p_ci, uT1);      // -[e0; e1] T [p_ci]x
                d3 E0t0, E0t1, E0r0, E0r1, E1t0, E1t1, E1r0, E1r1;
                if (kind == PROJ_K3) {
                    for (int k = 0; k < 6; k++) { VIS_PUT(k, 0.0, 0.0); VIS_PUT(8 + k, 0.0, 0.0); }
                    E0t0 = uC0; E0t1 = uC1; E0r0 = et0; E0r1 = et1; E1t0 = -uC0; E1t1 = -uC1; E1r0 = er0; E1r1 = er1;
                } else {
                    const double *C = s.lin + 27 * (2 * (j - a - 1) + cam);
                    VIS_U(C, uA0, uA1);
                    VIS_U(C + 9, uR0, uR1);
                    const d3 ir0 = cross3(p_bi, uR0), ir1 = cross3(p_bi, uR1);  // -[e] A Ri [p_bi]x
                    const d3 jr0 = cross3(uC0, p_bj), jr1 = cross3(uC1, p_bj);  //  [e] Rc^T [p_bj]x
                    VIS_PUT3(0, uA0, uA1); VIS_PUT3(3, ir0, ir1);
                    VIS_PUT3(8, -uA0, -uA1); VIS_PUT3(11, jr0, jr1);
                    wI[0] += uA0.x * l0 + uA1.x * l1; wI[1] += uA0.y * l0 + uA1.y * l1; wI[2] += uA0.z * l0 + uA1.z * l1;
                    wI[3] += ir0.x * l0 + ir1.x * l1; wI[4] += ir0.y * l0 + ir1.y * l1; wI[5] += ir0.z * l0 + ir1.z * l1;
                    wjv[0] = -(uA0.x * l0 + uA1.x * l1); wjv[1] = -(uA0.y * l0 + uA1.y * l1); wjv[2] = -(uA0.z * l0 + uA1.z * l1);
                    wjv[3] = jr0.x * l0 + jr1.x * l1; wjv[4] = jr0.y * l0 + jr1.y * l1; wjv[5] = jr0.z * l0 + jr1.z * l1;
                    if (kind == PROJ_K1) {
                        E0t0 = uR0 - uC0; E0t1 = uR1 - uC1; E0r0 = et0 + er0; E0r1 = et1 + er1;
                        E1t0 = mk3(0, 0, 0); E1t1 = E1t0; E1r0 = E1t0; E1r1 = E1t0;
                    } else {
                        E0t0 = uR0; E0t1 = uR1; E0r0 = et0; E0r1 = et1; E1t0 = -uC0; E1t1 = -uC1; E1r0 = er0; E1r1 = er1;
                    }
                }
                VIS_PUT3(14, E0t0, E0t1); VIS_PUT3(17, E0r0, E0r1); VIS_PUT3(20, E1t0, E1t1); VIS_PUT3(23, E1r0, E1r1);
                wE0[0] += E0t0.x * l0 + E0t1.x * l1; wE0[1] += E0t0.y * l0 + E0t1.y * l1; wE0[2] += E0t0.z * l0 + E0t1.z * l1;
                wE0[3] += E0r0.x * l0 + E0r1.x * l1; wE0[4] += E0r0.y * l0 + E0r1.y * l1; wE0[5] += E0r0.z * l0 + E0r1.z * l1;
                wE1[0] += E1t0.x * l0 + E1t1.x * l1; wE1[1] += E1t0.y * l0 + E1t1.y * l1; wE1[2] += E1t0.z * l0 + E1t1.z * l1;
                wE1[3] += E1r0.x * l0 + E1r1.x * l1; wE1[4] += E1r0.y * l0 + E1r1.y * l1; wE1[5] += E1r0.z * l0 + E1r1.z * l1;
#undef VIS_U
#undef VIS_PUT
#undef VIS_PUT3
            } else {
                for (int k = 0; k < VT_COLS; k++) { t0[k * VT_LD] = 0.0; t1[k * VT_LD] = 0.0; }
            }
            // W rows of frame j: camera 0 stores, camera 1 adds after the barrier (a K2 factor implies the K1 factor)
            const bool wrow = valid && j != a;
            if (wrow && cam == 0) for (int k = 0; k < 6; k++) W[(size_t)(6 * j + k) * F + f] = wjv[k] * (prescale ? s.sc[6 * j + k] * slf : 1.0);
            __syncthreads();
            PH_MARK(21);
            double wprev[6] = {0, 0, 0, 0, 0, 0};                       // loaded here, consumed after the tensor-core loop (L2 latency hidden)
            if (wrow && cam == 1) for (int k = 0; k < 6; k++) wprev[k] = W[(size_t)(6 * j + k) * F + f];
            { const int jn = j + 2; ov.stereo = 0; if (ev && jn < a + nobs) obs_fetch(obs, stereo, mo, off + (jn - a), cam, ov); }     // prefetch the next pass
            // --- Gram matrix.  Warp (jw = wid / 4, half = (wid / 2) & 1, par = wid & 1) contracts, for BOTH cameras of frame
            // j0 + jw, the k-steps (4 rows each) of parity `par` of row `half` of the factors: every warp issues the same number
            // of tensor-core instructions (camera-0 rows need 6 blocks, camera-1 rows 10), operands are fetched one k-step ahead. ---
            {
                const int jw = j0 + (wid >> 2), hw = (wid >> 1) & 1, par = wid & 1;
                const bool k3 = (jw == a);
                const int nkt = (nc + 3) >> 2;                                  // k-steps that hold valid features
                const bool work = jw < NFR && par < nkt;
                double acc[10][2];
                for (int k = 0; k < 10; k++) { acc[k][0] = 0.0; acc[k][1] = 0.0; }
                if (work) {
                    const int rb0 = 256 * hw + 64 * (wid >> 2) + 4 * par;       // camera 0 rows of this unit; camera 1: + 128
                    if (!k3) {                                                      // camera 0 (K1): groups g0, g1, g2
                        double v0 = tq[0][rb0], v1 = tv[1] ? tq[1][rb0] : 0.0, v2 = tv[2] ? tq[2][rb0] : 0.0;
                        for (int ks = par; ks < nkt; ks += 2) {
                            const int rn = rb0 + 4 * (ks + 2 - par);
                            const bool more = ks + 2 < nkt;
                            const double n0 = more ? tq[0][rn] : 0.0, n1 = (more && tv[1]) ? tq[1][rn] : 0.0, n2 = (more && tv[2]) ? tq[2][rn] : 0.0;
                            CERB_DMMA(acc[0][0], acc[0][1], v0, v0, acc[0][0], acc[0][1]);
                            CERB_DMMA(acc[1][0], acc[1][1], v0, v1, acc[1][0], acc[1][1]);
                            CERB_DMMA(acc[2][0], acc[2][1], v0, v2, acc[2][0], acc[2][1]);
                            CERB_DMMA(acc[4][0], acc[4][1], v1, v1, acc[4][0], acc[4][1]);
                            CERB_DMMA(acc[5][0], acc[5][1], v1, v2, acc[5][0], acc[5][1]);
                            CERB_DMMA(acc[7][0], acc[7][1], v2, v2, acc[7][0], acc[7][1]);
                            v0 = n0; v1 = n1; v2 = n2;
                        }
                    }
                    {                                                               // camera 1 (K2, or K3 in the anchor frame: no g1)
                        const int rb1 = rb0 + 128;
                        double v0 = tq[0][rb1], v1 = (!k3 && tv[1]) ? tq[1][rb1] : 0.0, v2 = tv[2] ? tq[2][rb1] : 0.0, v3 = tv[3] ? tq[3][rb1] : 0.0;
                        for (int ks = par; ks < nkt; ks += 2) {
                            const int rn = rb1 + 4 * (ks + 2 - par);
                            const bool more = ks + 2 < nkt;
                            const double n0 = more ? tq[0][rn] : 0.0, n1 = (more && !k3 && tv[1]) ? tq[1][rn] : 0.0, n2 = (more && tv[2]) ? tq[2][rn] : 0.0, n3 = (more && tv[3]) ? tq[3][rn] : 0.0;
                            CERB_DMMA(acc[0][0], acc[0][1], v0, v0, acc[0][0], acc[0][1]);
                            CERB_DMMA(acc[2][0], acc[2][1], v0, v2, acc[2][0], acc[2][1]);
                            CERB_DMMA(acc[3][0], acc[3][1], v0, v3, acc[3][0], acc[3][1]);
                            CERB_DMMA(acc[7][0], acc[7][1], v2, v2, acc[7][0], acc[7][1]);
                            CERB_DMMA(acc[8][0], acc[8][1], v2, v3, acc[8][0], acc[8][1]);
                            CERB_DMMA(acc[9][0], acc[9][1], v3, v3, acc[9][0], acc[9][1]);
                            if (!k3) {
                                CERB_DMMA(acc[1][0], acc[1][1], v0, v1, acc[1][0], acc[1][1]);
                                CERB_DMMA(acc[4][0], acc[4][1], v1, v1, acc[4][0], acc[4][1]);
                                CERB_DMMA(acc[5][0], acc[5][1], v1, v2, acc[5][0], acc[5][1]);
                                CERB_DMMA(acc[6][0], acc[6][1], v1, v3, acc[6][0], acc[6][1]);
                            }
                            v0 = n0; v1 = n1; v2 = n2; v3 = n3;
                        }
                    }
                    PH_MARK(28);
                    const int o = (lane >> 2) * 8 + 2 * (lane & 3);
                    pp[0 * 64 + o] += acc[0][0]; pp[0 * 64 + o + 1] += acc[0][1];      // (g0, g0)
                    pp[1 * 64 + o] += acc[2][0]; pp[1 * 64 + o + 1] += acc[2][1];      // (g0, g2)
                    pp[2 * 64 + o] += acc[3][0]; pp[2 * 64 + o + 1] += acc[3][1];      // (g0, g3)
                    pp[3 * 64 + o] += acc[7][0]; pp[3 * 64 + o + 1] += acc[7][1];      // (g2, g2)
                    pp[4 * 64 + o] += acc[8][0]; pp[4 * 64 + o + 1] += acc[8][1];      // (g2, g3)
                    pp[5 * 64 + o] += acc[9][0]; pp[5 * 64 + o + 1] += acc[9][1];      // (g3, g3)
                }
                {
                    const int o = wid * VJ_SZ + (lane >> 2) * 8 + 2 * (lane & 3);
                    jp[o] = acc[1][0]; jp[o + 1] = acc[1][1];                           // (g0, g1)
                    jp[64 + o] = acc[4][0]; jp[64 + o + 1] = acc[4][1];                 // (g1, g1)
                    jp[128 + o] = acc[5][0]; jp[128 + o + 1] = acc[5][1];               // (g1, g2)
                    jp[192 + o] = acc[6][0]; jp[192 + o + 1] = acc[6][1];               // (g1, g3)
                }
            }
            if (wrow && cam == 1) for (int k = 0; k < 6; k++) W[(size_t)(6 * j + k) * F + f] = wprev[k] + wjv[k] * (prescale ? s.sc[6 * j + k] * slf : 1.0);
            PH_MARK(29);
            __syncthreads();
            PH_MARK(22);
            // --- frame-dependent blocks: sum over the four warps of each frame (fixed order) and scatter ----------------------------
            // (thread tid owns entry el = tid of both frames; its destination is affine in (a, j): vis_jplan)
            if (jbase >= 0) {
                _Pragma("unroll")
                for (int fj = 0; fj < 2; fj++) {
                    const int jf = j0 + fj;
                    if (jf >= NFR || jf == a) continue;
                    const double *q = jp + (4 * fj) * VJ_SZ + tid;        // warps 4 fj .. 4 fj + 3 hold the partial blocks of frame j0 + fj
                    smem_base[jbase + jca * a + jcj * jf] += ((q[0] + q[VJ_SZ]) + q[2 * VJ_SZ]) + q[3 * VJ_SZ];
                }
            }
            PH_MARK(23);
        }
        __syncthreads();
        // --- end of the chunk: frame-independent blocks (sum over the 8 warps) and the per-feature lambda blocks ------------------------
        {
            double *ex = T;                                              // [21][256] exchange of the per-thread partial sums
            ex[0 * 256 + tid] = h; ex[1 * 256 + tid] = gq; ex[2 * 256 + tid] = wT;
            for (int k = 0; k < 6; k++) { ex[(3 + k) * 256 + tid] = wI[k]; ex[(9 + k) * 256 + tid] = wE0[k]; ex[(15 + k) * 256 + tid] = wE1[k]; }
        }
        __syncthreads();
        for (int e = tid; e < VP_SZ; e += SOLVE_THREADS) {
            double v = 0.0;
            for (int wq = 0; wq < 8; wq++) v += ((wq < 5) ? s.Ju + 8 * VJ_SZ + VP_SZ * wq : s.tile + VT_SZ + VP_SZ * (wq - 5))[e];
            const int blk = e >> 6, ra = (e >> 3) & 7, rb = e & 7;
            const int ga = blk < 3 ? 0 : (blk < 5 ? 2 : 3), gb = blk == 0 ? 0 : (blk == 1 || blk == 3 ? 2 : 3);
            vis_scatter(s, ga, gb, ra, rb, a, a, v);
        }
        if (tid < 64 && ev) {
            const double *ex = T;
            double q[21];
            for (int k = 0; k < 21; k++) q[k] = ((ex[k * 256 + tid] + ex[k * 256 + 64 + tid]) + ex[k * 256 + 128 + tid]) + ex[k * 256 + 192 + tid];
            hh[f] = q[0] * slf * slf; gl[f] = q[1] * slf;
            W[(size_t)X_TD * F + f] = q[2] * (prescale ? s.sc[X_TD] * slf : 1.0);
            for (int k = 0; k < 6; k++) {
                W[(size_t)(6 * a + k) * F + f] = q[3 + k] * (prescale ? s.sc[6 * a + k] * slf : 1.0);
                W[(size_t)(66 + k) * F + f] = q[9 + k] * (prescale ? s.sc[66 + k] * slf : 1.0);
                W[(size_t)(72 + k) * F + f] = q[15 + k] * (prescale ? s.sc[72 + k] * slf : 1.0);
            }
        }
        __syncthreads();
        PH_MARK(24);
    }
    return cost;
}

// ---- inertial part (IMU-leg factors + prior) ------------------------------------------------------------------
CERB_D void imu_lin_all(const SolveParams &P, Smem &s, int w, const double *x, bool want_jac, int tid) {
    if (tid < CERB_WINDOW) {
        const double *pre = P.pre + ((size_t)w * CERB_WINDOW + tid) * PRE_STRIDE;
        IMULegLin *L = reinterpret_cast<IMULegLin *>(s.lin + 96 * tid);
        imu_leg_linearize(pre, x + ST_POSE + 7 * tid, x + ST_SB + 9 * tid, x + ST_LB + 4 * tid, x + ST_POSE + 7 * (tid + 1),
                          x + ST_SB + 9 * (tid + 1), x + ST_LB + 4 * (tid + 1), P.G, want_jac, L);
    }
    __syncthreads();
}

// prior residual r = r0 + J0 dx into s.pr; returns this thread's share of 0.5 ||r||^2
CERB_D double prior_residual(const SolveParams &P, Smem &s, int w, const double *x, int tid) {
    const int *meta = P.prior_meta + (size_t)w * PRIOR_META_STRIDE;
    if (!meta[0]) return 0.0;
    const int n = meta[1], nb = meta[2];
    const double *J = P.prior_J + (size_t)w * PRIOR_LD * PRIOR_LD, *r0 = P.prior_r + (size_t)w * PRIOR_LD, *x0 = P.prior_x0 + (size_t)w * 16 * 9;
    if (tid < nb) {
        const int kind = meta[4 + 3 * tid], index = meta[5 + 3 * tid], col = meta[6 + 3 * tid];
        prior_block_dx(kind, x + prior_block_state_offset(kind, index), x0 + 9 * tid, s.pdx + col);
    }
    __syncthreads();
    // J0 dx with the column range cut into `parts` slices so that (almost) all threads stream J0 (coalesced over the rows)
    int parts = SOLVE_THREADS / n; if (parts > 4) parts = 4; if (parts < 1) parts = 1;
    const int kc = (n + parts - 1) / parts;
    double *part = s.red;                                               // [parts][PRIOR_LD]
    for (int e = tid; e < parts * n; e += SOLVE_THREADS) {
        const int p = e / n, i = e % n;
        const int k1 = (p + 1) * kc < n ? (p + 1) * kc : n;
        double t = 0.0;
        for (int k = p * kc; k < k1; k++) t += J[(size_t)k * n + i] * s.pdx[k];
        part[p * PRIOR_LD + i] = t;
    }
    __syncthreads();
    double cost = 0.0;
    for (int i = tid; i < n; i += SOLVE_THREADS) {
        double t = r0[i];
        for (int p = 0; p < parts; p++) t += part[p * PRIOR_LD + i];
        s.pr[i] = t; cost += 0.5 * t * t;
    }
    __syncthreads();
    return cost;
}

// cost only: 0.5 * sum || S r ||^2 over the valid factors + prior
CERB_NOINLINE double inertial_cost(const SolveParams &P, int w, const double *x, int tid) {
    CERB_DYN_SMEM(double, smem_base);
    Smem s; smem_carve(smem_base, s);
    imu_lin_all(P, s, w, x, false, tid);
    double cost = 0.0;
    for (int idx = tid; idx < CERB_WINDOW * 31; idx += SOLVE_THREADS) {
        const int i = idx / 31, r = idx % 31;
        const double *pre = P.pre + ((size_t)w * CERB_WINDOW + i) * PRE_STRIDE;
        if (pre[PRE_SUM_DT] > 10.0) continue;
        const double *ru = s.lin + 96 * i, *S = P.sinfo + ((size_t)w * CERB_WINDOW + i) * 961;
        double t = 0.0;
        for (int q = r; q < 31; q++) t += S[r * 31 + q] * ru[q];
        cost += 0.5 * t * t;
    }
    return cost + prior_residual(P, s, w, x, tid);
}

// destination of a local IMU-leg tangent column c (0..37) of factor i: x index (>=0) or -(1 + y index)
CERB_D int imu_col_dest(int i, int c) {
    if (c < 6) return 6 * i + c;
    if (c < 19) return -(1 + NYB * i + (c - 6));
    if (c < 25) return 6 * (i + 1) + (c - 19);
    return -(1 + NYB * (i + 1) + (c - 25));
}
// add v to H at (a, b) given destinations in the x / y numbering (a, b come from upper-triangular local order)
// addresses of H(a, b) (a1: the mirrored entry of a diagonal Hyy block, or null)
CERB_D void scatter_addr(const Smem &s, int da, int db, double **a0, double **a1) {
    *a1 = nullptr;
    if (da >= 0 && db >= 0) { *a0 = (da <= db) ? s.Hxx + da * NX + db : s.Hxx + db * NX + da; return; }
    if (da >= 0) { *a0 = s.Hxy + da * NY + (-db - 1); return; }
    if (db >= 0) { *a0 = s.Hxy + db * NY + (-da - 1); return; }
    const int ya = -da - 1, yb = -db - 1;
    const int fa = ya / NYB, fb = yb / NYB, ka = ya % NYB, kb = yb % NYB;
    if (fa == fb) { *a0 = s.Ad + fa * HBLK + ka * NYB + kb; if (ka != kb) *a1 = s.Ad + fa * HBLK + kb * NYB + ka; }
    else if (fb == fa + 1) *a0 = s.Bo + fa * HBLK + ka * NYB + kb;
    else *a0 = s.Bo + fb * HBLK + kb * NYB + ka;
}
CERB_D void scatter_H(Smem &s, int da, int db, double v) {
    if (da >= 0 && db >= 0) { if (da <= db) s.Hxx[da * NX + db] += v; else s.Hxx[db * NX + da] += v; return; }
    if (da >= 0) { s.Hxy[da * NY + (-db - 1)] += v; return; }
    if (db >= 0) { s.Hxy[db * NY + (-da - 1)] += v; return; }
    const int ya = -da - 1, yb = -db - 1;
    const int fa = ya / NYB, fb = yb / NYB, ka = ya % NYB, kb = yb % NYB;
    if (fa == fb) { s.Ad[fa * HBLK + ka * NYB + kb] += v; if (ka != kb) s.Ad[fa * HBLK + kb * NYB + ka] += v; }
    else if (fb == fa + 1) s.Bo[fa * HBLK + ka * NYB + kb] += v;
    else s.Bo[fb * HBLK + kb * NYB + ka] += v;
}

// Inertial linearisation.  Warps 0..2 each run whole IMU-leg factors on their own (warp-synchronous, no block barriers):
//   Ju (unwhitened 31 x 38 tangent Jacobian + residual column, expanded from IMULegLin) -> Jw = S Ju in place -> Gram matrix
//   Jw^T Jw (39 x 39: Hessian blocks, gradient column, cost corner) -> scatter into Hxx / Hxy / Hyy / g.
// Both products are dense contractions (32 x 32 x 40 and 40 x 32 x 40 after padding) on the fp64 tensor cores; the
// upper-triangular S is fetched from HBM/L2 straight into its A-fragment registers (one factor ahead), Ju / Jw live in a
// per-warp [32][44] tile.  Factors that share parameter blocks (i, i + 1) are never in flight together: round r handles
// factors {r, r + 4, r + 8}, rounds are separated by a barrier among the three warps.
// Warps 3..7 meanwhile evaluate the prior (r = r0 + J0 dx, g_prior = J0^T r into a separate vector that is added at the end;
// its constant Hessian is already part of the initial H).
enum { IMU_LDJ = 44, IMU_TILE = 32 * 44, IMU_WARPS = 3, PRIOR_THREADS = SOLVE_THREADS - 32 * IMU_WARPS };
CERB_NOINLINE double inertial_linearize(const SolveParams &P, int w, const double *x, int tid) {
    CERB_DYN_SMEM(double, smem_base);
    Smem s; smem_carve(smem_base, s);
    double cost = 0.0;
    PH_DECL();
    imu_lin_all(P, s, w, x, true, tid);                                  // (the asynchronous copy of the Hxy | Hyy image is in flight)
    PH_MARK(25);
    const int wid = tid >> 5, lane = tid & 31;
    CERB_CP_ASYNC_WAIT();
    double *gp = s.stp;                                                 // prior gradient [NRP]; stp | yv are idle during a linearisation (gn is not:
                                                                        // a rejected speculative linearisation is followed by the dogleg re-use path)
    double *ppart = s.yv;                                               // [2][PRIOR_LD] partial sums of J0 dx
    for (int k = tid; k < NRP; k += SOLVE_THREADS) gp[k] = 0.0;
    __syncthreads();
    if (wid < IMU_WARPS) {
        double *Jt = s.Ju + IMU_TILE * wid;
        // scatter plan of this lane (built once per launch), kept in registers: x = offset(i = 0), y = stride | (mirror delta + 256) << 12
        int plx[30], ply[30];
        {
            const int *plan = ws_carve(P).imu_plan;
            _Pragma("unroll")
            for (int q = 0; q < 30; q++) { plx[q] = __ldg(plan + (2 * q) * 32 + lane); ply[q] = __ldg(plan + (2 * q + 1) * 32 + lane); }
            // entries without a destination share a dummy slot per lane in the plan: give every IMU warp its own (no write-write hazard between warps)
            const int dummy = (int)(s.idg - smem_base) + lane;
            _Pragma("unroll")
            for (int q = 0; q < 30; q++) if (plx[q] == dummy && (ply[q] & 4095) == 0) plx[q] += 32 * wid;
        }
        double sa[20];
        auto load_S = [&](int i) {      // A-fragments of the upper-triangular sqrt_info: block row mi needs k-steps ks >= 2 mi
            const double *S = P.sinfo + ((size_t)w * CERB_WINDOW + i) * 961;
            int q = 0;
            _Pragma("unroll")
            for (int mi = 0; mi < 4; mi++)
                _Pragma("unroll")
                for (int ks = 2 * mi; ks < 8; ks++) {
                    const int r = 8 * mi + (lane >> 2), c = 4 * ks + (lane & 3);
                    sa[q++] = (r < 31 && c < 31 && c >= r) ? S[r * 31 + c] : 0.0;
                }
        };
        load_S(wid * 4);
        const int imu_mask = s.ti[TI_IMU_MASK];                           // 0: all factors (solve); marginalization: 1 only factor 0, 2 none
        double sdt[4];                                                    // sum_dt of this warp's factors, fetched up front
        _Pragma("unroll")
        for (int rnd = 0; rnd < 4; rnd++) { const int i = rnd + 4 * wid; sdt[rnd] = (i < CERB_WINDOW) ? P.pre[((size_t)w * CERB_WINDOW + i) * PRE_STRIDE + PRE_SUM_DT] : 1e30; }
        _Pragma("unroll")
        for (int rnd = 0; rnd < 4; rnd++) {
            const int i = rnd + 4 * wid;
            const double *pre = P.pre + ((size_t)w * CERB_WINDOW + (i < CERB_WINDOW ? i : 0)) * PRE_STRIDE;
            if (i < CERB_WINDOW && !(sdt[rnd] > 10.0) && (imu_mask == 0 || (imu_mask == 1 && i == 0))) {      // estimator.cpp:1119
                // ---- expand Ju ----------------------------------------------------------------------------------------------
                for (int k = lane; k < IMU_TILE; k += 32) Jt[k] = 0.0;
                __syncwarp();
                if (lane < 11) imu_leg_fill_ju_part(*reinterpret_cast<const IMULegLin *>(s.lin + 96 * i), pre, Jt, IMU_LDJ, lane);
                if (lane < 31) Jt[lane * IMU_LDJ + 38] = s.lin[96 * i + lane];          // residual column
                __syncwarp();
                PH_MARK(32);
                // ---- Jw = S Ju, one 8-column block at a time, in place --------------------------------------------------------
                for (int ni = 0; ni < 5; ni++) {
                    double b[8];
                    _Pragma("unroll")
                    for (int ks = 0; ks < 8; ks++) b[ks] = Jt[(4 * ks + (lane & 3)) * IMU_LDJ + 8 * ni + (lane >> 2)];
                    __syncwarp();
                    double c[4][2];
                    int q = 0;
                    _Pragma("unroll")
                    for (int mi = 0; mi < 4; mi++) {
                        c[mi][0] = 0.0; c[mi][1] = 0.0;
                        _Pragma("unroll")
                        for (int ks = 2 * mi; ks < 8; ks++) { CERB_DMMA(c[mi][0], c[mi][1], sa[q], b[ks], c[mi][0], c[mi][1]); q++; }
                    }
                    _Pragma("unroll")
                    for (int mi = 0; mi < 4; mi++) { double *o = Jt + (8 * mi + (lane >> 2)) * IMU_LDJ + 8 * ni + 2 * (lane & 3); o[0] = c[mi][0]; o[1] = c[mi][1]; }
                    __syncwarp();
                }
                PH_MARK(33);
                if (i + 1 < CERB_WINDOW && rnd < 3) load_S(i + 1);         // next round's factor (latency hidden behind the Gram pass)
                // ---- Gram matrix of Jw (40 x 40, 15 upper blocks, K = 32) -----------------------------------------------------------
                double acc[15][2];
                _Pragma("unroll")
                for (int k = 0; k < 15; k++) { acc[k][0] = 0.0; acc[k][1] = 0.0; }
                for (int ks = 0; ks < 8; ks++) {
                    double f[5];
                    _Pragma("unroll")
                    for (int n = 0; n < 5; n++) f[n] = Jt[(4 * ks + (lane & 3)) * IMU_LDJ + 8 * n + (lane >> 2)];
                    int q = 0;
                    _Pragma("unroll")
                    for (int mi = 0; mi < 5; mi++)
                        _Pragma("unroll")
                        for (int ni = mi; ni < 5; ni++) { CERB_DMMA(acc[q][0], acc[q][1], f[mi], f[ni], acc[q][0], acc[q][1]); q++; }
                }
                PH_MARK(34);
                // scatter through the per-lane plan (built once per launch: every destination is affine in the factor index i).  The
                // destinations of a lane (and of different lanes) are distinct, so each half is done as load all / add / store all
                // instead of 15 dependent read-modify-writes.
                // Branch-free and decode-free: entries without a destination (padding, lower triangle, the cost corner) point at a
                // per-lane dummy slot with stride 0; entries without a mirror have delta 0 (second store to the same address).
                if (lane == 27) cost += 0.5 * acc[14][0];                   // (38, 38): 0.5 ||S r||^2 of this factor
                _Pragma("unroll")
                for (int hq = 0; hq < 30; hq += 15) {
                    double cur[15];
                    _Pragma("unroll")
                    for (int t = 0; t < 15; t++) cur[t] = smem_base[plx[hq + t] + i * (ply[hq + t] & 4095)];
                    _Pragma("unroll")
                    for (int t = 0; t < 15; t++) {
                        const int o = plx[hq + t] + i * (ply[hq + t] & 4095);
                        const double nv = cur[t] + acc[(hq + t) >> 1][(hq + t) & 1];
                        smem_base[o] = nv;
                        smem_base[o + (ply[hq + t] >> 12) - 256] = nv;     // mirrored entry of a symmetric diagonal block (or the same address)
                    }
                }
                PH_MARK(35);
            } else if (i + 1 < CERB_WINDOW && rnd < 3) load_S(i + 1);
            CERB_BAR_SYNC(2, 32 * IMU_WARPS);
            PH_MARK(36);                             // factors of the next round touch the blocks of this one
        }
        PH_MARK(30);
    } else {
        // ---- prior: r = r0 + J0 dx, g_prior = J0^T r (threads 96..255) ----------------------------------------------------------------
        const int *meta = P.prior_meta + (size_t)w * PRIOR_META_STRIDE;
        if (meta[0]) {
            const int t5 = tid - 32 * IMU_WARPS, n = meta[1], nb = meta[2];
            const double *J = P.prior_J + (size_t)w * PRIOR_LD * PRIOR_LD, *r0 = P.prior_r + (size_t)w * PRIOR_LD, *x0 = P.prior_x0 + (size_t)w * 16 * 9;
            if (t5 < nb) {
                const int kind = meta[4 + 3 * t5], index = meta[5 + 3 * t5], col = meta[6 + 3 * t5];
                prior_block_dx(kind, x + prior_block_state_offset(kind, index), x0 + 9 * t5, s.pdx + col);
            }
            CERB_BAR_SYNC(3, PRIOR_THREADS);
            const int kc = (n + 1) / 2;
            for (int e = t5; e < 2 * n; e += PRIOR_THREADS) {
                const int p = e / n, i = e % n;
                const int k1 = (p + 1) * kc < n ? (p + 1) * kc : n;
                double t = 0.0;
                for (int k = p * kc; k < k1; k++) t += J[(size_t)k * n + i] * s.pdx[k];
                ppart[p * PRIOR_LD + i] = t;
            }
            CERB_BAR_SYNC(3, PRIOR_THREADS);
            for (int i = t5; i < n; i += PRIOR_THREADS) {
                const double t = (r0[i] + ppart[i]) + ppart[PRIOR_LD + i];
                s.pr[i] = t; cost += 0.5 * t * t;
            }
            CERB_BAR_SYNC(3, PRIOR_THREADS);
            // one warp per column of J0 (contiguous, coalesced), lanes stride the rows, fixed-order shuffle reduction
            for (int c = wid - IMU_WARPS; c < n; c += PRIOR_THREADS / 32) {
                double t = 0.0;
                for (int k = lane; k < n; k += 32) t += J[(size_t)c * n + k] * s.pr[k];
                for (int o = 16; o > 0; o >>= 1) t += __shfl_sync(0xffffffffu, t, (lane + o) & 31);
                const int d = s.ti[TI_PRIOR_MAP + c];                  // the kept blocks tile all n columns (validate_prior)
                if (lane == 0) gp[d >= 0 ? d : NX + (-d - 1)] += t;
            }
        }
        PH_MARK_T(31, 96);
    }
    __syncthreads();
    PH_MARK(26);
    for (int k = tid; k < NR; k += SOLVE_THREADS) s.g[k] += gp[k];
    __syncthreads();
    PH_MARK(27);
    return cost;
}

// x [+] delta -> xc ; lam + dlam -> lamc
CERB_D void apply_plus(const Smem &s, const double *delta, const double *lam, const double *dlam, double *lamc, int nF, bool ex_open, bool td_open, int tid) {
    if (tid < 11) pose_plus(s.xs + ST_POSE + 7 * tid, delta + 6 * tid, s.xc + ST_POSE + 7 * tid);
    else if (tid < 13) {
        const int e = tid - 11;
        if (ex_open) pose_plus(s.xs + ST_EX + 7 * e, delta + 66 + 6 * e, s.xc + ST_EX + 7 * e);
        else for (int k = 0; k < 7; k++) s.xc[ST_EX + 7 * e + k] = s.xs[ST_EX + 7 * e + k];     // constant block: bit-exact copy
    }
    for (int k = tid; k < 99; k += SOLVE_THREADS) { const int f = k / 9, c = k % 9; s.xc[ST_SB + k] = s.xs[ST_SB + k] + delta[NX + NYB * f + c]; }
    for (int k = tid; k < 44; k += SOLVE_THREADS) { const int f = k / 4, c = k % 4; s.xc[ST_LB + k] = s.xs[ST_LB + k] + delta[NX + NYB * f + 9 + c]; }
    if (tid == 0) s.xc[ST_TD] = td_open ? s.xs[ST_TD] + delta[X_TD] : s.xs[ST_TD];
    for (int f = tid; f < nF; f += SOLVE_THREADS) lamc[f] = lam[f] + dlam[f];
    __syncthreads();
}

// ambient squared norm of the active parameter blocks of `a` (or of a - b if b != null)
CERB_D double ambient_sq(const double *a, const double *b, const double *la, const double *lb, int nF, bool ex_open, bool lb_open, bool td_open, int tid) {
    double t = 0.0;
    for (int k = tid; k < ST_SIZE; k += SOLVE_THREADS) {
        if (k >= ST_LB && k < ST_EX && !lb_open) continue;
        if (k >= ST_EX && k < ST_TD && !ex_open) continue;
        if (k == ST_TD && !td_open) continue;
        const double v = b ? a[k] - b[k] : a[k];
        t += v * v;
    }
    for (int f = tid; f < nF; f += SOLVE_THREADS) { const double v = lb ? la[f] - lb[f] : la[f]; t += v * v; }
    return t;
}

// t +/- w_f . v for the column w_f = W[0..NX)[f] of the L2-resident W (pointer to W[0][f], row stride F), accumulated in row order.  The loads
// of a batch of rows are all issued before its first FMA: written as one loop, the body was compiled as load, FMA, load, ... (the next load
// re-used the register of the FMA operand), one L2 round trip per row -- 79 in a row for every feature.
template <bool SUB>
CERB_D double w_column_dot(const double *wf, int F, const double *v, double t) {
    constexpr int BATCH = 16;
    for (int a0 = 0; a0 < NX; a0 += BATCH) {
        double wr[BATCH];
        _Pragma("unroll")
        for (int u = 0; u < BATCH; u++) wr[u] = (a0 + u < NX) ? wf[(size_t)(a0 + u) * F] : 0.0;
        _Pragma("unroll")
        for (int u = 0; u < BATCH; u++) {
            if (a0 + u < NX) { if (SUB) t -= wr[u] * v[a0 + u]; else t += wr[u] * v[a0 + u]; }
        }
    }
    return t;
}

// ---- S' = S - T T^T for one warp (see the call site).  The 55 upper 8 x 8 blocks of the 80 x 80 Gram matrix of [T; gy'^T] are dealt to
// the 8 warps as rectangles of the block grid, so that a warp's 6-7 blocks share 4-7 fragment rows: 40 fragment loads per k-step
// and CTA instead of 110 (the row stride of T, 143 doubles, makes every fragment load a 4-way bank conflict, and the loop was bound
// by exactly that).  TT_ROWS: distinct block rows of warp W; TT_A / TT_B: the two block rows of each of its blocks (indices into
// TT_ROWS); everything is compile-time so that the fragments stay in registers.
template <int W> struct TTPlan;
#define CERB_TT_PLAN(W, NR_, NB_, ...) template <> struct TTPlan<W> { static constexpr int nr = NR_, nb = NB_; static CERB_HD int tab(int i) { constexpr int t[] = {__VA_ARGS__}; return t[i]; } };
//            rows (padded to 7)           block -> first row index      block -> second row index
CERB_TT_PLAN(0, 4, 7, 0, 1, 2, 3, 0, 0, 0,   0, 0, 1, 0, 1, 0, 1,   0, 1, 1, 2, 2, 3, 3)
CERB_TT_PLAN(1, 4, 7, 2, 3, 4, 5, 0, 0, 0,   0, 0, 1, 0, 1, 0, 1,   0, 1, 1, 2, 2, 3, 3)
CERB_TT_PLAN(2, 4, 7, 4, 5, 6, 7, 0, 0, 0,   0, 0, 1, 0, 1, 0, 1,   0, 1, 1, 2, 2, 3, 3)
CERB_TT_PLAN(3, 4, 7, 6, 7, 8, 9, 0, 0, 0,   0, 0, 1, 0, 1, 0, 1,   0, 1, 1, 2, 2, 3, 3)
CERB_TT_PLAN(4, 6, 7, 8, 9, 0, 1, 4, 5, 0,   0, 0, 1, 2, 3, 2, 3,   0, 1, 1, 4, 4, 5, 5)
CERB_TT_PLAN(5, 6, 7, 0, 1, 6, 7, 8, 9, 0,   0, 0, 0, 0, 1, 1, 1,   2, 3, 4, 5, 2, 3, 4)
CERB_TT_PLAN(6, 7, 7, 1, 9, 2, 6, 7, 8, 3,   0, 2, 2, 2, 2, 6, 6,   1, 3, 4, 5, 1, 3, 4)
CERB_TT_PLAN(7, 5, 6, 3, 4, 5, 8, 9, 0, 0,   0, 0, 1, 1, 2, 2, 0,   3, 4, 3, 4, 3, 4, 0)
template <int W> CERB_D void ttt_warp(Smem &s, int lane) {
    typedef TTPlan<W> PL;
    const double *pr[7];
    _Pragma("unroll")
    for (int u = 0; u < 7; u++) {
        const int r = 8 * PL::tab(u < PL::nr ? u : 0) + (lane >> 2);
        pr[u] = (r < NX ? s.Hxy + r * NY : s.yv + NX) + (lane & 3);      // rows 0..78 of T, row 79 = gy'
    }
    double acc[7][2], fv[7];
    _Pragma("unroll")
    for (int k = 0; k < 7; k++) { acc[k][0] = 0.0; acc[k][1] = 0.0; }
    _Pragma("unroll")
    for (int u = 0; u < 7; u++) fv[u] = (u < PL::nr) ? pr[u][0] : 0.0;
    for (int q0 = 0; q0 < NY; q0 += 4) {
        const int qn = q0 + 4;
        const bool take = qn < NY && qn + (lane & 3) < NY;                   // the last k-step holds 3 valid columns (K = 143)
        double fn[7];
        _Pragma("unroll")
        for (int u = 0; u < 7; u++) fn[u] = (u < PL::nr && take) ? pr[u][qn] : 0.0;
        _Pragma("unroll")
        for (int k = 0; k < 7; k++) if (k < PL::nb) CERB_DMMA(acc[k][0], acc[k][1], fv[PL::tab(7 + k)], fv[PL::tab(14 + k)], acc[k][0], acc[k][1]);
        _Pragma("unroll")
        for (int u = 0; u < 7; u++) fv[u] = fn[u];
    }
    _Pragma("unroll")
    for (int k = 0; k < 7; k++) {
        if (k >= PL::nb) continue;
        const int ba = PL::tab(PL::tab(7 + k)), bb = PL::tab(PL::tab(14 + k));        // block rows (ba <= bb)
        const int a = 8 * ba + (lane >> 2);
        for (int e = 0; e < 2; e++) {
            const int b = 8 * bb + 2 * (lane & 3) + e;
            if (a > b || a >= NX || b > NX) continue;
            if (b == NX) s.yv[a] -= acc[k][e];
            else s.Hxx[b * NX + a] -= acc[k][e];
        }
    }
}

// ---- inverse-depth elimination S -= W' W'^T on the tensor cores: the 55 upper 8 x 8 blocks of the 80 x 80 Gram matrix of a staged 80 x 32 tile,
// dealt to the seven warps 1..7 as row strips (8 blocks each, 7 for the last) so that a warp needs at most nine 8-row fragments per k-step.
// Everything is compile-time (like TTPlan): the fragments of a k-step sit in DISTINCT registers and the DMMAs issue back to back -- with a
// run-time block table ptxas re-used one register pair for the operands of all blocks and every DMMA waited for its own two LDS (~119 cycles
// per DMMA instead of 16 - 32, measured with the phase timers).
template <int W> struct SCPlan;
#define CERB_SC_PLAN(W, NR_, NB_, ...) template <> struct SCPlan<W> { static constexpr int nr = NR_, nb = NB_; static CERB_HD int tab(int i) { constexpr int t[] = {__VA_ARGS__}; return t[i]; } };
//            block rows (padded to 9)          block -> first row index     block -> second row index
CERB_SC_PLAN(0, 8, 8, 0, 1, 2, 3, 4, 5, 6, 7, 0,   0, 0, 0, 0, 0, 0, 0, 0,   0, 1, 2, 3, 4, 5, 6, 7)      // (0,0) .. (0,7)
CERB_SC_PLAN(1, 9, 8, 0, 8, 9, 1, 2, 3, 4, 5, 6,   0, 0, 3, 3, 3, 3, 3, 3,   1, 2, 3, 4, 5, 6, 7, 8)      // (0,8) (0,9) (1,1) .. (1,6)
CERB_SC_PLAN(2, 9, 8, 1, 7, 8, 9, 2, 3, 4, 5, 6,   0, 0, 0, 4, 4, 4, 4, 4,   1, 2, 3, 4, 5, 6, 7, 8)      // (1,7) .. (1,9) (2,2) .. (2,6)
CERB_SC_PLAN(3, 8, 8, 2, 7, 8, 9, 3, 4, 5, 6, 0,   0, 0, 0, 4, 4, 4, 4, 4,   1, 2, 3, 4, 5, 6, 7, 1)      // (2,7) .. (2,9) (3,3) .. (3,7)
CERB_SC_PLAN(4, 7, 8, 3, 8, 9, 4, 5, 6, 7, 0, 0,   0, 0, 3, 3, 3, 3, 3, 3,   1, 2, 3, 4, 5, 6, 1, 2)      // (3,8) (3,9) (4,4) .. (4,9)
CERB_SC_PLAN(5, 5, 8, 5, 6, 7, 8, 9, 0, 0, 0, 0,   0, 0, 0, 0, 0, 1, 1, 1,   0, 1, 2, 3, 4, 1, 2, 3)      // (5,5) .. (5,9) (6,6) .. (6,8)
CERB_SC_PLAN(6, 4, 7, 6, 7, 8, 9, 0, 0, 0, 0, 0,   0, 1, 1, 1, 2, 2, 3, 0,   3, 1, 2, 3, 2, 3, 3, 0)      // (6,9) (7,7) .. (7,9) (8,8) (8,9) (9,9)
enum { SC_LDW = 36 };
template <int W> CERB_D void schur_tile(const double *tw, double (&acc)[8][2], int lane) {
    typedef SCPlan<W> PL;
    const double *pr[9];
    _Pragma("unroll")
    for (int u = 0; u < 9; u++) pr[u] = tw + (8 * PL::tab(u < PL::nr ? u : 0) + (lane >> 2)) * SC_LDW + (lane & 3);
    double fv[9];
    _Pragma("unroll")
    for (int u = 0; u < 9; u++) fv[u] = (u < PL::nr) ? pr[u][0] : 0.0;
    _Pragma("unroll")
    for (int ks = 0; ks < 8; ks++) {
        double fn[9];
        _Pragma("unroll")
        for (int u = 0; u < 9; u++) fn[u] = (u < PL::nr && ks < 7) ? pr[u][4 * (ks + 1)] : 0.0;      // operands one k-step ahead
        _Pragma("unroll")
        for (int k = 0; k < 8; k++) if (k < PL::nb) CERB_DMMA(acc[k][0], acc[k][1], fv[PL::tab(9 + k)], fv[PL::tab(17 + k)], acc[k][0], acc[k][1]);
        _Pragma("unroll")
        for (int u = 0; u < 9; u++) fv[u] = fn[u];
    }
}
template <int W> CERB_D void schur_scatter(Smem &s, const double (&acc)[8][2], int lane) {
    typedef SCPlan<W> PL;
    _Pragma("unroll")
    for (int k = 0; k < 8; k++) {
        if (k >= PL::nb) continue;
        const int a = 8 * PL::tab(PL::tab(9 + k)) + (lane >> 2);
        for (int e = 0; e < 2; e++) {
            const int b = 8 * PL::tab(PL::tab(17 + k)) + 2 * (lane & 3) + e;
            if (a > b || a >= NX || b > NX) continue;
            if (b == NX) s.yv[a] -= acc[k][e];            // rhs_x
            else { s.Hxx[b * NX + a] -= acc[k][e]; if (a != b) s.Hxx[a * NX + b] -= acc[k][e]; }
        }
    }
}

// prior Hessian image (J0^T J0 scattered into the layout of Hxx | Hxy | Ad | Bo) in global memory: constant during the solve, every linearisation
// starts from it instead of from zero; + the column -> destination map of the prior in s.ti[TI_PRIOR_MAP + 0..n); returns whether the window has a prior
CERB_D bool build_prior_image(const SolveParams &P, Smem &s, int w, double *pimg, int tid) {
    const int *pmeta = P.prior_meta + (size_t)w * PRIOR_META_STRIDE;
    const bool has_prior = pmeta[0] != 0;
    if (has_prior) {
        const int n = pmeta[1], nb = pmeta[2];
        for (int k = tid; k < PIMG_SZ; k += SOLVE_THREADS) pimg[k] = 0.0;
        if (tid < nb) {
            const int kind = pmeta[4 + 3 * tid], index = pmeta[5 + 3 * tid], col = pmeta[6 + 3 * tid];
            const int local = (kind == 0 || kind == 3) ? 6 : prior_block_size(kind);
            for (int k = 0; k < local; k++) {
                int d;
                if (kind == 0) d = 6 * index + k;
                else if (kind == 3) d = 66 + 6 * index + k;
                else if (kind == 1) d = -(1 + NYB * index + k);
                else if (kind == 2) d = -(1 + NYB * index + 9 + k);
                else d = X_TD;
                s.ti[TI_PRIOR_MAP + col + k] = d;
            }
        }
        __syncthreads();
        Smem si = s; si.Hxx = pimg; si.Hxy = pimg + PIMG_HXY; si.Ad = pimg + PIMG_HXY + HXY_SZ; si.Bo = pimg + PIMG_HXY + HXY_SZ + AD_SZ;
        const double *Hp = P.prior_Hp + (size_t)w * PRIOR_LD * PRIOR_LD;
        for (int idx = tid; idx < n * n; idx += SOLVE_THREADS) {
            const int a = idx / n, b = idx % n;
            if (b < a) continue;
            scatter_H(si, s.ti[TI_PRIOR_MAP + a], s.ti[TI_PRIOR_MAP + b], Hp[a * PRIOR_LD + b]);
        }
    }
    return has_prior;
}

// ---- the prologue both kernels share ----------------------------------------------------------------------------
// Scatter plan of the 40 x 40 IMU-leg Gram matrix (inertial_linearize), built by warp 0 once per launch: lane `tid` holds, for block
// q = (mi, ni) and e = 0, 1, the entry (la, lb) = (8 mi + lane / 4, 8 ni + 2 (lane % 4) + e).  Its destination in Hxx / Hxy / Hyy / g is
// affine in the factor index i, so the plan stores two ints: offset(i = 0) and stride | (mirror delta + 256) << 12 (in doubles
// from the start of shared memory; the mirror is the transposed entry of a diagonal Hyy block).  Entries without a destination
// point at a per-lane dummy slot (idg[32 warp + lane], never read) with stride 0.
CERB_D void build_imu_plan(const Smem &s, const double *smem_base, int *plan, int tid) {
    if (tid >= 32) return;
    int q = 0;
    for (int mi = 0; mi < 5; mi++)
        for (int ni = mi; ni < 5; ni++, q++)
            for (int e = 0; e < 2; e++) {
                const int la = 8 * mi + (tid >> 2), lb = 8 * ni + 2 * (tid & 3) + e;
                int px = (int)(s.idg - smem_base) + tid, py = 256 << 12;         // default: dummy slot of this lane (idg is idle during a linearisation; each IMU warp adds 32 x its index), stride 0, delta 0
                if (la <= lb && lb <= 38 && la != 38) {
                    double *p0[2], *p1[2];
                    for (int i = 0; i < 2; i++) {
                        const int da = imu_col_dest(i, la);
                        if (lb == 38) { p0[i] = da >= 0 ? s.g + da : s.g + NX + (-da - 1); p1[i] = nullptr; }
                        else scatter_addr(s, da, imu_col_dest(i, lb), &p0[i], &p1[i]);
                    }
                    px = (int)(p0[0] - smem_base);
                    py = (int)(p0[1] - p0[0]) | (((p1[0] ? (int)(p1[0] - p0[0]) : 0) + 256) << 12);
                }
                plan[(2 * (q * 2 + e)) * 32 + tid] = px; plan[(2 * (q * 2 + e) + 1) * 32 + tid] = py;
            }
}
// feature chunks of the tracks [0, n_end) (anchor frames fstart) for vision_linearize (one thread): <= 64 consecutive tracks with the same anchor frame
CERB_D void build_chunks(const int *fstart, Smem &s, int *chunks, int n_end) {
    int n = 0, c0 = 0;
    while (c0 < n_end) {
        chunks[1 + n] = c0;
        const int a = fstart[c0];
        int e = c0 + 1;
        while (e < n_end && e < c0 + 64 && fstart[e] == a) e++;
        if (n < TI_CACHED_CHUNKS) { s.ti[TI_CHUNK_CACHE + 2 * n] = c0; s.ti[TI_CHUNK_CACHE + 2 * n + 1] = ((e - c0) << 8) | a; }   // also cached in shared memory
        n++; c0 = e;
    }
    chunks[1 + n] = n_end; chunks[0] = n; s.ti[TI_NCHUNKS] = n;
}
// ---- the solve kernel: the window of a CTA and the phases of one trust-region iteration ---------------------------
struct Win { int w, nF; bool ex_open, lb_open, td_open, has_prior, bulk_ok; double *lam; CtaWs ws; };     // lam: inverse depths of the current point
struct PriorCopy { unsigned par0, par1; bool hxx_prefetched; };    // prior-image copies: parities of the two bulk-copy mbarriers, Hxx part in flight
// linearisation at (xl, laml): H, g (Jacobi scaled), W, hh, gl; results S_LCOST (cost), S_LNORM (||x||), S_LGMAX (max |g|)
CERB_D void linearize(const SolveParams &P, Smem &s, const Win &c, PriorCopy &pc, const double *xl, const double *laml, bool first, int tid PH_ARG) {
    const int F = c.ws.F, nF = c.nF;
    double *sca = s.sca, *W = c.ws.W, *hh = c.ws.hh, *gl = c.ws.gl, *sl = c.ws.sl, *pimg = c.ws.pimg;
    // start from the prior Hessian image; its Hxx part was prefetched asynchronously when the previous factorisation of
    // Hxx had been consumed (the copy overlapped with the rest of that iteration), except for the first linearisation
    if (!c.has_prior) { for (int k = tid; k < HXX_SZ; k += SOLVE_THREADS) s.Hxx[k] = 0.0; }
    else if (c.bulk_ok) {
        if (!pc.hxx_prefetched) { __syncthreads(); if (tid == 0) CERB_BULK_G2S(s.Hxx, pimg, PIMG_HXY * 8, &s.mbar[0]); }
        CERB_MBAR_WAIT(&s.mbar[0], pc.par0); pc.par0 ^= 1;
    } else { if (!pc.hxx_prefetched) copy_g2s_async(s.Hxx, pimg, HXX_SZ, tid); CERB_CP_ASYNC_WAIT(); }
    pc.hxx_prefetched = false;
    for (int k = tid; k < NRP; k += SOLVE_THREADS) s.g[k] = 0.0;
    load_geometry(xl, s, tid);
    double part[2];
    PH_MARK(0);
    part[0] = vision_linearize(P, c.w, xl, laml, W, hh, gl, sl, !first, c.ws.chunks, tid);
    if (c.has_prior && c.bulk_ok) {                                                              // Hxy | Ad | Bo (contiguous; the tile aliased them):
        if (tid == 0) CERB_BULK_G2S(s.Hxy, pimg + PIMG_HXY, PIMG_REST * 8, &s.mbar[1]);            // one bulk copy (vision_linearize ended with a barrier)
        CERB_MBAR_WAIT(&s.mbar[1], pc.par1); pc.par1 ^= 1;
    } else if (c.has_prior) copy_g2s_async(s.Hxy, pimg + PIMG_HXY, PIMG_REST, tid);               // completed inside inertial_linearize
    else for (int k = tid; k < PIMG_REST; k += SOLVE_THREADS) s.Hxy[k] = 0.0;
    __syncthreads();
    PH_MARK(1);
    part[0] += inertial_linearize(P, c.w, xl, tid);
    PH_MARK(2);
    part[1] = ambient_sq(xl, nullptr, laml, nullptr, nF, c.ex_open, c.lb_open, c.td_open, tid);
    double tot[2];
    block_sum<2>(part, s.red, tot, tid);
    if (tid == 0) { sca[S_LCOST] = tot[0]; sca[S_LNORM] = sqrt(tot[1]); }
    // (Hxx holds its upper triangle; it is mirrored and scaled in one row-wise pass below)
    // gradient max norm over active dims (unscaled), Jacobi scale at the first linearisation
    if (first) {
        for (int k = tid; k < NR; k += SOLVE_THREADS) {
            double d;
            bool active = true;
            if (k < NX) { d = s.Hxx[k * NX + k]; if (k >= 66 && k < X_TD && !c.ex_open) active = false; if (k == X_TD && !c.td_open) active = false; }
            else { const int yk = k - NX, f = yk / NYB, q = yk % NYB; d = s.Ad[f * HBLK + q * NYB + q]; if (q >= 9 && !c.lb_open) active = false; }
            s.sc[k] = active ? 1.0 / (1.0 + sqrt(d)) : 0.0;
        }
        for (int f = tid; f < nF; f += SOLVE_THREADS) sl[f] = 1.0 / (1.0 + sqrt(hh[f]));
    }
    __syncthreads();
    if (P.dbg && c.w == P.dbg_window && first) {      // parity probe, ABI order
        for (int k = tid; k < NR; k += SOLVE_THREADS) {
            int dst; double d;
            if (k < NX) { dst = k < X_TD ? k : 221; d = s.Hxx[k * NX + k]; }      // ABI order: td after the leg biases
            else { const int yk = k - NX, f = yk / NYB, q = yk % NYB; dst = q < 9 ? 78 + 9 * f + q : 177 + 4 * f + (q - 9); d = s.Ad[f * HBLK + q * NYB + q]; }
            const bool act = s.sc[k] != 0.0;
            P.dbg[1 + dst] = act ? s.g[k] : 0.0; P.dbg[1 + NR + F + dst] = act ? d : 0.0;
        }
        for (int f = tid; f < nF; f += SOLVE_THREADS) { P.dbg[1 + NR + f] = gl[f]; P.dbg[1 + NR + F + NR + f] = hh[f]; }
        if (tid == 0) P.dbg[0] = sca[S_LCOST];
    }
    double gm = 0.0;
    for (int k = tid; k < NR; k += SOLVE_THREADS) if (s.sc[k] != 0.0) gm = fmax(gm, fabs(s.g[k]));
    for (int f = tid; f < nF; f += SOLVE_THREADS) gm = fmax(gm, fabs(!first ? gl[f] / sl[f] : gl[f]));   // unscaled gradient
    for (int o = 16; o > 0; o >>= 1) gm = fmax(gm, __shfl_sync(0xffffffffu, gm, (tid + o) & 31));
    if ((tid & 31) == 0) s.red[tid >> 5] = gm;
    __syncthreads();
    if (tid == 0) { double m8 = s.red[0]; for (int k = 1; k < SOLVE_THREADS / 32; k++) m8 = fmax(m8, s.red[k]); sca[S_LGMAX] = m8; }
    // apply the Jacobi scaling: H~ = S H S, g~ = S g, w~_f = s_f S_x w_f, h~ = s_f^2 h, gl~ = s_f gl.  Row-wise (a warp per
    // row: no index divisions); the Hxx pass also mirrors the upper triangle into the lower one.
    for (int a = tid >> 5; a < NX; a += SOLVE_THREADS / 32) {
        const double sa = s.sc[a];
        for (int b = a + (tid & 31); b < NX; b += 32) { const double v = s.Hxx[a * NX + b] * (sa * s.sc[b]); s.Hxx[a * NX + b] = v; s.Hxx[b * NX + a] = v; }
        for (int q = tid & 31; q < NY; q += 32) s.Hxy[a * NY + q] *= sa * s.sc[NX + q];
    }
    for (int k = tid; k < AD_SZ; k += SOLVE_THREADS) { const int f = k / HBLK, a = (k % HBLK) / NYB, b = k % NYB; s.Ad[k] *= s.sc[NX + NYB * f + a] * s.sc[NX + NYB * f + b]; }
    for (int k = tid; k < BO_SZ; k += SOLVE_THREADS) { const int f = k / HBLK, a = (k % HBLK) / NYB, b = k % NYB; s.Bo[k] *= s.sc[NX + NYB * f + a] * s.sc[NX + NYB * (f + 1) + b]; }
    for (int k = tid; k < NR; k += SOLVE_THREADS) s.g[k] *= s.sc[k];
    if (first) {      // later linearisations write W, hh, gl pre-scaled
        for (int k = tid; k < NX * nF; k += SOLVE_THREADS) { const int a = k / nF, f = k % nF; W[(size_t)a * F + f] *= s.sc[a] * sl[f]; }
        for (int f = tid; f < nF; f += SOLVE_THREADS) { hh[f] *= sl[f] * sl[f]; gl[f] *= sl[f]; }
    }
    __syncthreads();
}
// FinalizeIterationAndCheckIfMinimizerCanContinue; true: the minimizer stops
CERB_D bool finalize_iteration(const SolveParams &P, double *sca, int iteration, int tid) {
    if (tid == 0) {
        if (iteration >= P.max_iters) { sca[S_DONE] = 1; sca[S_TERM] = 1; }
        else if (sca[S_GMAX] <= P.gtol) { sca[S_DONE] = 1; sca[S_TERM] = 0; }
        else if (sca[S_RADIUS] <= P.min_radius) { sca[S_DONE] = 1; sca[S_TERM] = 0; }
        else if (!(sca[S_XCOST] == sca[S_XCOST]) || fabs(sca[S_XCOST]) > 1e300) { sca[S_DONE] = 1; sca[S_TERM] = 2; }
    }
    __syncthreads();
    return sca[S_DONE] != 0.0;
}
// dogleg diagonal D, gradient / D, scaled gradient v (kept in s.stp: the Cauchy point's v^T H v is finished in lambda_schur);
// ||gh||^2 and the Hyy part of v^T H v (Hyy is about to be factored in place)
CERB_D void dogleg_diagonal(Smem &s, const Win &c, int tid PH_ARG) {
    const int nF = c.nF;
    double *sca = s.sca, *Dl = c.ws.Dl, *ghl = c.ws.ghl, *stl = c.ws.stl;
    for (int k = tid; k < NR; k += SOLVE_THREADS) {
        const double d = (k < NX) ? s.Hxx[k * NX + k] : s.Ad[((k - NX) / NYB) * HBLK + ((k - NX) % NYB) * (NYB + 1)];
        const double D = sqrt(fmin(fmax(d, 1e-6), 1e32));
        s.D[k] = D; s.gh[k] = s.g[k] / D; s.stp[k] = s.gh[k] / D;
    }
    for (int f = tid; f < nF; f += SOLVE_THREADS) { const double D = sqrt(fmin(fmax(c.ws.hh[f], 1e-6), 1e32)); Dl[f] = D; ghl[f] = c.ws.gl[f] / D; stl[f] = ghl[f] / D; }
    __syncthreads();
    double part[2] = {0.0, 0.0};     // [0] v_y^T Hyy v_y  [1] ||gh||^2
    for (int k = tid; k < AD_SZ; k += SOLVE_THREADS) { const int f = k / HBLK, a = (k % HBLK) / NYB, b = k % NYB; part[0] += s.stp[NX + NYB * f + a] * s.Ad[k] * s.stp[NX + NYB * f + b]; }
    for (int k = tid; k < BO_SZ; k += SOLVE_THREADS) { const int f = k / HBLK, a = (k % HBLK) / NYB, b = k % NYB; part[0] += 2.0 * s.stp[NX + NYB * f + a] * s.Bo[k] * s.stp[NX + NYB * (f + 1) + b]; }
    for (int f = tid; f < nF; f += SOLVE_THREADS) part[1] += ghl[f] * ghl[f];
    for (int k = tid; k < NR; k += SOLVE_THREADS) part[1] += s.gh[k] * s.gh[k];
    double tot[2];
    block_sum<2>(part, s.red, tot, tid);
    if (tid == 0) { sca[S_GNORM2] = tot[1]; sca[S_VHV] = tot[0]; sca[S_OK] = 1; }      // S_OK: a failure below is an invalid step: mu *= 10, re-linearise
    PH_MARK(4);
}
// warp 0: block-bidiagonal Cholesky of Hyy: Ad[f] <- L_f (lower), Bo[f] <- M_f = B_f^T L_f^-T.  Lane r owns row r of the 13 x 13 block in
// registers; the column sweep exchanges pivots and column entries with shuffles (no shared-memory round trips on the dependency chain).
// Every finished block f is published through chain_done = f + 1.
CERB_D void chain_cholesky(Smem &s, int *chain_done, int lane PH_ARG) {
    const bool act = lane < NYB;
    const int r = act ? lane : 0;              // idle lanes shadow row 0 and never store
    double m[NYB];                             // row r of M_{f-1}
    _Pragma("unroll")
    for (int c = 0; c < NYB; c++) m[c] = 0.0;
    _Pragma("unroll 1")                        // keep the block body compact: it is re-used 11 times from the instruction cache
    for (int f = 0; f < NFR; f++) {
        double *A = s.Ad + f * HBLK;
        double a[NYB], invd[NYB], myinv = 1.0;
        _Pragma("unroll")
        for (int c = 0; c < NYB; c++) a[c] = A[r * NYB + c];
        if (f > 0) {
            const double *Mp = s.Bo + (f - 1) * HBLK;        // M[r][c], r: y_f index, c: y_{f-1} index
            _Pragma("unroll")
            for (int c = 0; c < NYB; c++) { double t = 0.0; _Pragma("unroll") for (int q = 0; q < NYB; q++) t += m[q] * Mp[c * NYB + q]; a[c] -= t; }
        }
        _Pragma("unroll")
        for (int j = 0; j < NYB; j++) {                     // right-looking column sweep
            double d = __shfl_sync(0xffffffffu, a[j], j);
            if (!(d > 0.0)) { if (lane == 0) s.sca[S_OK] = 0; d = 1.0; }
            const double inv = rsqrt(d);
            invd[j] = inv;
            if (lane == j) myinv = inv;
            const double l = (lane == j) ? d * inv : a[j] * inv;
            a[j] = l;
            // column j of L to all lanes through a double-buffered shared-memory line (1 store + 12 broadcast loads
            // instead of 12 two-instruction shuffles: the sweep is bound by the instruction issue of this one warp)
            double *colb = s.chain_col + 16 * (j & 1);
            if (act) colb[lane] = l;
            __syncwarp();
            _Pragma("unroll")
            for (int k = j + 1; k < NYB; k++) a[k] -= l * colb[k];
        }
        if (act) { _Pragma("unroll") for (int c = 0; c < NYB; c++) if (c <= r) A[r * NYB + c] = a[c]; s.idg[NYB * f + r] = myinv; }
        __syncwarp();
        if (f < NFR - 1) {
            double *B = s.Bo + f * HBLK;                     // in: B[k1][k2] = H(y_f[k1], y_{f+1}[k2]); out: M[r][c]
            double t[NYB];
            _Pragma("unroll")
            for (int c = 0; c < NYB; c++) t[c] = B[c * NYB + r];
            _Pragma("unroll")
            for (int c = 0; c < NYB; c++) {
                m[c] = t[c] * invd[c];
                _Pragma("unroll")
                for (int c2 = c + 1; c2 < NYB; c2++) t[c2] -= m[c] * A[c2 * NYB + c];
            }
            __syncwarp();
            if (act) { _Pragma("unroll") for (int c = 0; c < NYB; c++) B[r * NYB + c] = m[c]; }
            __syncwarp();
        }
        __threadfence_block(); __syncwarp();
        if (lane == 0) CERB_ST_RELEASE_S32(chain_done, f + 1);   // L_f, M_f and the inverse pivots of block f are in shared memory
    }
    PH_MARK(6);
}
// warp-uniform dispatch to the compile-time block plans (SCPlan, TTPlan)
CERB_D void schur_tile_w(int wq, const double *tw, double (&acc)[8][2], int lane) {
    switch (wq) { case 0: schur_tile<0>(tw, acc, lane); break; case 1: schur_tile<1>(tw, acc, lane); break; case 2: schur_tile<2>(tw, acc, lane); break;
                  case 3: schur_tile<3>(tw, acc, lane); break; case 4: schur_tile<4>(tw, acc, lane); break; case 5: schur_tile<5>(tw, acc, lane); break;
                  default: schur_tile<6>(tw, acc, lane); break; }
}
CERB_D void schur_scatter_w(int wq, Smem &s, const double (&acc)[8][2], int lane) {
    switch (wq) { case 0: schur_scatter<0>(s, acc, lane); break; case 1: schur_scatter<1>(s, acc, lane); break; case 2: schur_scatter<2>(s, acc, lane); break;
                  case 3: schur_scatter<3>(s, acc, lane); break; case 4: schur_scatter<4>(s, acc, lane); break; case 5: schur_scatter<5>(s, acc, lane); break;
                  default: schur_scatter<6>(s, acc, lane); break; }
}
CERB_D void ttt_warp_w(int wq, Smem &s, int lane) {
    switch (wq) { case 0: ttt_warp<0>(s, lane); break; case 1: ttt_warp<1>(s, lane); break; case 2: ttt_warp<2>(s, lane); break; case 3: ttt_warp<3>(s, lane); break;
                  case 4: ttt_warp<4>(s, lane); break; case 5: ttt_warp<5>(s, lane); break; case 6: ttt_warp<6>(s, lane); break; default: ttt_warp<7>(s, lane); break; }
}
// warps 1..7: the Cauchy point's v_x^T Hxx v_x + 2 v_x^T Hxy v_y + lambda terms (into s.lin[0..7)), the mu-regularised diagonal of Hxx,
// then the inverse depths are eliminated on the fp64 tensor cores:
//   S = Hxx - W' W'^T,  rhs_x -= W' (w g_l),  W'[a][f] = W[a][f] / sqrt(h_f + mu D_f^2)
// W' is staged through shared memory 32 features at a time as an 80-row tile whose row 78 carries
// g_l / sqrt(h + mu D^2) (so that column 78 of the Gram matrix is the rhs update) and row 79 is zero.
// The 55 upper 8x8 blocks of the 80x80 Gram matrix go to the 7 warps as row strips (SCPlan, compile-time).
CERB_D void lambda_schur(Smem &s, const CtaWs &ws, int nF, double mu, int tid PH_ARG) {
    const int F = ws.F;
    const double *W = ws.W, *hh = ws.hh, *gl = ws.gl, *Dl = ws.Dl, *stl = ws.stl;
    const int t2 = tid - 32, n2 = SOLVE_THREADS - 32;
    const int wq = (tid >> 5) - 1, lane = tid & 31;
    const int LDW = SC_LDW;
    double *tw = s.Ju;                         // 80 x 36 tile (aliases Ju .. red, unused during the solve)
    double *sinv = nF <= 1024 ? s.wj : ws.sinv;  // 1 / sqrt(h + mu D^2): shared memory (wj: 1024 doubles) up to the reference's NUM_OF_F,
                                                   // the ninth workspace vector for the larger synthetic stress windows
    {   // Cauchy point (H still unregularised / unfactored here)
        const double *v = s.stp;
        double pv = 0.0;
        for (int k = t2; k < NX * NX; k += n2) pv += v[k / NX] * s.Hxx[k] * v[k % NX];
        for (int k = t2; k < NX * NY; k += n2) pv += 2.0 * v[k / NY] * s.Hxy[k] * v[NX + k % NY];
        for (int f = t2; f < nF; f += n2) {
            const double wv = w_column_dot<false>(W + f, F, v, 0.0);
            pv += 2.0 * stl[f] * wv + hh[f] * stl[f] * stl[f];
        }
        for (int o = 16; o > 0; o >>= 1) pv += __shfl_sync(0xffffffffu, pv, (lane + o) & 31);
        if (lane == 0) s.lin[wq] = pv;
        CERB_BAR_SYNC(1, n2);
        for (int k = t2; k < NX; k += n2) s.Hxx[k * NX + k] += mu * s.D[k] * s.D[k];
    }
    PH_MARK_T(19, 32);
    for (int f = t2; f < nF; f += n2) sinv[f] = rsqrt(hh[f] + mu * Dl[f] * Dl[f]);
    double acc[8][2];
    _Pragma("unroll")
    for (int k = 0; k < 8; k++) { acc[k][0] = 0.0; acc[k][1] = 0.0; }
    CERB_BAR_SYNC(1, n2);
    // raw W / g_l values of a tile are fetched into registers one tile ahead (12 per thread: the loads are issued
    // together and stay in flight during the tensor-core loop), scaled and stored when the tile buffer is free
    double buf[12];
    auto fetch = [&](int f0) {
        const int nf = (nF - f0) < 32 ? (nF - f0) : 32;
        _Pragma("unroll")
        for (int u = 0; u < 12; u++) {
            const int e = t2 + u * n2, a = e >> 5, f = e & 31;
            buf[u] = (e < 80 * 32 && f < nf) ? (a < NX ? W[(size_t)a * F + f0 + f] : (a == NX ? gl[f0 + f] : 0.0)) : 0.0;
        }
    };
    fetch(0);
    PH_MARK_T(37, 32);
    for (int f0 = 0; f0 < nF; f0 += 32) {
        const int nf = (nF - f0) < 32 ? (nF - f0) : 32;
        _Pragma("unroll")
        for (int u = 0; u < 12; u++) {
            const int e = t2 + u * n2, a = e >> 5, f = e & 31;
            if (e < 80 * 32) tw[a * LDW + f] = (f < nf) ? buf[u] * sinv[f0 + f] : 0.0;
        }
        CERB_BAR_SYNC(1, n2);
        PH_MARK_T(38, 32);
        if (f0 + 32 < nF) fetch(f0 + 32);
        schur_tile_w(wq, tw, acc, lane);
        CERB_BAR_SYNC(1, n2);
        PH_MARK_T(39, 32);
    }
    schur_scatter_w(wq, s, acc, lane);
    PH_MARK_T(7, 32);
}
// T = L^-1 Hyx (row a of Hxy in place; row 79: the y part of the rhs), rows on threads 32..111: block f of the forward substitution
// starts as soon as warp 0 has published the factor of block f, so that the substitution finishes right behind the chain instead of after it
CERB_D void forward_subst(Smem &s, const int *chain_done, int t2) {
    if (t2 <= NX) {
        double *row = (t2 < NX) ? s.Hxy + t2 * NY : s.yv + NX;
        double tp[NYB];
        _Pragma("unroll")
        for (int k = 0; k < NYB; k++) tp[k] = 0.0;
        _Pragma("unroll 1")
        for (int f = 0; f < NFR; f++) {
            while (CERB_LD_ACQUIRE_S32(chain_done) <= f) { CERB_SPIN_PAUSE(); }
            __threadfence_block();
            const double *L = s.Ad + f * HBLK, *idg = s.idg + NYB * f;
            double *t = row + NYB * f;
            double tc[NYB];
            _Pragma("unroll")
            for (int r = 0; r < NYB; r++) tc[r] = t[r];
            if (f > 0) {
                const double *M = s.Bo + (f - 1) * HBLK;
                _Pragma("unroll")
                for (int r = 0; r < NYB; r++) { double acc = 0.0; _Pragma("unroll") for (int q = 0; q < NYB; q++) acc += M[r * NYB + q] * tp[q]; tc[r] -= acc; }
            }
            _Pragma("unroll")
            for (int c = 0; c < NYB; c++) {             // right-looking: the dependency chain is 13 (multiply, update) steps
                tc[c] *= idg[c];
                _Pragma("unroll")
                for (int r = c + 1; r < NYB; r++) tc[r] -= L[r * NYB + c] * tc[c];
            }
            _Pragma("unroll")
            for (int r = 0; r < NYB; r++) { t[r] = tc[r]; tp[r] = tc[r]; }
        }
    }
}
// dense Cholesky of the 79 x 79 lower triangle, rhs carried as row 79 (z = L^-1 rhs), blocked by panels of 8,
// with look-ahead: (a) warp 0 factors a diagonal block in registers (pivots / column entries exchanged by shuffles),
// (b) one thread per row below solves its 8 panel entries against L_kk, (c) the trailing lower triangle is updated
// block by block on the fp64 tensor cores (A_ij -= L_ik L_jk^T, K = 8) -- warp 0 takes only the block that becomes
// the next diagonal block and factors it right away, while warps 1..7 update the rest.  Two barriers per panel; the
// serial column sweeps of the diagonal blocks (the critical path) overlap with the trailing updates.
CERB_D void panel_cholesky(Smem &s, int tid PH_ARG) {
    const int wq = tid >> 5, lane = tid & 31;
    auto factor_diag = [&](int c0, int nb, double *Lkk) {      // warp 0: L_kk of the nb x nb block at (c0, c0); Lkk[64..72) = 1 / diag
        const bool act = lane < nb;
        const int r = act ? lane : 0;
        double a[8];
        _Pragma("unroll")
        for (int c = 0; c < 8; c++) a[c] = (c < nb && c <= r) ? s.Hxx[(c0 + r) * NX + c0 + c] : 0.0;
        double myinv = 1.0;
        _Pragma("unroll")
        for (int j = 0; j < 8; j++) {
            double d = __shfl_sync(0xffffffffu, a[j], j);
            if (j < nb && !(d > 0.0)) { if (lane == 0) s.sca[S_OK] = 0; }
            if (!(d > 0.0)) d = 1.0;
            const double inv = rsqrt(d);
            if (lane == j) myinv = inv;
            const double l = (lane == j) ? d * inv : a[j] * inv;
            a[j] = l;
            _Pragma("unroll")
            for (int k = j + 1; k < 8; k++) { const double lk = __shfl_sync(0xffffffffu, l, k); a[k] -= l * lk; }
        }
        if (act) {
            _Pragma("unroll")
            for (int c = 0; c < 8; c++) if (c <= r) { s.Hxx[(c0 + r) * NX + c0 + c] = a[c]; Lkk[r * 8 + c] = a[c]; }
            Lkk[64 + r] = myinv; s.idx[c0 + r] = myinv;
        }
    };
    auto trailing_block = [&](int c0, int b0, int b) {          // block b = (bi, bj), bj <= bi, of the rows / columns from 8 b0 on
        int bi = 0, idx = b;
        while (idx > bi) { idx -= bi + 1; bi++; }
        const int ri = 8 * (b0 + bi) + (lane >> 2), rj = 8 * (b0 + idx) + (lane >> 2);
        double a0 = 0.0, a1 = 0.0;
        for (int ks = 0; ks < 2; ks++) {
            const int cc = c0 + 4 * ks + (lane & 3);
            const double av = (ri < NX) ? s.Hxx[ri * NX + cc] : (ri == NX ? s.yv[cc] : 0.0);
            const double bv = (rj < NX) ? s.Hxx[rj * NX + cc] : 0.0;
            CERB_DMMA(a0, a1, av, bv, a0, a1);
        }
        const int cj = 8 * (b0 + idx) + 2 * (lane & 3);
        if (ri < NX) {
            if (cj <= ri && cj < NX) s.Hxx[ri * NX + cj] -= a0;
            if (cj + 1 <= ri && cj + 1 < NX) s.Hxx[ri * NX + cj + 1] -= a1;
        } else if (ri == NX) {
            if (cj < NX) s.yv[cj] -= a0;
            if (cj + 1 < NX) s.yv[cj + 1] -= a1;
        }
    };
    if (wq == 0) factor_diag(0, 8, s.red);
    __syncthreads();
    int pk = 0;
    for (int c0 = 0; c0 < NX; c0 += 8, pk ^= 1) {
        const int nb = (NX - c0) < 8 ? (NX - c0) : 8, c1 = c0 + nb;
        const double *Lkk = s.red + 80 * pk;            // factored diagonal block of this panel (+ inverse diagonal at [64..72))
        // (b) rows c1 .. NX (row NX = rhs, kept in yv)
        if (tid <= NX - c1) {
            const int i = c1 + tid;
            double *row = (i < NX) ? s.Hxx + i * NX + c0 : s.yv + c0;
            double t[8];
            _Pragma("unroll")
            for (int c = 0; c < 8; c++) t[c] = (c < nb) ? row[c] : 0.0;
            _Pragma("unroll")
            for (int c = 0; c < 8; c++) {
                if (c < nb) {
                    t[c] *= Lkk[64 + c];
                    _Pragma("unroll")
                    for (int c2 = c + 1; c2 < 8; c2++) if (c2 < nb) t[c2] -= t[c] * Lkk[c2 * 8 + c];
                }
            }
            _Pragma("unroll")
            for (int c = 0; c < 8; c++) if (c < nb) row[c] = t[c];
        }
        __syncthreads();
        PH_MARK(47);
        if (c1 >= NX) break;
        // (c) trailing update of rows / columns c1 .. NX (row NX = rhs) + look-ahead factorisation of the next diagonal block
        {
            const int b0 = c1 >> 3, nbt = 10 - b0;               // block rows b0 .. 9
            const int nblk = nbt * (nbt + 1) / 2;
            if (wq == 0) {
                trailing_block(c0, b0, 0);
                __syncwarp();
                factor_diag(c1, (NX - c1) < 8 ? (NX - c1) : 8, s.red + 80 * (pk ^ 1));
                PH_MARK(44);
            } else {
                for (int b = wq; b < nblk; b += 7) trailing_block(c0, b0, b);
                PH_MARK_T(45, 32);
            }
        }
        __syncthreads();
        PH_MARK(46);
    }
}
// The three parts of the Gauss-Newton step below are real calls, like vision_linearize: each gets its own register allocation.  Inlined
// into the kernel body (at the 255-register cap with spills) the per-feature loops over W were scheduled as load, FMA, load, ...
// Hyy chain factorisation (warp 0) | Cauchy point, inverse-depth Schur complement and forward substitution (warps 1..7)
CERB_NOINLINE void gn_eliminate(const SolveParams &P, int w, double mu, int tid PH_ARG) {
    CERB_DYN_SMEM(double, smem_base);
    Smem s; smem_carve(smem_base, s);
    int *chain_done = s.ti + TI_CHAIN_DONE;
    if (tid < 32) chain_cholesky(s, chain_done, tid PH_FWD);
    else { lambda_schur(s, ws_carve(P), P.n_features[w], mu, tid PH_FWD); forward_subst(s, chain_done, tid - 32); }
}
// S' = S - T T^T (lower), rhs'_x = rhs_x - T gy' : Gram matrix of the 79 x 143 matrix [T; gy'^T] on the fp64 tensor cores, K = 143
// padded to 144, block rectangles per warp (ttt_warp); then the dense Cholesky of S'
CERB_NOINLINE void gn_reduce_factor(int tid PH_ARG) {
    CERB_DYN_SMEM(double, smem_base);
    Smem s; smem_carve(smem_base, s);
    ttt_warp_w(tid >> 5, s, tid & 31);
    __syncthreads();
    PH_MARK(9);
    panel_cholesky(s, tid PH_FWD);
    PH_MARK(10);
}
// back substitutions for y_x, y_y and the inverse depths; the prior image's Hxx part is prefetched as soon as the factor of Hxx is dead
// (fail: report the solve as failed, the fault injection of the parity tests).  The inverse depths need only y_x: warps 5..7 start them
// as soon as y_x is solved, warps 1..4 join after their share of T^T y_x, while warp 0 runs the y substitution.
CERB_NOINLINE void back_substitution(const SolveParams &P, int w, bool has_prior, bool bulk_ok, double mu, bool fail, int tid PH_ARG) {
    CERB_DYN_SMEM(double, smem_base);
    Smem s; smem_carve(smem_base, s);
    const CtaWs ws = ws_carve(P);
    const int wq = tid >> 5, lane = tid & 31;
    if (wq == 0) {      // L^T y_x = z: lane holds y[lane], y[lane + 32], y[lane + 64] in registers; branch-free steps (selects), the L entries
                        // of the next step are loaded before the current shuffle completes
        double y0 = s.yv[lane], y1 = s.yv[32 + lane], y2 = (64 + lane < NX) ? s.yv[64 + lane] : 0.0;
        _Pragma("unroll 1")
        for (int k = NX - 1; k >= 0; k--) {
            const double *Lk = s.Hxx + k * NX;
            const double ik = s.idx[k];
            const double l0 = (lane < k) ? Lk[lane] : 0.0, l1 = (32 + lane < k) ? Lk[32 + lane] : 0.0, l2 = (64 + lane < k) ? Lk[64 + lane] : 0.0;
            const double src = (k >= 64) ? y2 : (k >= 32 ? y1 : y0);
            const double yk = __shfl_sync(0xffffffffu, src, k & 31) * ik;
            y0 = (lane == k) ? yk : y0 - l0 * yk;
            y1 = (32 + lane == k) ? yk : y1 - l1 * yk;
            y2 = (64 + lane == k) ? yk : y2 - l2 * yk;
        }
        s.yv[lane] = y0; s.yv[32 + lane] = y1; if (64 + lane < NX) s.yv[64 + lane] = y2;
    }
    __syncthreads();
    if (has_prior) {                                                                           // the factor of Hxx is dead from here on
        if (bulk_ok) { if (tid == 0) CERB_BULK_G2S(s.Hxx, ws.pimg, PIMG_HXY * 8, &s.mbar[0]); }
        else copy_g2s_async(s.Hxx, ws.pimg, HXX_SZ, tid);
    }
    PH_MARK(11);
    double bad = 0.0;
    if (wq < 5) {       // y part: u = gy' - T^T y_x (threads 0..142), then L^T y_y = u blockwise (warp 0)
        if (tid < NY) { double t = 0.0; for (int a = 0; a < NX; a++) t += s.Hxy[a * NY + tid] * s.yv[a]; s.yv[NX + tid] -= t; }
        CERB_BAR_SYNC(1, 160);
    }
    if (wq == 0) {      // lane r holds component r of the current block; one shuffle per substitution step
        const int r = lane < NYB ? lane : 0;
        double yn[NYB];                                  // solved block f + 1 (all lanes)
        _Pragma("unroll")
        for (int k = 0; k < NYB; k++) yn[k] = 0.0;
        _Pragma("unroll 1")
        for (int f = NFR - 1; f >= 0; f--) {
            const double *L = s.Ad + f * HBLK;
            double u = s.yv[NX + NYB * f + r];
            if (f < NFR - 1) {
                const double *M = s.Bo + f * HBLK;
                double t = 0.0;
                _Pragma("unroll")
                for (int k = 0; k < NYB; k++) t += M[k * NYB + r] * yn[k];
                u -= t;
            }
            double lc[NYB], ig[NYB];                          // column r of L^T and the inverse pivots: loaded before the chain
            _Pragma("unroll")
            for (int k = 0; k < NYB; k++) { lc[k] = (lane < k) ? L[k * NYB + r] : 0.0; ig[k] = s.idg[NYB * f + k]; }
            _Pragma("unroll")
            for (int k = NYB - 1; k >= 0; k--) {
                const double yk = __shfl_sync(0xffffffffu, u, k) * ig[k];
                yn[k] = yk;
                u = (lane == k) ? yk : u - lc[k] * yk;
            }
            if (lane < NYB) s.yv[NX + NYB * f + lane] = u;
        }
        __syncwarp();
        for (int k = lane; k < NR; k += 32) if (!(fabs(s.yv[k]) < 1e300)) bad = 1.0;
        PH_MARK(12);
    } else {            // warps 1..7: inverse depths y_l = (gl - w^T y_x) / (h + mu D^2)
        const int nF = P.n_features[w];
        for (int f = tid - 32; f < nF; f += SOLVE_THREADS - 32) {
            const double t = w_column_dot<true>(ws.W + f, ws.F, s.yv, ws.gl[f]);
            const double y = t / (ws.hh[f] + mu * ws.Dl[f] * ws.Dl[f]);
            ws.gnl[f] = y;
            if (!(fabs(y) < 1e300)) bad = 1.0;
        }
        PH_MARK_T(43, 32);
    }
    if (bad != 0.0) s.sca[S_OK] = 0;          // benign race: every writer stores 0
    if (fail) s.sca[S_OK] = 0;
    __syncthreads();
    PH_MARK(13);
}
// Gauss-Newton step (H~ + mu D^2) y = g~ -> gn = -D y (s.gn, gnl) and its norms; S_OK = 0 if it failed
CERB_D void gauss_newton_step(const SolveParams &P, Smem &s, const Win &c, PriorCopy &pc, int &gn_attempts, int tid PH_ARG) {
    const int nF = c.nF;
    const double mu = s.sca[S_MU];
    // rhs: yv[0..NR) = g~ ; regularise the diagonal of Hyy (that of Hxx: warps 1..7, after their share of v^T H v)
    for (int k = tid; k < NR; k += SOLVE_THREADS) {
        s.yv[k] = s.g[k];
        if (k >= NX) s.Ad[((k - NX) / NYB) * HBLK + ((k - NX) % NYB) * (NYB + 1)] += mu * s.D[k] * s.D[k];
    }
    if (tid == 0) s.ti[TI_CHAIN_DONE] = 0;
    __syncthreads();
    gn_eliminate(P, c.w, mu, tid PH_FWD);
    __syncthreads();
    if (tid == 0) {
        double vhv = s.sca[S_VHV];
        for (int k = 0; k < 7; k++) vhv += s.lin[k];
        s.sca[S_ALPHA] = s.sca[S_GNORM2] / vhv;
    }
    PH_MARK(5);
    __syncthreads();
    PH_MARK(8);
    gn_reduce_factor(tid PH_FWD);
    back_substitution(P, c.w, c.has_prior, c.bulk_ok, mu, gn_attempts < P.test_fail_factorizations, tid PH_FWD);
    if (c.has_prior) pc.hxx_prefetched = true;
    gn_attempts++;
    if (s.sca[S_OK] != 0.0) {      // gauss_newton_step = -D * y ; norms for the dogleg
        double part3[2] = {0.0, 0.0};    // ||gn||^2, gh . gn
        for (int k = tid; k < NR; k += SOLVE_THREADS) { const double v = -s.D[k] * s.yv[k]; s.gn[k] = v; part3[0] += v * v; part3[1] += s.gh[k] * v; }
        for (int f = tid; f < nF; f += SOLVE_THREADS) { const double v = -c.ws.Dl[f] * c.ws.gnl[f]; c.ws.gnl[f] = v; part3[0] += v * v; part3[1] += c.ws.ghl[f] * v; }
        double tot3[2];
        block_sum<2>(part3, s.red, tot3, tid);
        if (tid == 0) { s.sca[S_GNNORM2] = tot3[0]; s.sca[S_GDOTGN] = tot3[1]; }
        __syncthreads();
    }
}
// ComputeTraditionalDoglegStep: S_P, S_Q (step = (p gh + q gn) / D), its norm and the model cost change
CERB_D void dogleg_step(double *sca, int tid) {
    if (tid == 0) {
        const double radius = sca[S_RADIUS], alpha = sca[S_ALPHA];
        const double gradient_norm = sqrt(sca[S_GNORM2]), gauss_newton_norm = sqrt(sca[S_GNNORM2]);
        double p, q, nrm;
        if (gauss_newton_norm <= radius) { p = 0.0; q = 1.0; nrm = gauss_newton_norm; }
        else if (gradient_norm * alpha >= radius) { p = -(radius / gradient_norm); q = 0.0; nrm = radius; }
        else {
            const double b_dot_a = -alpha * sca[S_GDOTGN];
            const double a_squared_norm = (alpha * gradient_norm) * (alpha * gradient_norm);
            const double b_minus_a_squared_norm = a_squared_norm - 2 * b_dot_a + gauss_newton_norm * gauss_newton_norm;
            const double c = b_dot_a - a_squared_norm;
            const double d = sqrt(c * c + b_minus_a_squared_norm * (radius * radius - a_squared_norm));
            const double beta = (c <= 0) ? (d - c) / b_minus_a_squared_norm : (radius * radius - a_squared_norm) / (d + c);
            p = -alpha * (1.0 - beta); q = beta;
            nrm = sqrt(p * p * sca[S_GNORM2] + 2 * p * q * sca[S_GDOTGN] + q * q * sca[S_GNNORM2]);
        }
        sca[S_P] = p; sca[S_Q] = q; sca[S_DLNORM] = nrm;
        // model_cost_change = -(step^T g~ + 0.5 step^T H~ step) with step = (p gh + q gn) / D, using
        // H~ (gn/D) = -(g~ + mu D gn)  (the Gauss-Newton equations):
        const double mu = sca[S_MU], g2 = sca[S_GNORM2], gg = sca[S_GDOTGN], n2 = sca[S_GNNORM2];
        const double sTg = p * g2 + q * gg;
        const double sHs = p * p * (g2 / alpha) - 2.0 * p * q * (g2 + mu * gg) + q * q * (-gg - mu * n2);
        sca[S_MODEL] = -(sTg + 0.5 * sHs);
    }
    __syncthreads();
}
// HandleInvalidStep (LINEAR_SOLVER_FAILURE or a step without model decrease; the failed factorisation overwrote H, so the caller
// re-linearises at the same point); true: the minimizer stops
CERB_D bool handle_invalid_step(double *sca, int tid) {
    if (tid == 0) {
        sca[S_INVALID] += 1;
        if (sca[S_INVALID] >= 5) { sca[S_DONE] = 1; sca[S_TERM] = 2; }
        sca[S_MU] *= 10.0; sca[S_REUSE] = 0;      // StepIsInvalid
    }
    __syncthreads();
    return sca[S_DONE] != 0.0;
}
// candidate point x [+] delta, lam + dlam, its cost (S_CCOST) and ||delta|| (S_STEPNORM).  Speculative linearisation: if the previous step of
// this window was accepted, the candidate is linearised right away -- its cost is the candidate cost, and when the step is accepted (the common
// case) the linearisation of the next iteration is already there, so the separate cost-only pass is saved.  A rejected step leaves H / g / W at
// the candidate, which is harmless: the re-use path of the dogleg needs none of them.  Not done in the last allowed iteration (never needed).
CERB_D void evaluate_candidate(const SolveParams &P, Smem &s, const Win &c, PriorCopy &pc, bool speculate, int tid PH_ARG) {
    const int nF = c.nF;
    double *sca = s.sca, *stl = c.ws.stl, *lamc = c.ws.lamc;
    {   // delta = ((p gh + q gn) / D) * jacobi_scale
        const double p = sca[S_P], q = sca[S_Q];
        for (int k = tid; k < NR; k += SOLVE_THREADS) s.stp[k] = (p * s.gh[k] + q * s.gn[k]) / s.D[k] * s.sc[k];
        for (int f = tid; f < nF; f += SOLVE_THREADS) stl[f] = (p * c.ws.ghl[f] + q * c.ws.gnl[f]) / c.ws.Dl[f] * c.ws.sl[f];
    }
    __syncthreads();
    PH_MARK(14);
    apply_plus(s, s.stp, c.lam, stl, lamc, nF, c.ex_open, c.td_open, tid);
    double part[2];
    PH_MARK(15);
    if (speculate) { linearize(P, s, c, pc, s.xc, lamc, false, tid PH_FWD); part[0] = 0.0; }
    else {
        load_geometry(s.xc, s, tid);
        part[0] = vision_cost(P, c.w, s.xc, lamc, tid);
        PH_MARK(16);
        part[0] += inertial_cost(P, c.w, s.xc, tid);
    }
    PH_MARK(17);
    part[1] = ambient_sq(s.xs, s.xc, c.lam, lamc, nF, c.ex_open, c.lb_open, c.td_open, tid);
    double tot[2];
    block_sum<2>(part, s.red, tot, tid);
    if (tid == 0) {
        double cc = speculate ? sca[S_LCOST] : tot[0];
        if (!(cc == cc) || fabs(cc) > 1e300) cc = 1.7976931348623157e308;
        sca[S_CCOST] = cc; sca[S_STEPNORM] = sqrt(tot[1]);
    }
    __syncthreads();
}
// tolerances, then StepAccepted (S_OK = 2) / StepRejected; true: the minimizer stops
CERB_D bool accept_or_reject(const SolveParams &P, double *sca, int tid) {
    if (tid == 0) {
        const double x_cost = sca[S_XCOST], cand = sca[S_CCOST];
        if (sca[S_STEPNORM] <= P.ptol * (sca[S_XNORM] + P.ptol)) { sca[S_DONE] = 1; sca[S_TERM] = 0; }
        else if (fabs(x_cost - cand) <= P.ftol * x_cost) { sca[S_DONE] = 1; sca[S_TERM] = 0; }
        else {
            const double rel = (x_cost - cand) / sca[S_MODEL];
            if (rel > P.min_rel_dec) {            // StepAccepted
                if (rel < 0.25) sca[S_RADIUS] *= 0.5;
                if (rel > 0.75) sca[S_RADIUS] = fmax(sca[S_RADIUS], 3.0 * sca[S_DLNORM]);
                sca[S_MU] = fmax(1e-8, 2.0 * sca[S_MU] / 10.0);
                sca[S_REUSE] = 0; sca[S_NSUCC] += 1; sca[S_OK] = 2;     // 2 == accepted marker
                sca[S_XCOST] = cand;                                   // x_cost of the new point (re-evaluated by the next linearisation, if any)
            } else {                              // StepRejected
                sca[S_RADIUS] *= 0.5; sca[S_REUSE] = 1; sca[S_OK] = 1;
            }
        }
    }
    __syncthreads();
    return sca[S_DONE] != 0.0;
}

// ---- the kernel -----------------------------------------------------------------------------------------------
CERB_GLOBAL void __launch_bounds__(SOLVE_THREADS, CERB_SOLVE_MIN_BLOCKS) vilo_solve_kernel(CERB_GRID_CONSTANT SolveParams P) {
    CERB_DYN_SMEM(double, smem_base);
    Smem s; smem_carve(smem_base, s);
    const int tid = threadIdx.x;
    const CtaWs ws = ws_carve(P);
    double *sca = s.sca;
    PH_DECL();
    PriorCopy pc = {0, 0, false};
    if (tid == 0) { CERB_MBAR_INIT(&s.mbar[0]); CERB_MBAR_INIT(&s.mbar[1]); }
    build_imu_plan(s, smem_base, ws.imu_plan, tid);
    __syncthreads();
    for (int w = blockIdx.x; w < P.n_windows; w += gridDim.x) {
        Win c; c.w = w; c.nF = P.n_features[w]; c.ws = ws; c.lam = P.lam + (size_t)w * ws.F;
        c.ex_open = (P.flags[w] & 1) != 0; c.lb_open = P.optimize_leg_bias && (P.flags[w] & 4) == 0; c.td_open = (P.flags[w] & 2) != 0;
        if (tid == 0) build_chunks(P.feat_start + (size_t)w * ws.F, s, ws.chunks, c.nF);
        c.has_prior = build_prior_image(P, s, w, ws.pimg, tid);
        if (tid == 0) s.ti[TI_IMU_MASK] = 0;                             // all IMU-leg factors (the marginalization kernel restricts them)
        for (int k = tid; k < ST_STRIDE; k += SOLVE_THREADS) s.xs[k] = (k < ST_SIZE) ? P.state[(size_t)w * ST_STRIDE + k] : 0.0;
        if (tid == 0) {
            sca[S_RADIUS] = P.radius0; sca[S_MU] = P.test_initial_mu > 0.0 ? P.test_initial_mu : 1e-8; sca[S_REUSE] = 0; sca[S_DONE] = 0; sca[S_TERM] = 1; sca[S_ITER] = 0; sca[S_NSUCC] = 0;
            sca[S_INVALID] = 0; sca[S_DLNORM] = 0;
        }
        __syncthreads();
        c.bulk_ok = (reinterpret_cast<uintptr_t>(ws.pimg) & 15) == 0 && !P.no_bulk_copy;          // TMA bulk copies need 16-byte aligned sources (max_features even)
        pc.hxx_prefetched = false;
        bool need_linearize = true, last_accepted = true;
        int iteration = 0, gn_attempts = 0;
        while (true) {
            // Ceres evaluates the Jacobian at every accepted point, but when that point is the last one allowed by max_num_iterations the
            // evaluation is never used: FinalizeIterationAndCheckIfMinimizerCanContinue tests the iteration limit before the gradient
            // tolerance, so termination, states and costs are decided already.  That last linearisation is skipped.
            if (need_linearize && (iteration < P.max_iters || iteration == 0)) {
                linearize(P, s, c, pc, s.xs, c.lam, iteration == 0, tid PH_FWD);
                if (tid == 0) { sca[S_XCOST] = sca[S_LCOST]; sca[S_XNORM] = sca[S_LNORM]; sca[S_GMAX] = sca[S_LGMAX]; if (iteration == 0) sca[S_INIT_COST] = sca[S_LCOST]; }
                __syncthreads();
                need_linearize = false;
                PH_MARK(3);
            }
            if (finalize_iteration(P, sca, iteration, tid)) break;
            iteration++;
            // DoglegStrategy::ComputeStep.  ComputeGaussNewtonStep retries INSIDE one ComputeStep (`while (mu_ < max_mu_)`, Ceres 1.14
            // dogleg_strategy.cc): a failed factorisation / non-finite step multiplies mu by 10 and solves again at the same point -- no
            // iteration and no invalid step is consumed; only when mu reaches max_mu (1.0) does the strategy report LINEAR_SOLVER_FAILURE.
            // The factorisation here is in place, so a retry first rebuilds H / g at the same point.
            if (sca[S_REUSE] == 0.0) {
                for (;;) {
                    if (!(sca[S_MU] < 1.0)) {                 // while (mu_ < max_mu_) not entered: LINEAR_SOLVER_FAILURE without a solve
                        __syncthreads();
                        if (tid == 0) { sca[S_OK] = 0; sca[S_REUSE] = 1; }
                        __syncthreads();
                        break;
                    }
                    dogleg_diagonal(s, c, tid PH_FWD);
                    gauss_newton_step(P, s, c, pc, gn_attempts, tid PH_FWD);
                    if (tid == 0) sca[S_REUSE] = 1;
                    __syncthreads();
                    if (sca[S_OK] != 0.0) break;              // the Gauss-Newton step is there
                    __syncthreads();
                    if (tid == 0) sca[S_MU] *= 10.0;           // mu_ *= mu_increase_factor_; continue;
                    __syncthreads();
                    if (!(sca[S_MU] < 1.0)) break;            // LINEAR_SOLVER_FAILURE (S_OK == 0)
                    linearize(P, s, c, pc, s.xs, c.lam, false, tid PH_FWD);      // the failed in-place factorisation overwrote H: rebuild it
                }
            }
            if (sca[S_OK] == 0.0) { if (handle_invalid_step(sca, tid)) break; need_linearize = true; continue; }      // LINEAR_SOLVER_FAILURE
            dogleg_step(sca, tid);
            if (!(sca[S_MODEL] > 0.0)) { if (handle_invalid_step(sca, tid)) break; need_linearize = true; continue; }
            if (tid == 0) sca[S_INVALID] = 0;
            const bool speculate = last_accepted && iteration < P.max_iters;
            evaluate_candidate(P, s, c, pc, speculate, tid PH_FWD);
            if (accept_or_reject(P, sca, tid)) break;
            const bool accepted = (sca[S_OK] == 2.0);
            __syncthreads();
            if (accepted) {      // the candidate becomes the current point
                for (int k = tid; k < ST_STRIDE; k += SOLVE_THREADS) s.xs[k] = s.xc[k];
                for (int f = tid; f < c.nF; f += SOLVE_THREADS) c.lam[f] = ws.lamc[f];
                if (tid == 0) { sca[S_OK] = 1; if (speculate) { sca[S_XNORM] = sca[S_LNORM]; sca[S_GMAX] = sca[S_LGMAX]; } }
                __syncthreads();
                need_linearize = !speculate;                     // a speculative linearisation is the linearisation at the new point
            }
            last_accepted = accepted;
            PH_MARK(18);
        }
        // ---- write back ---------------------------------------------------------------------------------
        if (c.bulk_ok && pc.hxx_prefetched) { CERB_MBAR_WAIT(&s.mbar[0], pc.par0); pc.par0 ^= 1; }   // drain a prefetch of the prior image that was never consumed
        CERB_CP_ASYNC_WAIT();
        for (int k = tid; k < ST_SIZE; k += SOLVE_THREADS) P.state[(size_t)w * ST_STRIDE + k] = s.xs[k];
        if (tid == 0) {
            P.rep_i[4 * w + 0] = iteration; P.rep_i[4 * w + 1] = (int)sca[S_NSUCC]; P.rep_i[4 * w + 2] = (int)sca[S_TERM];
            P.rep_i[4 * w + 3] = (sca[S_XCOST] == sca[S_XCOST] && fabs(sca[S_XCOST]) < 1e300) ? 0 : 4;
            P.rep_d[2 * w + 0] = sca[S_INIT_COST]; P.rep_d[2 * w + 1] = sca[S_XCOST];
        }
        __syncthreads();
    }
}

// ---- marginalization: A = sum J^T J, b = sum J^T r over the factors that touch the dropped blocks ----------------------------------
// MarginalizationInfo::{addResidualBlockInfo, preMarginalize, marginalize} up to ThreadsConstructA (marginalization_factor.cpp:98-279)
// for the factor set Estimator::optimization() hands it (estimator.cpp:1247-1376 MARGIN_OLD: the old prior, the IMU-leg factor 0 -> 1
// unless sum_dt > 10, every projection factor of the tracks anchored at frame 0 with the Huber corrector of ResidualBlockInfo::Evaluate;
// :1377-1455 MARGIN_SECOND_NEW: the old prior only).  The linearisation is the solve kernel's own (vision_linearize restricted to the
// anchor-0 chunks, inertial_linearize restricted to factor 0, the prior image): H and g in the solver's x | y | lambda partition are then
// scattered into the reference's [dropped | kept] order:
//   dropped: pose0, speedbias0, legbias0 (those that occur), the inverse depths of the anchor-0 tracks in the caller's order
//            (MARGIN_SECOND_NEW: para_Pose[WINDOW_SIZE - 1] of the old prior)
//   kept   : poses ascending, speed bias, leg bias, ex0, ex1, td (those that occur)
// The eps-clamped eigen Schur complement then runs in marg_schur_kernel on A / b in place (no host round trip).
struct MargParams {
    const int *flags;                // [n] 0: MARGIN_OLD, 1: MARGIN_SECOND_NEW
    const double *state, *lam;       // [n][ST_STRIDE], [n][maxF] (device feature order): the states the reference calls vector2double() on
    double *A, *b;                   // [n][posmax * posmax] row-major (leading dimension pos of the window), [n][posmax]
    int posmax;
    int *dims;                       // [n][4]: m, n, status (1: prior produced, 0: none (m == 0), 2: old prior carried over unchanged), number of kept blocks
    int *blocks;                     // [n][16][4]: kind, index AFTER the address shift of the slide, column, index in the window being marginalized, of every kept block
};
enum { MARG_OLD = 0, MARG_SECOND_NEW = 1 };

CERB_GLOBAL void __launch_bounds__(SOLVE_THREADS, 1) marg_assemble_kernel(CERB_GRID_CONSTANT SolveParams P, CERB_GRID_CONSTANT MargParams M) {
    CERB_DYN_SMEM(double, smem_base);
    Smem s; smem_carve(smem_base, s);
    const int tid = threadIdx.x, F = P.maxF;
    const CtaWs ws = ws_carve(P);
    int *colx = reinterpret_cast<int *>(s.idx);           // [79] column of x index a in A (-1: block absent), then [26] of the y indices of frames 0 / 1
                                                          // (idx: 80 doubles that only the Gauss-Newton step of the solver uses; idg holds the dummy slots of the IMU scatter)
    int *coly = colx + 80;
    int *misc = coly + 32;                                // [0] n0, [1] m, [2] n, [3] status, [4] stereo seen, [5] longest anchor-0 track
    build_imu_plan(s, smem_base, ws.imu_plan, tid);
    __syncthreads();
    for (int w = blockIdx.x; w < P.n_windows; w += gridDim.x) {
        const int nF = P.n_features[w], flag = M.flags[w];
        const double *lam = M.lam + (size_t)w * F;
        const int *pmeta = P.prior_meta + (size_t)w * PRIOR_META_STRIDE;
        const int *fstart = P.feat_start + (size_t)w * F, *fnobs = P.feat_nobs + (size_t)w * F, *foff = P.feat_off + (size_t)w * F;
        const int *stereo = P.obs_stereo + (size_t)w * P.maxObs;
        // ---- tracks anchored at frame 0 (the device order is sorted by anchor: they are the first n0 slots, in the caller's order) ----
        if (tid == 0) {
            int n0 = 0;
            if (flag == MARG_OLD) while (n0 < nF && fstart[n0] == 0) n0++;
            build_chunks(fstart, s, ws.chunks, n0);                  // all anchored at frame 0: chunks of 64
            s.ti[TI_IMU_MASK] = flag == MARG_OLD ? 1 : 2;
            misc[0] = n0; misc[4] = 0; misc[5] = 0;
        }
        const bool has_prior = build_prior_image(P, s, w, ws.pimg, tid);
        for (int k = tid; k < ST_STRIDE; k += SOLVE_THREADS) s.xs[k] = (k < ST_SIZE) ? M.state[(size_t)w * ST_STRIDE + k] : 0.0;
        __syncthreads();
        const int n0 = misc[0];
        {   // which of ex1 / pose_j occur among the visual factors: any stereo observation, the longest anchor-0 track
            int st = 0, len = 0;
            for (int f = tid; f < n0; f += SOLVE_THREADS) { const int nb = fnobs[f]; len = nb > len ? nb : len; for (int k = 0; k < nb; k++) st |= (stereo[foff[f] + k] != 0); }
            s.red[tid] = (double)(len | (st << 8));
            __syncthreads();
            if (tid == 0) { int l = 0, q = 0; for (int k = 0; k < SOLVE_THREADS; k++) { const int v = (int)s.red[k]; l = (v & 255) > l ? (v & 255) : l; q |= v >> 8; } misc[4] = q; misc[5] = l; }
            __syncthreads();
        }
        // ---- linearise: prior image | visual factors of the anchor-0 tracks | IMU-leg factor 0 | prior gradient ---------------------
        if (!has_prior) { for (int k = tid; k < HXX_SZ; k += SOLVE_THREADS) s.Hxx[k] = 0.0; }
        else copy_g2s(s.Hxx, ws.pimg, HXX_SZ, tid);
        for (int k = tid; k < NRP; k += SOLVE_THREADS) s.g[k] = 0.0;
        load_geometry(s.xs, s, tid);
        if (n0 > 0) vision_linearize(P, w, s.xs, lam, ws.W, ws.hh, ws.gl, ws.sl, false, ws.chunks, tid);
        __syncthreads();
        if (has_prior) copy_g2s(s.Hxy, ws.pimg + PIMG_HXY, PIMG_REST, tid);
        else for (int k = tid; k < PIMG_REST; k += SOLVE_THREADS) s.Hxy[k] = 0.0;
        __syncthreads();
        inertial_linearize(P, w, s.xs, tid);
        // ---- block presence and the [dropped | kept] column map ---------------------------------------------------------------
        if (tid == 0) {
            bool pose[NFR] = {false}, sb[2] = {false, false}, lb[2] = {false, false}, ex[2] = {false, false}, td = false;
            if (has_prior) for (int b = 0; b < pmeta[2]; b++) {
                const int kind = pmeta[4 + 3 * b], index = pmeta[5 + 3 * b];
                if (kind == 0) pose[index] = true; else if (kind == 1) sb[index ? 1 : 0] = true; else if (kind == 2) lb[index ? 1 : 0] = true;
                else if (kind == 3) ex[index] = true; else td = true;
            }
            const bool noleg = (P.flags[w] & 4) != 0;
            if (flag == MARG_OLD) {
                if (!(P.pre[(size_t)w * CERB_WINDOW * PRE_STRIDE + PRE_SUM_DT] > 10.0)) { pose[0] = pose[1] = true; sb[0] = sb[1] = true; if (!noleg) lb[0] = lb[1] = true; }
                if (n0 > 0) { pose[0] = true; ex[0] = true; td = true; if (misc[4]) ex[1] = true; for (int j = 1; j < misc[5] && j < NFR; j++) pose[j] = true; }
            }
            for (int k = 0; k < 80 + 32; k++) colx[k] = -1;
            int m = 0, n = 0, status = 1, nblk = 0;
            int *blk = M.blocks + (size_t)w * 64;
#define MARG_BLK(kind_, shifted_, src_) do { blk[4 * nblk] = (kind_); blk[4 * nblk + 1] = (shifted_); blk[4 * nblk + 2] = n; blk[4 * nblk + 3] = (src_); nblk++; } while (0)
            if (flag == MARG_OLD) {
                if (pose[0]) { for (int k = 0; k < 6; k++) colx[k] = m + k; m += 6; }
                if (sb[0]) { for (int k = 0; k < 9; k++) coly[k] = m + k; m += 9; }
                if (lb[0]) { for (int k = 0; k < 4; k++) coly[9 + k] = m + k; m += 4; }
                m += n0;                                                   // lambda k -> column (m - n0) + k
                if (m == 0) status = 0;                                    // MarginalizationInfo::valid = false (marginalization_factor.cpp:205-210)
                for (int j = 1; j < NFR; j++) if (pose[j]) { for (int k = 0; k < 6; k++) colx[6 * j + k] = m + n + k; MARG_BLK(0, j - 1, j); n += 6; }
                if (sb[1]) { for (int k = 0; k < 9; k++) coly[13 + k] = m + n + k; MARG_BLK(1, 0, 1); n += 9; }
                if (lb[1]) { for (int k = 0; k < 4; k++) coly[13 + 9 + k] = m + n + k; MARG_BLK(2, 0, 1); n += 4; }
            } else {
                if (!has_prior || !pose[CERB_WINDOW - 1]) status = 2;       // prior carried over unchanged (estimator.cpp:1380-1381)
                else {
                    for (int k = 0; k < 6; k++) colx[6 * (CERB_WINDOW - 1) + k] = k;
                    m = 6;
                    for (int j = 0; j < NFR; j++) if (pose[j] && j != CERB_WINDOW - 1) {
                        for (int k = 0; k < 6; k++) colx[6 * j + k] = m + n + k;
                        MARG_BLK(0, (j == CERB_WINDOW) ? j - 1 : j, j); n += 6;
                    }
                    if (sb[0]) { for (int k = 0; k < 9; k++) coly[k] = m + n + k; MARG_BLK(1, 0, 0); n += 9; }
                    if (lb[0]) { for (int k = 0; k < 4; k++) coly[9 + k] = m + n + k; MARG_BLK(2, 0, 0); n += 4; }
                }
            }
            if (status == 1) {
                for (int e = 0; e < 2; e++) if (ex[e]) { for (int k = 0; k < 6; k++) colx[66 + 6 * e + k] = m + n + k; MARG_BLK(3, e, e); n += 6; }
                if (td) { colx[X_TD] = m + n; MARG_BLK(4, 0, 0); n += 1; }
            }
#undef MARG_BLK
            misc[1] = m; misc[2] = n; misc[3] = status;
            int *dm = M.dims + 4 * w; dm[0] = m; dm[1] = n; dm[2] = status; dm[3] = nblk;
        }
        __syncthreads();
        if (misc[3] == 1) {
            const int m = misc[1], n = misc[2], pos = m + n, l0 = m - n0;      // l0: column of lambda 0 (MARGIN_OLD)
            double *A = M.A + (size_t)w * M.posmax * M.posmax, *b = M.b + (size_t)w * M.posmax;
            for (int e = tid; e < pos * pos; e += SOLVE_THREADS) A[e] = 0.0;
            __syncthreads();
            for (int e = tid; e < NX * NX; e += SOLVE_THREADS) {             // x - x (Hxx holds its upper triangle)
                const int a = e / NX, c = e % NX; if (c < a) continue;
                const int ca = colx[a], cc = colx[c]; if (ca < 0 || cc < 0) continue;
                const double v = s.Hxx[a * NX + c];
                A[(size_t)ca * pos + cc] = v; A[(size_t)cc * pos + ca] = v;
            }
            for (int e = tid; e < NX * 26; e += SOLVE_THREADS) {             // x - y (frames 0, 1)
                const int a = e / 26, q = e % 26, ca = colx[a], cq = coly[q]; if (ca < 0 || cq < 0) continue;
                const double v = s.Hxy[a * NY + q];
                A[(size_t)ca * pos + cq] = v; A[(size_t)cq * pos + ca] = v;
            }
            for (int e = tid; e < 26 * 26; e += SOLVE_THREADS) {             // y - y
                const int q = e / 26, r = e % 26, cq = coly[q], cr = coly[r]; if (cq < 0 || cr < 0) continue;
                const int fq = q / NYB, fr = r / NYB, kq = q % NYB, kr = r % NYB;
                A[(size_t)cq * pos + cr] = fq == fr ? s.Ad[fq * HBLK + kq * NYB + kr] : (fq < fr ? s.Bo[kq * NYB + kr] : s.Bo[kr * NYB + kq]);
            }
            for (int e = tid; e < NX * n0; e += SOLVE_THREADS) {             // x - lambda
                const int a = e / n0, k = e % n0, ca = colx[a]; if (ca < 0) continue;
                const double v = ws.W[(size_t)a * F + k];
                A[(size_t)ca * pos + l0 + k] = v; A[(size_t)(l0 + k) * pos + ca] = v;
            }
            for (int k = tid; k < n0; k += SOLVE_THREADS) { A[(size_t)(l0 + k) * pos + l0 + k] = ws.hh[k]; b[l0 + k] = ws.gl[k]; }
            for (int a = tid; a < NX; a += SOLVE_THREADS) if (colx[a] >= 0) b[colx[a]] = s.g[a];
            for (int q = tid; q < 26; q += SOLVE_THREADS) if (coly[q] >= 0) b[coly[q]] = s.g[NX + q];
        }
        __syncthreads();
    }
}

}  // namespace cerb

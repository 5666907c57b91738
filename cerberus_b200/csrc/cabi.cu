// cabi.cu -- implementation of the C ABI of include/cerberus_b200.h on top of the sm_90a kernels.
// Host side only packs the reference-shaped descriptors (AoS, Eigen column-major) into the device
// layout (planar observations, compact preintegration records), moves them through pinned staging
// buffers on the handle's stream and launches kernels.  There is no CPU compute path: if no CUDA
// device is present cerb_create fails with CERB_ERR_NO_DEVICE.
#include "../../include/cerberus_b200.h"
#include "solve_kernel.cuh"
#include "preint_kernel.cuh"
#include "feature_kernels.cuh"
#include "marg_kernels.cuh"
#include "pack_kernels.cuh"
#include "resident_kernels.cuh"
#include <string>
#include <vector>
#include <thread>
#include <cstring>
#include <cstdio>
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstdint>
#include <utility>

using namespace cerb;

static thread_local std::string g_err;
static int fail(int code, const std::string &msg) { g_err = msg; return code; }
#define CUDA_TRY(expr)                                                                                         \
    do {                                                                                                       \
        cudaError_t e_ = (expr);                                                                               \
        if (e_ != cudaSuccess) return fail(CERB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_)); \
    } while (0)
// cudaMemcpyAsync between host and device, counted in the handle's traffic totals (cerb_traffic)
#define COPY_TRY(h, dst, src, bytes, kind, s)                                                          \
    do {                                                                                               \
        (h)->traffic.count((kind), (bytes));                                                           \
        CUDA_TRY(cudaMemcpyAsync((dst), (src), (bytes), (kind), (s)));                                 \
    } while (0)
struct Traffic {
    int64_t h2d = 0, d2h = 0, ops = 0, staged = 0;
    void count(cudaMemcpyKind kind, size_t bytes) { if (kind == cudaMemcpyDeviceToDevice) return; (kind == cudaMemcpyHostToDevice ? h2d : d2h) += (int64_t)bytes; ops++; }
};

// One array of the resident batch: `per` elements per window, window w at at(w); `h` is its pinned host mirror of the same shape, where it has one
// (the staging of a caller's descriptors, the landing place of the results).
template <typename T> struct Resident {
    T *d = nullptr, *h = nullptr;
    size_t per = 0;
    T *at(size_t w) const { return d + w * per; }
    T *h_at(size_t w) const { return h + w * per; }
    size_t bytes(size_t n_windows) const { return n_windows * per * sizeof(T); }
};

struct CerbHandle {
    CerbSolverConfig cfg;
    int sm_count = 0, grid = 0;
    enum { MAX_CHUNKS = 32, LANES = 4 };
    cudaStream_t stream = nullptr, copy_stream = nullptr;
    cudaStream_t lane[LANES] = {};       // compute lanes of the chunked pipeline: lane[0] == stream; each has its own slice of d_ws
    cudaEvent_t ev_lane[LANES] = {};
    cudaEvent_t ev_copy[MAX_CHUNKS] = {};
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool ev_pending = false;
    double last_ms = 0; int last_launches = 0, last_dma_ops = 0; size_t last_staged_bytes = 0;
    int B = 0, F = 0, O = 0;          // capacities
    int n = 0;                        // windows currently resident
    // The resident batch, sized and allocated by create_impl.  The caller's descriptors as they are (filled by DMA, through the pinned mirror
    // for sources that are not in registered memory) ...
    Resident<CerbWindowDesc> rdesc; Resident<CerbFeature> rfeat; Resident<CerbObservation> robs; Resident<CerbWindowState> rstate;
    Resident<double> rpre, rlam;
    // ... the solver's layout (written by pack_kernel; the prior matrix and residuals by DMA) and its results ...
    Resident<int> n_features, feat_start, feat_nobs, feat_off, flags, obs_stereo, prior_meta, rep_i, perm;
    Resident<double> obs, pre, sinfo, prior_J, prior_r, prior_x0, prior_Hp, state, state0, lam, lam0, rep_d;
    // ... and the results in the caller's layout (unpack_kernel), with pinned mirrors
    Resident<double> olam, ostate; Resident<CerbSolveReport> orep;
    double *d_ws = nullptr, *d_dbg = nullptr, *h_dbg = nullptr, *d_G = nullptr, *d_probe_repd = nullptr;
    int *d_probe_repi = nullptr;
    std::vector<void *> dev_bufs, host_bufs;    // everything create_impl allocated (cudaMalloc / cudaMallocHost): freed by cerb_destroy
    std::vector<std::pair<uintptr_t, size_t>> regs;   // host ranges registered with cerb_register_host_buffer: DMA straight out of them
    std::vector<int> nfeat, n0;       // [B] n_features / number of tracks anchored at frame 0 of the resident windows
    int test_fail_factorizations = 0; double test_initial_mu = 0.0;   // fault injection of the parity tests (environment, read by cerb_create)
    bool solved = false;              // the device states are the solved ones (else: the uploaded initial states)
    std::vector<int> h_perm; bool perm_valid = false;     // [B][F] device feature slot -> index in the caller's feature array (fetched on demand)
    long ws_stride = 0;
    size_t smem_bytes = 0;
    // scratch arena of the evaluator / feature / preintegration entry points: grows to the high-water mark, then no more cudaMalloc per call
    std::vector<std::pair<char *, size_t>> arena; size_t arena_chunk = 0, arena_used = 0;
    Traffic traffic;                  // host <-> device copies issued since cerb_create
    // resident sliding window (cerb_resident_*): robs / rpre / the prior of windows [0, res_n) are edited in place instead of uploaded
    // Per window of the store: robs, rpre, the prior inside rdesc, prior_J, prior_r, res_extent, res_prior_valid, res_leg.  Per row of the
    // batch the last resident upload named (cerb_resident_upload_windows: row i reads store window res_win[i]): everything else.
    int res_n = 0;
    Resident<int> pre_slot;           // one copy per upload of n rows: [n][CERB_WINDOW_SIZE] row of rpre that holds interval i -> i + 1, then [n] res_win
    std::vector<int> res_win;         // [n] store window of each batch row
    std::vector<int> res_extent;      // [B] observations of robs a pack has to read: up to the highest slot ever put
    std::vector<char> res_prior_valid;
    std::vector<char> res_leg;        // [B] record kind of the window's preintegration slots: 1 CerbIMULegPreint, 0 CerbIMUPreint
    Resident<double> step_J, step_r;  // the priors of a compact batch by row (prior_gather_kernel; allocated with the first one)
    bool prior_gathered = false;      // the batch reads its priors from step_J / step_r instead of prior_J / prior_r
    bool prior_gather_due = false;    // ... and they have not been gathered yet (the per-feature passes read no prior: only a solve or a marginalization gathers)
    std::vector<unsigned char> res_mark;      // [B][O] scratch of the duplicate checks of put / edit (all zero between calls)
};

static int create_impl(CerbHandle *h, const CerbSolverConfig *cfg, const cudaDeviceProp &prop);
// every entry point re-selects the handle's device: the host application (or torch) may have changed the current device, and two
// handles on different GPUs may be driven from one thread
#define CERB_DEVICE(h) do { if (h) { cudaError_t e_ = cudaSetDevice((h)->cfg.device); if (e_ != cudaSuccess) return fail(CERB_ERR_CUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(e_)); } } while (0)

extern "C" {

const char *cerb_last_error(void) { return g_err.c_str(); }
const char *cerb_version(void) {
#if defined(CERB_CUSIM)
    return "cerberus_b200 0.1 (cusim test build)";
#else
    return "cerberus_b200 0.1 (sm_90a)";
#endif
}

void cerb_default_config(CerbSolverConfig *c) {
    std::memset(c, 0, sizeof(*c));
    c->device = 0; c->max_batch = 1024; c->max_features = 160; c->max_obs = 160 * CERB_NUM_FRAMES;
    c->max_num_iterations = 12; c->optimize_leg_bias = 1;
    c->g[0] = 0; c->g[1] = 0; c->g[2] = 9.805;
    c->visual_sqrt_info = 460.0 / 1.5; c->huber_delta = 1.0;
    c->initial_trust_region_radius = 1e4; c->max_trust_region_radius = 1e16; c->min_trust_region_radius = 1e-32;
    c->min_relative_decrease = 1e-3; c->function_tolerance = 1e-6; c->gradient_tolerance = 1e-10; c->parameter_tolerance = 1e-8;
}

void cerb_default_preint_config(CerbPreintConfig *p) {
    std::memset(p, 0, sizeof(*p));
    p->acc_n = 0.9; p->acc_n_z = 2.5; p->gyr_n = 0.05; p->acc_w = 0.0004; p->gyr_w = 0.0002;
    p->phi_n = 1e-5; p->dphi_n = 1e-5; p->rho_c_n = 1e-8; p->rho_nc_n = 1e-11;
    p->v_n_min_xy = 1e-3; p->v_n_min_z = 5e-3; p->v_n_min = 5e-3; p->v_n_max = 900.0;
    p->v_n_force_thres_ratio = 0.8; p->v_n_term1_steep = 10; p->v_n_term2_var_rescale = 1e-6; p->v_n_term3_distance_rescale = 1e-3;
    p->contact_sensor_type = 0;
    const double ox[4] = {0.1805, 0.1805, -0.1805, -0.1805}, oy[4] = {0.047, -0.047, 0.047, -0.047}, d[4] = {0.0838, -0.0838, 0.0838, -0.0838};
    for (int l = 0; l < 4; l++) { p->rho_fix[l][0] = ox[l]; p->rho_fix[l][1] = oy[l]; p->rho_fix[l][2] = d[l]; p->rho_fix[l][3] = 0.21; }
    p->R_br[0] = p->R_br[4] = p->R_br[8] = 1.0;
}


int cerb_create(const CerbSolverConfig *cfg, CerbHandle **out) {
    if (!cfg || !out) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_create: null argument");
    if (cfg->max_batch < 1 || cfg->max_features < 1 || cfg->max_features > CERB_MAX_FEATURES || cfg->max_obs < 1)
        return fail(CERB_ERR_BAD_ARGUMENT, "cerb_create: bad capacities");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= cfg->device)
        return fail(CERB_ERR_NO_DEVICE, "cerb_create: no CUDA device (this library has no CPU fallback)");
    CUDA_TRY(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
    CerbHandle *h = new CerbHandle();
    const int rc = create_impl(h, cfg, prop);
    if (rc != CERB_OK) { const std::string keep = g_err; cerb_destroy(h); g_err = keep; return rc; }      // no leak of streams / buffers on a failed create
    *out = h;
    return CERB_OK;
}

}  // extern "C"

template <typename T> static cudaError_t dmalloc(CerbHandle *h, T **p, size_t n) {
    const cudaError_t e = cudaMalloc((void **)p, n * sizeof(T));
    if (e == cudaSuccess) h->dev_bufs.push_back(*p);
    return e;
}
template <typename T> static cudaError_t hmalloc(CerbHandle *h, T **p, size_t n) {
    const cudaError_t e = cudaMallocHost((void **)p, n * sizeof(T));
    if (e == cudaSuccess) h->host_bufs.push_back(*p);
    return e;
}
// B windows of `per` elements, and the pinned mirror if `mirror`
template <typename T> static cudaError_t alloc(CerbHandle *h, Resident<T> &a, size_t per, bool mirror = false) {
    a.per = per;
    const cudaError_t e = dmalloc(h, &a.d, (size_t)h->B * per);
    return (e != cudaSuccess || !mirror) ? e : hmalloc(h, &a.h, (size_t)h->B * per);
}

static int create_impl(CerbHandle *h, const CerbSolverConfig *cfg, const cudaDeviceProp &prop) {
    h->cfg = *cfg; h->sm_count = prop.multiProcessorCount;
    // Test hooks of the Ceres LINEAR_SOLVER_FAILURE path (tests/test_solver_failure.py); unset in production.  A factorisation of
    // J^T J + 1e-8 D^2 practically never fails in fp64, so the in-step mu retry of DoglegStrategy can only be exercised by injection.
    if (const char *e = std::getenv("CERB_TEST_FAIL_FACTORIZATIONS")) h->test_fail_factorizations = std::atoi(e);
    if (const char *e = std::getenv("CERB_TEST_INITIAL_MU")) h->test_initial_mu = std::atof(e);
    h->B = cfg->max_batch; h->F = cfg->max_features; h->O = cfg->max_obs;
    h->grid = std::min(h->B, h->sm_count);
    h->smem_bytes = (size_t)SMEM_DOUBLES * sizeof(double);
    if (h->smem_bytes > prop.sharedMemPerBlockOptin) return fail(CERB_ERR_CUDA, "solve kernel needs more shared memory than the device offers");
    CUDA_TRY(cudaFuncSetAttribute(vilo_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_bytes));
    CUDA_TRY(cudaFuncSetAttribute(prior_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(PRIOR_TROWS * PRIOR_TLD * sizeof(double))));
    CUDA_TRY(cudaStreamCreate(&h->stream));
    CUDA_TRY(cudaStreamCreate(&h->copy_stream));
    h->lane[0] = h->stream;
    for (int k = 1; k < CerbHandle::LANES; k++) CUDA_TRY(cudaStreamCreate(&h->lane[k]));
    for (int k = 0; k < CerbHandle::LANES; k++) CUDA_TRY(cudaEventCreate(&h->ev_lane[k]));
    for (int k = 0; k < CerbHandle::MAX_CHUNKS; k++) CUDA_TRY(cudaEventCreate(&h->ev_copy[k]));
    CUDA_TRY(cudaEventCreate(&h->ev0)); CUDA_TRY(cudaEventCreate(&h->ev1));
    const size_t F = h->F, O = h->O;
    h->ws_stride = ws_size(h->F);
    // the resident batch: elements per window, and whether the array has a pinned mirror
    CUDA_TRY(alloc(h, h->rdesc, 1, true)); CUDA_TRY(alloc(h, h->rfeat, F, true)); CUDA_TRY(alloc(h, h->robs, O, true)); CUDA_TRY(alloc(h, h->rstate, 1, true));
    CUDA_TRY(alloc(h, h->rpre, CERB_WINDOW_SIZE * RAW_PRE_STRIDE, true)); CUDA_TRY(alloc(h, h->rlam, F, true)); CUDA_TRY(alloc(h, h->perm, F));
    CUDA_TRY(alloc(h, h->olam, F, true)); CUDA_TRY(alloc(h, h->ostate, ST_STRIDE, true)); CUDA_TRY(alloc(h, h->orep, 1, true));
    CUDA_TRY(alloc(h, h->n_features, 1)); CUDA_TRY(alloc(h, h->feat_start, F)); CUDA_TRY(alloc(h, h->feat_nobs, F)); CUDA_TRY(alloc(h, h->feat_off, F));
    CUDA_TRY(alloc(h, h->flags, 1)); CUDA_TRY(alloc(h, h->obs_stereo, O)); CUDA_TRY(alloc(h, h->prior_meta, PRIOR_META_STRIDE)); CUDA_TRY(alloc(h, h->rep_i, 4));
    CUDA_TRY(alloc(h, h->obs, NOBS_PLANES * O)); CUDA_TRY(alloc(h, h->pre, CERB_WINDOW_SIZE * PRE_STRIDE)); CUDA_TRY(alloc(h, h->sinfo, CERB_WINDOW_SIZE * 961));
    CUDA_TRY(alloc(h, h->prior_J, PRIOR_LD * PRIOR_LD, true)); CUDA_TRY(alloc(h, h->prior_r, PRIOR_LD, true)); CUDA_TRY(alloc(h, h->prior_x0, CERB_MAX_PRIOR_BLOCKS * 9));
    CUDA_TRY(alloc(h, h->prior_Hp, PRIOR_LD * PRIOR_LD));
    CUDA_TRY(alloc(h, h->state, ST_STRIDE)); CUDA_TRY(alloc(h, h->state0, ST_STRIDE)); CUDA_TRY(alloc(h, h->lam, F)); CUDA_TRY(alloc(h, h->lam0, F)); CUDA_TRY(alloc(h, h->rep_d, 2));
    CUDA_TRY(dmalloc(h, &h->d_ws, (size_t)CerbHandle::LANES * h->grid * h->ws_stride)); CUDA_TRY(dmalloc(h, &h->d_dbg, 2 * (NR + F) + 8)); CUDA_TRY(dmalloc(h, &h->d_G, 4));
    CUDA_TRY(dmalloc(h, &h->d_probe_repi, 4)); CUDA_TRY(dmalloc(h, &h->d_probe_repd, 2)); CUDA_TRY(hmalloc(h, &h->h_dbg, 2 * (NR + F) + 8));
    CUDA_TRY(alloc(h, h->pre_slot, CERB_WINDOW_SIZE + 1, true));
    h->nfeat.assign(h->B, 0); h->n0.assign(h->B, 0); h->res_extent.assign(h->B, 0); h->res_prior_valid.assign(h->B, 0); h->res_leg.assign(h->B, 1);
    CUDA_TRY(cudaMemcpy(h->d_G, cfg->g, 3 * sizeof(double), cudaMemcpyHostToDevice));
    return CERB_OK;
}

extern "C" {

void cerb_destroy(CerbHandle *h) {
    if (!h) return;
    cudaSetDevice(h->cfg.device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    for (void *p : h->dev_bufs) cudaFree(p);
    for (auto &c : h->arena) cudaFree(c.first);
    for (auto &r : h->regs) cudaHostUnregister((void *)r.first);
    for (void *p : h->host_bufs) cudaFreeHost(p);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    for (int k = 0; k < CerbHandle::MAX_CHUNKS; k++) if (h->ev_copy[k]) cudaEventDestroy(h->ev_copy[k]);
    for (int k = 0; k < CerbHandle::LANES; k++) if (h->ev_lane[k]) cudaEventDestroy(h->ev_lane[k]);
    for (int k = 1; k < CerbHandle::LANES; k++) if (h->lane[k]) cudaStreamDestroy(h->lane[k]);
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

}  // extern "C"

// ---- host side of an upload: validation + DMA of the caller's arrays as they are ---------------------------------------
// The descriptors are reference-shaped AoS; csrc/pack_kernels.cuh turns them into the solver's HBM layout on the device.  What the host
// does per window is (1) validate the descriptor (the device trusts it), (2) get the bytes across PCIe: straight out of the caller's
// buffers when they lie in memory registered with cerb_register_host_buffer (zero CPU copies; uniformly strided per-window arrays go
// as ONE 2-D copy per array and chunk), else through pinned staging filled with plain memcpy on a few threads.
struct StageJob { void *dst; const void *src; size_t bytes; };
struct DmaOp { void *dst; size_t dpitch; const void *src; size_t spitch, width, height; };
struct UploadPlan { std::vector<StageJob> stage; std::vector<DmaOp> dma; };

static bool in_registered(const CerbHandle *h, const void *p, size_t bytes) {
    const uintptr_t a = (uintptr_t)p;
    for (const auto &r : h->regs) if (a >= r.first && a + bytes <= r.first + r.second) return true;
    return false;
}

// One logical array of windows [w0, w0 + cn): window w holds `rows` rows of width_of(w) bytes, row r at src_of(w) + r * spitch.  Each window's
// slice of the resident array a is split into `rows` rows of equal pitch; the row lands `col` bytes into its device row (or, staged, into the
// same place of the pinned mirror).
template <class T, class SrcOf, class WidthOf>
static void plan_rows(const CerbHandle *h, UploadPlan &pl, int w0, int cn, const Resident<T> &a, size_t col, int rows, size_t spitch, SrcOf src_of, WidthOf width_of) {
    char *dst = (char *)a.at(w0) + col, *stage = (char *)a.h_at(w0) + col;
    const size_t dpitch = a.per * sizeof(T) / rows;
    size_t maxw = 0; bool all_reg = true, uniform = true; int nact = 0;
    ptrdiff_t delta = 0;
    for (int i = 0; i < cn; i++) {
        const size_t wd = width_of(w0 + i);
        if (wd == 0) { uniform = false; continue; }
        nact++;
        maxw = std::max(maxw, wd);
        const char *p = (const char *)src_of(w0 + i);
        if (!in_registered(h, p, (rows - 1) * spitch + wd)) all_reg = false;
        if (i > 0 && width_of(w0 + i - 1) != 0) {
            const ptrdiff_t dl = p - (const char *)src_of(w0 + i - 1);
            if (i == 1) delta = dl; else if (dl != delta) uniform = false;
        }
    }
    if (nact == 0) return;
    if (all_reg) {
        const char *p0 = (const char *)src_of(w0);
        if (uniform && cn > 1 && nact == cn && delta > 0) {
            if (rows == 1 && (size_t)delta >= maxw && in_registered(h, p0, (size_t)delta * (cn - 1) + maxw)) { pl.dma.push_back({dst, dpitch, p0, (size_t)delta, maxw, (size_t)cn}); return; }
            if (rows > 1 && (size_t)delta == rows * spitch && in_registered(h, p0, (size_t)delta * cn - spitch + maxw)) { pl.dma.push_back({dst, dpitch, p0, spitch, maxw, (size_t)rows * cn}); return; }
        }
        for (int i = 0; i < cn; i++) { const size_t wd = width_of(w0 + i); if (wd) pl.dma.push_back({dst + (size_t)i * rows * dpitch, dpitch, src_of(w0 + i), rows > 1 ? spitch : wd, wd, (size_t)rows}); }
        return;
    }
    for (int i = 0; i < cn; i++) {
        const size_t wd = width_of(w0 + i); if (!wd) continue;
        const char *p = (const char *)src_of(w0 + i);
        for (int r = 0; r < rows; r++) pl.stage.push_back({stage + ((size_t)i * rows + r) * dpitch, p + (size_t)r * spitch, wd});
    }
    pl.dma.push_back({dst, dpitch, stage, dpitch, maxw, (size_t)rows * cn});
}

static int validate_prior(const CerbPrior &pr) {
    if (!pr.valid) return CERB_OK;
    if (pr.n < 1 || pr.n > CERB_MAX_PRIOR_DIM || pr.num_blocks < 1 || pr.num_blocks > CERB_MAX_PRIOR_BLOCKS || !pr.linearized_jacobians || !pr.linearized_residuals)
        return fail(CERB_ERR_BAD_ARGUMENT, "prior: bad n / num_blocks / null matrices");
    bool covered[CERB_MAX_PRIOR_DIM] = {false};          // the kept blocks must tile [0, n) exactly once (the solver's column -> destination map is built from them)
    for (int b = 0; b < pr.num_blocks; b++) {
        for (int c = 0; c < b; c++) if (pr.block_kind[c] == pr.block_kind[b] && pr.block_index[c] == pr.block_index[b]) return fail(CERB_ERR_BAD_ARGUMENT, "prior: duplicate parameter block");
        const int kind = pr.block_kind[b], index = pr.block_index[b];
        if (kind < 0 || kind > 4 || index < 0 || index > 10 || ((kind == CERB_BLOCK_EX_POSE) && index > 1)) return fail(CERB_ERR_BAD_ARGUMENT, "prior: bad block");
        // the solver keeps Hyy block tridiagonal: a prior may only keep the speed/leg bias of frame 0 (what
        // MARGIN_OLD / MARGIN_SECOND_NEW produce, estimator.cpp:1253-1401)
        if ((kind == CERB_BLOCK_SPEEDBIAS || kind == CERB_BLOCK_LEGBIAS) && index != 0) return fail(CERB_ERR_BAD_ARGUMENT, "prior keeps a speed/leg bias block of a frame other than 0");
        const int size = prior_block_size(kind), local = size == 7 ? 6 : size;
        if (pr.block_col[b] < 0 || pr.block_col[b] + local > pr.n) return fail(CERB_ERR_BAD_ARGUMENT, "prior: block column out of range");
        for (int k = 0; k < local; k++) { if (covered[pr.block_col[b] + k]) return fail(CERB_ERR_BAD_ARGUMENT, "prior: overlapping block columns"); covered[pr.block_col[b] + k] = true; }
    }
    for (int k = 0; k < pr.n; k++) if (!covered[k]) return fail(CERB_ERR_BAD_ARGUMENT, "prior: the kept blocks do not cover all n columns");
    return CERB_OK;
}

// the tracks of a feature list against an observation array of obs_bound records; *n_anchor0: tracks anchored at frame 0
static int validate_tracks(const CerbWindowDesc &d, int obs_bound, int *n_anchor0) {
    int n0 = 0;
    for (int f = 0; f < d.n_features; f++) {
        const CerbFeature &ft = d.features[f];
        if (ft.start_frame < 0 || ft.n_obs < 1 || ft.start_frame + ft.n_obs > CERB_NUM_FRAMES || ft.obs_offset < 0 || ft.obs_offset + ft.n_obs > obs_bound)
            return fail(CERB_ERR_BAD_ARGUMENT, "window: malformed feature track");
        n0 += ft.start_frame == 0;
    }
    if (n_anchor0) *n_anchor0 = n0;
    return CERB_OK;
}
static int validate_window(const CerbHandle *h, const CerbWindowDesc &d, const CerbWindowState &st, int *n_anchor0) {
    if (d.n_features < 0 || d.n_features > h->F) return fail(CERB_ERR_BAD_ARGUMENT, "window: n_features over capacity");
    if (d.n_obs < 0 || d.n_obs > h->O) return fail(CERB_ERR_BAD_ARGUMENT, "window: n_obs over capacity");
    if ((d.n_features && (!d.features || !d.obs || !st.para_Feature)) || (!d.preint && !d.imu_preint)) return fail(CERB_ERR_BAD_ARGUMENT, "window: null pointer");
    const int rc = validate_tracks(d, d.n_obs, n_anchor0); if (rc) return rc;
    return validate_prior(d.prior);
}

// fn(k) for k in [0, n), round robin over min(hardware threads, 16) host threads, or on the calling thread alone unless `wide`.  A thread stops
// at its first failure (non-zero return); the first failing thread's code and message are returned.
template <class Fn> static int fan_out(int n, bool wide, Fn fn) {
    const unsigned hw = wide ? std::thread::hardware_concurrency() : 1;       // a system call: kept off the per-chunk path when nothing is staged
    const int nth = (int)std::min<unsigned>(hw ? hw : 1, 16u);
    std::vector<int> rcs(nth, CERB_OK); std::vector<std::string> errs(nth);
    auto work = [&](int t) { for (int k = t; k < n; k += nth) { const int rc = fn(k); if (rc) { rcs[t] = rc; errs[t] = g_err; return; } } };
    std::vector<std::thread> th;
    for (int t = 1; t < nth; t++) th.emplace_back(work, t);
    work(0);
    for (auto &t : th) t.join();
    for (int t = 0; t < nth; t++) if (rcs[t]) return fail(rcs[t], errs[t]);
    return CERB_OK;
}

static void run_stage_jobs(const std::vector<StageJob> &jobs) {
    if (jobs.empty()) return;
    size_t total = 0; for (const auto &j : jobs) total += j.bytes;
    fan_out((int)jobs.size(), total >= (4u << 20), [&](int k) { std::memcpy(jobs[k].dst, jobs[k].src, jobs[k].bytes); return (int)CERB_OK; });
}

// stage what the plan stages, then issue its DMA operations on stream s
static int run_plan(CerbHandle *h, const UploadPlan &pl, cudaStream_t s, double *t_stage_ms) {
    const auto t0 = std::chrono::steady_clock::now();
    run_stage_jobs(pl.stage);
    if (t_stage_ms) *t_stage_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    for (const DmaOp &op : pl.dma) {
        h->traffic.count(cudaMemcpyHostToDevice, op.width * op.height);
        if (op.height == 1) CUDA_TRY(cudaMemcpyAsync(op.dst, op.src, op.width, cudaMemcpyHostToDevice, s));
        else CUDA_TRY(cudaMemcpy2DAsync(op.dst, op.dpitch, op.src, op.spitch, op.width, op.height, cudaMemcpyHostToDevice, s));
    }
    const size_t staged = [&] { size_t t = 0; for (const auto &j : pl.stage) t += j.bytes; return t; }();
    h->last_dma_ops += (int)pl.dma.size(); h->last_staged_bytes += staged; h->traffic.staged += (int64_t)staged;
    return CERB_OK;
}

// validate windows [w0, w0 + cn), move their raw descriptors to the device on stream s (staging only what is not registered)
static int upload_raw(CerbHandle *h, int w0, int cn, const CerbWindowDesc *descs, const CerbWindowState *states, cudaStream_t s, double *t_stage_ms) {
    for (int w = w0; w < w0 + cn; w++) { int rc = validate_window(h, descs[w], states[w], &h->n0[w]); if (rc) return rc; h->nfeat[w] = descs[w].n_features; }
    h->res_n = 0; h->prior_gathered = h->prior_gather_due = false;       // robs / rpre / the prior are overwritten: the resident sliding window, if there was one, is gone
    UploadPlan pl;
    plan_rows(h, pl, w0, cn, h->rdesc, 0, 1, 0, [&](int w) { return (const void *)&descs[w]; }, [&](int) { return sizeof(CerbWindowDesc); });
    plan_rows(h, pl, w0, cn, h->rstate, 0, 1, 0, [&](int w) { return (const void *)&states[w]; }, [&](int) { return sizeof(CerbWindowState); });
    plan_rows(h, pl, w0, cn, h->rfeat, 0, 1, 0,
              [&](int w) { return (const void *)descs[w].features; }, [&](int w) { return (size_t)descs[w].n_features * sizeof(CerbFeature); });
    plan_rows(h, pl, w0, cn, h->robs, 0, 1, 0,
              [&](int w) { return (const void *)descs[w].obs; }, [&](int w) { return (size_t)descs[w].n_obs * sizeof(CerbObservation); });
    plan_rows(h, pl, w0, cn, h->rlam, 0, 1, 0,
              [&](int w) { return (const void *)states[w].para_Feature; }, [&](int w) { return (size_t)descs[w].n_features * 8; });
    // preintegration results, one row per factor: the members IMULegFactor::Evaluate reads -- head (33 doubles) and, contiguous in the struct,
    // jacobian columns 21..30 + covariance
    const size_t tail_off = (size_t)(RAW_PRE_HEAD + RAW_PRE_JCOL0 * 31) * 8, tail_w = sizeof(CerbIMULegPreint) - tail_off;
    static_assert(sizeof(CerbIMULegPreint) == (33 + 2 * 961) * 8, "CerbIMULegPreint layout");
    static_assert(sizeof(CerbIMUPreint) == 467 * 8 && sizeof(CerbIMUPreint) <= RAW_PRE_STRIDE * 8, "CerbIMUPreint layout");
    plan_rows(h, pl, w0, cn, h->rpre, 0, CERB_WINDOW_SIZE, sizeof(CerbIMULegPreint),
              [&](int w) { return (const void *)descs[w].preint; }, [&](int w) { return descs[w].preint ? (size_t)RAW_PRE_HEAD * 8 : (size_t)0; });
    plan_rows(h, pl, w0, cn, h->rpre, RAW_PRE_HEAD * 8, CERB_WINDOW_SIZE, sizeof(CerbIMULegPreint),
              [&](int w) { return (const void *)((const char *)descs[w].preint + tail_off); }, [&](int w) { return descs[w].preint ? tail_w : (size_t)0; });
    plan_rows(h, pl, w0, cn, h->rpre, 0, CERB_WINDOW_SIZE, sizeof(CerbIMUPreint),
              [&](int w) { return (const void *)descs[w].imu_preint; }, [&](int w) { return descs[w].preint ? (size_t)0 : sizeof(CerbIMUPreint); });
    plan_rows(h, pl, w0, cn, h->prior_J, 0, 1, 0,
              [&](int w) { return (const void *)descs[w].prior.linearized_jacobians; }, [&](int w) { return descs[w].prior.valid ? (size_t)descs[w].prior.n * descs[w].prior.n * 8 : (size_t)0; });
    plan_rows(h, pl, w0, cn, h->prior_r, 0, 1, 0,
              [&](int w) { return (const void *)descs[w].prior.linearized_residuals; }, [&](int w) { return descs[w].prior.valid ? (size_t)descs[w].prior.n * 8 : (size_t)0; });
    return run_plan(h, pl, s, t_stage_ms);
}

// device pack of windows [w0, w0 + cn) (after their raw descriptors have arrived) on stream s
static int enqueue_pack(CerbHandle *h, int w0, int cn, cudaStream_t s) {
    PackParams P;
    P.n = cn; P.maxF = h->F; P.maxObs = h->O;
    P.rdesc = h->rdesc.at(w0); P.rfeat = h->rfeat.at(w0); P.robs = h->robs.at(w0); P.rpre = h->rpre.at(w0); P.rstate = h->rstate.at(w0); P.rlam = h->rlam.at(w0);
    P.n_features = h->n_features.at(w0); P.feat_start = h->feat_start.at(w0); P.feat_nobs = h->feat_nobs.at(w0); P.feat_off = h->feat_off.at(w0); P.flags = h->flags.at(w0);
    P.obs_stereo = h->obs_stereo.at(w0); P.prior_meta = h->prior_meta.at(w0); P.perm = h->perm.at(w0);
    P.obs = h->obs.at(w0); P.pre = h->pre.at(w0); P.prior_x0 = h->prior_x0.at(w0); P.state0 = h->state0.at(w0); P.lam0 = h->lam0.at(w0);
    if (h->res_n) { P.pre_slot = h->pre_slot.d; P.window = h->pre_slot.d + (size_t)cn * CERB_WINDOW_SIZE; }      // a resident batch is packed whole (w0 = 0)
    CERB_LAUNCH(pack_kernel, std::min(cn, 8 * h->sm_count), PACK_THREADS, 0, s, P);
    CUDA_TRY(cudaGetLastError());
    return CERB_OK;
}
static int upload(CerbHandle *h, int n, const CerbWindowDesc *descs, const CerbWindowState *states) {
    h->last_dma_ops = 0; h->last_staged_bytes = 0;
    int rc = upload_raw(h, 0, n, descs, states, h->stream, nullptr); if (rc) return rc;
    rc = enqueue_pack(h, 0, n, h->stream); if (rc) return rc;
    h->n = n; h->solved = false; h->perm_valid = false;
    return CERB_OK;
}
// device slot -> caller's feature index of the resident batch (computed by the pack kernel; fetched on demand by the probes / feature passes)
static int ensure_perm(CerbHandle *h) {
    if (h->perm_valid) return CERB_OK;
    h->h_perm.resize((size_t)h->B * h->perm.per);
    CUDA_TRY(cudaMemcpyAsync(h->h_perm.data(), h->perm.d, h->perm.bytes(h->n), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    h->perm_valid = true;
    return CERB_OK;
}

// the prior matrices and residuals of the batch by row: the store, or the per-step copy of a compact batch of resident windows
static const Resident<double> &batch_prior_J(const CerbHandle *h) { return h->prior_gathered ? h->step_J : h->prior_J; }
static const Resident<double> &batch_prior_r(const CerbHandle *h) { return h->prior_gathered ? h->step_r : h->prior_r; }

static SolveParams make_params(CerbHandle *h, int w0, int n, int max_iters, double *dbg, int dbg_window) {
    SolveParams P;
    std::memset(&P, 0, sizeof(P));
    const CerbSolverConfig &c = h->cfg;
    P.n_windows = n; P.maxF = h->F; P.maxObs = h->O; P.max_iters = max_iters; P.optimize_leg_bias = c.optimize_leg_bias;
    for (int k = 0; k < 3; k++) P.G[k] = c.g[k];
    P.sqrt_info = c.visual_sqrt_info; P.huber = c.huber_delta;
    P.radius0 = c.initial_trust_region_radius; P.max_radius = c.max_trust_region_radius; P.min_radius = c.min_trust_region_radius;
    P.min_rel_dec = c.min_relative_decrease; P.ftol = c.function_tolerance; P.gtol = c.gradient_tolerance; P.ptol = c.parameter_tolerance;
    P.n_features = h->n_features.at(w0); P.feat_start = h->feat_start.at(w0); P.feat_nobs = h->feat_nobs.at(w0); P.feat_off = h->feat_off.at(w0); P.flags = h->flags.at(w0);
    P.obs = h->obs.at(w0); P.obs_stereo = h->obs_stereo.at(w0); P.pre = h->pre.at(w0); P.sinfo = h->sinfo.at(w0);
    P.prior_J = batch_prior_J(h).at(w0); P.prior_r = batch_prior_r(h).at(w0); P.prior_x0 = h->prior_x0.at(w0); P.prior_Hp = h->prior_Hp.at(w0); P.prior_meta = h->prior_meta.at(w0);
    P.state = h->state.at(w0); P.lam = h->lam.at(w0); P.rep_i = h->rep_i.at(w0); P.rep_d = h->rep_d.at(w0); P.ws = h->d_ws; P.ws_stride = h->ws_stride;
    P.dbg = dbg; P.dbg_window = dbg_window;
    P.test_fail_factorizations = h->test_fail_factorizations; P.test_initial_mu = h->test_initial_mu;
    P.no_bulk_copy = std::getenv("CERB_NO_TMA") != nullptr;
    return P;
}

// sqrt_info of the IMU-leg factors and the Gram matrix of the prior of windows [w0, w0 + n), on stream s
static void enqueue_prepare(CerbHandle *h, int w0, int n, cudaStream_t s) {
    const int nfac = n * CERB_WINDOW_SIZE;
    CERB_LAUNCH(imu_leg_prepare_kernel, (nfac + 1) / 2, 64, 0, s, nfac, (const double *)h->pre.at(w0), h->sinfo.at(w0));
    CERB_LAUNCH(prior_prepare_kernel, n, 256, (size_t)PRIOR_TROWS * PRIOR_TLD * sizeof(double), s, (const double *)batch_prior_J(h).at(w0), (const int *)h->prior_meta.at(w0), h->prior_Hp.at(w0));
}

// a compact batch of resident windows: the listed windows' priors into the per-step area, once per upload, on stream s
static int gather_priors(CerbHandle *h, cudaStream_t s) {
    if (!h->prior_gather_due) return CERB_OK;
    const int n = h->n;
    CERB_LAUNCH(prior_gather_kernel, std::min(n, 8 * h->sm_count), 256, 0, s, n, (const int *)(h->pre_slot.d + (size_t)n * CERB_WINDOW_SIZE), (const CerbWindowDesc *)h->rdesc.d,
                (const double *)h->prior_J.d, (const double *)h->prior_r.d, h->step_J.d, h->step_r.d);
    CUDA_TRY(cudaGetLastError());
    h->prior_gather_due = false;
    return CERB_OK;
}

// restore the initial states of windows [w0, w0 + n), prepare (sqrt_info, prior Gram matrix) and solve; asynchronous on the stream
static int enqueue_solve(CerbHandle *h, int w0, int n, int max_iters, double *dbg, int dbg_window, bool restore = true, bool probe = false, int lane = 0) {
    cudaStream_t s = h->lane[lane];
    if (restore) {
        CUDA_TRY(cudaMemcpyAsync(h->state.at(w0), h->state0.at(w0), h->state.bytes(n), cudaMemcpyDeviceToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(h->lam.at(w0), h->lam0.at(w0), h->lam.bytes(n), cudaMemcpyDeviceToDevice, s));
    }
    int rc = gather_priors(h, s); if (rc) return rc;
    enqueue_prepare(h, w0, n, s);
    SolveParams P = make_params(h, w0, n, max_iters, dbg, dbg_window);
    P.ws = h->d_ws + (size_t)lane * h->grid * h->ws_stride;                      // kernels of different lanes run concurrently: one workspace slice each
    if (probe) { P.rep_i = h->d_probe_repi; P.rep_d = h->d_probe_repd; }       // a probe leaves the reports of the batch alone
    if (max_iters > 0) h->solved = true;
    CERB_LAUNCH(vilo_solve_kernel, std::min(n, h->grid), SOLVE_THREADS, h->smem_bytes, s, P);
    CUDA_TRY(cudaGetLastError());
    return CERB_OK;
}
static int launch_solve(CerbHandle *h, int max_iters, double *dbg, int dbg_window, bool timed) {
    const int n = h->n;
    if (n < 1) return fail(CERB_ERR_BAD_ARGUMENT, "no resident batch");
    if (timed) CUDA_TRY(cudaEventRecord(h->ev0, h->stream));
    int rc = enqueue_solve(h, 0, n, max_iters, dbg, dbg_window); if (rc) return rc;
    if (timed) { CUDA_TRY(cudaEventRecord(h->ev1, h->stream)); h->ev_pending = true; h->last_launches = 3; }
    return CERB_OK;
}

static int collect_time(CerbHandle *h) {
    if (h->ev_pending) {
        CUDA_TRY(cudaEventSynchronize(h->ev1));
        float ms = 0; CUDA_TRY(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
        h->last_ms = ms; h->ev_pending = false;
    }
    return CERB_OK;
}

// a batch of states in device layout: state [n][ST_STRIDE], lam [n][F] in device feature order
struct States { Resident<double> state, lam; };
// the current states of the resident batch: the solved ones after a solve, else the uploaded (or cerb_batch_update_states') initial ones
static States resident_states(const CerbHandle *h) { return h->solved ? States{h->state, h->lam} : States{h->state0, h->lam0}; }

static int download(CerbHandle *h, CerbWindowState *states, CerbSolveReport *reports) {
    const int n = h->n;
    cudaStream_t s = h->stream;
    const States cur = resident_states(h);
    UnpackParams U;
    U.n = n; U.maxF = h->F; U.n_features = h->n_features.d; U.perm = h->perm.d; U.rep_i = h->rep_i.d; U.rep_d = h->rep_d.d;
    U.lam = cur.lam.d; U.state = cur.state.d;
    U.olam = h->olam.d; U.orep = h->orep.d; U.ostate = h->ostate.d;
    CERB_LAUNCH(unpack_kernel, std::min(n, 8 * h->sm_count), PACK_THREADS, 0, s, U);
    CUDA_TRY(cudaGetLastError());
    COPY_TRY(h, h->ostate.h, h->ostate.d, h->ostate.bytes(n), cudaMemcpyDeviceToHost, s);
    COPY_TRY(h, h->olam.h, h->olam.d, h->olam.bytes(n), cudaMemcpyDeviceToHost, s);
    COPY_TRY(h, h->orep.h, h->orep.d, h->orep.bytes(n), cudaMemcpyDeviceToHost, s);
    CUDA_TRY(cudaStreamSynchronize(s));
    int rc = collect_time(h); if (rc) return rc;
    int status = CERB_OK;
    for (int w = 0; w < n; w++) {
        if (states) {
            std::memcpy(&states[w], h->ostate.h_at(w), ST_SIZE * sizeof(double));        // para_Pose .. para_Td: contiguous, same order
            if (states[w].para_Feature && h->nfeat[w]) std::memcpy(states[w].para_Feature, h->olam.h_at(w), (size_t)h->nfeat[w] * sizeof(double));
        }
        if (reports) reports[w] = h->orep.h[w];
        if (h->orep.h[w].status != 0) status = CERB_ERR_NON_FINITE;
    }
    if (status) return fail(status, "at least one window produced a non-finite cost (see reports[].status)");
    return CERB_OK;
}

extern "C" {

int cerb_register_host_buffer(CerbHandle *h, void *ptr, size_t bytes) {
    if (!h || !ptr || !bytes) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_register_host_buffer: null argument");
    CERB_DEVICE(h);
    CUDA_TRY(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
    h->regs.emplace_back((uintptr_t)ptr, bytes);
    return CERB_OK;
}
int cerb_unregister_host_buffer(CerbHandle *h, void *ptr) {
    if (!h || !ptr) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_unregister_host_buffer: null argument");
    CERB_DEVICE(h);
    for (size_t k = 0; k < h->regs.size(); k++) if (h->regs[k].first == (uintptr_t)ptr) {
        CUDA_TRY(cudaStreamSynchronize(h->stream)); CUDA_TRY(cudaStreamSynchronize(h->copy_stream));
        CUDA_TRY(cudaHostUnregister(ptr));
        h->regs.erase(h->regs.begin() + k);
        return CERB_OK;
    }
    return fail(CERB_ERR_BAD_ARGUMENT, "cerb_unregister_host_buffer: not registered with this handle");
}

int cerb_batch_upload(CerbHandle *h, int32_t n, const CerbWindowDesc *descs, const CerbWindowState *states) {
    if (!h || !descs || !states) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    CERB_DEVICE(h);
    if (n < 1 || n > h->B) return fail(CERB_ERR_BAD_ARGUMENT, "batch size over capacity");
    CUDA_TRY(cudaStreamSynchronize(h->stream));          // staging buffers may still be in flight
    return upload(h, n, descs, states);
}
int cerb_batch_solve_resident(CerbHandle *h) {
    if (!h) return fail(CERB_ERR_BAD_ARGUMENT, "null handle");
    CERB_DEVICE(h);
    int rc = collect_time(h); if (rc) return rc;
    return launch_solve(h, h->cfg.max_num_iterations, nullptr, -1, true);
}
int cerb_batch_download(CerbHandle *h, CerbWindowState *states, CerbSolveReport *reports) {
    if (!h) return fail(CERB_ERR_BAD_ARGUMENT, "null handle");
    CERB_DEVICE(h);
    return download(h, states, reports);
}
int cerb_sync(CerbHandle *h) {
    if (!h) return fail(CERB_ERR_BAD_ARGUMENT, "null handle");
    CERB_DEVICE(h);
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    return collect_time(h);
}
int cerb_last_solve_stats(CerbHandle *h, double *kernel_ms, int32_t *kernel_launches) {
    if (!h) return fail(CERB_ERR_BAD_ARGUMENT, "null handle");
    CERB_DEVICE(h);
    int rc = collect_time(h); if (rc) return rc;
    if (kernel_ms) *kernel_ms = h->last_ms;
    if (kernel_launches) *kernel_launches = h->last_launches;
    return CERB_OK;
}
int cerb_last_upload_stats(CerbHandle *h, int32_t *dma_ops, int64_t *staged_bytes) {
    if (!h) return fail(CERB_ERR_BAD_ARGUMENT, "null handle");
    if (dma_ops) *dma_ops = h->last_dma_ops;
    if (staged_bytes) *staged_bytes = (int64_t)h->last_staged_bytes;
    return CERB_OK;
}
int cerb_solve_batch(CerbHandle *h, int32_t n, const CerbWindowDesc *descs, CerbWindowState *states, CerbSolveReport *reports) {
    if (!h || !descs || !states) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    CERB_DEVICE(h);
    if (n < 1 || n > h->B) return fail(CERB_ERR_BAD_ARGUMENT, "batch size over capacity");
    CUDA_TRY(cudaStreamSynchronize(h->stream)); CUDA_TRY(cudaStreamSynchronize(h->copy_stream));
    for (int l = 1; l < CerbHandle::LANES; l++) CUDA_TRY(cudaStreamSynchronize(h->lane[l]));       // only busy after a call that failed half way
    int rc = collect_time(h); if (rc) return rc;
    // Pipeline in chunks: the copy stream moves chunk c + 1 (and the host stages it, if its buffers are not registered) while the compute lanes pack
    // and solve the chunks that have arrived.  Three lanes (streams) take the chunks round-robin and their kernels run concurrently, so a chunk's CTAs
    // fill the SMs as earlier windows retire -- no wave alignment, whatever the batch size is relative to the SM count.  Chunk sizes ramp up (64, 64,
    // 128, 256, 256, ...): the GPU starts after the first 64 windows (19 MB at F = 150) are across, and every later chunk arrives before the SMs run dry
    // while the number of launches / DMA operations stays small (measured: sixteen equal chunks of 64 lose more to their prepare kernels than they gain).
    const int MAXC = CerbHandle::MAX_CHUNKS;
    int NL = 3, first = 64;
    if (const char *e = std::getenv("CERB_PIPE_LANES")) NL = std::min((int)CerbHandle::LANES, std::max(1, std::atoi(e)));       // tuning knobs of the measurement in DESIGN.md 2.4
    if (const char *e = std::getenv("CERB_PIPE_FIRST")) first = std::max(1, std::atoi(e));
    int bounds[CerbHandle::MAX_CHUNKS + 1], nch = 0; bounds[0] = 0;
    if (const char *e = std::getenv("CERB_TEST_CHUNK")) {              // test hook: the multi-chunk / multi-lane path on a handful of windows
        const int per = std::max(std::max(1, std::atoi(e)), (n + MAXC - 1) / MAXC);
        for (int pos = 0; pos < n; ) { pos = std::min(n, pos + per); bounds[++nch] = pos; }
    } else if (n <= first + first / 2) { bounds[1] = n; nch = 1; }
    else {
        int cap = 4 * first;
        if ((n + cap - 1) / cap > MAXC - 8) cap = (((n + MAXC - 9) / (MAXC - 8)) + first - 1) / first * first;
        int pos = 0, sz = first, k = 0;
        while (pos < n) {
            int take = std::min(sz, n - pos);
            if (n - pos - take < first / 2 || nch == MAXC - 1) take = n - pos;  // no crumbs; never more than MAXC chunks
            pos += take; bounds[++nch] = pos;
            if (++k >= 2) sz = std::min(cap, 2 * sz);
        }
    }
    h->n = n; h->perm_valid = false;
    h->last_dma_ops = 0; h->last_staged_bytes = 0;
    const bool trace = std::getenv("CERB_TRACE") != nullptr;            // host timeline of the pipeline on stderr (diagnostics)
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_begin = now(); double t_stage = 0.0;
    CUDA_TRY(cudaEventRecord(h->ev0, h->stream));
    for (int l = 1; l < NL; l++) CUDA_TRY(cudaStreamWaitEvent(h->lane[l], h->ev0, 0));
    // a descriptor rejected in a later chunk: drain what the earlier chunks have in flight before the caller sees the error (its buffers may go away)
    auto drain = [&](int code) { for (int l = 0; l < NL; l++) cudaStreamSynchronize(h->lane[l]); cudaStreamSynchronize(h->copy_stream); return code; };
    for (int c = 0; c < nch; c++) {
        const int w0 = bounds[c], cn = bounds[c + 1] - bounds[c], l = c % NL;
        rc = upload_raw(h, w0, cn, descs, states, h->copy_stream, &t_stage); if (rc) return drain(rc);
        CUDA_TRY(cudaEventRecord(h->ev_copy[c], h->copy_stream));
        CUDA_TRY(cudaStreamWaitEvent(h->lane[l], h->ev_copy[c], 0));
        rc = enqueue_pack(h, w0, cn, h->lane[l]); if (rc) return drain(rc);
        rc = enqueue_solve(h, w0, cn, h->cfg.max_num_iterations, nullptr, -1, true, false, l); if (rc) return drain(rc);
    }
    for (int l = 1; l < NL; l++) { CUDA_TRY(cudaEventRecord(h->ev_lane[l], h->lane[l])); CUDA_TRY(cudaStreamWaitEvent(h->stream, h->ev_lane[l], 0)); }
    CUDA_TRY(cudaEventRecord(h->ev1, h->stream)); h->ev_pending = true; h->last_launches = 4 * nch + 1;      // + the unpack kernel of the download
    const double t_issued = now();
    rc = download(h, states, reports);
    if (trace) std::fprintf(stderr, "[cerb_solve_batch] n=%d chunks=%d dma ops %d, staged %.1f MB in %.2f ms, all issued at %.2f ms, done at %.2f ms\n", n, nch, h->last_dma_ops,
                            h->last_staged_bytes / 1e6, t_stage, t_issued - t_begin, now() - t_begin);
    return rc;
}
int cerb_solve_window(CerbHandle *h, const CerbWindowDesc *desc, CerbWindowState *state, CerbSolveReport *report) {
    return cerb_solve_batch(h, 1, desc, state, report);
}

int cerb_debug_linearize(CerbHandle *h, int32_t w, double *cost, double *gradient, double *jtj_diag, int32_t n_alloc) {
    if (!h || w < 0 || w >= h->n) return fail(CERB_ERR_BAD_ARGUMENT, "bad window index");
    CERB_DEVICE(h);
    const int nf = h->nfeat[w], F = h->F;
    if (n_alloc < NR + nf) return fail(CERB_ERR_BAD_ARGUMENT, "n_alloc too small");
    int rc = ensure_perm(h); if (rc) return rc;
    const size_t cnt = 2 * (size_t)(NR + F) + 8;
    CUDA_TRY(cudaMemsetAsync(h->d_dbg, 0, cnt * sizeof(double), h->stream));
    // Read-only with respect to the resident batch: only window w is linearised, at the solved states if the batch has been solved
    // (else at the uploaded initial states, which are first copied into place), with the reports going to scratch.
    rc = enqueue_solve(h, w, 1, 0, h->d_dbg, 0, !h->solved, true); if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(h->h_dbg, h->d_dbg, cnt * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    if (cost) *cost = h->h_dbg[0];
    const int *perm = h->h_perm.data() + (size_t)w * F;
    for (int k = 0; k < NR + nf; k++) {
        const int dst = k < NR ? k : NR + perm[k - NR];          // device feature slot -> caller's feature index
        if (gradient) gradient[dst] = h->h_dbg[1 + k];
        if (jtj_diag) jtj_diag[dst] = h->h_dbg[1 + NR + F + k];
    }
    return CERB_OK;
}

#if defined(CERB_PHASE_TIMING) && !defined(CERB_CUSIM)
// tools/phase_profile.py only (separate library build): read and reset the per-phase cycle counters of the solve kernel
extern "C" int cerb_prof_phase_cycles(unsigned long long *out48) {
    unsigned long long z[48] = {0};
    if (cudaMemcpyFromSymbol(out48, g_phase_cycles, sizeof(z)) != cudaSuccess) return CERB_ERR_CUDA;
    if (cudaMemcpyToSymbol(g_phase_cycles, z, sizeof(z)) != cudaSuccess) return CERB_ERR_CUDA;
    return CERB_OK;
}
#endif

// ---- factor-family evaluators ----------------------------------------------------------------------------------
struct DevBuf {   // bump allocator over the handle's scratch arena (reset per entry point; chunks are kept, so steady state does no cudaMalloc)
    CerbHandle *h;
    explicit DevBuf(CerbHandle *h_) : h(h_) { h->arena_chunk = 0; h->arena_used = 0; }
    void *raw(size_t bytes) {
        bytes = (std::max<size_t>(bytes, 8) + 255) & ~(size_t)255;
        while (h->arena_chunk < h->arena.size() && h->arena_used + bytes > h->arena[h->arena_chunk].second) { h->arena_chunk++; h->arena_used = 0; }
        if (h->arena_chunk == h->arena.size()) {
            const size_t sz = std::max<size_t>(bytes, (size_t)16 << 20);
            char *p = nullptr; if (cudaMalloc((void **)&p, sz) != cudaSuccess) return nullptr;
            h->arena.emplace_back(p, sz); h->arena_used = 0;
        }
        void *r = h->arena[h->arena_chunk].first + h->arena_used; h->arena_used += bytes;
        return r;
    }
    double *up(const double *src, size_t n, cudaStream_t s) {
        double *d = (double *)raw(n * sizeof(double)); if (!d) return nullptr;
        if (src) { h->traffic.count(cudaMemcpyHostToDevice, n * sizeof(double)); cudaMemcpyAsync(d, src, n * sizeof(double), cudaMemcpyHostToDevice, s); }
        return d;
    }
    int *upi(const int *src, size_t n, cudaStream_t s) {
        int *d = (int *)raw(n * sizeof(int)); if (!d) return nullptr;
        if (src) { h->traffic.count(cudaMemcpyHostToDevice, n * sizeof(int)); cudaMemcpyAsync(d, src, n * sizeof(int), cudaMemcpyHostToDevice, s); }
        return d;
    }
};

// host views of the device pack functions (one source of truth for the record layout): used by the evaluator entry points
static void pack_preint(const CerbIMULegPreint &p, double *o) {
    const double *sdb = reinterpret_cast<const double *>(&p);
    std::vector<double> raw(RAW_PRE_STRIDE);
    for (int k = 0; k < RAW_PRE_STRIDE; k++) raw[k] = k < RAW_PRE_HEAD ? sdb[k] : sdb[k + RAW_PRE_JCOL0 * 31];
    for (int k = 0; k < PRE_STRIDE; k++) o[k] = pack_pre_leg(raw.data(), k);
}
static void pack_imu_preint(const CerbIMUPreint &p, double *o) {
    const double *raw = reinterpret_cast<const double *>(&p);
    for (int k = 0; k < PRE_STRIDE; k++) o[k] = pack_pre_imu(raw, k);
}
static const int kImuTo31[15] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 21, 22, 23, 24, 25, 26};
// the prior's record on the device apart from its matrix and residuals: meta (PRIOR_META_STRIDE ints: valid, n, num_blocks, -, then kind /
// index / column of block b at 4 + 3 b) and x0 (9 doubles per block)
static void encode_prior(const CerbPrior &pr, int *meta, double *x0) {
    std::memset(meta, 0, PRIOR_META_STRIDE * sizeof(int));
    if (!pr.valid) return;
    meta[0] = 1; meta[1] = pr.n; meta[2] = pr.num_blocks;
    for (int b = 0; b < pr.num_blocks; b++) {
        meta[4 + 3 * b] = pr.block_kind[b]; meta[5 + 3 * b] = pr.block_index[b]; meta[6 + 3 * b] = pr.block_col[b];
        for (int k = 0; k < 9; k++) x0[9 * b + k] = pr.block_x0[b][k];
    }
}
static void decode_prior(const int *meta, const double *x0, CerbPrior &pr) {
    pr.valid = 0; pr.n = 0; pr.num_blocks = 0;
    if (!meta[0]) return;
    pr.valid = 1; pr.n = meta[1]; pr.num_blocks = meta[2];
    for (int b = 0; b < pr.num_blocks; b++) {
        pr.block_kind[b] = meta[4 + 3 * b]; pr.block_index[b] = meta[5 + 3 * b]; pr.block_col[b] = meta[6 + 3 * b];
        for (int k = 0; k < 9; k++) pr.block_x0[b][k] = x0[9 * b + k];
    }
}


int cerb_eval_projection(CerbHandle *h, int32_t kind, int32_t n, const double *pose_i, const double *pose_j, const double *ex0, const double *ex1,
                         const double *inv_dep, const double *td, const double *pts_i, const double *pts_j, const double *vel_i, const double *vel_j,
                         const double *td_i, const double *td_j, double *residuals, double *jacobians) {
    if (!h || n < 1 || kind < 0 || kind > 2 || !ex0 || !inv_dep || !td || !pts_i || !pts_j || !vel_i || !vel_j || !td_i || !td_j) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_eval_projection: bad argument");
    CERB_DEVICE(h);
    if (kind != CERB_PROJ_ONE_FRAME_TWO_CAM && (!pose_i || !pose_j)) return fail(CERB_ERR_BAD_ARGUMENT, "poses required");
    if (kind != CERB_PROJ_TWO_FRAME_ONE_CAM && !ex1) return fail(CERB_ERR_BAD_ARGUMENT, "ex1 required");
    cudaStream_t s = h->stream; DevBuf B(h); const size_t N = n;
    const int JS = kind == 0 ? 46 : (kind == 1 ? 60 : 32);
    double *dpi = pose_i ? B.up(pose_i, 7 * N, s) : nullptr, *dpj = pose_j ? B.up(pose_j, 7 * N, s) : nullptr;
    double *de0 = B.up(ex0, 7 * N, s), *de1 = ex1 ? B.up(ex1, 7 * N, s) : nullptr;
    double *dl = B.up(inv_dep, N, s), *dtd = B.up(td, N, s), *dpti = B.up(pts_i, 3 * N, s), *dptj = B.up(pts_j, 3 * N, s);
    double *dvi = B.up(vel_i, 2 * N, s), *dvj = B.up(vel_j, 2 * N, s), *dti = B.up(td_i, N, s), *dtj = B.up(td_j, N, s);
    double *dr = B.up(nullptr, 2 * N, s), *dJ = jacobians ? B.up(nullptr, JS * N, s) : nullptr;
    if (!dr || !dtj) return fail(CERB_ERR_CUDA, "device allocation failed");
    CERB_LAUNCH(projection_eval_kernel, (n + 127) / 128, 128, 0, s, (int)kind, (int)n, (const double *)dpi, (const double *)dpj, (const double *)de0, (const double *)de1,
                (const double *)dl, (const double *)dtd, (const double *)dpti, (const double *)dptj, (const double *)dvi, (const double *)dvj, (const double *)dti,
                (const double *)dtj, h->cfg.visual_sqrt_info, dr, dJ);
    CUDA_TRY(cudaGetLastError());
    if (residuals) CUDA_TRY(cudaMemcpyAsync(residuals, dr, 2 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (jacobians) CUDA_TRY(cudaMemcpyAsync(jacobians, dJ, JS * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return CERB_OK;
}

// IMU-leg factors of n packed preintegration records (PRE_STRIDE each) and parameter rows (40 each): residuals [n][31], Jacobians [n][31 x 40]
// and sqrt_info [n][961] into the host arrays that are not null
static int eval_imu_leg_packed(CerbHandle *h, int n, const double *packed, const double *params, double *residuals, double *jacobians, double *sqrt_info) {
    cudaStream_t s = h->stream; DevBuf B(h); const size_t N = n;
    double *dpre = B.up(packed, N * PRE_STRIDE, s), *dsi = B.up(nullptr, N * 961, s), *dpar = B.up(params, 40 * N, s);
    double *dr = B.up(nullptr, 31 * N, s), *dJ = jacobians ? B.up(nullptr, 31 * 40 * N, s) : nullptr;
    if (!dpre || !dsi || !dpar || !dr) return fail(CERB_ERR_CUDA, "device allocation failed");
    CERB_LAUNCH(imu_leg_prepare_kernel, (n + 1) / 2, 64, 0, s, (int)n, (const double *)dpre, dsi);
    CERB_LAUNCH(imu_leg_eval_kernel, n, 128, 0, s, (int)n, (const double *)dpre, (const double *)dsi, (const double *)dpar, (const double *)h->d_G, dr, dJ);
    CUDA_TRY(cudaGetLastError());
    if (residuals) CUDA_TRY(cudaMemcpyAsync(residuals, dr, 31 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (jacobians) CUDA_TRY(cudaMemcpyAsync(jacobians, dJ, 31 * 40 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (sqrt_info) CUDA_TRY(cudaMemcpyAsync(sqrt_info, dsi, 961 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return CERB_OK;
}

int cerb_eval_imu_leg(CerbHandle *h, int32_t n, const CerbIMULegPreint *preint, const double *params, double *residuals, double *jacobians, double *sqrt_info) {
    if (!h || n < 1 || !preint || !params) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_eval_imu_leg: bad argument");
    CERB_DEVICE(h);
    std::vector<double> packed((size_t)n * PRE_STRIDE, 0.0);
    for (int k = 0; k < n; k++) pack_preint(preint[k], packed.data() + (size_t)k * PRE_STRIDE);
    return eval_imu_leg_packed(h, n, packed.data(), params, residuals, jacobians, sqrt_info);
}

int cerb_eval_imu(CerbHandle *h, int32_t n, const CerbIMUPreint *preint, const double *params, double *residuals, double *jacobians, double *sqrt_info) {
    if (!h || n < 1 || !preint || !params) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_eval_imu: bad argument");
    CERB_DEVICE(h);
    const size_t N = n;
    std::vector<double> packed(N * PRE_STRIDE), p40(N * 40, 0.0);
    for (int k = 0; k < n; k++) {
        pack_imu_preint(preint[k], packed.data() + (size_t)k * PRE_STRIDE);
        const double *q = params + (size_t)k * 32; double *o = p40.data() + (size_t)k * 40;
        std::memcpy(o, q, 16 * sizeof(double)); std::memcpy(o + 20, q + 16, 16 * sizeof(double));     // leg-bias slots stay 0
    }
    std::vector<double> hr(31 * N), hj(jacobians ? 31 * 40 * N : 0), hs(961 * N);
    int rc = eval_imu_leg_packed(h, n, packed.data(), p40.data(), hr.data(), jacobians ? hj.data() : nullptr, hs.data()); if (rc) return rc;
    // gather the 15 rows P, R, V, BA, BG and the blocks pose_i, speedbias_i, pose_j, speedbias_j
    const int boff31[4] = {0, 7, 20, 27}, bsz[4] = {7, 9, 7, 9}, boff15[4] = {0, 7, 16, 23};
    for (int k = 0; k < n; k++) {
        for (int r = 0; r < 15; r++) {
            const int R = kImuTo31[r];
            if (residuals) residuals[(size_t)k * 15 + r] = hr[(size_t)k * 31 + R];
            if (sqrt_info) for (int c = 0; c < 15; c++) sqrt_info[(size_t)k * 225 + r * 15 + c] = hs[(size_t)k * 961 + R * 31 + kImuTo31[c]];
            if (jacobians) for (int b = 0; b < 4; b++) for (int c = 0; c < bsz[b]; c++)
                jacobians[(size_t)k * 15 * 32 + 15 * boff15[b] + r * bsz[b] + c] = hj[(size_t)k * 31 * 40 + 31 * boff31[b] + R * bsz[b] + c];
        }
    }
    return CERB_OK;
}

int cerb_eval_prior(CerbHandle *h, const CerbPrior *prior, const CerbWindowState *state, double *residuals, double *jacobians) {
    if (!h || !prior || !state || !prior->valid || !residuals) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_eval_prior: bad argument");
    CERB_DEVICE(h);
    std::vector<int> meta(PRIOR_META_STRIDE); std::vector<double> J(PRIOR_LD * PRIOR_LD, 0.0), r(PRIOR_LD, 0.0), x0(16 * 9, 0.0), st(ST_STRIDE, 0.0);
    int rc = validate_prior(*prior); if (rc) return rc;
    encode_prior(*prior, meta.data(), x0.data());
    std::memcpy(J.data(), prior->linearized_jacobians, sizeof(double) * prior->n * prior->n);
    std::memcpy(r.data(), prior->linearized_residuals, sizeof(double) * prior->n);
    std::memcpy(st.data() + ST_POSE, state->para_Pose, sizeof(state->para_Pose)); std::memcpy(st.data() + ST_SB, state->para_SpeedBias, sizeof(state->para_SpeedBias));
    std::memcpy(st.data() + ST_LB, state->para_LegBias, sizeof(state->para_LegBias)); std::memcpy(st.data() + ST_EX, state->para_Ex_Pose, sizeof(state->para_Ex_Pose));
    st[ST_TD] = state->para_Td[0];
    size_t jtot = 0; for (int b = 0; b < prior->num_blocks; b++) jtot += (size_t)prior->n * prior_block_size(prior->block_kind[b]);
    cudaStream_t s = h->stream; DevBuf B(h);
    double *dJ = B.up(J.data(), J.size(), s), *dr0 = B.up(r.data(), r.size(), s), *dx0 = B.up(x0.data(), x0.size(), s), *dst = B.up(st.data(), st.size(), s);
    double *dres = B.up(nullptr, PRIOR_LD, s), *djac = jacobians ? B.up(nullptr, jtot, s) : nullptr;
    int *dmeta = B.upi(meta.data(), PRIOR_META_STRIDE, s);
    if (!dJ || !dr0 || !dx0 || !dst || !dres || !dmeta || (jacobians && !djac)) return fail(CERB_ERR_CUDA, "device allocation failed");
    CERB_LAUNCH(prior_eval_kernel, 1, 128, 0, s, (const double *)dJ, (const double *)dr0, (const int *)dmeta, (const double *)dx0, (const double *)dst, dres, djac);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(residuals, dres, prior->n * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (jacobians) CUDA_TRY(cudaMemcpyAsync(jacobians, djac, jtot * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return CERB_OK;
}

int cerb_a1_kinematics(CerbHandle *h, int32_t n, const double *q, const double *rho_opt, const double *rho_fix, double *fk, double *jac, double *dfk_drho,
                       double *dJ_dq, double *dJ_drho) {
    if (!h || n < 1 || !q || !rho_opt || !rho_fix) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_a1_kinematics: bad argument");
    CERB_DEVICE(h);
    cudaStream_t s = h->stream; DevBuf B(h); const size_t N = n;
    double *dq = B.up(q, 3 * N, s), *dro = B.up(rho_opt, N, s), *drf = B.up(rho_fix, 4 * N, s);
    double *dfk = fk ? B.up(nullptr, 3 * N, s) : nullptr, *dj = jac ? B.up(nullptr, 9 * N, s) : nullptr, *ddf = dfk_drho ? B.up(nullptr, 3 * N, s) : nullptr;
    double *djq = dJ_dq ? B.up(nullptr, 27 * N, s) : nullptr, *djr = dJ_drho ? B.up(nullptr, 9 * N, s) : nullptr;
    CERB_LAUNCH(a1_kinematics_kernel, (n + 127) / 128, 128, 0, s, (int)n, (const double *)dq, (const double *)dro, (const double *)drf, dfk, dj, ddf, djq, djr);
    CUDA_TRY(cudaGetLastError());
    if (fk) CUDA_TRY(cudaMemcpyAsync(fk, dfk, 3 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (jac) CUDA_TRY(cudaMemcpyAsync(jac, dj, 9 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (dfk_drho) CUDA_TRY(cudaMemcpyAsync(dfk_drho, ddf, 3 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (dJ_dq) CUDA_TRY(cudaMemcpyAsync(dJ_dq, djq, 27 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (dJ_drho) CUDA_TRY(cudaMemcpyAsync(dJ_drho, djr, 9 * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return CERB_OK;
}

// ---- per-feature steps on the resident batch ------------------------------------------------------------------------
// One pass over the features of the resident batch at its current states: launch(s, blocks, threads, states, out) enqueues the pass kernel,
// which writes `planes` planes of [n][F] doubles in device slot order.  They come back in the caller's feature order: store(q, v, N) is called
// for entry q = w * F + f of the first nfeat[w] features of each window w (plane p at v[p * N + q]).  The caller's entries past nfeat[w] are
// left as they are.
}  // extern "C"
template <class Launch, class Store> static int feature_pass(CerbHandle *h, int planes, Launch launch, Store store) {
    CERB_DEVICE(h);
    if (h->n < 1) return fail(CERB_ERR_BAD_ARGUMENT, "no resident batch");
    const int n = h->n, F = h->F;
    const size_t N = (size_t)n * F;
    cudaStream_t s = h->stream; DevBuf B(h);
    double *d_out = B.up(nullptr, planes * N, s), *d_perm_out = B.up(nullptr, planes * N, s);
    if (!d_out || !d_perm_out) return fail(CERB_ERR_CUDA, "device allocation failed");
    const int threads = 128, blocks = (int)((N + threads - 1) / threads);
    launch(s, blocks, threads, resident_states(h), d_out);
    CERB_LAUNCH(unpermute_kernel, blocks, threads, 0, s, n, F, planes, (const int *)h->n_features.d, (const int *)h->perm.d, (const double *)d_out, d_perm_out);   // device slot -> caller's feature index
    CUDA_TRY(cudaGetLastError());
    std::vector<double> tmp(planes * N);
    COPY_TRY(h, tmp.data(), d_perm_out, tmp.size() * sizeof(double), cudaMemcpyDeviceToHost, s);
    CUDA_TRY(cudaStreamSynchronize(s));
    for (int w = 0; w < n; w++)
        for (int f = 0; f < h->nfeat[w]; f++) store((size_t)w * F + f, tmp.data(), N);
    return CERB_OK;
}
extern "C" {

int cerb_batch_outlier_errors(CerbHandle *h, double focal_length, double *ave_err, int32_t *remove) {
    if (!h || !ave_err) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    return feature_pass(h, 1, [&](cudaStream_t s, int blocks, int threads, const States &cur, double *out) {
        CERB_LAUNCH(outlier_error_kernel, blocks, threads, 0, s, h->n, h->F, h->O, (const int *)h->n_features.d, (const int *)h->feat_start.d, (const int *)h->feat_nobs.d,
                    (const int *)h->feat_off.d, (const double *)h->obs.d, (const int *)h->obs_stereo.d, (const double *)cur.state.d, (const double *)cur.lam.d, out);
    }, [&](size_t q, const double *v, size_t) { ave_err[q] = v[q]; if (remove) remove[q] = (v[q] * focal_length > 3.0) ? 1 : 0; });
}
int cerb_batch_triangulate(CerbHandle *h, double init_depth, double *depth) {
    if (!h || !depth) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    return feature_pass(h, 1, [&](cudaStream_t s, int blocks, int threads, const States &cur, double *out) {
        CERB_LAUNCH(triangulate_kernel, blocks, threads, 0, s, h->n, h->F, h->O, (const int *)h->n_features.d, (const int *)h->feat_start.d, (const int *)h->feat_nobs.d,
                    (const int *)h->feat_off.d, (const double *)h->obs.d, (const int *)h->obs_stereo.d, (const double *)cur.state.d, (const double *)cur.lam.d, init_depth, out);
    }, [&](size_t q, const double *v, size_t) { depth[q] = v[q]; });
}
int cerb_batch_shift_depth(CerbHandle *h, double init_depth, int32_t *new_start_frame, double *depth, int32_t *keep) {
    if (!h || !new_start_frame || !depth || !keep) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    return feature_pass(h, 3, [&](cudaStream_t s, int blocks, int threads, const States &cur, double *out) {
        CERB_LAUNCH(shift_depth_kernel, blocks, threads, 0, s, h->n, h->F, h->O, (const int *)h->n_features.d, (const int *)h->feat_start.d, (const int *)h->feat_nobs.d,
                    (const int *)h->feat_off.d, (const double *)h->obs.d, (const double *)cur.state.d, (const double *)cur.lam.d, init_depth, out);
    }, [&](size_t q, const double *v, size_t N) { new_start_frame[q] = (int32_t)v[q]; depth[q] = v[N + q]; keep[q] = (int32_t)v[2 * N + q]; });
}
// test hook: CERB_TEST_MARG_SMEM=<bytes> shrinks the shared-memory budget of the eigen-solver's memory plan (split / global layouts on small matrices)
static size_t marg_smem_limit() {
    const char *e = std::getenv("CERB_TEST_MARG_SMEM");
    if (!e) return MARG_SMEM_MAX;
    const long v = std::atol(e);
    return (v >= 4096 && (size_t)v <= MARG_SMEM_MAX) ? (size_t)v : MARG_SMEM_MAX;
}
int cerb_marginalize_schur(CerbHandle *h, int32_t n_windows, int32_t m, int32_t n, const double *A, const double *b, double eps,
                           double *linearized_jacobians, double *linearized_residuals, int32_t *sweeps) {
    if (!h || !A || !b || !linearized_jacobians || !linearized_residuals) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    CERB_DEVICE(h);
    if (n_windows < 1 || m < 1 || n < 1 || m > 19 + CERB_MAX_FEATURES || n > CERB_MAX_PRIOR_DIM) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_marginalize_schur: bad sizes");      // m: what a window can drop (also keeps the kernel's multiply-high divisions exact)
    const size_t pos = (size_t)m + n, N = n_windows;
    const size_t lim = marg_smem_limit();
    int grid = std::min<int>(n_windows, marg_ctas_per_sm(m, n, lim) * h->sm_count);
    grid = (int)std::max<size_t>(1, std::min<size_t>(grid, ((size_t)4 << 30) / (marg_ws_doubles(m, n, lim) * sizeof(double))));      // <= 4 GB of per-CTA workspace
    CUDA_TRY(cudaFuncSetAttribute(marg_schur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)marg_smem_bytes(m, n, lim)));
    cudaStream_t s = h->stream; DevBuf B(h);
    double *dA = B.up(A, N * pos * pos, s), *db = B.up(b, N * pos, s), *dws = B.up(nullptr, (size_t)grid * marg_ws_doubles(m, n, lim), s);
    double *dJ = B.up(nullptr, N * n * n, s), *dr = B.up(nullptr, N * n, s), *dsw = B.up(nullptr, N, s);     // dsw: 2 ints per window
    if (!dA || !db || !dws || !dJ || !dr || !dsw) return fail(CERB_ERR_CUDA, "device allocation failed");
    CERB_LAUNCH(marg_schur_kernel, grid, marg_threads(m, n, lim), marg_smem_bytes(m, n, lim), s, (int)n_windows, (int)m, (int)n, (const int *)nullptr, (const double *)dA, 0L, (const double *)db, 0L, eps, dws, dJ, 0L, dr, 0L, (int *)dsw, (int)lim);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(linearized_jacobians, dJ, N * n * n * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(linearized_residuals, dr, N * n * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (sweeps) CUDA_TRY(cudaMemcpyAsync(sweeps, dsw, N * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return CERB_OK;
}

// ---- marginalization of the resident batch ----------------------------------------------------------------------------------
CERB_GLOBAL void permute_lam_kernel(int n, int F, const int *n_features, const int *perm, const double *lam_caller, double *lam_dev) {
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long)n * F) return;
    const int w = (int)(idx / F), k = (int)(idx % F);
    if (k < n_features[w]) lam_dev[idx] = lam_caller[(size_t)w * F + perm[idx]];
}

// The caller's states of the resident batch into dst: para_Pose .. para_Td as they are, para_Feature in device feature order.  `who` names the
// entry point in the error messages.  hst receives the host image of dst.state; the copies are done when this returns.
static int states_to_device(CerbHandle *h, DevBuf &B, const CerbWindowState *states, const char *who, const States &dst, std::vector<double> &hst) {
    const int n = h->n, F = h->F;
    cudaStream_t s = h->stream;
    hst.assign(n * dst.state.per, 0.0);
    std::vector<double> hl(n * dst.lam.per, 0.0);
    for (int w = 0; w < n; w++) {
        std::memcpy(hst.data() + w * dst.state.per, &states[w], ST_SIZE * sizeof(double));
        if (h->nfeat[w]) {
            if (!states[w].para_Feature) return fail(CERB_ERR_BAD_ARGUMENT, std::string(who) + ": null para_Feature");
            std::memcpy(hl.data() + w * dst.lam.per, states[w].para_Feature, (size_t)h->nfeat[w] * 8);
        }
    }
    double *dlc = B.up(hl.data(), hl.size(), s);
    if (!dlc) return fail(CERB_ERR_CUDA, "device allocation failed");
    COPY_TRY(h, dst.state.d, hst.data(), dst.state.bytes(n), cudaMemcpyHostToDevice, s);
    CERB_LAUNCH(permute_lam_kernel, (int)(((size_t)n * F + 127) / 128), 128, 0, s, n, F, (const int *)h->n_features.d, (const int *)h->perm.d, (const double *)dlc, dst.lam.d);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(s));               // hst / hl are read by the asynchronous copies
    return CERB_OK;
}

// cerb_batch_marginalize (priors: the new priors return to the host) and cerb_resident_marginalize (priors == NULL: they become the priors of
// the resident windows on the device, valid [n] returns)
static int marginalize_impl(CerbHandle *h, const int32_t *flags, const CerbWindowState *states, CerbPrior *priors, int32_t *sweeps, int32_t *valid) {
    const int n = h->n;
    if (n < 1) return fail(CERB_ERR_BAD_ARGUMENT, "no resident batch");
    for (int w = 0; w < n; w++) {
        if (flags[w] != 0 && flags[w] != 1) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_marginalize: flag must be 0 (MARGIN_OLD) or 1 (MARGIN_SECOND_NEW)");
        if (priors && (!priors[w].linearized_jacobians || !priors[w].linearized_residuals)) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_marginalize: priors[w] needs storage for linearized_jacobians / linearized_residuals");
    }
    cudaStream_t s = h->stream; DevBuf B(h);
    int mmax = 19;
    const int nmax = MARG_N_STRUCT;            // what a window can keep (the kernel skips a window that claims more); the prior arrays keep the stride CERB_MAX_PRIOR_DIM
    for (int w = 0; w < n; w++) if (flags[w] == 0) mmax = std::max(mmax, 19 + h->n0[w]);
    const int posmax = mmax + CERB_MAX_PRIOR_DIM;
    // states to linearise at: the caller's (after double2vector + vector2double), or the resident ones; hst is their host image
    std::vector<double> hst;
    States lin = resident_states(h);
    if (states) {
        lin.state.d = B.up(nullptr, n * lin.state.per, s); lin.lam.d = B.up(nullptr, n * lin.lam.per, s);
        if (!lin.state.d || !lin.lam.d) return fail(CERB_ERR_CUDA, "device allocation failed");
        int rc = states_to_device(h, B, states, "cerb_batch_marginalize", lin, hst); if (rc) return rc;
    } else {
        hst.resize(n * lin.state.per);
        COPY_TRY(h, hst.data(), lin.state.d, lin.state.bytes(n), cudaMemcpyDeviceToHost, s);
    }
    std::vector<int> hflags(flags, flags + n);
    int *dflags = B.upi(hflags.data(), n, s), *ddims = B.upi(nullptr, (size_t)n * 4, s), *dblocks = B.upi(nullptr, (size_t)n * 64, s), *dsw = B.upi(nullptr, (size_t)n * 2, s);
    // the new priors, laid out as the resident one: they come back through its pinned mirrors
    const size_t jper = h->prior_J.per, rper = h->prior_r.per;
    double *dJ = B.up(nullptr, n * jper, s), *dr = B.up(nullptr, n * rper, s);
    // A / b of a sub-batch and the per-CTA workspace of the eigen-solver: bounded device memory whatever the batch size
    const size_t a_bytes = (size_t)posmax * posmax * 8, budget = (size_t)3 << 30;
    const int per = (int)std::max<size_t>(1, std::min<size_t>(n, budget / a_bytes));
    double *dA = B.up(nullptr, (size_t)per * posmax * posmax, s), *db = B.up(nullptr, (size_t)per * posmax, s);
    const size_t lim = marg_smem_limit();
    int sgrid = std::min(per, marg_ctas_per_sm(mmax, nmax, lim) * h->sm_count);
    CUDA_TRY(cudaFuncSetAttribute(marg_schur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)marg_smem_bytes(mmax, nmax, lim)));
    sgrid = (int)std::max<size_t>(1, std::min<size_t>(sgrid, ((size_t)2 << 30) / (marg_ws_doubles(mmax, nmax, lim) * sizeof(double))));
    double *dws = B.up(nullptr, (size_t)sgrid * marg_ws_doubles(mmax, nmax, lim), s);
    if (!dflags || !ddims || !dblocks || !dsw || !dJ || !dr || !dA || !db || !dws) return fail(CERB_ERR_CUDA, "device allocation failed");
    CUDA_TRY(cudaMemsetAsync(dsw, 0, (size_t)n * 2 * sizeof(int), s));
    CUDA_TRY(cudaFuncSetAttribute(marg_assemble_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_bytes));
    int rc = gather_priors(h, s); if (rc) return rc;
    for (int w0 = 0; w0 < n; w0 += per) {
        const int cn = std::min(per, n - w0);
        enqueue_prepare(h, w0, cn, s);         // a solve leaves sqrt_info and the prior's Gram matrix behind; a bare upload does not
        SolveParams P = make_params(h, w0, cn, 0, nullptr, -1);
        MargParams M;
        M.flags = dflags + w0; M.state = lin.state.at(w0); M.lam = lin.lam.at(w0); M.A = dA; M.b = db; M.posmax = posmax;
        M.dims = ddims + (size_t)w0 * 4; M.blocks = dblocks + (size_t)w0 * 64;
        CERB_LAUNCH(marg_assemble_kernel, std::min(cn, h->grid), SOLVE_THREADS, h->smem_bytes, s, P, M);
        CERB_LAUNCH(marg_schur_kernel, std::min(cn, sgrid), marg_threads(mmax, nmax, lim), marg_smem_bytes(mmax, nmax, lim), s, cn, mmax, nmax, (const int *)(ddims + (size_t)w0 * 4), (const double *)dA, (long)posmax * posmax,
                    (const double *)db, (long)posmax, 1e-8, dws, dJ + w0 * jper, (long)jper, dr + w0 * rper, (long)rper, dsw + (size_t)w0 * 2, (int)lim);
        CUDA_TRY(cudaGetLastError());
    }
    std::vector<int> hdims((size_t)n * 4), hblocks((size_t)n * 64), hsw((size_t)n * 2);
    if (!priors) {
        // the old prior was an input of the kernels above: it is replaced only now, by a kernel behind them on the stream
        COPY_TRY(h, hdims.data(), ddims, hdims.size() * sizeof(int), cudaMemcpyDeviceToHost, s);
        CUDA_TRY(cudaStreamSynchronize(s));
        for (int w = 0; w < n; w++) if (hdims[4 * w + 2] == 1 && (hdims[4 * w] > mmax || hdims[4 * w + 1] > nmax)) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_resident_marginalize: a window exceeds the structural size of the kept / dropped blocks");
        CERB_LAUNCH(prior_handover_kernel, std::min(n, 8 * h->sm_count), 256, 0, s, n, (const int *)(h->pre_slot.d + (size_t)n * CERB_WINDOW_SIZE), (const int *)ddims, (const int *)dblocks,
                    (const double *)lin.state.d, (const double *)dJ, (long)jper, (const double *)dr, (long)rper, h->rdesc.d, h->prior_J.d, h->prior_r.d);
        CUDA_TRY(cudaGetLastError());
        for (int w = 0; w < n; w++) {
            const int status = hdims[4 * w + 2];
            char &v = h->res_prior_valid[h->res_win[w]];
            if (status != 2) v = status == 1;
            valid[w] = v;
        }
        return CERB_OK;
    }
    COPY_TRY(h, hdims.data(), ddims, hdims.size() * sizeof(int), cudaMemcpyDeviceToHost, s);
    COPY_TRY(h, hblocks.data(), dblocks, hblocks.size() * sizeof(int), cudaMemcpyDeviceToHost, s);
    COPY_TRY(h, hsw.data(), dsw, hsw.size() * sizeof(int), cudaMemcpyDeviceToHost, s);
    // the pinned staging of the prior upload is idle here: D2H at PCIe rate instead of through pageable memory
    COPY_TRY(h, h->prior_J.h, dJ, h->prior_J.bytes(n), cudaMemcpyDeviceToHost, s);
    COPY_TRY(h, h->prior_r.h, dr, h->prior_r.bytes(n), cudaMemcpyDeviceToHost, s);
    // a prior that is carried over unchanged comes back from the device copy of the old one
    std::vector<int> hmeta(n * h->prior_meta.per); std::vector<double> hx0(n * h->prior_x0.per);
    COPY_TRY(h, hmeta.data(), h->prior_meta.d, h->prior_meta.bytes(n), cudaMemcpyDeviceToHost, s);
    COPY_TRY(h, hx0.data(), h->prior_x0.d, h->prior_x0.bytes(n), cudaMemcpyDeviceToHost, s);
    CUDA_TRY(cudaStreamSynchronize(s));
    std::vector<StageJob> out_jobs; out_jobs.reserve(n);
    for (int w = 0; w < n; w++) if (hdims[4 * w + 2] == 1 && (hdims[4 * w] > mmax || hdims[4 * w + 1] > nmax)) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_marginalize: a window exceeds the structural size of the kept / dropped blocks");
    for (int w = 0; w < n; w++) {
        CerbPrior &pr = priors[w];
        double *Jout = const_cast<double *>(pr.linearized_jacobians), *rout = const_cast<double *>(pr.linearized_residuals);
        const int status = hdims[4 * w + 2];
        if (sweeps) { sweeps[2 * w] = hsw[2 * w]; sweeps[2 * w + 1] = hsw[2 * w + 1]; }
        pr.valid = 0; pr.n = 0; pr.num_blocks = 0;
        if (status == 0) continue;
        if (status == 2) {                       // MARGIN_SECOND_NEW without para_Pose[WINDOW_SIZE - 1] in the old prior: unchanged (estimator.cpp:1380-1381)
            decode_prior(hmeta.data() + w * h->prior_meta.per, hx0.data() + w * h->prior_x0.per, pr);
            if (!pr.valid) continue;
            COPY_TRY(h, Jout, batch_prior_J(h).at(w), (size_t)pr.n * pr.n * 8, cudaMemcpyDeviceToHost, s);
            COPY_TRY(h, rout, batch_prior_r(h).at(w), (size_t)pr.n * 8, cudaMemcpyDeviceToHost, s);
            continue;
        }
        const int nn = hdims[4 * w + 1], nb = hdims[4 * w + 3];
        pr.valid = 1; pr.n = nn; pr.num_blocks = nb;
        const double *st = hst.data() + w * h->state.per;
        for (int b = 0; b < nb; b++) {
            const int *q = hblocks.data() + (size_t)w * 64 + 4 * b;
            pr.block_kind[b] = q[0]; pr.block_index[b] = q[1]; pr.block_col[b] = q[2];
            const int size = prior_block_size(q[0]);
            const double *x = st + prior_block_state_offset(q[0], q[3]);          // keep_block_data: the state the factors were linearised at
            for (int k = 0; k < 9; k++) pr.block_x0[b][k] = k < size ? x[k] : 0.0;
        }
        out_jobs.push_back({Jout, h->prior_J.h_at(w), (size_t)nn * nn * 8});       // 59 KB per window: copied by a few threads below
        std::memcpy(rout, h->prior_r.h_at(w), (size_t)nn * 8);
    }
    CUDA_TRY(cudaStreamSynchronize(s));          // the carried-over priors
    run_stage_jobs(out_jobs);
    return CERB_OK;
}

int cerb_batch_marginalize(CerbHandle *h, const int32_t *flags, const CerbWindowState *states, CerbPrior *priors, int32_t *sweeps) {
    if (!h || !flags || !priors) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_marginalize: null argument");
    CERB_DEVICE(h);
    return marginalize_impl(h, flags, states, priors, sweeps, nullptr);
}

int cerb_batch_update_states(CerbHandle *h, int32_t n, const CerbWindowState *states) {
    if (!h || !states) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    CERB_DEVICE(h);
    if (h->n < 1 || n != h->n) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_update_states: n must be the size of the resident batch");
    DevBuf B(h); std::vector<double> hst;
    int rc = states_to_device(h, B, states, "cerb_batch_update_states", States{h->state0, h->lam0}, hst); if (rc) return rc;
    h->solved = false;                                 // the per-feature passes and a resident solve start from these states
    return CERB_OK;
}

// ---- leg-contact and plain IMU preintegration -----------------------------------------------------------------------
// Job j integrates under cfgs[cfg_of[j]] into the record kind imu_only[j] (0: IMULegIntegrationBase, 1: IntegrationBase), all in one
// preintegrate_kernel launch.  where (resident sliding window): [n][2] window, slot -- the results stay in rpre and only sum_dt [n] returns;
// else out[j] / out_imu[j] receive them by kind.  The caller has validated cfg_of and where.
static int preintegrate_impl(CerbHandle *h, int32_t n_cfg, const CerbPreintConfig *cfgs, int32_t n, const CerbPreintJob *jobs, const int32_t *cfg_of,
                             const std::vector<int> &imu_only, CerbIMULegPreint *out, CerbIMUPreint *out_imu, const int *where = nullptr, double *sum_dt = nullptr) {
    CERB_DEVICE(h);
    std::vector<PreintParams> table((size_t)2 * n_cfg);      // entry 2 c + imu_only: configuration c with the record kind
    for (int c = 0; c < 2 * n_cfg; c++) {
        const CerbPreintConfig *cfg = &cfgs[c / 2];
        PreintParams &P = table[c];
        std::memset(&P, 0, sizeof(P));
        P.imu_only = c % 2;
        P.acc_n = cfg->acc_n; P.acc_n_z = cfg->acc_n_z; P.gyr_n = cfg->gyr_n; P.acc_w = cfg->acc_w; P.gyr_w = cfg->gyr_w; P.phi_n = cfg->phi_n; P.dphi_n = cfg->dphi_n;
        P.rho_c_n = cfg->rho_c_n; P.rho_nc_n = cfg->rho_nc_n; P.v_n_min_xy = cfg->v_n_min_xy; P.v_n_min_z = cfg->v_n_min_z; P.v_n_min = cfg->v_n_min; P.v_n_max = cfg->v_n_max;
        P.v_n_force_thres_ratio = cfg->v_n_force_thres_ratio; P.v_n_term1_steep = cfg->v_n_term1_steep; P.v_n_term2_var_rescale = cfg->v_n_term2_var_rescale;
        P.v_n_term3_distance_rescale = cfg->v_n_term3_distance_rescale; P.contact_sensor_type = cfg->contact_sensor_type;
        for (int l = 0; l < 4; l++) for (int k = 0; k < 4; k++) P.rho_fix[4 * l + k] = cfg->rho_fix[l][k];
        for (int k = 0; k < 3; k++) P.p_br[k] = cfg->p_br[k];
        for (int k = 0; k < 9; k++) P.R_br[k] = cfg->R_br[k];
    }
    size_t total = 0;
    for (int j = 0; j < n; j++) { if (jobs[j].n_samples < 0 || (jobs[j].n_samples && !jobs[j].samples)) return fail(CERB_ERR_BAD_ARGUMENT, "bad job"); total += jobs[j].n_samples; }
    std::vector<double> hj((size_t)n * PJ_STRIDE), hs(std::max<size_t>(total, 1) * SAMPLE_STRIDE);
    std::vector<int> hi((size_t)n * 3);
    size_t off = 0;
    for (int j = 0; j < n; j++) {
        const CerbPreintJob &q = jobs[j];
        double *o = hj.data() + (size_t)j * PJ_STRIDE;
        std::memcpy(o, q.acc_0, 24); std::memcpy(o + 3, q.gyr_0, 24); std::memcpy(o + 6, q.phi_0, 96); std::memcpy(o + 18, q.dphi_0, 96); std::memcpy(o + 30, q.c_0, 32);
        std::memcpy(o + 34, q.linearized_ba, 24); std::memcpy(o + 37, q.linearized_bg, 24); std::memcpy(o + 40, q.linearized_rho, 32);
        hi[3 * j] = q.n_samples; hi[3 * j + 1] = (int)off; hi[3 * j + 2] = 2 * cfg_of[j] + imu_only[j];
        for (int k = 0; k < q.n_samples; k++) {
            const CerbIMULegSample &m = q.samples[k];
            double *so = hs.data() + (off + k) * SAMPLE_STRIDE;
            so[0] = m.dt; std::memcpy(so + 1, m.acc, 24); std::memcpy(so + 4, m.gyr, 24); std::memcpy(so + 7, m.phi, 96); std::memcpy(so + 19, m.dphi, 96); std::memcpy(so + 31, m.c, 32);
        }
        off += q.n_samples;
    }
    cudaStream_t s = h->stream; DevBuf B(h);
    double *dj = B.up(hj.data(), hj.size(), s), *ds = B.up(hs.data(), hs.size(), s), *dout = B.up(nullptr, (size_t)n * PRE_STRIDE, s), *dfull = B.up(nullptr, (size_t)n * 1922, s);
    int *di = B.upi(hi.data(), hi.size(), s);
    PreintParams *dparams = (PreintParams *)B.raw(table.size() * sizeof(PreintParams));
    if (!dj || !ds || !dout || !dfull || !di || !dparams) return fail(CERB_ERR_CUDA, "device allocation failed");
    COPY_TRY(h, dparams, table.data(), table.size() * sizeof(PreintParams), cudaMemcpyHostToDevice, s);
    CERB_LAUNCH(preintegrate_kernel, n, 128, 0, s, (const PreintParams *)dparams, (int)n, (const double *)dj, (const int *)di, (const double *)ds, dout, dfull);
    CUDA_TRY(cudaGetLastError());
    if (where) {
        std::vector<int> where3((size_t)n * 3);
        for (int j = 0; j < n; j++) { where3[3 * j] = where[2 * j]; where3[3 * j + 1] = where[2 * j + 1]; where3[3 * j + 2] = imu_only[j]; }
        int *dwhere = B.upi(where3.data(), where3.size(), s); double *dsum = B.up(nullptr, n, s);
        if (!dwhere || !dsum) return fail(CERB_ERR_CUDA, "device allocation failed");
        CERB_LAUNCH(preint_store_kernel, n, 128, 0, s, (int)n, (const int *)dwhere, (const double *)dout, (const double *)dfull, h->rpre.d, dsum);
        CUDA_TRY(cudaGetLastError());
        std::vector<double> hsum(n);
        COPY_TRY(h, hsum.data(), dsum, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, s);
        CUDA_TRY(cudaStreamSynchronize(s));
        if (sum_dt) std::memcpy(sum_dt, hsum.data(), (size_t)n * sizeof(double));
        return CERB_OK;
    }
    std::vector<double> ho((size_t)n * PRE_STRIDE), hf((size_t)n * 1922);
    COPY_TRY(h, ho.data(), dout, ho.size() * sizeof(double), cudaMemcpyDeviceToHost, s);
    COPY_TRY(h, hf.data(), dfull, hf.size() * sizeof(double), cudaMemcpyDeviceToHost, s);
    CUDA_TRY(cudaStreamSynchronize(s));
    for (int j = 0; j < n; j++) {
        const double *o = ho.data() + (size_t)j * PRE_STRIDE, *f = hf.data() + (size_t)j * 1922;
        if (imu_only[j]) {
            CerbIMUPreint &r = out_imu[j];
            r.sum_dt = o[PRE_SUM_DT];
            for (int k = 0; k < 3; k++) { r.delta_p[k] = o[PRE_DP + k]; r.delta_v[k] = o[PRE_DV + k]; r.linearized_ba[k] = o[PRE_BA + k]; r.linearized_bg[k] = o[PRE_BG + k]; }
            for (int k = 0; k < 4; k++) r.delta_q[k] = o[PRE_DQ + k];
            for (int a = 0; a < 15; a++) for (int b = 0; b < 15; b++) { r.jacobian[b * 15 + a] = f[kImuTo31[a] * 31 + kImuTo31[b]]; r.covariance[b * 15 + a] = f[961 + kImuTo31[a] * 31 + kImuTo31[b]]; }
            continue;
        }
        CerbIMULegPreint &r = out[j];
        r.sum_dt = o[PRE_SUM_DT];
        for (int k = 0; k < 3; k++) { r.delta_p[k] = o[PRE_DP + k]; r.delta_v[k] = o[PRE_DV + k]; r.linearized_ba[k] = o[PRE_BA + k]; r.linearized_bg[k] = o[PRE_BG + k]; }
        for (int k = 0; k < 4; k++) { r.delta_q[k] = o[PRE_DQ + k]; r.linearized_rho[k] = o[PRE_RHO + k]; }
        for (int k = 0; k < 12; k++) r.delta_epsilon[k] = o[PRE_DEPS + k];
        for (int a = 0; a < 31; a++) for (int b = 0; b < 31; b++) { r.jacobian[b * 31 + a] = f[a * 31 + b]; r.covariance[b * 31 + a] = f[961 + a * 31 + b]; }
    }
    return CERB_OK;
}

// the arguments every preintegration entry point shares: jobs and their configuration indices
static int check_preint_args(CerbHandle *h, int32_t n_cfg, const CerbPreintConfig *cfgs, int32_t n, const CerbPreintJob *jobs, const int32_t *cfg_of, const char *who) {
    if (!h || n_cfg < 1 || !cfgs || n < 1 || !jobs || !cfg_of) return fail(CERB_ERR_BAD_ARGUMENT, std::string(who) + ": bad argument");
    for (int j = 0; j < n; j++) if (cfg_of[j] < 0 || cfg_of[j] >= n_cfg) return fail(CERB_ERR_BAD_ARGUMENT, std::string(who) + ": cfg_of out of range");
    return CERB_OK;
}

int cerb_preintegrate_mixed(CerbHandle *h, int32_t n_cfg, const CerbPreintConfig *cfgs, const int32_t *use_leg, int32_t n, const CerbPreintJob *jobs,
                            const int32_t *cfg_of, CerbIMULegPreint *out, CerbIMUPreint *out_imu) {
    int rc = check_preint_args(h, n_cfg, cfgs, n, jobs, cfg_of, "cerb_preintegrate"); if (rc) return rc;
    if (!use_leg) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_preintegrate: bad argument");
    std::vector<int> imu_only(n);
    for (int j = 0; j < n; j++) {
        imu_only[j] = use_leg[cfg_of[j]] ? 0 : 1;
        if (imu_only[j] ? !out_imu : !out) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_preintegrate: no output array for a job's record kind");
    }
    return preintegrate_impl(h, n_cfg, cfgs, n, jobs, cfg_of, imu_only, out, out_imu);
}
int cerb_preintegrate_batch(CerbHandle *h, const CerbPreintConfig *cfg, int32_t n, const CerbPreintJob *jobs, CerbIMULegPreint *out) {
    const int32_t leg = 1; const std::vector<int32_t> cfg_of(std::max(n, 0), 0);
    return cerb_preintegrate_mixed(h, 1, cfg, &leg, n, jobs, cfg_of.data(), out, nullptr);
}
int cerb_preintegrate_imu_batch(CerbHandle *h, const CerbPreintConfig *cfg, int32_t n, const CerbPreintJob *jobs, CerbIMUPreint *out) {
    const int32_t leg = 0; const std::vector<int32_t> cfg_of(std::max(n, 0), 0);
    return cerb_preintegrate_mixed(h, 1, cfg, &leg, n, jobs, cfg_of.data(), nullptr, out);
}

// ---- host-side gauge re-anchoring: Estimator::double2vector (estimator.cpp:903-957) ----------------------------------
static void r2ypr(const m33 &R, double ypr[3]) {   // Utility::R2ypr, degrees
    const double nx = R.m[0], ny = R.m[3], nz = R.m[6], ox = R.m[1], oy = R.m[4], ax = R.m[2], ay = R.m[5];
    const double y = atan2(ny, nx);
    const double p = atan2(-nz, nx * cos(y) + ny * sin(y));
    const double r = atan2(ax * sin(y) - ay * cos(y), -ox * sin(y) + oy * cos(y));
    ypr[0] = y / M_PI * 180.0; ypr[1] = p / M_PI * 180.0; ypr[2] = r / M_PI * 180.0;
}
void cerb_double2vector(const CerbWindowState *before, const CerbWindowState *after, double *Ps, double *Rs, double *Vs) {
    const m33 Rs0 = qtoR(ldq(before->para_Pose[0] + 3));
    const m33 R00 = qtoR(ldq(after->para_Pose[0] + 3));
    double o0[3], o00[3];
    r2ypr(Rs0, o0); r2ypr(R00, o00);
    const double yd = (o0[0] - o00[0]) / 180.0 * M_PI;
    m33 rot = ident33();
    rot.m[0] = cos(yd); rot.m[1] = -sin(yd); rot.m[3] = sin(yd); rot.m[4] = cos(yd);
    if (fabs(fabs(o0[1]) - 90) < 1.0 || fabs(fabs(o00[1]) - 90) < 1.0) rot = mul33(Rs0, tr33(R00));
    const d3 P0 = ld3(after->para_Pose[0]), origin = ld3(before->para_Pose[0]);
    for (int i = 0; i < CERB_NUM_FRAMES; i++) {
        const m33 R = mul33(rot, qtoR(qnormalized(ldq(after->para_Pose[i] + 3))));
        const d3 P = mv33(rot, ld3(after->para_Pose[i]) - P0) + origin;
        const d3 V = mv33(rot, ld3(after->para_SpeedBias[i]));
        st3(Ps + 3 * i, P); st3(Vs + 3 * i, V);
        for (int k = 0; k < 9; k++) Rs[9 * i + k] = R.m[k];
    }
}

}  // extern "C"

#include "resident_host.inl"
#include "replay_host.inl"

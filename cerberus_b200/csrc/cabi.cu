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

template <typename T> static cudaError_t dmalloc(T **p, size_t n) { return cudaMalloc((void **)p, n * sizeof(T)); }
template <typename T> static cudaError_t hmalloc(T **p, size_t n) { return cudaMallocHost((void **)p, n * sizeof(T)); }

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
    // device: the caller's descriptors as they are (filled by DMA) ...
    CerbWindowDesc *d_rdesc = nullptr; CerbFeature *d_rfeat = nullptr; CerbObservation *d_robs = nullptr; CerbWindowState *d_rstate = nullptr;
    double *d_rpre = nullptr, *d_rlam = nullptr;
    // ... and the solver's layout (written by pack_kernel)
    int *d_nfeat = nullptr, *d_fstart = nullptr, *d_fnobs = nullptr, *d_foff = nullptr, *d_flags = nullptr, *d_stereo = nullptr, *d_pmeta = nullptr, *d_repi = nullptr, *d_perm = nullptr;
    double *d_obs = nullptr, *d_pre = nullptr, *d_sinfo = nullptr, *d_pJ = nullptr, *d_pr = nullptr, *d_px0 = nullptr, *d_pHp = nullptr;
    double *d_state = nullptr, *d_state0 = nullptr, *d_lam = nullptr, *d_lam0 = nullptr, *d_repd = nullptr, *d_ws = nullptr, *d_dbg = nullptr, *d_G = nullptr, *d_probe_repd = nullptr;
    int *d_probe_repi = nullptr;
    double *d_olam = nullptr, *d_ostate = nullptr; CerbSolveReport *d_orep = nullptr;      // results in the caller's layout (unpack_kernel)
    // pinned staging (used for sources that are not in registered memory, and for the results)
    CerbWindowDesc *h_rdesc = nullptr; CerbFeature *h_rfeat = nullptr; CerbObservation *h_robs = nullptr; CerbWindowState *h_rstate = nullptr;
    double *h_rpre = nullptr, *h_rlam = nullptr, *h_pJ = nullptr, *h_pr = nullptr, *h_state = nullptr, *h_lam = nullptr, *h_dbg = nullptr;
    CerbSolveReport *h_orep = nullptr;
    std::vector<std::pair<uintptr_t, size_t>> regs;   // host ranges registered with cerb_register_host_buffer: DMA straight out of them
    std::vector<int> nfeat, n0;       // [B] n_features / number of tracks anchored at frame 0 of the resident windows
    int test_fail_factorizations = 0; double test_initial_mu = 0.0;   // fault injection of the parity tests (environment, read by cerb_create)
    bool solved = false;              // the device states are the solved ones (else: the uploaded initial states)
    std::vector<int> h_perm; bool perm_valid = false;     // [B][F] device feature slot -> index in the caller's feature array (fetched on demand)
    long ws_stride = 0;
    size_t smem_bytes = 0;
    // scratch arena of the evaluator / feature / preintegration entry points: grows to the high-water mark, then no more cudaMalloc per call
    std::vector<std::pair<char *, size_t>> arena; size_t arena_chunk = 0, arena_used = 0;
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
    const size_t B = h->B, F = h->F, O = h->O;
    h->ws_stride = ws_size(h->F);
    CUDA_TRY(dmalloc(&h->d_rdesc, B)); CUDA_TRY(dmalloc(&h->d_rfeat, B * F)); CUDA_TRY(dmalloc(&h->d_robs, B * O)); CUDA_TRY(dmalloc(&h->d_rstate, B));
    CUDA_TRY(dmalloc(&h->d_rpre, B * 10 * RAW_PRE_STRIDE)); CUDA_TRY(dmalloc(&h->d_rlam, B * F)); CUDA_TRY(dmalloc(&h->d_perm, B * F));
    CUDA_TRY(dmalloc(&h->d_olam, B * F)); CUDA_TRY(dmalloc(&h->d_ostate, B * ST_STRIDE)); CUDA_TRY(dmalloc(&h->d_orep, B));
    CUDA_TRY(dmalloc(&h->d_nfeat, B)); CUDA_TRY(dmalloc(&h->d_fstart, B * F)); CUDA_TRY(dmalloc(&h->d_fnobs, B * F)); CUDA_TRY(dmalloc(&h->d_foff, B * F));
    CUDA_TRY(dmalloc(&h->d_flags, B)); CUDA_TRY(dmalloc(&h->d_stereo, B * O)); CUDA_TRY(dmalloc(&h->d_pmeta, B * PRIOR_META_STRIDE)); CUDA_TRY(dmalloc(&h->d_repi, B * 4));
    CUDA_TRY(dmalloc(&h->d_obs, B * NOBS_PLANES * O)); CUDA_TRY(dmalloc(&h->d_pre, B * 10 * PRE_STRIDE)); CUDA_TRY(dmalloc(&h->d_sinfo, B * 10 * 961));
    CUDA_TRY(dmalloc(&h->d_pJ, B * PRIOR_LD * PRIOR_LD)); CUDA_TRY(dmalloc(&h->d_pr, B * PRIOR_LD)); CUDA_TRY(dmalloc(&h->d_px0, B * 16 * 9)); CUDA_TRY(dmalloc(&h->d_pHp, B * PRIOR_LD * PRIOR_LD));
    CUDA_TRY(dmalloc(&h->d_state, B * ST_STRIDE)); CUDA_TRY(dmalloc(&h->d_state0, B * ST_STRIDE)); CUDA_TRY(dmalloc(&h->d_lam, B * F)); CUDA_TRY(dmalloc(&h->d_lam0, B * F));
    CUDA_TRY(dmalloc(&h->d_repd, B * 2)); CUDA_TRY(dmalloc(&h->d_ws, (size_t)CerbHandle::LANES * h->grid * h->ws_stride)); CUDA_TRY(dmalloc(&h->d_dbg, 2 * (NR + F) + 8)); CUDA_TRY(dmalloc(&h->d_G, 4));
    CUDA_TRY(dmalloc(&h->d_probe_repi, 4)); CUDA_TRY(dmalloc(&h->d_probe_repd, 2));
    CUDA_TRY(hmalloc(&h->h_rdesc, B)); CUDA_TRY(hmalloc(&h->h_rfeat, B * F)); CUDA_TRY(hmalloc(&h->h_robs, B * O)); CUDA_TRY(hmalloc(&h->h_rstate, B));
    CUDA_TRY(hmalloc(&h->h_rpre, B * 10 * RAW_PRE_STRIDE)); CUDA_TRY(hmalloc(&h->h_rlam, B * F));
    CUDA_TRY(hmalloc(&h->h_pJ, B * PRIOR_LD * PRIOR_LD)); CUDA_TRY(hmalloc(&h->h_pr, B * PRIOR_LD));
    CUDA_TRY(hmalloc(&h->h_state, B * ST_STRIDE)); CUDA_TRY(hmalloc(&h->h_lam, B * F)); CUDA_TRY(hmalloc(&h->h_orep, B)); CUDA_TRY(hmalloc(&h->h_dbg, 2 * (NR + F) + 8));
    h->nfeat.assign(B, 0); h->n0.assign(B, 0);
    CUDA_TRY(cudaMemcpy(h->d_G, cfg->g, 3 * sizeof(double), cudaMemcpyHostToDevice));
#if !defined(CERB_CUSIM)
    // The per-CTA workspace (W, the prior Hessian image: ~290 KB x one CTA per SM) is re-read every iteration while ~300 KB of inputs per
    // window stream through once per linearisation; a persisting access-policy window on the compute stream can keep the workspace in L2.
    // The solve is fp64-latency bound with DRAM nearly idle, so the carve-out mostly takes L2 away from the inputs: opt-in
    // (CERB_L2_PERSIST=1), off by default.
    {
        const size_t ws_bytes = (size_t)h->grid * h->ws_stride * sizeof(double);
        const size_t want = std::min<size_t>(ws_bytes, (size_t)prop.persistingL2CacheMaxSize);
        if (want > 0 && std::getenv("CERB_L2_PERSIST") != nullptr) {
            if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) == cudaSuccess) {
                cudaStreamAttrValue av;
                std::memset(&av, 0, sizeof(av));
                av.accessPolicyWindow.base_ptr = h->d_ws;
                av.accessPolicyWindow.num_bytes = std::min<size_t>(ws_bytes, (size_t)prop.accessPolicyMaxWindowSize);
                av.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)want / (double)av.accessPolicyWindow.num_bytes);
                av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
                av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
                if (cudaStreamSetAttribute(h->stream, cudaStreamAttributeAccessPolicyWindow, &av) != cudaSuccess) cudaGetLastError();   // an optimisation only
            } else cudaGetLastError();
        }
    }
#endif
    return CERB_OK;
}

extern "C" {

void cerb_destroy(CerbHandle *h) {
    if (!h) return;
    cudaSetDevice(h->cfg.device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    void *dev[] = {h->d_rdesc, h->d_rfeat, h->d_robs, h->d_rstate, h->d_rpre, h->d_rlam, h->d_perm, h->d_olam, h->d_ostate, h->d_orep,
                   h->d_nfeat, h->d_fstart, h->d_fnobs, h->d_foff, h->d_flags, h->d_stereo, h->d_pmeta, h->d_repi, h->d_obs, h->d_pre, h->d_sinfo, h->d_pJ, h->d_pr,
                   h->d_px0, h->d_pHp, h->d_state, h->d_state0, h->d_lam, h->d_lam0, h->d_repd, h->d_ws, h->d_dbg, h->d_G, h->d_probe_repi, h->d_probe_repd};
    for (void *p : dev) if (p) cudaFree(p);
    for (auto &c : h->arena) cudaFree(c.first);
    for (auto &r : h->regs) cudaHostUnregister((void *)r.first);
    void *hst[] = {h->h_rdesc, h->h_rfeat, h->h_robs, h->h_rstate, h->h_rpre, h->h_rlam, h->h_pJ, h->h_pr, h->h_state, h->h_lam, h->h_orep, h->h_dbg};
    for (void *p : hst) if (p) cudaFreeHost(p);
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

// One logical array of windows [w0, w0 + cn): window w holds `rows` rows of width_of(w) bytes, row r at src_of(w) + r * spitch;
// device row (w - w0) * rows + r at dst + that * dpitch (stage: the pinned mirror of dst).
template <class SrcOf, class WidthOf>
static void plan_rows(const CerbHandle *h, UploadPlan &pl, int w0, int cn, char *dst, char *stage, size_t dpitch, int rows, size_t spitch, SrcOf src_of, WidthOf width_of) {
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

static int validate_window(const CerbHandle *h, const CerbWindowDesc &d, const CerbWindowState &st, int *n_anchor0) {
    if (d.n_features < 0 || d.n_features > h->F) return fail(CERB_ERR_BAD_ARGUMENT, "window: n_features over capacity");
    if (d.n_obs < 0 || d.n_obs > h->O) return fail(CERB_ERR_BAD_ARGUMENT, "window: n_obs over capacity");
    if ((d.n_features && (!d.features || !d.obs || !st.para_Feature)) || (!d.preint && !d.imu_preint)) return fail(CERB_ERR_BAD_ARGUMENT, "window: null pointer");
    int n0 = 0;
    for (int f = 0; f < d.n_features; f++) {
        const CerbFeature &ft = d.features[f];
        if (ft.start_frame < 0 || ft.n_obs < 1 || ft.start_frame + ft.n_obs > CERB_NUM_FRAMES || ft.obs_offset < 0 || ft.obs_offset + ft.n_obs > d.n_obs)
            return fail(CERB_ERR_BAD_ARGUMENT, "window: malformed feature track");
        n0 += ft.start_frame == 0;
    }
    if (n_anchor0) *n_anchor0 = n0;
    return validate_prior(d.prior);
}

static void run_stage_jobs(const std::vector<StageJob> &jobs) {
    if (jobs.empty()) return;
    size_t total = 0; for (const auto &j : jobs) total += j.bytes;
    unsigned hw = std::thread::hardware_concurrency();
    int nth = (int)std::min<unsigned>(hw ? hw : 1, 16u);
    if (total < (4u << 20)) nth = 1;
    auto work = [&](int t) { for (size_t k = t; k < jobs.size(); k += nth) std::memcpy(jobs[k].dst, jobs[k].src, jobs[k].bytes); };
    std::vector<std::thread> th;
    for (int t = 1; t < nth; t++) th.emplace_back(work, t);
    work(0);
    for (auto &t : th) t.join();
}

// validate windows [w0, w0 + cn), move their raw descriptors to the device on stream s (staging only what is not registered)
static int upload_raw(CerbHandle *h, int w0, int cn, const CerbWindowDesc *descs, const CerbWindowState *states, cudaStream_t s, double *t_stage_ms) {
    for (int w = w0; w < w0 + cn; w++) { int rc = validate_window(h, descs[w], states[w], &h->n0[w]); if (rc) return rc; h->nfeat[w] = descs[w].n_features; }
    UploadPlan pl;
    const size_t F = h->F, O = h->O, W0 = (size_t)w0;
    auto dv = [&](void *base, size_t per) { return (char *)base + W0 * per; };
    plan_rows(h, pl, w0, cn, dv(h->d_rdesc, sizeof(CerbWindowDesc)), dv(h->h_rdesc, sizeof(CerbWindowDesc)), sizeof(CerbWindowDesc), 1, 0,
              [&](int w) { return (const void *)&descs[w]; }, [&](int) { return sizeof(CerbWindowDesc); });
    plan_rows(h, pl, w0, cn, dv(h->d_rstate, sizeof(CerbWindowState)), dv(h->h_rstate, sizeof(CerbWindowState)), sizeof(CerbWindowState), 1, 0,
              [&](int w) { return (const void *)&states[w]; }, [&](int) { return sizeof(CerbWindowState); });
    plan_rows(h, pl, w0, cn, dv(h->d_rfeat, F * sizeof(CerbFeature)), dv(h->h_rfeat, F * sizeof(CerbFeature)), F * sizeof(CerbFeature), 1, 0,
              [&](int w) { return (const void *)descs[w].features; }, [&](int w) { return (size_t)descs[w].n_features * sizeof(CerbFeature); });
    plan_rows(h, pl, w0, cn, dv(h->d_robs, O * sizeof(CerbObservation)), dv(h->h_robs, O * sizeof(CerbObservation)), O * sizeof(CerbObservation), 1, 0,
              [&](int w) { return (const void *)descs[w].obs; }, [&](int w) { return (size_t)descs[w].n_obs * sizeof(CerbObservation); });
    plan_rows(h, pl, w0, cn, dv(h->d_rlam, F * 8), dv(h->h_rlam, F * 8), F * 8, 1, 0,
              [&](int w) { return (const void *)states[w].para_Feature; }, [&](int w) { return (size_t)descs[w].n_features * 8; });
    // preintegration results: the members IMULegFactor::Evaluate reads -- head (33 doubles) and, contiguous in the struct, jacobian columns 21..30 + covariance
    const size_t pre_pitch = (size_t)RAW_PRE_STRIDE * 8, tail_off = (size_t)(RAW_PRE_HEAD + RAW_PRE_JCOL0 * 31) * 8, tail_w = sizeof(CerbIMULegPreint) - tail_off;
    static_assert(sizeof(CerbIMULegPreint) == (33 + 2 * 961) * 8, "CerbIMULegPreint layout");
    static_assert(sizeof(CerbIMUPreint) == 467 * 8 && sizeof(CerbIMUPreint) <= RAW_PRE_STRIDE * 8, "CerbIMUPreint layout");
    plan_rows(h, pl, w0, cn, dv(h->d_rpre, 10 * pre_pitch), dv(h->h_rpre, 10 * pre_pitch), pre_pitch, CERB_WINDOW_SIZE, sizeof(CerbIMULegPreint),
              [&](int w) { return (const void *)descs[w].preint; }, [&](int w) { return descs[w].preint ? (size_t)RAW_PRE_HEAD * 8 : (size_t)0; });
    plan_rows(h, pl, w0, cn, dv(h->d_rpre, 10 * pre_pitch) + RAW_PRE_HEAD * 8, dv(h->h_rpre, 10 * pre_pitch) + RAW_PRE_HEAD * 8, pre_pitch, CERB_WINDOW_SIZE, sizeof(CerbIMULegPreint),
              [&](int w) { return (const void *)((const char *)descs[w].preint + tail_off); }, [&](int w) { return descs[w].preint ? tail_w : (size_t)0; });
    plan_rows(h, pl, w0, cn, dv(h->d_rpre, 10 * pre_pitch), dv(h->h_rpre, 10 * pre_pitch), pre_pitch, CERB_WINDOW_SIZE, sizeof(CerbIMUPreint),
              [&](int w) { return (const void *)descs[w].imu_preint; }, [&](int w) { return descs[w].preint ? (size_t)0 : sizeof(CerbIMUPreint); });
    const size_t pj_pitch = (size_t)PRIOR_LD * PRIOR_LD * 8;
    plan_rows(h, pl, w0, cn, dv(h->d_pJ, pj_pitch), dv(h->h_pJ, pj_pitch), pj_pitch, 1, 0,
              [&](int w) { return (const void *)descs[w].prior.linearized_jacobians; }, [&](int w) { return descs[w].prior.valid ? (size_t)descs[w].prior.n * descs[w].prior.n * 8 : (size_t)0; });
    plan_rows(h, pl, w0, cn, dv(h->d_pr, PRIOR_LD * 8), dv(h->h_pr, PRIOR_LD * 8), (size_t)PRIOR_LD * 8, 1, 0,
              [&](int w) { return (const void *)descs[w].prior.linearized_residuals; }, [&](int w) { return descs[w].prior.valid ? (size_t)descs[w].prior.n * 8 : (size_t)0; });
    const auto t0 = std::chrono::steady_clock::now();
    run_stage_jobs(pl.stage);
    if (t_stage_ms) *t_stage_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    for (const DmaOp &op : pl.dma) {
        if (op.height == 1) CUDA_TRY(cudaMemcpyAsync(op.dst, op.src, op.width, cudaMemcpyHostToDevice, s));
        else CUDA_TRY(cudaMemcpy2DAsync(op.dst, op.dpitch, op.src, op.spitch, op.width, op.height, cudaMemcpyHostToDevice, s));
    }
    h->last_dma_ops += (int)pl.dma.size(); h->last_staged_bytes += [&] { size_t t = 0; for (const auto &j : pl.stage) t += j.bytes; return t; }();
    return CERB_OK;
}

// device pack of windows [w0, w0 + cn) (after their raw descriptors have arrived) on stream s
static int enqueue_pack(CerbHandle *h, int w0, int cn, cudaStream_t s) {
    PackParams P;
    const size_t W0 = (size_t)w0, F = h->F, O = h->O;
    P.n = cn; P.maxF = h->F; P.maxObs = h->O;
    P.rdesc = h->d_rdesc + W0; P.rfeat = h->d_rfeat + W0 * F; P.robs = h->d_robs + W0 * O; P.rpre = h->d_rpre + W0 * 10 * RAW_PRE_STRIDE; P.rstate = h->d_rstate + W0; P.rlam = h->d_rlam + W0 * F;
    P.n_features = h->d_nfeat + W0; P.feat_start = h->d_fstart + W0 * F; P.feat_nobs = h->d_fnobs + W0 * F; P.feat_off = h->d_foff + W0 * F; P.flags = h->d_flags + W0;
    P.obs_stereo = h->d_stereo + W0 * O; P.prior_meta = h->d_pmeta + W0 * PRIOR_META_STRIDE; P.perm = h->d_perm + W0 * F;
    P.obs = h->d_obs + W0 * NOBS_PLANES * O; P.pre = h->d_pre + W0 * 10 * PRE_STRIDE; P.prior_x0 = h->d_px0 + W0 * 16 * 9; P.state0 = h->d_state0 + W0 * ST_STRIDE; P.lam0 = h->d_lam0 + W0 * F;
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
    h->h_perm.resize((size_t)h->B * h->F);
    CUDA_TRY(cudaMemcpyAsync(h->h_perm.data(), h->d_perm, (size_t)h->n * h->F * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    h->perm_valid = true;
    return CERB_OK;
}

static SolveParams make_params(CerbHandle *h, int w0, int n, int max_iters, double *dbg, int dbg_window) {
    SolveParams P;
    std::memset(&P, 0, sizeof(P));
    const CerbSolverConfig &c = h->cfg;
    P.n_windows = n; P.maxF = h->F; P.maxObs = h->O; P.max_iters = max_iters; P.optimize_leg_bias = c.optimize_leg_bias;
    for (int k = 0; k < 3; k++) P.G[k] = c.g[k];
    P.sqrt_info = c.visual_sqrt_info; P.huber = c.huber_delta;
    P.radius0 = c.initial_trust_region_radius; P.max_radius = c.max_trust_region_radius; P.min_radius = c.min_trust_region_radius;
    P.min_rel_dec = c.min_relative_decrease; P.ftol = c.function_tolerance; P.gtol = c.gradient_tolerance; P.ptol = c.parameter_tolerance;
    const size_t W0 = (size_t)w0, F = h->F, O = h->O;
    P.n_features = h->d_nfeat + W0; P.feat_start = h->d_fstart + W0 * F; P.feat_nobs = h->d_fnobs + W0 * F; P.feat_off = h->d_foff + W0 * F; P.flags = h->d_flags + W0;
    P.obs = h->d_obs + W0 * NOBS_PLANES * O; P.obs_stereo = h->d_stereo + W0 * O; P.pre = h->d_pre + W0 * 10 * PRE_STRIDE; P.sinfo = h->d_sinfo + W0 * 10 * 961;
    P.prior_J = h->d_pJ + W0 * PRIOR_LD * PRIOR_LD; P.prior_r = h->d_pr + W0 * PRIOR_LD; P.prior_x0 = h->d_px0 + W0 * 16 * 9; P.prior_Hp = h->d_pHp + W0 * PRIOR_LD * PRIOR_LD;
    P.prior_meta = h->d_pmeta + W0 * PRIOR_META_STRIDE;
    P.state = h->d_state + W0 * ST_STRIDE; P.lam = h->d_lam + W0 * F; P.rep_i = h->d_repi + W0 * 4; P.rep_d = h->d_repd + W0 * 2; P.ws = h->d_ws; P.ws_stride = h->ws_stride;
    P.dbg = dbg; P.dbg_window = dbg_window;
    P.test_fail_factorizations = h->test_fail_factorizations; P.test_initial_mu = h->test_initial_mu;
    P.no_bulk_copy = std::getenv("CERB_NO_TMA") != nullptr;
    return P;
}

// restore the initial states of windows [w0, w0 + n), prepare (sqrt_info, prior Gram matrix) and solve; asynchronous on the stream
static int enqueue_solve(CerbHandle *h, int w0, int n, int max_iters, double *dbg, int dbg_window, bool restore = true, bool probe = false, int lane = 0) {
    cudaStream_t s = h->lane[lane];
    const size_t W0 = (size_t)w0;
    if (restore) {
        CUDA_TRY(cudaMemcpyAsync(h->d_state + W0 * ST_STRIDE, h->d_state0 + W0 * ST_STRIDE, (size_t)n * ST_STRIDE * sizeof(double), cudaMemcpyDeviceToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(h->d_lam + W0 * h->F, h->d_lam0 + W0 * h->F, (size_t)n * h->F * sizeof(double), cudaMemcpyDeviceToDevice, s));
    }
    const int nfac = n * 10;
    CERB_LAUNCH(imu_leg_prepare_kernel, (nfac + 1) / 2, 64, 0, s, nfac, (const double *)(h->d_pre + W0 * 10 * PRE_STRIDE), h->d_sinfo + W0 * 10 * 961);
    CERB_LAUNCH(prior_prepare_kernel, n, 256, (size_t)PRIOR_TROWS * PRIOR_TLD * sizeof(double), s, (const double *)(h->d_pJ + W0 * PRIOR_LD * PRIOR_LD), (const int *)(h->d_pmeta + W0 * PRIOR_META_STRIDE), h->d_pHp + W0 * PRIOR_LD * PRIOR_LD);
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

static int download(CerbHandle *h, CerbWindowState *states, CerbSolveReport *reports) {
    const int n = h->n; const size_t F = h->F;
    cudaStream_t s = h->stream;
    UnpackParams U;
    U.n = n; U.maxF = h->F; U.n_features = h->d_nfeat; U.perm = h->d_perm; U.rep_i = h->d_repi; U.rep_d = h->d_repd;
    U.lam = h->solved ? h->d_lam : h->d_lam0; U.state = h->solved ? h->d_state : h->d_state0;
    U.olam = h->d_olam; U.orep = h->d_orep; U.ostate = h->d_ostate;
    CERB_LAUNCH(unpack_kernel, std::min(n, 8 * h->sm_count), PACK_THREADS, 0, s, U);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(h->h_state, h->d_ostate, (size_t)n * ST_STRIDE * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(h->h_lam, h->d_olam, n * F * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(h->h_orep, h->d_orep, (size_t)n * sizeof(CerbSolveReport), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    int rc = collect_time(h); if (rc) return rc;
    int status = CERB_OK;
    for (int w = 0; w < n; w++) {
        if (states) {
            std::memcpy(&states[w], h->h_state + (size_t)w * ST_STRIDE, ST_SIZE * sizeof(double));        // para_Pose .. para_Td: contiguous, same order
            if (states[w].para_Feature && h->nfeat[w]) std::memcpy(states[w].para_Feature, h->h_lam + (size_t)w * F, (size_t)h->nfeat[w] * sizeof(double));
        }
        if (reports) reports[w] = h->h_orep[w];
        if (h->h_orep[w].status != 0) status = CERB_ERR_NON_FINITE;
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
        if (src) cudaMemcpyAsync(d, src, n * sizeof(double), cudaMemcpyHostToDevice, s);
        return d;
    }
    int *upi(const int *src, size_t n, cudaStream_t s) {
        int *d = (int *)raw(n * sizeof(int)); if (!d) return nullptr;
        if (src) cudaMemcpyAsync(d, src, n * sizeof(int), cudaMemcpyHostToDevice, s);
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
static int pack_prior(const CerbPrior &pr, int *meta, double *J, double *r, double *x0) {
    std::memset(meta, 0, PRIOR_META_STRIDE * sizeof(int));
    if (!pr.valid) return CERB_OK;
    int rc = validate_prior(pr); if (rc) return rc;
    meta[0] = 1; meta[1] = pr.n; meta[2] = pr.num_blocks;
    for (int b = 0; b < pr.num_blocks; b++) {
        meta[4 + 3 * b] = pr.block_kind[b]; meta[5 + 3 * b] = pr.block_index[b]; meta[6 + 3 * b] = pr.block_col[b];
        for (int k = 0; k < 9; k++) x0[9 * b + k] = pr.block_x0[b][k];
    }
    std::memcpy(J, pr.linearized_jacobians, sizeof(double) * pr.n * pr.n);
    std::memcpy(r, pr.linearized_residuals, sizeof(double) * pr.n);
    return CERB_OK;
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

int cerb_eval_imu_leg(CerbHandle *h, int32_t n, const CerbIMULegPreint *preint, const double *params, double *residuals, double *jacobians, double *sqrt_info) {
    if (!h || n < 1 || !preint || !params) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_eval_imu_leg: bad argument");
    CERB_DEVICE(h);
    cudaStream_t s = h->stream; DevBuf B(h); const size_t N = n;
    std::vector<double> packed(N * PRE_STRIDE, 0.0);
    for (int k = 0; k < n; k++) pack_preint(preint[k], packed.data() + (size_t)k * PRE_STRIDE);
    double *dpre = B.up(packed.data(), N * PRE_STRIDE, s), *dsi = B.up(nullptr, N * 961, s), *dpar = B.up(params, 40 * N, s);
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

int cerb_eval_imu(CerbHandle *h, int32_t n, const CerbIMUPreint *preint, const double *params, double *residuals, double *jacobians, double *sqrt_info) {
    if (!h || n < 1 || !preint || !params) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_eval_imu: bad argument");
    CERB_DEVICE(h);
    cudaStream_t s = h->stream; DevBuf B(h); const size_t N = n;
    std::vector<double> packed(N * PRE_STRIDE), p40(N * 40, 0.0);
    for (int k = 0; k < n; k++) {
        pack_imu_preint(preint[k], packed.data() + (size_t)k * PRE_STRIDE);
        const double *q = params + (size_t)k * 32; double *o = p40.data() + (size_t)k * 40;
        std::memcpy(o, q, 16 * sizeof(double)); std::memcpy(o + 20, q + 16, 16 * sizeof(double));     // leg-bias slots stay 0
    }
    double *dpre = B.up(packed.data(), N * PRE_STRIDE, s), *dsi = B.up(nullptr, N * 961, s), *dpar = B.up(p40.data(), 40 * N, s);
    double *dr = B.up(nullptr, 31 * N, s), *dJ = jacobians ? B.up(nullptr, 31 * 40 * N, s) : nullptr;
    if (!dpre || !dsi || !dpar || !dr) return fail(CERB_ERR_CUDA, "device allocation failed");
    CERB_LAUNCH(imu_leg_prepare_kernel, (n + 1) / 2, 64, 0, s, (int)n, (const double *)dpre, dsi);
    CERB_LAUNCH(imu_leg_eval_kernel, n, 128, 0, s, (int)n, (const double *)dpre, (const double *)dsi, (const double *)dpar, (const double *)h->d_G, dr, dJ);
    CUDA_TRY(cudaGetLastError());
    std::vector<double> hr(31 * N), hj(jacobians ? 31 * 40 * N : 0), hs(961 * N);
    CUDA_TRY(cudaMemcpyAsync(hr.data(), dr, hr.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (jacobians) CUDA_TRY(cudaMemcpyAsync(hj.data(), dJ, hj.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(hs.data(), dsi, hs.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
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
    int rc = pack_prior(*prior, meta.data(), J.data(), r.data(), x0.data()); if (rc) return rc;
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
static int feature_pass(CerbHandle *h, int which, double param, double *out, int32_t *remove) {
    if (!h || !out) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    CERB_DEVICE(h);
    if (h->n < 1) return fail(CERB_ERR_BAD_ARGUMENT, "no resident batch");
    const int n = h->n, F = h->F;
    cudaStream_t s = h->stream; DevBuf B(h);
    double *d_out = B.up(nullptr, (size_t)n * F, s), *d_perm_out = B.up(nullptr, (size_t)n * F, s);
    if (!d_out || !d_perm_out) return fail(CERB_ERR_CUDA, "device allocation failed");
    const int threads = 128, blocks = (n * F + threads - 1) / threads;
    const double *d_st = h->solved ? h->d_state : h->d_state0, *d_lm = h->solved ? h->d_lam : h->d_lam0;
    if (which == 0)
        CERB_LAUNCH(outlier_error_kernel, blocks, threads, 0, s, n, F, h->O, (const int *)h->d_nfeat, (const int *)h->d_fstart, (const int *)h->d_fnobs, (const int *)h->d_foff,
                    (const double *)h->d_obs, (const int *)h->d_stereo, d_st, d_lm, d_out);
    else
        CERB_LAUNCH(triangulate_kernel, blocks, threads, 0, s, n, F, h->O, (const int *)h->d_nfeat, (const int *)h->d_fstart, (const int *)h->d_fnobs, (const int *)h->d_foff,
                    (const double *)h->d_obs, (const int *)h->d_stereo, d_st, d_lm, param, d_out);
    CERB_LAUNCH(unpermute_kernel, blocks, threads, 0, s, n, F, 1, (const int *)h->d_nfeat, (const int *)h->d_perm, (const double *)d_out, d_perm_out);      // device slot -> caller's feature index
    CUDA_TRY(cudaGetLastError());
    std::vector<double> tmp((size_t)n * F);
    CUDA_TRY(cudaMemcpyAsync(tmp.data(), d_perm_out, tmp.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    for (int w = 0; w < n; w++)
        for (int f = 0; f < h->nfeat[w]; f++) {
            const double v = tmp[(size_t)w * F + f];
            out[(size_t)w * F + f] = v;
            if (remove) remove[(size_t)w * F + f] = (v * param > 3.0) ? 1 : 0;
        }
    return CERB_OK;
}
int cerb_batch_outlier_errors(CerbHandle *h, double focal_length, double *ave_err, int32_t *remove) { return feature_pass(h, 0, focal_length, ave_err, remove); }
int cerb_batch_triangulate(CerbHandle *h, double init_depth, double *depth) { return feature_pass(h, 1, init_depth, depth, nullptr); }
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

int cerb_batch_marginalize(CerbHandle *h, const int32_t *flags, const CerbWindowState *states, CerbPrior *priors, int32_t *sweeps) {
    if (!h || !flags || !priors) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_marginalize: null argument");
    CERB_DEVICE(h);
    const int n = h->n, F = h->F;
    if (n < 1) return fail(CERB_ERR_BAD_ARGUMENT, "no resident batch");
    for (int w = 0; w < n; w++) {
        if (flags[w] != 0 && flags[w] != 1) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_marginalize: flag must be 0 (MARGIN_OLD) or 1 (MARGIN_SECOND_NEW)");
        if (!priors[w].linearized_jacobians || !priors[w].linearized_residuals) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_marginalize: priors[w] needs storage for linearized_jacobians / linearized_residuals");
    }
    cudaStream_t s = h->stream; DevBuf B(h);
    int mmax = 19;
    const int nmax = MARG_N_STRUCT;            // what a window can keep (the kernel skips a window that claims more); the prior arrays keep the stride CERB_MAX_PRIOR_DIM
    for (int w = 0; w < n; w++) if (flags[w] == 0) mmax = std::max(mmax, 19 + h->n0[w]);
    const int posmax = mmax + CERB_MAX_PRIOR_DIM;
    // states to linearise at: the caller's (after double2vector + vector2double), or the resident ones
    std::vector<double> hst((size_t)n * ST_STRIDE, 0.0);
    const double *d_st, *d_lm;
    if (states) {
        std::vector<double> hl((size_t)n * F, 0.0);
        for (int w = 0; w < n; w++) {
            std::memcpy(hst.data() + (size_t)w * ST_STRIDE, &states[w], ST_SIZE * sizeof(double));
            if (h->nfeat[w]) { if (!states[w].para_Feature) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_marginalize: null para_Feature"); std::memcpy(hl.data() + (size_t)w * F, states[w].para_Feature, (size_t)h->nfeat[w] * 8); }
        }
        double *ds = B.up(hst.data(), hst.size(), s), *dlc = B.up(hl.data(), hl.size(), s), *dl = B.up(nullptr, (size_t)n * F, s);
        if (!ds || !dlc || !dl) return fail(CERB_ERR_CUDA, "device allocation failed");
        CERB_LAUNCH(permute_lam_kernel, (int)(((size_t)n * F + 127) / 128), 128, 0, s, n, F, (const int *)h->d_nfeat, (const int *)h->d_perm, (const double *)dlc, dl);
        CUDA_TRY(cudaStreamSynchronize(s));               // hl / hst are read by the asynchronous copies
        d_st = ds; d_lm = dl;
    } else {
        d_st = h->solved ? h->d_state : h->d_state0; d_lm = h->solved ? h->d_lam : h->d_lam0;
        CUDA_TRY(cudaMemcpyAsync(hst.data(), d_st, hst.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    std::vector<int> hflags(flags, flags + n);
    int *dflags = B.upi(hflags.data(), n, s), *ddims = B.upi(nullptr, (size_t)n * 4, s), *dblocks = B.upi(nullptr, (size_t)n * 64, s), *dsw = B.upi(nullptr, (size_t)n * 2, s);
    double *dJ = B.up(nullptr, (size_t)n * PRIOR_LD * PRIOR_LD, s), *dr = B.up(nullptr, (size_t)n * PRIOR_LD, s);
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
    for (int w0 = 0; w0 < n; w0 += per) {
        const int cn = std::min(per, n - w0);
        // sqrt_info of the IMU-leg factors and the Gram matrix of the old prior (a solve leaves them behind; a bare upload does not)
        const int nfac = cn * 10;
        CERB_LAUNCH(imu_leg_prepare_kernel, (nfac + 1) / 2, 64, 0, s, nfac, (const double *)(h->d_pre + (size_t)w0 * 10 * PRE_STRIDE), h->d_sinfo + (size_t)w0 * 10 * 961);
        CERB_LAUNCH(prior_prepare_kernel, cn, 256, (size_t)PRIOR_TROWS * PRIOR_TLD * sizeof(double), s, (const double *)(h->d_pJ + (size_t)w0 * PRIOR_LD * PRIOR_LD), (const int *)(h->d_pmeta + (size_t)w0 * PRIOR_META_STRIDE), h->d_pHp + (size_t)w0 * PRIOR_LD * PRIOR_LD);
        SolveParams P = make_params(h, w0, cn, 0, nullptr, -1);
        MargParams M;
        M.flags = dflags + w0; M.state = d_st + (size_t)w0 * ST_STRIDE; M.lam = d_lm + (size_t)w0 * F; M.A = dA; M.b = db; M.posmax = posmax;
        M.dims = ddims + (size_t)w0 * 4; M.blocks = dblocks + (size_t)w0 * 64;
        CERB_LAUNCH(marg_assemble_kernel, std::min(cn, h->grid), SOLVE_THREADS, h->smem_bytes, s, P, M);
        CERB_LAUNCH(marg_schur_kernel, std::min(cn, sgrid), marg_threads(mmax, nmax, lim), marg_smem_bytes(mmax, nmax, lim), s, cn, mmax, nmax, (const int *)(ddims + (size_t)w0 * 4), (const double *)dA, (long)posmax * posmax,
                    (const double *)db, (long)posmax, 1e-8, dws, dJ + (size_t)w0 * PRIOR_LD * PRIOR_LD, (long)PRIOR_LD * PRIOR_LD, dr + (size_t)w0 * PRIOR_LD, (long)PRIOR_LD, dsw + (size_t)w0 * 2, (int)lim);
        CUDA_TRY(cudaGetLastError());
    }
    std::vector<int> hdims((size_t)n * 4), hblocks((size_t)n * 64), hsw((size_t)n * 2);
    double *hJ = h->h_pJ, *hr = h->h_pr;       // the pinned staging of the prior upload is idle here: D2H at PCIe rate instead of through pageable memory
    CUDA_TRY(cudaMemcpyAsync(hdims.data(), ddims, hdims.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(hblocks.data(), dblocks, hblocks.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(hsw.data(), dsw, hsw.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(hJ, dJ, (size_t)n * PRIOR_LD * PRIOR_LD * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(hr, dr, (size_t)n * PRIOR_LD * sizeof(double), cudaMemcpyDeviceToHost, s));
    // a prior that is carried over unchanged comes back from the device copy of the old one
    std::vector<int> hmeta((size_t)n * PRIOR_META_STRIDE); std::vector<double> hx0((size_t)n * 16 * 9);
    CUDA_TRY(cudaMemcpyAsync(hmeta.data(), h->d_pmeta, hmeta.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(hx0.data(), h->d_px0, hx0.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    std::vector<double> oldJ, oldr;
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
            const int *meta = hmeta.data() + (size_t)w * PRIOR_META_STRIDE;
            if (!meta[0]) continue;
            pr.valid = 1; pr.n = meta[1]; pr.num_blocks = meta[2];
            for (int b = 0; b < pr.num_blocks; b++) {
                pr.block_kind[b] = meta[4 + 3 * b]; pr.block_index[b] = meta[5 + 3 * b]; pr.block_col[b] = meta[6 + 3 * b];
                for (int k = 0; k < 9; k++) pr.block_x0[b][k] = hx0[(size_t)w * 144 + 9 * b + k];
            }
            oldJ.resize((size_t)pr.n * pr.n); oldr.resize(pr.n);
            CUDA_TRY(cudaMemcpy(oldJ.data(), h->d_pJ + (size_t)w * PRIOR_LD * PRIOR_LD, oldJ.size() * 8, cudaMemcpyDeviceToHost));
            CUDA_TRY(cudaMemcpy(oldr.data(), h->d_pr + (size_t)w * PRIOR_LD, oldr.size() * 8, cudaMemcpyDeviceToHost));
            std::memcpy(Jout, oldJ.data(), oldJ.size() * 8); std::memcpy(rout, oldr.data(), oldr.size() * 8);
            continue;
        }
        const int nn = hdims[4 * w + 1], nb = hdims[4 * w + 3];
        pr.valid = 1; pr.n = nn; pr.num_blocks = nb;
        const double *st = hst.data() + (size_t)w * ST_STRIDE;
        for (int b = 0; b < nb; b++) {
            const int *q = hblocks.data() + (size_t)w * 64 + 4 * b;
            pr.block_kind[b] = q[0]; pr.block_index[b] = q[1]; pr.block_col[b] = q[2];
            const int size = prior_block_size(q[0]);
            const double *x = st + prior_block_state_offset(q[0], q[3]);          // keep_block_data: the state the factors were linearised at
            for (int k = 0; k < 9; k++) pr.block_x0[b][k] = k < size ? x[k] : 0.0;
        }
        out_jobs.push_back({Jout, hJ + (size_t)w * PRIOR_LD * PRIOR_LD, (size_t)nn * nn * 8});       // 59 KB per window: copied by a few threads below
        std::memcpy(rout, hr + (size_t)w * PRIOR_LD, (size_t)nn * 8);
    }
    run_stage_jobs(out_jobs);
    return CERB_OK;
}

int cerb_batch_update_states(CerbHandle *h, int32_t n, const CerbWindowState *states) {
    if (!h || !states) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    CERB_DEVICE(h);
    if (h->n < 1 || n != h->n) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_update_states: n must be the size of the resident batch");
    const int F = h->F;
    cudaStream_t s = h->stream; DevBuf B(h);
    std::vector<double> hst((size_t)n * ST_STRIDE, 0.0), hl((size_t)n * F, 0.0);
    for (int w = 0; w < n; w++) {
        std::memcpy(hst.data() + (size_t)w * ST_STRIDE, &states[w], ST_SIZE * sizeof(double));
        if (h->nfeat[w]) { if (!states[w].para_Feature) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_batch_update_states: null para_Feature"); std::memcpy(hl.data() + (size_t)w * F, states[w].para_Feature, (size_t)h->nfeat[w] * 8); }
    }
    double *ds = B.up(hst.data(), hst.size(), s), *dlc = B.up(hl.data(), hl.size(), s);
    if (!ds || !dlc) return fail(CERB_ERR_CUDA, "device allocation failed");
    CUDA_TRY(cudaMemcpyAsync(h->d_state0, ds, hst.size() * sizeof(double), cudaMemcpyDeviceToDevice, s));
    CERB_LAUNCH(permute_lam_kernel, (int)(((size_t)n * F + 127) / 128), 128, 0, s, n, F, (const int *)h->d_nfeat, (const int *)h->d_perm, (const double *)dlc, h->d_lam0);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(s));               // hst / hl are read by the asynchronous copies
    h->solved = false;                                 // the per-feature passes and a resident solve start from these states
    return CERB_OK;
}

int cerb_batch_shift_depth(CerbHandle *h, double init_depth, int32_t *new_start_frame, double *depth, int32_t *keep) {
    if (!h || !new_start_frame || !depth || !keep) return fail(CERB_ERR_BAD_ARGUMENT, "null argument");
    CERB_DEVICE(h);
    if (h->n < 1) return fail(CERB_ERR_BAD_ARGUMENT, "no resident batch");
    const int n = h->n, F = h->F;
    const size_t N = (size_t)n * F;
    cudaStream_t s = h->stream; DevBuf B(h);
    double *d_out = B.up(nullptr, 3 * N, s), *d_perm_out = B.up(nullptr, 3 * N, s);
    if (!d_out || !d_perm_out) return fail(CERB_ERR_CUDA, "device allocation failed");
    const double *d_st = h->solved ? h->d_state : h->d_state0, *d_lm = h->solved ? h->d_lam : h->d_lam0;
    CERB_LAUNCH(shift_depth_kernel, (int)((N + 127) / 128), 128, 0, s, n, F, h->O, (const int *)h->d_nfeat, (const int *)h->d_fstart, (const int *)h->d_fnobs, (const int *)h->d_foff,
                (const double *)h->d_obs, d_st, d_lm, init_depth, d_out);
    CERB_LAUNCH(unpermute_kernel, (int)((N + 127) / 128), 128, 0, s, n, F, 3, (const int *)h->d_nfeat, (const int *)h->d_perm, (const double *)d_out, d_perm_out);
    CUDA_TRY(cudaGetLastError());
    std::vector<double> tmp(3 * N);
    CUDA_TRY(cudaMemcpyAsync(tmp.data(), d_perm_out, tmp.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    for (int w = 0; w < n; w++)
        for (int f = 0; f < h->nfeat[w]; f++) {
            const size_t q = (size_t)w * F + f;
            new_start_frame[q] = (int32_t)tmp[q]; depth[q] = tmp[N + q]; keep[q] = (int32_t)tmp[2 * N + q];
        }
    return CERB_OK;
}

// ---- leg-contact preintegration ------------------------------------------------------------------------------------
static int preintegrate_impl(CerbHandle *h, const CerbPreintConfig *cfg, int32_t n, const CerbPreintJob *jobs, CerbIMULegPreint *out, CerbIMUPreint *out_imu) {
    if (!h || !cfg || n < 1 || !jobs || (!out && !out_imu)) return fail(CERB_ERR_BAD_ARGUMENT, "cerb_preintegrate: bad argument");
    CERB_DEVICE(h);
    PreintParams P;
    P.imu_only = out_imu ? 1 : 0;
    P.acc_n = cfg->acc_n; P.acc_n_z = cfg->acc_n_z; P.gyr_n = cfg->gyr_n; P.acc_w = cfg->acc_w; P.gyr_w = cfg->gyr_w; P.phi_n = cfg->phi_n; P.dphi_n = cfg->dphi_n;
    P.rho_c_n = cfg->rho_c_n; P.rho_nc_n = cfg->rho_nc_n; P.v_n_min_xy = cfg->v_n_min_xy; P.v_n_min_z = cfg->v_n_min_z; P.v_n_min = cfg->v_n_min; P.v_n_max = cfg->v_n_max;
    P.v_n_force_thres_ratio = cfg->v_n_force_thres_ratio; P.v_n_term1_steep = cfg->v_n_term1_steep; P.v_n_term2_var_rescale = cfg->v_n_term2_var_rescale;
    P.v_n_term3_distance_rescale = cfg->v_n_term3_distance_rescale; P.contact_sensor_type = cfg->contact_sensor_type;
    for (int l = 0; l < 4; l++) for (int k = 0; k < 4; k++) P.rho_fix[4 * l + k] = cfg->rho_fix[l][k];
    for (int k = 0; k < 3; k++) P.p_br[k] = cfg->p_br[k];
    for (int k = 0; k < 9; k++) P.R_br[k] = cfg->R_br[k];
    size_t total = 0;
    for (int j = 0; j < n; j++) { if (jobs[j].n_samples < 0 || (jobs[j].n_samples && !jobs[j].samples)) return fail(CERB_ERR_BAD_ARGUMENT, "bad job"); total += jobs[j].n_samples; }
    std::vector<double> hj((size_t)n * PJ_STRIDE), hs(std::max<size_t>(total, 1) * SAMPLE_STRIDE);
    std::vector<int> hi((size_t)n * 2);
    size_t off = 0;
    for (int j = 0; j < n; j++) {
        const CerbPreintJob &q = jobs[j];
        double *o = hj.data() + (size_t)j * PJ_STRIDE;
        std::memcpy(o, q.acc_0, 24); std::memcpy(o + 3, q.gyr_0, 24); std::memcpy(o + 6, q.phi_0, 96); std::memcpy(o + 18, q.dphi_0, 96); std::memcpy(o + 30, q.c_0, 32);
        std::memcpy(o + 34, q.linearized_ba, 24); std::memcpy(o + 37, q.linearized_bg, 24); std::memcpy(o + 40, q.linearized_rho, 32);
        hi[2 * j] = q.n_samples; hi[2 * j + 1] = (int)off;
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
    if (!dj || !ds || !dout || !dfull || !di) return fail(CERB_ERR_CUDA, "device allocation failed");
    CERB_LAUNCH(preintegrate_kernel, n, 128, 0, s, P, (int)n, (const double *)dj, (const int *)di, (const double *)ds, dout, dfull);
    CUDA_TRY(cudaGetLastError());
    std::vector<double> ho((size_t)n * PRE_STRIDE), hf((size_t)n * 1922);
    CUDA_TRY(cudaMemcpyAsync(ho.data(), dout, ho.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(hf.data(), dfull, hf.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    for (int j = 0; j < n; j++) {
        const double *o = ho.data() + (size_t)j * PRE_STRIDE, *f = hf.data() + (size_t)j * 1922;
        if (out_imu) {
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

int cerb_preintegrate_batch(CerbHandle *h, const CerbPreintConfig *cfg, int32_t n, const CerbPreintJob *jobs, CerbIMULegPreint *out) {
    return preintegrate_impl(h, cfg, n, jobs, out, nullptr);
}
int cerb_preintegrate_imu_batch(CerbHandle *h, const CerbPreintConfig *cfg, int32_t n, const CerbPreintJob *jobs, CerbIMUPreint *out) {
    return preintegrate_impl(h, cfg, n, jobs, nullptr, out);
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

#include "replay_host.inl"

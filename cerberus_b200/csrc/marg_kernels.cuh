// marg_kernels.cuh -- the dense tail of MarginalizationInfo::marginalize() on the device, one CTA per window:
//   reference src/factor/marginalization_factor.cpp:281-305
//     Amm = 0.5 (A_mm + A_mm^T); SelfAdjointEigenSolver(Amm); Amm_inv = V diag(lambda > eps ? 1 / lambda : 0) V^T
//     A   = Arr - Arm Amm_inv Amr;  b = brr - Arm Amm_inv bmm
//     SelfAdjointEigenSolver(A) (lower triangle);  S = lambda > eps ? lambda : 0;  S_inv = lambda > eps ? 1 / lambda : 0
//     linearized_jacobians = diag(sqrt S) V^T;  linearized_residuals = diag(sqrt S_inv) V^T b
// The eigen-solver is a parallel two-sided Jacobi iteration (round-robin pair ordering: kp / 2 disjoint rotations per round, applied to both
// sides in one pass over 2 x 2 blocks), in fp64, on PACKED symmetric matrices that live in SHARED memory (m = 19 + tracks anchored at frame 0 ->
// 169 x 169 for the 150-feature configuration = 112 KB, 86 x 86 for the kept block; m > ~235 falls back to the L2-resident workspace).  Rotation
// formulas as in the CPU restatement (oracle/ref_math.h sym_eig_jacobi), different pair order; the rows of linearized_jacobians come out in the
// order the eigenvalues sit on the diagonal (J^T J and J^T r, the only things MarginalizationFactor uses, do not depend on it).
#pragma once
#include "compat.h"

namespace cerb {

#if defined(CERB_CUSIM)
constexpr int MARG_THREADS = 64;      // the CPU simulator pays ~ one futex wake-up per thread and barrier; two warps still exercise every path
#else
constexpr int MARG_THREADS = 512;      // upper bound of the block size (128 registers per thread); the launch picks marg_threads(m, n)
#endif
constexpr int MARG_MAX_SWEEPS = 60;

// Memory plan of one CTA.  The symmetric matrices are PACKED (upper triangle by columns: (i, j), i <= j, at j (j + 1) / 2 + i): one copy of every
// entry, so a rotation task writes 4 values instead of 8 and the 169 x 169 matrix of the 150-feature configuration (112 KB) leaves room for T.
//   phase 1  M1 (m x m packed) in SHARED memory when it fits, else in the global workspace;
//            T = V1^T [Amr | bm] (m x (n + 1), row-major): the rotations are applied to its rows as they are applied to the rows of M1, so V1
//            itself is never formed:  Arm Amm_inv [Amr | bm] = T^T diag(lambda > eps ? 1 / lambda : 0) T.  Columns [0, ncs) of T live in
//            shared memory behind M1, the remaining ncg = n + 1 - ncs columns (0 for m <= ~165; 3 at m = 169) in the global workspace (L2)
//   phase 2  M2 (n x n packed) over the dead M1, V2 (n x n) behind it over the dead T
constexpr size_t MARG_SMEM_MAX = 232448;               // 227 KB: the opt-in limit of dynamic shared memory per block on sm_90 (the kernel has no static shared memory)
constexpr size_t MARG_SMEM_TWO = 115712;               // 113 KB: two CTAs of 256 threads per SM below this
constexpr int MARG_N_STRUCT = 86;                      // kept dimension of a VILO window: 10 poses + speed-bias + leg bias + 2 extrinsics + td (SURVEY 8(a) a12)
CERB_HD int marg_ld(int k) { return k | 1; }
CERB_HD size_t marg_tri(int k) { return (size_t)k * (k + 1) / 2; }
CERB_HD size_t marg_fixed_doubles(int m, int n) { const int k = m > n ? m : n; return 2 * (size_t)((k + 3) & ~1) + 4 + 2 * ((size_t)(k + 2) / 4 + 1); }   // (c, s) tables x 2 (1 / lambda aliases the first) | flags | pair tables x 2 (ints)
struct MargPlan { int m1_smem, ncs; size_t t_off, body, ws; };
CERB_HD MargPlan marg_plan(int m, int n, size_t limit = MARG_SMEM_MAX) {      // limit < MARG_SMEM_MAX: test hook (forces the split / global layouts on small matrices)
    MargPlan P;
    const size_t avail = limit / sizeof(double) > marg_fixed_doubles(m, n) + 64 ? limit / sizeof(double) - marg_fixed_doubles(m, n) : 64;
    const size_t p2 = marg_tri(n) + (size_t)n * marg_ld(n);                                  // phase 2: M2 | V2
    P.t_off = marg_tri(m) > marg_tri(n) ? marg_tri(m) : marg_tri(n);                          // T behind both M1 and M2 (M2 is built while T is read)
    P.m1_smem = marg_tri(m) <= avail;
    P.ncs = 0;
    if (P.m1_smem && avail > P.t_off) { const size_t c = (avail - P.t_off) / (size_t)m; P.ncs = c > (size_t)(n + 1) ? n + 1 : (int)c; }
    const size_t p1 = P.m1_smem ? (P.ncs ? P.t_off + (size_t)m * P.ncs : marg_tri(m)) : 0;
    P.body = p1 > p2 ? p1 : p2;
    P.ws = (size_t)m * (n + 1 - P.ncs) + 1 + (P.m1_smem ? 0 : marg_tri(m)) + (size_t)n + 8;   // per-CTA global workspace in doubles: T tail | M1 (if not in shared memory) | br
    return P;
}
CERB_HD size_t marg_smem_bytes(int m, int n, size_t limit = MARG_SMEM_MAX) { return (marg_fixed_doubles(m, n) + marg_plan(m, n, limit).body) * sizeof(double); }
CERB_HD size_t marg_ws_doubles(int m, int n, size_t limit = MARG_SMEM_MAX) { return marg_plan(m, n, limit).ws; }
// launch shape: two CTAs of 256 threads per SM when the shared memory allows it (the passes are bound by shared-memory bandwidth and by
// the two barriers of a round: a second CTA fills the gaps), else one CTA of 512 threads
CERB_HD int marg_threads(int m, int n, size_t limit = MARG_SMEM_MAX) {
#if defined(CERB_CUSIM)
    return 64;
#else
    return marg_smem_bytes(m, n, limit) <= MARG_SMEM_TWO ? 256 : 512;
#endif
}
CERB_HD int marg_ctas_per_sm(int m, int n, size_t limit = MARG_SMEM_MAX) { return marg_smem_bytes(m, n, limit) <= MARG_SMEM_TWO ? 2 : 1; }

// pair t (0 .. kp / 2 - 1) of round r (0 .. kp - 2) of a round-robin tournament over kp (even) players, p < q
CERB_D void jacobi_pair(int t, int r, int kp, int &p, int &q) {
    const int md = kp - 1;
    int a, b;
    if (t == 0) { a = md; b = r; }
    else { a = r + t; if (a >= md) a -= md; b = r - t; if (b < 0) b += md; }          // r, t < md
    p = a < b ? a : b; q = a < b ? b : a;
}

// e / d for 0 <= e < 2^16, 0 < d < 2^12 by one multiply-high: magic = ceil(2^32 / d)  (exact while e * d < 2^32; d == 1: magic 0 = "no division")
CERB_HD unsigned marg_magic(int d) { return d <= 1 ? 0u : (unsigned)((0x100000000ull + (unsigned)d - 1) / (unsigned)d); }
CERB_HD int marg_div(int e, unsigned magic) { return magic ? (int)(((unsigned long long)(unsigned)e * magic) >> 32) : e; }

struct alignas(16) MargCS { double c, s; };      // one rotation: a single 16-byte shared-memory load

// rotation angles of round r from M as it stands, pairs t0, t0 + ts, ...; (c, s) -> cs, the pair -> pq (p | q << 16; the passes of the
// round read it instead of redoing the modulo arithmetic), a non-trivial rotation raises *flag.  The smaller root of t^2 + 2 theta t - 1 = 0,
// theta = (aqq - app) / (2 apq), written with one square root, one division and one reciprocal square root on the dependency chain
// (t = sgn(d) e / (|d| + sqrt(d^2 + e^2)), d = aqq - app, e = 2 apq): the angles are the serial part of a round.
CERB_D void jacobi_angles(const double *M, int k, int kp, int r, MargCS *cs, int *pq, int *flag, int t0, int ts) {
    for (int t = t0; t < kp / 2; t += ts) {
        int p, q; jacobi_pair(t, r, kp, p, q);
        MargCS o; o.c = 1.0; o.s = 0.0;
        if (q < k) {
            const int tp = p * (p + 1) / 2, tq = q * (q + 1) / 2;
            const double apq = M[tq + p], app = M[tp + p], aqq = M[tq + q];
            if (apq * apq > 1e-30 * fabs(app * aqq)) {
                const double d = aqq - app, e = 2.0 * apq;
                const double tt = (d >= 0.0 ? e : -e) / (fabs(d) + sqrt(d * d + e * e));
                o.c = rsqrt(tt * tt + 1.0); o.s = tt * o.c;
                if (o.s != 0.0) *flag = 1;
            }
        }
        cs[t] = o; pq[t] = p | (q << 16);
    }
}

// (x, y) <- (c x - s y, s x + c y) on two contiguous vectors of length len, by one warp: the loads of four 32-element chunks are issued before
// the first store (x and y of different pairs never alias, but the compiler cannot know)
CERB_D void marg_rot2(double *x, double *y, int len, double c, double s, int lane) {
    for (int i0 = lane; i0 < len; i0 += 128) {
        double f[4], g[4];
        _Pragma("unroll")
        for (int u = 0; u < 4; u++) { const int i = i0 + 32 * u; if (i < len) { f[u] = x[i]; g[u] = y[i]; } else { f[u] = 0.0; g[u] = 0.0; } }
        _Pragma("unroll")
        for (int u = 0; u < 4; u++) { const int i = i0 + 32 * u; if (i < len) { x[i] = c * f[u] - s * g[u]; y[i] = s * f[u] + c * g[u]; } }
    }
}
// the same in two halves for vectors of <= 96 elements (what the kept block and the rows of T are): load now, rotate + store later, so that the
// loads of several pairs are in flight together; longer vectors finish through marg_rot2
enum { MARG_SCH = 3 };
CERB_D void marg_rot_load(const double *x, const double *y, bool on, int len, int lane, double (&f)[MARG_SCH], double (&g)[MARG_SCH]) {
    _Pragma("unroll")
    for (int v = 0; v < MARG_SCH; v++) { const int i = lane + 32 * v; const bool ok = on && i < len; f[v] = ok ? x[i] : 0.0; g[v] = ok ? y[i] : 0.0; }
}
CERB_D void marg_rot_store(double *x, double *y, bool on, double c, double s, int len, int lane, const double (&f)[MARG_SCH], const double (&g)[MARG_SCH]) {
    if (!on) return;
    _Pragma("unroll")
    for (int v = 0; v < MARG_SCH; v++) { const int i = lane + 32 * v; if (i < len) { x[i] = c * f[v] - s * g[v]; y[i] = s * f[v] + c * g[v]; } }
    if (len > 32 * MARG_SCH) marg_rot2(x + 32 * MARG_SCH, y + 32 * MARG_SCH, len - 32 * MARG_SCH, c, s, lane);
}

#if defined(CERB_PHASE_TIMING) && !defined(CERB_CUSIM)
#define MPH_DECL() long long mph_t = clock64()
#define MPH(id, thr) do { if ((int)threadIdx.x == (thr)) { const long long mph_n = clock64(); atomicAdd(&g_phase_cycles[id], (unsigned long long)(mph_n - mph_t)); mph_t = mph_n; } } while (0)
#else
#define MPH_DECL()
#define MPH(id, thr)
#endif

// Eigen-decomposition of the symmetric k x k matrix M (packed upper triangle): on return the eigenvalues are on the diagonal of M.
// V (optional, k x k, leading dimension ldv, set to the identity here): the eigenvectors as columns.  T (optional, k rows): replaced by
// V^T T (its rows are rotated like the rows of M); columns [0, ncs) of row i at Ts + i * ncs, the other ncg columns at Tg + i * ncg (global
// memory).  Called by all threads of the CTA; returns the number of sweeps.  cs0/cs1, pq0/pq1: the rotation tables of the current and of
// the next round (double-buffered); flag: 3 ints, flag[sweep % 3] collects "some rotation of this sweep was non-trivial".
//
// A round applies its kp / 2 disjoint rotations J to both sides, M <- J^T M J, in ONE pass over 2 x 2 blocks: the task (a, b), a <= b,
// owns the entries {p_a, q_a} x {p_b, q_b}, rotates their columns by pair b and their rows by pair a in registers and writes them back
// (one copy of every entry: M is symmetric by construction, no re-symmetrisation pass, half the arithmetic of a column pass + a row pass
// over the full matrix); no task reads what another one writes (no barrier inside the pass).  The rotated pair itself (a == b) gets an
// exact zero.  Two CTA barriers per round:
//     X: M blocks (all threads)                                   | barrier
//     Y: the last warps: angles of the NEXT round from the new M  || the other warps: columns of V, rows of T with THIS round's table | barrier
// The passes are bound by shared-memory bandwidth (128 B / clock / SM; measured with clock64 phase timers, tools/marg_phase.py) and by the
// latency of dependent shared-memory loads (table -> pair -> element), so every thread works on two tasks (X) / every warp on two pairs (Y)
// at a time, all loads before the first store.  The global tail of T (if any) is loaded before X and rotated / stored in Y: the L2 round
// trip hides behind the block pass.
CERB_D int jacobi_eig(double *M, int k, double *V, int ldv, double *Ts, int ncs, double *Tg, int ncg, MargCS *cs0, MargCS *cs1, int *pq0, int *pq1, int *flag) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const int kp = k + (k & 1), half = kp / 2, rounds = kp - 1;
    int nA = (half + 31) & ~31; if (nA > nt / 2) nA = nt / 2;       // the angle threads: the last nA (whole warps)
    const int nY = nt - nA;
    if (V) for (int j = tid >> 5; j < k; j += nt >> 5) for (int i = tid & 31; i < k; i += 32) V[i + j * ldv] = (i == j) ? 1.0 : 0.0;
    if (tid < 3) flag[tid] = 0;
    __syncthreads();
    jacobi_angles(M, k, kp, 0, cs0, pq0, flag, tid, nt);
    __syncthreads();
    const int nblk = ((half + 1) / 2) * (half + 1), ngt = (Tg && ncg > 0) ? half * ncg : 0;
    const unsigned mg_blk = marg_magic(half + 1), mg_ncg = marg_magic(ncg > 0 ? ncg : 1);
    const int lane = tid & 31, wid = tid >> 5, nwY = nY >> 5;
    const bool yw = tid < nY;                                        // this warp rotates V / T in Y
    int sweeps = 0, cur = 0;
    for (; sweeps < MARG_MAX_SWEEPS; sweeps++) {
        for (int r = 0; r < rounds; r++) {
            const MargCS *cs = cur ? cs1 : cs0; const int *pq = cur ? pq1 : pq0;
            MPH_DECL();
            double ga[2], gb[2];                                     // global tail of T: the first two tasks of this thread, in flight during X
            if (ngt && yw) {
                _Pragma("unroll")
                for (int u = 0; u < 2; u++) {
                    const int e = tid + u * nY;
                    ga[u] = 0.0; gb[u] = 0.0;
                    if (e < ngt) { const int t = marg_div(e, mg_ncg), j = e - t * ncg; if (cs[t].s != 0.0) { ga[u] = Tg[(size_t)(pq[t] & 0xffff) * ncg + j]; gb[u] = Tg[(size_t)(pq[t] >> 16) * ncg + j]; } }
                }
            }
            MPH(46, 0);
            // ---- X: 2 x 2 blocks.  Row a (half - a tasks) is folded with row half - 1 - a (a + 1 tasks): half + 1 tasks per folded row
            for (int e0 = tid; e0 < nblk; e0 += 2 * nt) {
                MargCS ra[2], rb[2];
                int o11[2], o12[2], o21[2], o22[2];
                bool on[2], va[2], vb[2], dg[2];
                _Pragma("unroll")
                for (int u = 0; u < 2; u++) {
                    const int e1 = e0 + u * nt;
                    bool ok = e1 < nblk;
                    const int e = ok ? e1 : 0;
                    const int af = marg_div(e, mg_blk), c = e - af * (half + 1);
                    int a, b;
                    if (c < half - af) { a = af; b = af + c; }
                    else { a = half - 1 - af; b = a + (c - (half - af)); if (a == af) ok = false; }
                    ra[u] = cs[a]; rb[u] = cs[b];
                    const int wa = pq[a], wb = pq[b];
                    const int pa = wa & 0xffff, qa = wa >> 16, pb = wb & 0xffff, qb = wb >> 16;       // pa < qa, pb < qb
                    va[u] = qa < k; vb[u] = qb < k;                                // the padding player of an odd k never rotates (s == 0)
                    on[u] = ok && !(ra[u].s == 0.0 && rb[u].s == 0.0); dg[u] = a == b;
                    // packed offsets of (pa, pb), (pa, qb), (qa, pb), (qa, qb): the larger index selects the column
                    const int tpa = pa * (pa + 1) / 2, tqa = qa * (qa + 1) / 2, tpb = pb * (pb + 1) / 2, tqb = qb * (qb + 1) / 2;
                    o11[u] = pa <= pb ? tpb + pa : tpa + pb; o12[u] = pa <= qb ? tqb + pa : tpa + qb;
                    o21[u] = qa <= pb ? tpb + qa : tqa + pb; o22[u] = qa <= qb ? tqb + qa : tqa + qb;
                }
                double x11[2], x12[2], x21[2], x22[2];
                _Pragma("unroll")
                for (int u = 0; u < 2; u++) {
                    x11[u] = on[u] ? M[o11[u]] : 0.0; x12[u] = (on[u] && vb[u]) ? M[o12[u]] : 0.0;
                    x21[u] = (on[u] && va[u]) ? M[o21[u]] : 0.0; x22[u] = (on[u] && va[u] && vb[u]) ? M[o22[u]] : 0.0;
                }
                _Pragma("unroll")
                for (int u = 0; u < 2; u++) {
                    if (!on[u]) continue;
                    const double ca = ra[u].c, sa = ra[u].s, cb = rb[u].c, sb = rb[u].s;
                    const double y11 = cb * x11[u] - sb * x12[u], y12 = sb * x11[u] + cb * x12[u], y21 = cb * x21[u] - sb * x22[u], y22 = sb * x21[u] + cb * x22[u];
                    double z11 = ca * y11 - sa * y21, z21 = sa * y11 + ca * y21, z12 = ca * y12 - sa * y22, z22 = sa * y12 + ca * y22;
                    if (dg[u]) { z12 = 0.0; z21 = 0.0; }                          // the annihilated entry (sa != 0 here); o21 == o12
                    M[o11[u]] = z11; if (vb[u]) M[o12[u]] = z12; if (va[u] && !dg[u]) M[o21[u]] = z21; if (va[u] && vb[u]) M[o22[u]] = z22;
                }
            }
            MPH(40, 0); MPH(47, nY);
            __syncthreads();
            MPH(41, 0); MPH(47, nY);
            // ---- Y
            if (!yw) {
                const int sw = (r + 1 < rounds) ? sweeps : sweeps + 1;
                jacobi_angles(M, k, kp, (r + 1 < rounds) ? r + 1 : 0, cur ? cs0 : cs1, cur ? pq0 : pq1, flag + sw % 3, tid - nY, nA);
            } else {
                if (r == 0 && tid == 0) flag[(sweeps + 2) % 3] = 0;                // last read at the end of sweep - 1, next written at the end of sweep + 1
                if (V || (Ts && ncs > 0)) for (int t0 = wid; t0 < half; t0 += 2 * nwY) {      // two pairs per warp at a time: columns of V, rows of T
                    const int t1 = t0 + nwY;
                    const bool in1 = t1 < half;
                    const MargCS r0 = cs[t0], r1 = cs[in1 ? t1 : t0];
                    const int w0 = pq[t0], w1 = pq[in1 ? t1 : t0];
                    const bool on0 = r0.s != 0.0, on1 = in1 && r1.s != 0.0;
                    const int p0 = w0 & 0xffff, q0 = on0 ? w0 >> 16 : p0, p1 = w1 & 0xffff, q1 = on1 ? w1 >> 16 : p1;
                    double f0[MARG_SCH], g0[MARG_SCH], f1[MARG_SCH], g1[MARG_SCH];
                    if (V) {
                        marg_rot_load(V + p0 * ldv, V + q0 * ldv, on0, k, lane, f0, g0);
                        marg_rot_load(V + p1 * ldv, V + q1 * ldv, on1, k, lane, f1, g1);
                        marg_rot_store(V + p0 * ldv, V + q0 * ldv, on0, r0.c, r0.s, k, lane, f0, g0);
                        marg_rot_store(V + p1 * ldv, V + q1 * ldv, on1, r1.c, r1.s, k, lane, f1, g1);
                    }
                    if (Ts && ncs > 0) {
                        marg_rot_load(Ts + p0 * ncs, Ts + q0 * ncs, on0, ncs, lane, f0, g0);
                        marg_rot_load(Ts + p1 * ncs, Ts + q1 * ncs, on1, ncs, lane, f1, g1);
                        marg_rot_store(Ts + p0 * ncs, Ts + q0 * ncs, on0, r0.c, r0.s, ncs, lane, f0, g0);
                        marg_rot_store(Ts + p1 * ncs, Ts + q1 * ncs, on1, r1.c, r1.s, ncs, lane, f1, g1);
                    }
                }
                if (ngt) {
                    _Pragma("unroll")
                    for (int u = 0; u < 2; u++) {
                        const int e = tid + u * nY;
                        if (e < ngt) {
                            const int t = marg_div(e, mg_ncg), j = e - t * ncg;
                            const MargCS rr = cs[t];
                            if (rr.s != 0.0) { Tg[(size_t)(pq[t] & 0xffff) * ncg + j] = rr.c * ga[u] - rr.s * gb[u]; Tg[(size_t)(pq[t] >> 16) * ncg + j] = rr.s * ga[u] + rr.c * gb[u]; }
                        }
                    }
                    for (int e0 = tid + 2 * nY; e0 < ngt; e0 += 4 * nY) {            // the rest (T entirely in global memory: m too large for shared memory), four in flight
                        double f[4], g[4];
                        _Pragma("unroll")
                        for (int u = 0; u < 4; u++) {
                            const int e = e0 + u * nY;
                            f[u] = 0.0; g[u] = 0.0;
                            if (e < ngt) { const int t = marg_div(e, mg_ncg), j = e - t * ncg; if (cs[t].s != 0.0) { f[u] = Tg[(size_t)(pq[t] & 0xffff) * ncg + j]; g[u] = Tg[(size_t)(pq[t] >> 16) * ncg + j]; } }
                        }
                        _Pragma("unroll")
                        for (int u = 0; u < 4; u++) {
                            const int e = e0 + u * nY;
                            if (e < ngt) {
                                const int t = marg_div(e, mg_ncg), j = e - t * ncg;
                                const MargCS rr = cs[t];
                                if (rr.s != 0.0) { Tg[(size_t)(pq[t] & 0xffff) * ncg + j] = rr.c * f[u] - rr.s * g[u]; Tg[(size_t)(pq[t] >> 16) * ncg + j] = rr.s * f[u] + rr.c * g[u]; }
                            }
                        }
                    }
                }
            }
            MPH(42, 0); MPH(44, nY);
            __syncthreads();
            MPH(43, 0); MPH(45, nY);
            cur ^= 1;
        }
        if (!flag[sweeps % 3]) break;
    }
    return sweeps;
}

// A [n_windows][(m + n)^2] row-major (dropped block first), b [n_windows][m + n]; lin_J [n_windows][n * n] column-major,
// lin_r [n_windows][n]; ws [gridDim.x][marg_ws_doubles(m, n)]; sweeps [n_windows][2] (diagnostics, may be null)
// dims (optional): per-window sizes [n_windows][4] = m, n, status (only status == 1 windows are processed), -; then mmax / nmax bound them
// and A / b / lin_J / lin_r are strided by A_stride / b_stride / J_stride / r_stride doubles per window (0: tight, from m and n)
CERB_GLOBAL void __launch_bounds__(MARG_THREADS, 1) marg_schur_kernel(int n_windows, int mmax, int nmax, const int *dims, const double *A_all, long A_stride, const double *b_all, long b_stride, double eps,
                                   double *ws_all, double *lin_J, long J_stride, double *lin_r, long r_stride, int *sweeps, int smem_limit) {
    CERB_DYN_SMEM(double, sm);
    const int tid = threadIdx.x, nt = blockDim.x;
    const int kmax = mmax > nmax ? mmax : nmax;
    const int tbl = (kmax + 3) & ~1;                                                      // doubles per (c, s) table: 16-byte aligned entries
    MargCS *cs0 = reinterpret_cast<MargCS *>(sm), *cs1 = reinterpret_cast<MargCS *>(sm + tbl);
    double *inv = sm;                                                                      // 1 / lambda: over the dead tables
    int *flag = reinterpret_cast<int *>(sm + 2 * tbl), *pq0 = flag + 8, *pq1 = pq0 + 2 * ((kmax + 2) / 4 + 1);
    double *body = sm + marg_fixed_doubles(mmax, nmax);
    const MargPlan plan = marg_plan(mmax, nmax, (size_t)smem_limit);
    double *wsp = ws_all + (size_t)blockIdx.x * plan.ws;
    double *Tg = wsp, *M1g = Tg + (size_t)mmax * (nmax + 1 - plan.ncs) + 1, *br = M1g + (plan.m1_smem ? 0 : marg_tri(mmax));
    for (int w = blockIdx.x; w < n_windows; w += gridDim.x) {
        const int m = dims ? dims[4 * w] : mmax, n = dims ? dims[4 * w + 1] : nmax;
        if (dims && (dims[4 * w + 2] != 1 || m > mmax || n > nmax)) continue;
        const int pos = m + n, nc = n + 1, ld2 = marg_ld(n);
        const int ncs = plan.ncs < nc ? plan.ncs : nc, ncg = nc - ncs;                       // columns of T in shared / in global memory
        const double *A = A_all + (size_t)w * (A_stride ? A_stride : (long)pos * pos), *b = b_all + (size_t)w * (b_stride ? b_stride : (long)pos);
        // ---- phase 1: Amm = 0.5 (Amm + Amm^T) = V1 diag(lambda) V1^T;  T = V1^T [Amr | bm] --------------------------------------
        double *M1 = plan.m1_smem ? body : M1g;
        double *Ts = body + (marg_tri(m) > marg_tri(n) ? marg_tri(m) : marg_tri(n));
        for (int j = tid / 32; j < m; j += nt / 32) for (int i = tid & 31; i <= j; i += 32) M1[marg_tri(j) + i] = 0.5 * (A[(size_t)i * pos + j] + A[(size_t)j * pos + i]);
        for (int e = tid; e < m * nc; e += nt) {
            const int c = e % nc, i = e / nc;
            const double v = c < n ? A[(size_t)i * pos + m + c] : b[i];
            if (c < ncs) Ts[i * ncs + c] = v; else Tg[(size_t)i * ncg + (c - ncs)] = v;
        }
        __syncthreads();
        // two instantiations: with the matrix in shared memory the compiler sees the address space (LDS / STS with 32-bit addresses instead of
        // generic 64-bit loads)
        int sw1;
        if (plan.m1_smem) sw1 = jacobi_eig(body, m, nullptr, 0, Ts, ncs, Tg, ncg, cs0, cs1, pq0, pq1, flag);
        else sw1 = jacobi_eig(M1g, m, nullptr, 0, nullptr, 0, Tg, ncg, cs0, cs1, pq0, pq1, flag);
        for (int i = tid; i < m; i += nt) { const double lam = M1[marg_tri(i) + i]; inv[i] = lam > eps ? 1.0 / lam : 0.0; }
        __syncthreads();
        // ---- [Ar | br] = [Arr | brr] - T^T diag(inv) T (the triangle c <= r) ------------------------------------------------------------------
        double *M2 = body;
        for (int e = tid; e < n * nc; e += nt) {
            const int r = e % n, c = e / n;
            if (c < n && c > r) continue;
            const double *tr = r < ncs ? Ts + r : Tg + (r - ncs), *tc = c < ncs ? Ts + c : Tg + (c - ncs);
            const int sr = r < ncs ? ncs : ncg, sc = c < ncs ? ncs : ncg;
            double acc = 0.0;
            for (int i = 0; i < m; i++) acc += tr[(size_t)i * sr] * inv[i] * tc[(size_t)i * sc];
            if (c < n) M2[marg_tri(r) + c] = A[(size_t)(m + r) * pos + m + c] - acc;        // (c, r), c <= r
            else br[r] = b[m + r] - acc;
        }
        __syncthreads();
        // ---- phase 2: A = V2 diag(lambda) V2^T;  linearized_jacobians = sqrt(S) V2^T, linearized_residuals = sqrt(S_inv) V2^T b ----------
        double *V2 = M2 + marg_tri(n);                                                     // over the dead T
        const int sw2 = jacobi_eig(M2, n, V2, ld2, nullptr, 0, nullptr, 0, cs0, cs1, pq0, pq1, flag);
        double *Jo = lin_J + (size_t)w * (J_stride ? J_stride : (long)n * n), *ro = lin_r + (size_t)w * (r_stride ? r_stride : (long)n);
        for (int e = tid; e < n * n; e += nt) {
            const int kk = e % n, j = e / n;
            const double lam = M2[marg_tri(kk) + kk];
            Jo[e] = lam > eps ? sqrt(lam) * V2[j + (size_t)kk * ld2] : 0.0;
        }
        for (int kk = tid; kk < n; kk += nt) {
            const double lam = M2[marg_tri(kk) + kk];
            double acc = 0.0;
            if (lam > eps) { const double *v = V2 + (size_t)kk * ld2; for (int i = 0; i < n; i++) acc += v[i] * br[i]; acc *= sqrt(1.0 / lam); }
            ro[kk] = acc;
        }
        if (sweeps && tid == 0) { sweeps[2 * w] = sw1; sweeps[2 * w + 1] = sw2; }
        __syncthreads();
    }
}

}  // namespace cerb

// preint_kernel.cuh -- leg-contact preintegration on device: the IMULegIntegrationBase::push_back loop
// (src/factor/imu_leg_integration_base.cpp:49-59 -> propagate :88-136 -> midPointIntegration :138-470)
// for a batch of independent inter-frame intervals, one CTA per interval.
//
// Per IMU/leg sample: midpoint IMU integration, per-leg body-velocity integration through the A1
// kinematics, then jacobian <- F jacobian, covariance <- F cov F^T + V diag(N) V^T with F 31x31,
// V 31x46 (ILStateOrder / ILNoiseStateOrder, parameters.h:135-172).  State lives in shared memory for
// the whole interval; only the 35-double samples stream from HBM.
#pragma once
#include "factors.cuh"

namespace cerb {

struct PreintParams {   // mirror of CerbPreintConfig plus the record kind; a launch reads one entry of a table of them per job
    double acc_n, acc_n_z, gyr_n, acc_w, gyr_w, phi_n, dphi_n, rho_c_n, rho_nc_n;
    double v_n_min_xy, v_n_min_z, v_n_min, v_n_max, v_n_force_thres_ratio, v_n_term1_steep, v_n_term2_var_rescale, v_n_term3_distance_rescale;
    int contact_sensor_type;
    int imu_only;             // 1: plain IntegrationBase (integration_base.h): no legs, acc_n on all three axes
    double rho_fix[16], p_br[3], R_br[9];
};

// device job table: per job [0..2] acc_0 [3..5] gyr_0 [6..17] phi_0 [18..29] dphi_0 [30..33] c_0
//                   [34..36] lin_ba [37..39] lin_bg [40..43] lin_rho ; n_samples, sample offset, entry of the parameter table in ints
enum { PJ_STRIDE = 44, SAMPLE_STRIDE = 35 };   // sample: dt, acc3, gyr3, phi12, dphi12, c4
enum { NO_Ai = 0, NO_Gi = 3, NO_Ai1 = 6, NO_Gi1 = 9, NO_BA = 12, NO_BG = 15, NO_PHIi = 18, NO_PHIi1 = 21, NO_DPHIi = 24, NO_DPHIi1 = 27, NO_V1 = 30, NO_NRHO1 = 42 };

struct LegStep {   // per-leg quantities of one midpoint step
    d3 fi, fi1, vi, vi1, gi, gi1;
    m33 Ji, Ji1, hi, hi1;
};

CERB_D void set_block(double *M, int ld, int r0, int c0, const m33 &B) {
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) M[(r0 + a) * ld + c0 + b] = B.m[3 * a + b];
}
CERB_D m33 colmajor33(const double *a) { m33 r; for (int c = 0; c < 3; c++) for (int rr = 0; rr < 3; rr++) r.m[3 * rr + c] = a[c * 3 + rr]; return r; }

// out (compact device preint layout, PRE_STRIDE doubles): nominal + jacobian sub-blocks + covariance;
// out_full (optional, 2*961 doubles): full jacobian and covariance, row-major (for the host ABI struct).
// job_ints [n_jobs][3] = n_samples, sample offset, p: job j integrates under params[p], so one launch serves jobs of several configurations
// and of both record kinds.  grid = n_jobs, block = 128.
CERB_GLOBAL void preintegrate_kernel(const PreintParams *params, int n_jobs, const double *jobs, const int *job_ints, const double *samples,
                                     double *out, double *out_full) {
    const int LD = 33, LDV = 47;
    __shared__ double jac[31 * 33], cov[31 * 33], F[31 * 33], T[31 * 33], V[31 * 47], Nn[48];
    __shared__ double nom[64];          // [0..2] dp [3..6] dq(xyzw) [7..9] dv [10..21] deps [22] sum_dt [23..25] ba [26..28] bg [29..32] rho
    __shared__ double cur[40], nxt[40]; // sample 0 / 1: acc3 gyr3 phi12 dphi12 c4  (offsets 0,3,6,18,30)
    __shared__ double stp[48];          // [0..3] result dq, [4..6] result dp, [7..9] result dv, [10..18] R0, [19..27] R1, [28] dt
    __shared__ LegStep legs[4];
    __shared__ double filt[4 * 12];     // type-2 contact filter state per leg: min, max, thr, var, idx, window[5]
    __shared__ int flag[4];
    const int job = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const PreintParams &P = params[job_ints[3 * job + 2]];
    const double *jb = jobs + (size_t)job * PJ_STRIDE;
    const int n_samples = job_ints[3 * job], s_off = job_ints[3 * job + 1];

    for (int i = tid; i < 31 * 33; i += nt) { const int r = i / 33, c = i % 33; jac[i] = (r == c) ? 1.0 : 0.0; cov[i] = 0.0; }
    if (tid < 34) cur[tid] = jb[tid];
    if (tid == 0) {
        for (int k = 0; k < 23; k++) nom[k] = 0.0;
        nom[6] = 1.0;   // identity quaternion (x,y,z,w)
        for (int k = 0; k < 3; k++) { nom[23 + k] = jb[34 + k]; nom[26 + k] = jb[37 + k]; }
        for (int k = 0; k < 4; k++) nom[29 + k] = jb[40 + k];
        for (int k = 0; k < 48; k++) filt[k] = 0.0;
    }
    __syncthreads();

    for (int s = 0; s < n_samples; s++) {
        const double *smp = samples + (size_t)(s_off + s) * SAMPLE_STRIDE;
        if (tid < 34) nxt[tid] = smp[1 + tid];
        __syncthreads();
        // ---- 1a: IMU midpoint (imu_leg_integration_base.cpp:152-160) --------------------------------
        if (tid == 0) {
            const double dt = smp[0];
            const quat dq = ldq(nom + 3);
            const d3 ba = ld3(nom + 23), bg = ld3(nom + 26);
            const d3 un_acc_0 = qrot(dq, ld3(cur) - ba);
            const d3 un_gyr = 0.5 * (ld3(cur + 3) + ld3(nxt + 3)) - bg;
            const quat rq = qmul(dq, mkq(un_gyr.x * dt / 2, un_gyr.y * dt / 2, un_gyr.z * dt / 2, 1.0));
            const d3 un_acc_1 = qrot(rq, ld3(nxt) - ba);
            const d3 un_acc = 0.5 * (un_acc_0 + un_acc_1);
            const d3 dp = ld3(nom), dv = ld3(nom + 7);
            stp[0] = rq.x; stp[1] = rq.y; stp[2] = rq.z; stp[3] = rq.w;
            st3(stp + 4, dp + dt * dv + (0.5 * dt * dt) * un_acc);
            st3(stp + 7, dv + dt * un_acc);
            const m33 R0 = qtoR(dq), R1 = qtoR(rq);
            for (int k = 0; k < 9; k++) { stp[10 + k] = R0.m[k]; stp[19 + k] = R1.m[k]; }
            stp[28] = dt;
        }
        // contact flag (:182-229); one thread per leg
        if (tid < 4) {
            const int j = tid;
            if (P.contact_sensor_type == 0 || P.contact_sensor_type == 1) {
                flag[j] = (nxt[30 + j] >= 0.5) ? 1 : 0;
            } else {
                double *fs = filt + 12 * j;   // min, max, thr, var, idx, window[5]
                const double force_mag = 0.5 * (cur[30 + j] + nxt[30 + j]);
                if (force_mag < fs[0]) fs[0] = 0.9 * fs[0] + 0.1 * force_mag;
                if (force_mag > fs[1]) fs[1] = 0.9 * fs[1] + 0.1 * force_mag;
                fs[0] *= 0.9991; fs[1] *= 0.997;
                fs[2] = fs[0] + P.v_n_force_thres_ratio * (fs[1] - fs[0]);
                flag[j] = (int)(1.0 / (1 + exp(-P.v_n_term1_steep * (force_mag - fs[2]))));   // Vector4i truncation (quirk a8')
                int idx = ((int)fs[4] + 1) % 5; fs[4] = (double)idx; fs[5 + idx] = force_mag;
                double mean = 0; for (int k = 0; k < 5; k++) mean += fs[5 + k]; mean /= 5;
                double var = 0; for (int k = 0; k < 5; k++) var += (fs[5 + k] - mean) * (fs[5 + k] - mean);
                fs[3] = var / 4;
            }
        }
        __syncthreads();
        // ---- 1b: per-leg kinematics and velocity (:232-286); one thread per leg ---------------------
        if (tid < 4 && P.imu_only) {
            LegStep &L = legs[tid];
            L.fi = L.fi1 = L.vi = L.vi1 = L.gi = L.gi1 = mk3(0, 0, 0);
            for (int k = 0; k < 9; k++) { L.Ji.m[k] = 0; L.Ji1.m[k] = 0; L.hi.m[k] = 0; L.hi1.m[k] = 0; }
        }
        if (tid < 4 && !P.imu_only) {
            const int j = tid;
            const double lc = nom[29 + j];
            const double *fix = P.rho_fix + 4 * j;
            const m33 R_br = ldm33(P.R_br), R0 = ldm33(stp + 10), R1 = ldm33(stp + 19);
            const d3 p_br = ld3(P.p_br), bg = ld3(nom + 26);
            const m33 W0 = skew33(ld3(cur + 3) - bg), W1 = skew33(ld3(nxt + 3) - bg);
            LegStep &L = legs[j];
            double t3[3], t9[9], t27[27];
            const A1Trig tr0 = a1_trig(cur + 6 + 3 * j), tr1 = a1_trig(nxt + 6 + 3 * j);
            const d3 dphi0 = ld3(cur + 18 + 3 * j), dphi1 = ld3(nxt + 18 + 3 * j);
            a1_fk(tr0, lc, fix, t3); L.fi = ld3(t3);
            a1_fk(tr1, lc, fix, t3); L.fi1 = ld3(t3);
            a1_jac(tr0, lc, fix, t9); L.Ji = colmajor33(t9);
            a1_jac(tr1, lc, fix, t9); L.Ji1 = colmajor33(t9);
            L.vi = -mv33(R_br, mv33(L.Ji, dphi0)) - mv33(W0, p_br + mv33(R_br, L.fi));
            L.vi1 = -mv33(R_br, mv33(L.Ji1, dphi1)) - mv33(W1, p_br + mv33(R_br, L.fi1));
            // g = -R (R_br (dphi^T (x) I) dJ/drho + [w]x R_br df/drho)
            a1_dJ_drho(tr0, t9); a1_dfk_drho(tr0, t3);
            d3 kd = mk3(dphi0.x * t9[0] + dphi0.y * t9[3] + dphi0.z * t9[6], dphi0.x * t9[1] + dphi0.y * t9[4] + dphi0.z * t9[7], dphi0.x * t9[2] + dphi0.y * t9[5] + dphi0.z * t9[8]);
            L.gi = -mv33(R0, mv33(R_br, kd) + mv33(W0, mv33(R_br, ld3(t3))));
            a1_dJ_drho(tr1, t9); a1_dfk_drho(tr1, t3);
            kd = mk3(dphi1.x * t9[0] + dphi1.y * t9[3] + dphi1.z * t9[6], dphi1.x * t9[1] + dphi1.y * t9[4] + dphi1.z * t9[7], dphi1.x * t9[2] + dphi1.y * t9[5] + dphi1.z * t9[8]);
            L.gi1 = -mv33(R1, mv33(R_br, kd) + mv33(W1, mv33(R_br, ld3(t3))));
            // h = R (R_br (dphi^T (x) I) dJ/dphi + [w]x R_br J)
            m33 K;
            a1_dJ_dq(tr0, lc, fix, t27);
            for (int m = 0; m < 3; m++) for (int r = 0; r < 3; r++) K.m[3 * r + m] = dphi0.x * t27[m * 9 + r] + dphi0.y * t27[m * 9 + 3 + r] + dphi0.z * t27[m * 9 + 6 + r];
            L.hi = mul33(R0, add33(mul33(R_br, K), mul33(W0, mul33(R_br, L.Ji))));
            a1_dJ_dq(tr1, lc, fix, t27);
            for (int m = 0; m < 3; m++) for (int r = 0; r < 3; r++) K.m[3 * r + m] = dphi1.x * t27[m * 9 + r] + dphi1.y * t27[m * 9 + 3 + r] + dphi1.z * t27[m * 9 + 6 + r];
            L.hi1 = mul33(R1, add33(mul33(R_br, K), mul33(W1, mul33(R_br, L.Ji1))));
        }
        for (int i = tid; i < 31 * 33; i += nt) F[i] = 0.0;
        for (int i = tid; i < 31 * 47; i += nt) V[i] = 0.0;
        __syncthreads();
        // ---- 2: noise diag, F and V (:290-465) -----------------------------------------------------------
        const double dt = stp[28];
        if (tid == 0) {
            const m33 R0 = ldm33(stp + 10), R1 = ldm33(stp + 19), I3 = ident33();
            const d3 ba = ld3(nom + 23), bg = ld3(nom + 26);
            const m33 R_w = skew33(0.5 * (ld3(cur + 3) + ld3(nxt + 3)) - bg);
            const m33 R_a0 = skew33(ld3(cur) - ba), R_a1 = skew33(ld3(nxt) - ba);
            const m33 k7 = sub33(I3, scale33(R_w, dt));
            const m33 k1 = add33(scale33(mul33(R0, R_a0), -0.5 * dt), scale33(mul33(mul33(R1, R_a1), k7), -0.5 * dt));
            const m33 R1a1 = mul33(R1, R_a1), R01 = add33(R0, R1);
            set_block(F, LD, ILO_P, ILO_P, I3);
            set_block(F, LD, ILO_P, ILO_R, scale33(k1, 0.5 * dt));
            set_block(F, LD, ILO_P, ILO_V, scale33(I3, dt));
            set_block(F, LD, ILO_P, ILO_BA, scale33(R01, -0.25 * dt * dt));
            set_block(F, LD, ILO_P, ILO_BG, scale33(R1a1, 0.25 * dt * dt * dt));
            set_block(F, LD, ILO_R, ILO_R, k7);
            set_block(F, LD, ILO_R, ILO_BG, scale33(I3, -dt));
            set_block(F, LD, ILO_V, ILO_R, k1);
            set_block(F, LD, ILO_V, ILO_V, I3);
            set_block(F, LD, ILO_V, ILO_BA, scale33(R01, -0.5 * dt));
            set_block(F, LD, ILO_V, ILO_BG, scale33(R1a1, 0.5 * dt * dt));
            set_block(F, LD, ILO_BA, ILO_BA, I3);
            set_block(F, LD, ILO_BG, ILO_BG, I3);
            for (int j = 0; j < 4; j++) F[(ILO_RHO1 + j) * LD + ILO_RHO1 + j] = 1.0;
            set_block(V, LDV, ILO_P, NO_Ai, scale33(R0, 0.25 * dt * dt));
            const m33 vpg = scale33(R1a1, -0.25 * dt * dt * 0.5 * dt);
            set_block(V, LDV, ILO_P, NO_Gi, vpg);
            set_block(V, LDV, ILO_P, NO_Ai1, scale33(R1, 0.25 * dt * dt));
            set_block(V, LDV, ILO_P, NO_Gi1, vpg);
            set_block(V, LDV, ILO_R, NO_Gi, scale33(I3, 0.5 * dt));
            set_block(V, LDV, ILO_R, NO_Gi1, scale33(I3, 0.5 * dt));
            set_block(V, LDV, ILO_V, NO_Ai, scale33(R0, 0.5 * dt));
            const m33 vvg = scale33(R1a1, -0.5 * dt * 0.5 * dt);
            set_block(V, LDV, ILO_V, NO_Gi, vvg);
            set_block(V, LDV, ILO_V, NO_Ai1, scale33(R1, 0.5 * dt));
            set_block(V, LDV, ILO_V, NO_Gi1, vvg);
            set_block(V, LDV, ILO_BA, NO_BA, scale33(I3, -dt));
            set_block(V, LDV, ILO_BG, NO_BG, scale33(I3, -dt));
            for (int j = 0; j < 4; j++) V[(ILO_RHO1 + j) * LDV + NO_NRHO1 + j] = -dt;
            // noise (:360-374)
            const double an = P.acc_n * P.acc_n, anz = P.imu_only ? P.acc_n * P.acc_n : P.acc_n_z * P.acc_n_z, gn = P.gyr_n * P.gyr_n;
            const double aw = P.acc_w * P.acc_w, gw = P.gyr_w * P.gyr_w, pn = P.phi_n * P.phi_n, dn = P.dphi_n * P.dphi_n;
            Nn[0] = an; Nn[1] = an; Nn[2] = anz; Nn[6] = an; Nn[7] = an; Nn[8] = anz;
            for (int k = 0; k < 3; k++) { Nn[3 + k] = gn; Nn[9 + k] = gn; Nn[12 + k] = aw; Nn[15 + k] = gw; }
            for (int k = 0; k < 6; k++) { Nn[18 + k] = pn; Nn[24 + k] = dn; }
            const int fsum = flag[0] + flag[1] + flag[2] + flag[3];
            for (int j = 0; j < 4; j++) {
                double u[3];
                if (P.contact_sensor_type == 0 || P.contact_sensor_type == 1) {
                    const double n_xy = P.v_n_max * (1 - flag[j]) + flag[j] * P.v_n_min_xy;
                    const double n_z = P.v_n_max * (1 - flag[j]) + flag[j] * P.v_n_min_z;
                    u[0] = n_xy; u[1] = n_xy; u[2] = n_z;
                } else {
                    const double n1 = P.v_n_max * (1 - flag[j]) + P.v_n_min, n2 = P.v_n_term2_var_rescale * filt[12 * j + 3];
                    const d3 lo = 0.5 * (mv33(R0, legs[j].vi) + mv33(R1, legs[j].vi1));
                    const d3 tmp = lo - ld3(nom + 7);
                    u[0] = n1 + n2 + P.v_n_term3_distance_rescale * tmp.x * tmp.x;
                    u[1] = n1 + n2 + P.v_n_term3_distance_rescale * tmp.y * tmp.y;
                    u[2] = n1 + n2 + P.v_n_term3_distance_rescale * tmp.z * tmp.z;
                }
                double ru = P.rho_c_n * flag[j] + P.rho_nc_n;
                if (fsum < 1) { ru = P.rho_nc_n; u[0] = u[1] = u[2] = 10e10; }   // all feet off the ground (:354-358)
                Nn[30 + 3 * j] = u[0]; Nn[31 + 3 * j] = u[1]; Nn[32 + 3 * j] = u[2];
                Nn[42 + j] = ru;
            }
        }
        if (tid >= 32 && tid < 36) {   // per-leg rows of F and V (:405-413, :452-460), one thread per leg, another warp
            const int j = tid - 32, e = ILO_EPS1 + 3 * j;
            if (P.imu_only) { set_block(F, LD, e, e, ident33()); }
            else {
            const LegStep &L = legs[j];
            const m33 R0 = ldm33(stp + 10), R1 = ldm33(stp + 19), I3 = ident33(), R_br = ldm33(P.R_br);
            const d3 p_br = ld3(P.p_br), bg = ld3(nom + 26);
            const m33 k7 = sub33(I3, scale33(skew33(0.5 * (ld3(cur + 3) + ld3(nxt + 3)) - bg), dt));
            const m33 R1v1 = mul33(R1, skew33(L.vi1));
            const m33 R0p0 = mul33(R0, skew33(p_br + mv33(R_br, L.fi))), R1p1 = mul33(R1, skew33(p_br + mv33(R_br, L.fi1)));
            set_block(F, LD, e, ILO_R, add33(scale33(mul33(R0, skew33(L.vi)), -0.5 * dt), scale33(mul33(R1v1, k7), -0.5 * dt)));
            set_block(F, LD, e, e, I3);
            set_block(F, LD, e, ILO_BG, sub33(scale33(R1v1, 0.5 * dt * dt), scale33(add33(R0p0, R1p1), 0.5 * dt)));
            const d3 gc = (0.5 * dt) * (L.gi + L.gi1);
            F[(e + 0) * LD + ILO_RHO1 + j] = gc.x; F[(e + 1) * LD + ILO_RHO1 + j] = gc.y; F[(e + 2) * LD + ILO_RHO1 + j] = gc.z;
            set_block(V, LDV, e, NO_Gi, add33(scale33(R1v1, -0.25 * dt * dt), scale33(R0p0, 0.5 * dt)));
            set_block(V, LDV, e, NO_Gi1, add33(scale33(R1v1, -0.25 * dt * dt), scale33(R1p1, 0.5 * dt)));
            set_block(V, LDV, e, NO_PHIi, scale33(L.hi, -0.5 * dt));
            set_block(V, LDV, e, NO_PHIi1, scale33(L.hi1, -0.5 * dt));
            set_block(V, LDV, e, NO_DPHIi, scale33(mul33(mul33(R0, R_br), L.Ji), -0.5 * dt));
            set_block(V, LDV, e, NO_DPHIi1, scale33(mul33(mul33(R1, R_br), L.Ji1), -0.5 * dt));
            set_block(V, LDV, e, NO_V1 + 3 * j, scale33(I3, -dt));
            }
        }
        __syncthreads();
        // ---- 3: jacobian = F jacobian ; covariance = F cov F^T + V N V^T (:467-468) ----------------------
        for (int i = tid; i < 31 * 31; i += nt) {
            const int r = i / 31, c = i % 31;
            double s = 0.0;
            for (int k = 0; k < 31; k++) s += F[r * LD + k] * jac[k * LD + c];
            T[r * LD + c] = s;
        }
        __syncthreads();
        for (int i = tid; i < 31 * 31; i += nt) {
            const int r = i / 31, c = i % 31;
            jac[r * LD + c] = T[r * LD + c];
            double s = 0.0;
            for (int k = 0; k < 31; k++) s += F[r * LD + k] * cov[k * LD + c];
            T[r * LD + c] = s;       // F * cov   (T is read by nobody else until the barrier below)
        }
        __syncthreads();
        for (int i = tid; i < 31 * 31; i += nt) {
            const int r = i / 31, c = i % 31;
            double s = 0.0;
            for (int k = 0; k < 31; k++) s += T[r * LD + k] * F[c * LD + k];
            for (int k = 0; k < 46; k++) s += V[r * LDV + k] * Nn[k] * V[c * LDV + k];
            cov[r * LD + c] = s;
        }
        // ---- 4: commit the nominal state (:125-135) ------------------------------------------------------
        if (tid == 0) {
            const quat rq = qnormalized(ldq(stp));
            const m33 R0 = ldm33(stp + 10), R1 = ldm33(stp + 19);
            for (int j = 0; j < 4; j++) {
                const d3 e = ld3(nom + 10 + 3 * j) + (0.5 * dt) * (mv33(R0, legs[j].vi) + mv33(R1, legs[j].vi1));   // :245 (delta_q * v == R v)
                st3(nom + 10 + 3 * j, e);
            }
            st3(nom, ld3(stp + 4)); st3(nom + 7, ld3(stp + 7));
            nom[3] = rq.x; nom[4] = rq.y; nom[5] = rq.z; nom[6] = rq.w;
            nom[22] += dt;
        }
        __syncthreads();
        if (tid < 34) cur[tid] = nxt[tid];
        __syncthreads();
    }
    // ---- write out -----------------------------------------------------------------------------------------
    double *o = out + (size_t)job * PRE_STRIDE;
    if (tid == 0) {
        o[PRE_SUM_DT] = nom[22];
        for (int k = 0; k < 3; k++) { o[PRE_DP + k] = nom[k]; o[PRE_DV + k] = nom[7 + k]; o[PRE_BA + k] = nom[23 + k]; o[PRE_BG + k] = nom[26 + k]; }
        for (int k = 0; k < 4; k++) { o[PRE_DQ + k] = nom[3 + k]; o[PRE_RHO + k] = nom[29 + k]; }
        for (int k = 0; k < 12; k++) o[PRE_DEPS + k] = nom[10 + k];
        for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) {
            o[PRE_DP_DBA + 3 * a + b] = jac[(ILO_P + a) * LD + ILO_BA + b];
            o[PRE_DP_DBG + 3 * a + b] = jac[(ILO_P + a) * LD + ILO_BG + b];
            o[PRE_DQ_DBG + 3 * a + b] = jac[(ILO_R + a) * LD + ILO_BG + b];
            o[PRE_DV_DBA + 3 * a + b] = jac[(ILO_V + a) * LD + ILO_BA + b];
            o[PRE_DV_DBG + 3 * a + b] = jac[(ILO_V + a) * LD + ILO_BG + b];
            for (int k = 0; k < 4; k++) o[PRE_DEP_DBG + 9 * k + 3 * a + b] = jac[(ILO_EPS1 + 3 * k + a) * LD + ILO_BG + b];
        }
        for (int k = 0; k < 4; k++) for (int a = 0; a < 3; a++) o[PRE_DEP_DRHO + 3 * k + a] = jac[(ILO_EPS1 + 3 * k + a) * LD + ILO_RHO1 + k];
    }
    for (int i = tid; i < 31 * 31; i += nt) {
        const int r = i / 31, c = i % 31;
        o[PRE_INFO + i] = cov[r * LD + c];
        if (out_full) { out_full[(size_t)job * 1922 + i] = jac[r * LD + c]; out_full[(size_t)job * 1922 + 961 + i] = cov[r * LD + c]; }
    }
}

}  // namespace cerb

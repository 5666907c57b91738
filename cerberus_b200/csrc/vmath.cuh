// vmath.cuh -- fp64 3-vector / 3x3 / quaternion helpers for the sm_90a kernels.
// Everything is __host__ __device__ so the same source also builds in the CPU kernel simulator used
// by the non-GPU tests (tests/cusim); the shipped library only ever instantiates the device side.
#pragma once
#include "compat.h"

namespace cerb {

struct d3 { double x, y, z; };
struct m33 { double m[9]; };   // row-major
struct quat { double x, y, z, w; };   // Eigen coeffs order (same as the para_Pose layout, estimator.cpp:852-859)

// read-only global load (ld.global.nc): unlike a plain load it may be hoisted above stores through pointers the compiler
// cannot disambiguate, so sequences of such loads are issued back to back instead of one L2 round trip at a time
CERB_HD double ldro(const double *p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}
CERB_HD d3 mk3(double x, double y, double z) { d3 r; r.x = x; r.y = y; r.z = z; return r; }
CERB_HD d3 ld3(const double *p) { return mk3(p[0], p[1], p[2]); }
CERB_HD void st3(double *p, d3 v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }
CERB_HD d3 operator+(d3 a, d3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
CERB_HD d3 operator-(d3 a, d3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
CERB_HD d3 operator-(d3 a) { return mk3(-a.x, -a.y, -a.z); }
CERB_HD d3 operator*(double s, d3 a) { return mk3(s * a.x, s * a.y, s * a.z); }
CERB_HD d3 operator*(d3 a, double s) { return mk3(s * a.x, s * a.y, s * a.z); }
CERB_HD double dot3(d3 a, d3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
CERB_HD d3 cross3(d3 a, d3 b) { return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
CERB_HD double get3(d3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }

CERB_HD m33 ident33() { m33 r; for (int i = 0; i < 9; i++) r.m[i] = 0.0; r.m[0] = r.m[4] = r.m[8] = 1.0; return r; }
CERB_HD m33 ldm33(const double *p) { m33 r; for (int i = 0; i < 9; i++) r.m[i] = p[i]; return r; }
CERB_HD d3 ld3ro(const double *p) { return mk3(ldro(p), ldro(p + 1), ldro(p + 2)); }
CERB_HD m33 ldm33ro(const double *p) { m33 r; for (int i = 0; i < 9; i++) r.m[i] = ldro(p + i); return r; }
CERB_HD m33 mul33(const m33 &a, const m33 &b) {
    m33 r;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
        r.m[3 * i + j] = a.m[3 * i] * b.m[j] + a.m[3 * i + 1] * b.m[3 + j] + a.m[3 * i + 2] * b.m[6 + j];
    return r;
}
CERB_HD m33 mulT33(const m33 &a, const m33 &b) {   // a^T * b
    m33 r;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
        r.m[3 * i + j] = a.m[i] * b.m[j] + a.m[3 + i] * b.m[3 + j] + a.m[6 + i] * b.m[6 + j];
    return r;
}
CERB_HD m33 tr33(const m33 &a) { m33 r; for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r.m[3 * i + j] = a.m[3 * j + i]; return r; }
CERB_HD d3 mv33(const m33 &a, d3 v) {
    return mk3(a.m[0] * v.x + a.m[1] * v.y + a.m[2] * v.z, a.m[3] * v.x + a.m[4] * v.y + a.m[5] * v.z, a.m[6] * v.x + a.m[7] * v.y + a.m[8] * v.z);
}
CERB_HD d3 mTv33(const m33 &a, d3 v) {   // a^T v
    return mk3(a.m[0] * v.x + a.m[3] * v.y + a.m[6] * v.z, a.m[1] * v.x + a.m[4] * v.y + a.m[7] * v.z, a.m[2] * v.x + a.m[5] * v.y + a.m[8] * v.z);
}
CERB_HD m33 scale33(const m33 &a, double s) { m33 r; for (int i = 0; i < 9; i++) r.m[i] = s * a.m[i]; return r; }
CERB_HD m33 add33(const m33 &a, const m33 &b) { m33 r; for (int i = 0; i < 9; i++) r.m[i] = a.m[i] + b.m[i]; return r; }
CERB_HD m33 sub33(const m33 &a, const m33 &b) { m33 r; for (int i = 0; i < 9; i++) r.m[i] = a.m[i] - b.m[i]; return r; }
// Utility::skewSymmetric (src/utils/utility.h:43-51)
CERB_HD m33 skew33(d3 q) {
    m33 r;
    r.m[0] = 0.0;  r.m[1] = -q.z; r.m[2] = q.y;
    r.m[3] = q.z;  r.m[4] = 0.0;  r.m[5] = -q.x;
    r.m[6] = -q.y; r.m[7] = q.x;  r.m[8] = 0.0;
    return r;
}

CERB_HD quat mkq(double x, double y, double z, double w) { quat q; q.x = x; q.y = y; q.z = z; q.w = w; return q; }
CERB_HD quat ldq(const double *p) { return mkq(p[0], p[1], p[2], p[3]); }   // from para_Pose[.][3..6]
CERB_HD quat qmul(quat a, quat b) {
    return mkq(a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
               a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
               a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x,
               a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z);
}
CERB_HD quat qinv(quat q) {   // conjugate / squaredNorm, like Eigen's inverse()
    double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    return mkq(-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2);
}
CERB_HD quat qnormalized(quat q) {
    double n = sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    return mkq(q.x / n, q.y / n, q.z / n, q.w / n);
}
CERB_HD d3 qvec(quat q) { return mk3(q.x, q.y, q.z); }
CERB_HD d3 qrot(quat q, d3 v) {   // q * v for a unit quaternion
    d3 u = qvec(q);
    d3 uv = cross3(u, v);
    uv = uv + uv;
    return v + q.w * uv + cross3(u, uv);
}
CERB_HD m33 qtoR(quat q) {
    m33 r;
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    r.m[0] = 1 - (tyy + tzz); r.m[1] = txy - twz;       r.m[2] = txz + twy;
    r.m[3] = txy + twz;       r.m[4] = 1 - (txx + tzz); r.m[5] = tyz - twx;
    r.m[6] = txz - twy;       r.m[7] = tyz + twx;       r.m[8] = 1 - (txx + tyy);
    return r;
}
// Utility::deltaQ (utility.h:28-41): (1, theta/2), NOT normalised
CERB_HD quat qdelta(d3 th) { return mkq(th.x * 0.5, th.y * 0.5, th.z * 0.5, 1.0); }
// bottom-right 3x3 of Utility::Qleft(q) / Qright(q)  (utility.h:63-83)
CERB_HD m33 qleft_br(quat q) { m33 r = skew33(qvec(q)); r.m[0] += q.w; r.m[4] += q.w; r.m[8] += q.w; return r; }
CERB_HD m33 qright_br(quat q) { m33 r = scale33(skew33(qvec(q)), -1.0); r.m[0] += q.w; r.m[4] += q.w; r.m[8] += q.w; return r; }
// (Qleft(a) * Qright(b)).bottomRightCorner<3,3>()
CERB_HD m33 qleft_qright_br(quat a, quat b) {
    m33 r = mul33(qleft_br(a), qright_br(b));
    d3 av = qvec(a), bv = qvec(b);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r.m[3 * i + j] -= get3(av, i) * get3(bv, j);
    return r;
}
// PoseLocalParameterization::Plus (pose_local_parameterization.cpp:12-30): x (7) [+] delta (6) -> out (7)
CERB_HD void pose_plus(const double *x, const double *delta, double *out) {
    out[0] = x[0] + delta[0]; out[1] = x[1] + delta[1]; out[2] = x[2] + delta[2];
    quat r = qnormalized(qmul(ldq(x + 3), qdelta(mk3(delta[3], delta[4], delta[5]))));
    out[3] = r.x; out[4] = r.y; out[5] = r.z; out[6] = r.w;
}

}  // namespace cerb

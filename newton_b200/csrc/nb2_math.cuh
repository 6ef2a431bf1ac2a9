// nb2_math.cuh - fp32 vector / quaternion / rigid-transform algebra for the sm_90a kernels.
//
// The operation order inside each helper follows NVIDIA Warp's built-ins (the arithmetic the reference
// kernels are written against: wp.quat_rotate, wp.transform_point, wp.normalize ...; SURVEY.md §8(c)), so
// results track the reference's to rounding.  Everything is __forceinline__ device code operating on
// registers; loads/stores of the reference's packed AoS elements (28-byte transforms, 24-byte spatial
// vectors) are explicit so each kernel controls its own memory traffic.
#pragma once
#include <stdint.h>
#ifdef __CUDACC__
#include <cuda_runtime.h>
#define NB2_DEV __host__ __device__ __forceinline__
#define NB2_CALL __host__ __device__ __noinline__  // one shared copy of a big routine (code size matters for 1-warp CTAs)
#else
// Host-only compilation (g++): lets the test suite compile the convex-contact routines of nb2_convex.cuh
// (see DESIGN.md section 5) with -ffp-contract=off, i.e. the arithmetic of the strict-fp CUDA build, and compare them
// with the oracle's own restatement on the CPU.
#include <cmath>
#define NB2_DEV inline
#define NB2_CALL inline
#ifndef NB2_STRICT_FP
#define NB2_STRICT_FP 1
#endif
#endif

namespace nb2 {

struct V3 {
    float x, y, z;
    NB2_DEV V3() : x(0.f), y(0.f), z(0.f) {}
    NB2_DEV V3(float a, float b, float c) : x(a), y(b), z(c) {}
    NB2_DEV float get(int i) const { return i == 0 ? x : (i == 1 ? y : z); }
    NB2_DEV void set(int i, float v) {
        if (i == 0) x = v;
        else if (i == 1) y = v;
        else z = v;
    }
};
NB2_DEV V3 operator+(V3 a, V3 b) { return V3(a.x + b.x, a.y + b.y, a.z + b.z); }
NB2_DEV V3 operator-(V3 a, V3 b) { return V3(a.x - b.x, a.y - b.y, a.z - b.z); }
NB2_DEV V3 operator-(V3 a) { return V3(-a.x, -a.y, -a.z); }
NB2_DEV V3 operator*(V3 a, float s) { return V3(a.x * s, a.y * s, a.z * s); }
NB2_DEV V3 operator*(float s, V3 a) { return V3(a.x * s, a.y * s, a.z * s); }
NB2_DEV V3 operator/(V3 a, float s) { return V3(a.x / s, a.y / s, a.z / s); }
NB2_DEV void operator+=(V3& a, V3 b) { a = a + b; }
NB2_DEV void operator-=(V3& a, V3 b) { a = a - b; }
NB2_DEV void operator*=(V3& a, float s) { a = a * s; }
NB2_DEV float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
NB2_DEV V3 cross(V3 a, V3 b) { return V3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
NB2_DEV float len2(V3 a) { return dot(a, a); }
NB2_DEV float len(V3 a) { return sqrtf(dot(a, a)); }
NB2_DEV V3 unit(V3 a) {  // wp.normalize: zero vector stays zero
    float l = len(a);
    return l > 0.f ? V3(a.x / l, a.y / l, a.z / l) : V3();
}
NB2_DEV float fmin_w(float a, float b) { return a < b ? a : b; }  // wp.min / wp.max select semantics
NB2_DEV float fmax_w(float a, float b) { return a > b ? a : b; }
NB2_DEV float clamp_w(float x, float lo, float hi) { return fmin_w(fmax_w(lo, x), hi); }
NB2_DEV V3 vmin(V3 a, V3 b) { return V3(fmin_w(a.x, b.x), fmin_w(a.y, b.y), fmin_w(a.z, b.z)); }
NB2_DEV V3 vmax(V3 a, V3 b) { return V3(fmax_w(a.x, b.x), fmax_w(a.y, b.y), fmax_w(a.z, b.z)); }
NB2_DEV V3 vabs(V3 a) { return V3(fabsf(a.x), fabsf(a.y), fabsf(a.z)); }
NB2_DEV V3 cmul(V3 a, V3 b) { return V3(a.x * b.x, a.y * b.y, a.z * b.z); }

// Inverse trig used by the swing-twist joint rows.  NB2_STRICT_FP selects correctly-rounded results (double
// evaluation rounded to fp32), which together with -fmad=false makes the kernels bit-reproduce the CPU oracle.
#ifdef NB2_STRICT_FP
NB2_DEV float asin_w(float x) { return (float)asin((double)x); }
NB2_DEV float acos_w(float x) { return (float)acos((double)x); }
NB2_DEV float sin_w(float x) { return (float)sin((double)x); }
NB2_DEV float cos_w(float x) { return (float)cos((double)x); }
NB2_DEV float atan2_w(float y, float x) { return (float)atan2((double)y, (double)x); }
#else
NB2_DEV float asin_w(float x) { return asinf(x); }
NB2_DEV float acos_w(float x) { return acosf(x); }
NB2_DEV float sin_w(float x) { return sinf(x); }
NB2_DEV float cos_w(float x) { return cosf(x); }
NB2_DEV float atan2_w(float y, float x) { return atan2f(y, x); }
#endif

struct Q4 {
    float x, y, z, w;
    NB2_DEV Q4() : x(0.f), y(0.f), z(0.f), w(1.f) {}
    NB2_DEV Q4(float a, float b, float c, float d) : x(a), y(b), z(c), w(d) {}
};
NB2_DEV Q4 qmul(Q4 a, Q4 b) {
    return Q4(a.w * b.x + b.w * a.x + a.y * b.z - b.y * a.z, a.w * b.y + b.w * a.y + a.z * b.x - b.z * a.x,
              a.w * b.z + b.w * a.z + a.x * b.y - b.x * a.y, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z);
}
NB2_DEV Q4 qadd(Q4 a, Q4 b) { return Q4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
NB2_DEV Q4 qscale(Q4 a, float s) { return Q4(a.x * s, a.y * s, a.z * s, a.w * s); }
NB2_DEV Q4 qconj(Q4 q) { return Q4(-q.x, -q.y, -q.z, q.w); }
NB2_DEV float qdot(Q4 a, Q4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
NB2_DEV Q4 qunit(Q4 q) {
    float l = sqrtf(qdot(q, q));
    if (l > 0.f) {
        float inv = 1.0f / l;
        return Q4(q.x * inv, q.y * inv, q.z * inv, q.w * inv);
    }
    return Q4(0.f, 0.f, 0.f, 1.f);
}
// v(2w^2-1) + 2(q.v)q +/- 2w(q x v)
// The reference formula multiplies each cross term by q.w and then by 2; (t * q.w) * 2 == t * (2 * q.w) bit for bit (scaling by a
// power of two commutes with rounding outside the subnormal range), so 2 * q.w is formed once per quaternion and shared with `c`.
NB2_DEV V3 qrot(Q4 q, V3 v) {
    const float w2 = 2.0f * q.w;
    float c = w2 * q.w - 1.0f;
    float d = 2.0f * (q.x * v.x + q.y * v.y + q.z * v.z);
    return V3(v.x * c + q.x * d + (q.y * v.z - q.z * v.y) * w2, v.y * c + q.y * d + (q.z * v.x - q.x * v.z) * w2,
              v.z * c + q.z * d + (q.x * v.y - q.y * v.x) * w2);
}
NB2_DEV V3 qrot_inv(Q4 q, V3 v) {
    const float w2 = 2.0f * q.w;
    float c = w2 * q.w - 1.0f;
    float d = 2.0f * (q.x * v.x + q.y * v.y + q.z * v.z);
    return V3(v.x * c + q.x * d - (q.y * v.z - q.z * v.y) * w2, v.y * c + q.y * d - (q.z * v.x - q.x * v.z) * w2,
              v.z * c + q.z * d - (q.x * v.y - q.y * v.x) * w2);
}

struct M33 {
    float a[9];  // row-major
    NB2_DEV float at(int r, int c) const { return a[3 * r + c]; }
};
NB2_DEV M33 m33_zero() {
    M33 m;
#pragma unroll
    for (int i = 0; i < 9; ++i) m.a[i] = 0.f;
    return m;
}
NB2_DEV V3 mv(const M33& m, V3 v) {  // sum of columns scaled by components
    V3 r(m.a[0] * v.x, m.a[3] * v.x, m.a[6] * v.x);
    r += V3(m.a[1] * v.y, m.a[4] * v.y, m.a[7] * v.y);
    r += V3(m.a[2] * v.z, m.a[5] * v.z, m.a[8] * v.z);
    return r;
}
NB2_DEV V3 mtv(const M33& m, V3 v) {  // transpose(m) * v
    V3 r(m.a[0] * v.x, m.a[1] * v.x, m.a[2] * v.x);
    r += V3(m.a[3] * v.y, m.a[4] * v.y, m.a[5] * v.y);
    r += V3(m.a[6] * v.z, m.a[7] * v.z, m.a[8] * v.z);
    return r;
}
NB2_DEV M33 mscale(float s, const M33& m) {
    M33 r;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.a[i] = m.a[i] * s;
    return r;
}
NB2_DEV M33 qmat(Q4 q) {  // columns = rotated basis vectors
    V3 c0 = qrot(q, V3(1.f, 0.f, 0.f)), c1 = qrot(q, V3(0.f, 1.f, 0.f)), c2 = qrot(q, V3(0.f, 0.f, 1.f));
    M33 m;
    m.a[0] = c0.x; m.a[1] = c1.x; m.a[2] = c2.x;
    m.a[3] = c0.y; m.a[4] = c1.y; m.a[5] = c2.y;
    m.a[6] = c0.z; m.a[7] = c1.z; m.a[8] = c2.z;
    return m;
}

struct Xf {
    V3 p;
    Q4 q;
    NB2_DEV Xf() {}
    NB2_DEV Xf(V3 p_, Q4 q_) : p(p_), q(q_) {}
};
NB2_DEV V3 xpoint(const Xf& t, V3 v) { return t.p + qrot(t.q, v); }
NB2_DEV V3 xvec(const Xf& t, V3 v) { return qrot(t.q, v); }
NB2_DEV Xf xmul(const Xf& a, const Xf& b) { return Xf(qrot(a.q, b.p) + a.p, qmul(a.q, b.q)); }
NB2_DEV Xf xinv(const Xf& t) {
    Q4 qi = qconj(t.q);
    return Xf(-qrot(qi, t.p), qi);
}

// ---- packed AoS element access (reference layouts) -------------------------------------------
NB2_DEV V3 ld3(const float* p) { return V3(p[0], p[1], p[2]); }
NB2_DEV void st3(float* p, V3 v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }
NB2_DEV Xf ldx(const float* p) { return Xf(V3(p[0], p[1], p[2]), Q4(p[3], p[4], p[5], p[6])); }
NB2_DEV void stx(float* p, const Xf& t) {
    p[0] = t.p.x; p[1] = t.p.y; p[2] = t.p.z; p[3] = t.q.x; p[4] = t.q.y; p[5] = t.q.z; p[6] = t.q.w;
}
NB2_DEV M33 ldm(const float* p) {
    M33 m;
#pragma unroll
    for (int i = 0; i < 9; ++i) m.a[i] = p[i];
    return m;
}

}  // namespace nb2

// nb2_spatial.cuh - spatial-vector algebra and joint-axis helpers shared by the articulated-body kernels
// (nb2_featherstone.cu: SolverFeatherstone.step, eval_fk / eval_ik; nb2_dynamics.cu: Jacobians, mass matrices, inverse
// dynamics).  Operation order follows the Warp built-ins of the reference, so the strict-fp build stays bit-exact.
#pragma once
#include "nb2_math.cuh"

namespace nb2 {

enum { FJ_PRISMATIC = 0, FJ_REVOLUTE = 1, FJ_BALL = 2, FJ_FIXED = 3, FJ_FREE = 4, FJ_DISTANCE = 5, FJ_D6 = 6 };

struct S6 {
    float v[6];
    NB2_DEV S6() {
#pragma unroll
        for (int i = 0; i < 6; ++i) v[i] = 0.f;
    }
    NB2_DEV S6(V3 a, V3 b) { v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = b.x; v[4] = b.y; v[5] = b.z; }
    NB2_DEV V3 top() const { return V3(v[0], v[1], v[2]); }
    NB2_DEV V3 bot() const { return V3(v[3], v[4], v[5]); }
};
NB2_DEV S6 ld6(const float* p) {
    S6 s;
#pragma unroll
    for (int i = 0; i < 6; ++i) s.v[i] = p[i];
    return s;
}
NB2_DEV void st6(float* p, const S6& s) {
#pragma unroll
    for (int i = 0; i < 6; ++i) p[i] = s.v[i];
}
NB2_DEV S6 operator+(const S6& a, const S6& b) {
    S6 r;
#pragma unroll
    for (int i = 0; i < 6; ++i) r.v[i] = a.v[i] + b.v[i];
    return r;
}
NB2_DEV S6 operator-(const S6& a, const S6& b) {
    S6 r;
#pragma unroll
    for (int i = 0; i < 6; ++i) r.v[i] = a.v[i] - b.v[i];
    return r;
}
NB2_DEV S6 operator*(const S6& a, float s) {
    S6 r;
#pragma unroll
    for (int i = 0; i < 6; ++i) r.v[i] = a.v[i] * s;
    return r;
}
NB2_DEV float dot6(const S6& a, const S6& b) {
    return a.v[0] * b.v[0] + a.v[1] * b.v[1] + a.v[2] * b.v[2] + a.v[3] * b.v[3] + a.v[4] * b.v[4] + a.v[5] * b.v[5];
}
NB2_DEV S6 twist_xf(const Xf& t, const S6& x) {  // math/spatial.py:82-105
    V3 w = qrot(t.q, x.bot());
    V3 v = qrot(t.q, x.top()) + cross(t.p, w);
    return S6(v, w);
}
NB2_DEV S6 scross(const S6& a, const S6& b) {
    V3 w = cross(a.bot(), b.bot());
    V3 v = cross(a.bot(), b.top()) + cross(a.top(), b.bot());
    return S6(v, w);
}
NB2_DEV S6 scross_dual(const S6& a, const S6& b) {
    V3 w = cross(a.bot(), b.bot()) + cross(a.top(), b.top());
    V3 v = cross(a.bot(), b.top());
    return S6(v, w);
}
NB2_DEV S6 m66v(const float* I, const S6& b) {  // dense 6x6 (row-major in shared memory) times vector, column order
    S6 r;
#pragma unroll
    for (int i = 0; i < 6; ++i) r.v[i] = I[6 * i] * b.v[0];
#pragma unroll
    for (int c = 1; c < 6; ++c)
#pragma unroll
        for (int i = 0; i < 6; ++i) r.v[i] += I[6 * i + c] * b.v[c];
    return r;
}
NB2_DEV Q4 q_axis_angle(V3 axis, float angle) {
    float half = angle * 0.5f;
    float w = cos_w(half), s = sin_w(half);
    V3 v = axis * s;
    return Q4(v.x, v.y, v.z, w);
}

// transform_spatial_inertia (kernels.py:66-138) for I = blockdiag(m 1, Ic): T^T I T with T = [[R, S], [0, R]],
// R / S from the inverse transform.  Sums follow the dense k-order of the reference with structural zeros dropped.
NB2_DEV void spatial_inertia(const Xf& t, float mass, const M33& Ic, float* out) {
    const Xf ti = xinv(t);
    const M33 R = qmat(ti.q);
    const V3 p = ti.p;
    M33 S;  // skew(p) @ R
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        S.a[0 + j] = (-p.z) * R.a[3 + j] + p.y * R.a[6 + j];
        S.a[3 + j] = p.z * R.a[0 + j] + (-p.x) * R.a[6 + j];
        S.a[6 + j] = (-p.y) * R.a[0 + j] + p.x * R.a[3 + j];
    }
    float A[6][6];  // A = T^T I
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            A[i][j] = R.a[3 * j + i] * mass;
            A[i][j + 3] = 0.0f;
            A[i + 3][j] = S.a[3 * j + i] * mass;
            float s = R.a[0 + i] * Ic.a[0 + j];
            s += R.a[3 + i] * Ic.a[3 + j];
            s += R.a[6 + i] * Ic.a[6 + j];
            A[i + 3][j + 3] = s;
        }
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float s = A[i][0] * R.a[0 + j];
            s += A[i][1] * R.a[3 + j];
            s += A[i][2] * R.a[6 + j];
            out[6 * i + j] = s;
            float u = A[i][0] * S.a[0 + j];
            u += A[i][1] * S.a[3 + j];
            u += A[i][2] * S.a[6 + j];
            if (i >= 3) {
                u += A[i][3] * R.a[0 + j];
                u += A[i][4] * R.a[3 + j];
                u += A[i][5] * R.a[6 + j];
            }
            out[6 * i + j + 3] = u;
        }
}

NB2_DEV float joint_force(float q, float qd, float tq, float tqd, float ke, float kd, float lo, float up, float lke, float lkd, float damping) {
    float limit_f = 0.0f, damping_f = 0.0f;
    float target_f = ke * (tq - q) + kd * (tqd - qd);
    if (q < lo) {
        limit_f = lke * (lo - q);
        damping_f = -lkd * qd;
        target_f = 0.0f;
    } else if (q > up) {
        limit_f = lke * (up - q);
        damping_f = -lkd * qd;
        target_f = 0.0f;
    }
    float passive_f = -damping * qd;
    return limit_f + damping_f + target_f + passive_f;
}

// wp.quat_from_matrix of the matrix whose COLUMNS are c0, c1, c2 (trace branch, else the largest diagonal element; normalized)
NB2_DEV Q4 q_from_cols(V3 c0, V3 c1, V3 c2) {
    const float m00 = c0.x, m10 = c0.y, m20 = c0.z, m01 = c1.x, m11 = c1.y, m21 = c1.z, m02 = c2.x, m12 = c2.y, m22 = c2.z;
    const float tr = m00 + m11 + m22;
    float x, y, z, w, h;
    if (tr >= 0.0f) {
        h = sqrtf(tr + 1.0f);
        w = 0.5f * h;
        h = 0.5f / h;
        x = (m21 - m12) * h;
        y = (m02 - m20) * h;
        z = (m10 - m01) * h;
    } else {
        int md = 0;
        if (m11 > m00) md = 1;
        if (m22 > (md == 0 ? m00 : m11)) md = 2;
        if (md == 0) {
            h = sqrtf((m00 - (m11 + m22)) + 1.0f);
            x = 0.5f * h;
            h = 0.5f / h;
            y = (m01 + m10) * h;
            z = (m20 + m02) * h;
            w = (m21 - m12) * h;
        } else if (md == 1) {
            h = sqrtf((m11 - (m22 + m00)) + 1.0f);
            y = 0.5f * h;
            h = 0.5f / h;
            z = (m12 + m21) * h;
            x = (m01 + m10) * h;
            w = (m02 - m20) * h;
        } else {
            h = sqrtf((m22 - (m00 + m11)) + 1.0f);
            z = 0.5f * h;
            h = 0.5f / h;
            x = (m20 + m02) * h;
            y = (m12 + m21) * h;
            w = (m10 - m01) * h;
        }
    }
    return qunit(Q4(x, y, z, w));
}
// transform_2d_rotational_axes (sim/articulation.py:37-58): D6 joints with exactly two angular axes
NB2_DEV void axes2(V3 a0, V3 a1, float q0, V3& o0, V3& o1) {
    const Q4 q_off = q_from_cols(a0, a1, cross(a0, a1));
    const V3 l0 = qrot(q_off, V3(1.f, 0.f, 0.f)), l1 = qrot(q_off, V3(0.f, 1.f, 0.f));
    o0 = l0;
    o1 = qrot(q_axis_angle(l0, q0), l1);
}
NB2_DEV void axes3(V3 a0, V3 a1, V3 a2, float q0, float q1, V3& o0, V3& o1, V3& o2) {  // transform_3d_rotational_axes
    Q4 q_0 = q_axis_angle(a0, q0);
    V3 a1w = qrot(q_0, a1);
    Q4 q_1 = q_axis_angle(a1w, q1);
    V3 a2w = qrot(qmul(q_1, q_0), a2);
    o0 = a0; o1 = a1w; o2 = a2w;
}

NB2_DEV float twist_angle_signed(V3 axis, Q4 q) {  // wp.quat_twist_angle_signed: 2 atan2(q.xyz . axis, q.w), range (-2 pi, 2 pi]
    return 2.0f * atan2_w(dot(V3(q.x, q.y, q.z), axis), q.w);
}

// newton.math.quat_decompose (math/spatial.py:150-175): wp.quat_to_euler(q, 2, 1, 0), each angle wrapped to [-pi, pi); for
// q = qx(a) qy(b) qz(c) the result is (a, b, c)
NB2_DEV float wrap_pm_pi(float theta) {
    const float pi = 3.14159265358979323846f, two_pi = 2.0f * pi;
    float wrapped = fmodf(theta + pi, two_pi);
    if (wrapped < 0.0f) wrapped += two_pi;
    return wrapped - pi;
}
NB2_DEV V3 q_decompose(Q4 q) {
    const float a = q.w - q.y, b = q.z - q.x, c = q.y + q.w, d = -q.x - q.z;
    const float n_ab = a * a + b * b;
    float theta2 = acos_w(2.0f * n_ab / (n_ab + c * c + d * d) - 1.0f);
    const float theta_plus = atan2_w(b, a), theta_minus = atan2_w(d, c);
    const float theta1 = theta_plus - theta_minus;
    float theta3 = theta_plus + theta_minus;
    theta3 = -theta3;
    theta2 -= 1.57079632679489661923f;
    return V3(wrap_pm_pi(theta3), wrap_pm_pi(theta2), wrap_pm_pi(theta1));
}

}  // namespace nb2

// oracle_featherstone.h - TEST INFRASTRUCTURE ONLY.
// CPU restatement of the reference SolverFeatherstone.step (solvers/featherstone/solver_featherstone.py:461-1066):
// one function per Warp kernel of solvers/featherstone/kernels.py, run serially in thread-id order, including the
// dense 6nj x 6nj mass matrix and the one-thread-per-articulation dense GEMMs exactly as the reference executes them.
#pragma once
#include <cstdio>
#include <cstring>
#include <vector>

#include "../include/newton_b200.h"
#include "oracle_math.h"
#include "oracle_xpbd.h"

namespace orc {

struct sv6 {  // Newton spatial vector (linear, angular) as a flat 6-vector
    float v[6];
    sv6() { for (float& x : v) x = 0.f; }
    sv6(vec3 a, vec3 b) { v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = b.x; v[4] = b.y; v[5] = b.z; }
    vec3 top() const { return vec3(v[0], v[1], v[2]); }
    vec3 bot() const { return vec3(v[3], v[4], v[5]); }
    static sv6 load(const float* f) { sv6 s; for (int i = 0; i < 6; ++i) s.v[i] = f[i]; return s; }
    void store(float* f) const { for (int i = 0; i < 6; ++i) f[i] = v[i]; }
};
inline sv6 operator+(const sv6& a, const sv6& b) { sv6 r; for (int i = 0; i < 6; ++i) r.v[i] = a.v[i] + b.v[i]; return r; }
inline sv6 operator-(const sv6& a, const sv6& b) { sv6 r; for (int i = 0; i < 6; ++i) r.v[i] = a.v[i] - b.v[i]; return r; }
inline sv6 operator-(const sv6& a) { sv6 r; for (int i = 0; i < 6; ++i) r.v[i] = -a.v[i]; return r; }
inline sv6 operator*(const sv6& a, float s) { sv6 r; for (int i = 0; i < 6; ++i) r.v[i] = a.v[i] * s; return r; }
inline float dot6(const sv6& a, const sv6& b) {
    return a.v[0] * b.v[0] + a.v[1] * b.v[1] + a.v[2] * b.v[2] + a.v[3] * b.v[3] + a.v[4] * b.v[4] + a.v[5] * b.v[5];
}
struct mat66 {
    float m[6][6];
    mat66() { std::memset(m, 0, sizeof(m)); }
};
inline mat66 mul66(const mat66& a, const mat66& b) {  // warp/native/mat.h mul(mat, mat)
    mat66 t;
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j)
            for (int k = 0; k < 6; ++k) t.m[i][j] += a.m[i][k] * b.m[k][j];
    return t;
}
inline mat66 transpose66(const mat66& a) {
    mat66 t;
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) t.m[i][j] = a.m[j][i];
    return t;
}
inline sv6 mul66v(const mat66& a, const sv6& b) {  // warp/native/mat.h mul(mat, vec): columns scaled, left to right
    sv6 r;
    for (int i = 0; i < 6; ++i) r.v[i] = a.m[i][0] * b.v[0];
    for (int c = 1; c < 6; ++c)
        for (int i = 0; i < 6; ++i) r.v[i] += a.m[i][c] * b.v[c];
    return r;
}

// newton.math.transform_twist (math/spatial.py:82-105): w' = R w, v' = R v + p x w'
inline sv6 transform_twist(const transform& t, const sv6& x) {
    vec3 w = quat_rotate(t.q, x.bot());
    vec3 v = quat_rotate(t.q, x.top()) + cross(t.p, w);
    return sv6(v, w);
}
inline sv6 spatial_cross(const sv6& a, const sv6& b) {  // kernels.py:731-742
    vec3 w = cross(a.bot(), b.bot());
    vec3 v = cross(a.bot(), b.top()) + cross(a.top(), b.bot());
    return sv6(v, w);
}
inline sv6 spatial_cross_dual(const sv6& a, const sv6& b) {  // kernels.py:745-756
    vec3 w = cross(a.bot(), b.bot()) + cross(a.top(), b.top());
    vec3 v = cross(a.bot(), b.top());
    return sv6(v, w);
}
// kernels.py:66-138
inline mat66 transform_spatial_inertia(const transform& t, const mat66& I) {
    transform t_inv = transform_inverse(t);
    quat q = t_inv.q;
    vec3 p = t_inv.p;
    vec3 r1 = quat_rotate(q, vec3(1.f, 0.f, 0.f)), r2 = quat_rotate(q, vec3(0.f, 1.f, 0.f)), r3 = quat_rotate(q, vec3(0.f, 0.f, 1.f));
    mat33 R(r1.x, r2.x, r3.x, r1.y, r2.y, r3.y, r1.z, r2.z, r3.z);
    mat33 skew(0.f, -p.z, p.y, p.z, 0.f, -p.x, -p.y, p.x, 0.f);
    mat33 S = skew * R;
    mat66 T;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            T.m[i][j] = R.m[i][j];
            T.m[i][j + 3] = S.m[i][j];
            T.m[i + 3][j + 3] = R.m[i][j];
        }
    return mul66(mul66(transpose66(T), I), T);
}
// semi_implicit/kernels_body.py:17-51
inline float joint_force(float q, float qd, float target_q, float target_qd, float target_ke, float target_kd, float lower,
                         float upper, float limit_ke, float limit_kd, float damping) {
    float limit_f = 0.0f, damping_f = 0.0f;
    float target_f = target_ke * (target_q - q) + target_kd * (target_qd - qd);
    if (q < lower) {
        limit_f = limit_ke * (lower - q);
        damping_f = -limit_kd * qd;
        target_f = 0.0f;
    } else if (q > upper) {
        limit_f = limit_ke * (upper - q);
        damping_f = -limit_kd * qd;
        target_f = 0.0f;
    }
    float passive_f = -damping * qd;
    return limit_f + damping_f + target_f + passive_f;
}
// sim/articulation.py:37-82 transform_2d_rotational_axes / compute_2d_rotational_dofs: the two axes are orthonormalised through
// q_off = quat_from_matrix([axis_0 axis_1 axis_0 x axis_1]); axis 1 is carried through the rotation about axis 0.
inline void transform_2d_rotational_axes(vec3 axis_0, vec3 axis_1, float q0, vec3& a0, vec3& a1) {
    quat q_off = quat_from_matrix(matrix_from_cols(axis_0, axis_1, cross(axis_0, axis_1)));
    vec3 local_0 = quat_rotate(q_off, vec3(1.f, 0.f, 0.f));
    vec3 local_1 = quat_rotate(q_off, vec3(0.f, 1.f, 0.f));
    a0 = local_0;
    quat q_0 = quat_from_axis_angle(a0, q0);
    a1 = quat_rotate(q_0, local_1);
}
inline void compute_2d_rotational_dofs(vec3 axis_0, vec3 axis_1, float q0, float q1, float qd0, float qd1, quat& rot, vec3& vel) {
    vec3 a0, a1;
    transform_2d_rotational_axes(axis_0, axis_1, q0, a0, a1);
    quat q_0 = quat_from_axis_angle(a0, q0), q_1 = quat_from_axis_angle(a1, q1);
    rot = q_1 * q_0;
    vel = a0 * qd0 + a1 * qd1;
}
// sim/articulation.py transform_3d_rotational_axes / compute_3d_rotational_dofs
inline void transform_3d_rotational_axes(vec3 a0, vec3 a1, vec3 a2, float q0, float q1, vec3& o0, vec3& o1, vec3& o2) {
    quat q_0 = quat_from_axis_angle(a0, q0);
    vec3 a1w = quat_rotate(q_0, a1);
    quat q_1 = quat_from_axis_angle(a1w, q1);
    vec3 a2w = quat_rotate(q_1 * q_0, a2);
    o0 = a0; o1 = a1w; o2 = a2w;
}
inline void compute_3d_rotational_dofs(vec3 a0, vec3 a1, vec3 a2, float q0, float q1, float q2, float qd0, float qd1, float qd2,
                                       quat& rot, vec3& vel) {
    vec3 w0, w1, w2;
    transform_3d_rotational_axes(a0, a1, a2, q0, q1, w0, w1, w2);
    quat q_0 = quat_from_axis_angle(w0, q0), q_1 = quat_from_axis_angle(w1, q1), q_2 = quat_from_axis_angle(w2, q2);
    rot = q_2 * q_1 * q_0;
    vel = w0 * qd0 + w1 * qd1 + w2 * qd2;
}

struct FsScratch {  // the per-solver aux arrays of solver_featherstone.py:361-459
    std::vector<float> body_q_com, body_qd_fk, body_solve_origin, body_I_s, body_v_s, body_a_s, body_f_s, body_f_ext, body_ft_s;
    std::vector<float> joint_S_s, joint_qd_in, joint_qd_out, joint_f_internal, joint_tau, joint_qdd;
    std::vector<float> J, M, P, H, L;
    std::vector<int> J_start, M_start, H_start;
    std::vector<float> body_q_prev;  // _featherstone_body_q_prev (solver_featherstone.py:514-516)
    int step = 0;
    bool mass_matrix_dirty = false;  // _mass_matrix_dirty (solver_featherstone.py:190, 284-288)
    bool init = false;
};

// notify_model_changed (solver_featherstone.py:284-288): body or dof properties changed -> form H on the next step
enum { MODEL_JOINT_DOF_PROPERTIES = 1 << 1, MODEL_BODY_PROPERTIES = 1 << 2 };  // ModelFlags (sim/enums.py:19-22)
inline void fs_notify_model_changed(FsScratch& s, int flags) {
    if (flags & (MODEL_JOINT_DOF_PROPERTIES | MODEL_BODY_PROPERTIES)) s.mass_matrix_dirty = true;
}

// descendant_free_distance_mask (solver_featherstone.py:225-262): FREE / DISTANCE joints with a parent and a non-kinematic child
inline bool descendant_free_distance(const nb2_model_desc& m, int j) {
    const int t = m.joint_type[j];
    return (t == JT_FREE || t == JT_DISTANCE) && m.joint_parent[j] >= 0 && !(m.body_flags[m.joint_child[j]] & BODY_KINEMATIC);
}

// kernels.py:142-238
inline transform jcalc_transform(const nb2_model_desc& m, int type, int axis_start, int lin, int ang, const float* joint_q, int q_start) {
    if (type == JT_PRISMATIC) return transform(load3(m.joint_axis + 3 * axis_start) * joint_q[q_start], quat_identity());
    if (type == JT_REVOLUTE) return transform(vec3(), quat_from_axis_angle(load3(m.joint_axis + 3 * axis_start), joint_q[q_start]));
    if (type == JT_BALL) return transform(vec3(), quat(joint_q[q_start], joint_q[q_start + 1], joint_q[q_start + 2], joint_q[q_start + 3]));
    if (type == JT_FIXED) return transform_identity();
    if (type == JT_FREE || type == JT_DISTANCE)
        return transform(vec3(joint_q[q_start], joint_q[q_start + 1], joint_q[q_start + 2]),
                         quat(joint_q[q_start + 3], joint_q[q_start + 4], joint_q[q_start + 5], joint_q[q_start + 6]));
    if (type == JT_D6) {
        vec3 pos(0.f);
        quat rot = quat_identity();
        for (int k = 0; k < 3; ++k)
            if (lin > k) pos += load3(m.joint_axis + 3 * (axis_start + k)) * joint_q[q_start + k];
        int ia = axis_start + lin, iq = q_start + lin;
        if (ang == 1) rot = quat_from_axis_angle(load3(m.joint_axis + 3 * ia), joint_q[iq]);
        if (ang == 2) {
            vec3 vel;
            compute_2d_rotational_dofs(load3(m.joint_axis + 3 * ia), load3(m.joint_axis + 3 * (ia + 1)), joint_q[iq], joint_q[iq + 1], 0.f, 0.f, rot,
                                       vel);
        }
        if (ang == 3) {
            vec3 vel;
            compute_3d_rotational_dofs(load3(m.joint_axis + 3 * ia), load3(m.joint_axis + 3 * (ia + 1)), load3(m.joint_axis + 3 * (ia + 2)),
                                       joint_q[iq], joint_q[iq + 1], joint_q[iq + 2], 0.f, 0.f, 0.f, rot, vel);
        }
        return transform(pos, rot);
    }
    return transform_identity();
}

// kernels.py:242-379; writes joint_S_s, returns v_j_s and the apparent-derivative term c_app_s
inline void jcalc_motion(const nb2_model_desc& m, int type, const float* joint_q, int lin, int ang, const transform& X_sc,
                         const float* joint_qd, int q_start, int qd_start, float* joint_S_s, sv6& v_j_s, sv6& c_app_s) {
    v_j_s = sv6();
    c_app_s = sv6();
    auto axis = [&](int i) { return load3(m.joint_axis + 3 * i); };
    if (type == JT_PRISMATIC) {
        sv6 S = transform_twist(X_sc, sv6(axis(qd_start), vec3()));
        v_j_s = S * joint_qd[qd_start];
        S.store(joint_S_s + 6 * qd_start);
        return;
    }
    if (type == JT_REVOLUTE) {
        sv6 S = transform_twist(X_sc, sv6(vec3(), axis(qd_start)));
        v_j_s = S * joint_qd[qd_start];
        S.store(joint_S_s + 6 * qd_start);
        return;
    }
    if (type == JT_D6) {
        vec3 c_app_ang;
        for (int k = 0; k < 3; ++k)
            if (lin > k) {
                sv6 S = transform_twist(X_sc, sv6(axis(qd_start + k), vec3()));
                v_j_s = v_j_s + S * joint_qd[qd_start + k];
                S.store(joint_S_s + 6 * (qd_start + k));
            }
        int iqd = qd_start + lin, iq = q_start + lin;
        if (ang == 1) {
            sv6 S = transform_twist(X_sc, sv6(vec3(), axis(iqd)));
            v_j_s = v_j_s + S * joint_qd[iqd];
            S.store(joint_S_s + 6 * iqd);
        }
        if (ang == 2) {  // kernels.py:301-311
            vec3 a0, a1;
            transform_2d_rotational_axes(axis(iqd), axis(iqd + 1), joint_q[iq], a0, a1);
            sv6 S0 = transform_twist(X_sc, sv6(vec3(), a0)), S1 = transform_twist(X_sc, sv6(vec3(), a1));
            float qd0 = joint_qd[iqd], qd1 = joint_qd[iqd + 1];
            v_j_s = v_j_s + (S0 * qd0 + S1 * qd1);
            S0.store(joint_S_s + 6 * iqd);
            S1.store(joint_S_s + 6 * (iqd + 1));
            c_app_ang += cross(a0, a1) * (qd0 * qd1);
        }
        if (ang == 3) {
            vec3 a0, a1, a2;
            transform_3d_rotational_axes(axis(iqd), axis(iqd + 1), axis(iqd + 2), joint_q[iq], joint_q[iq + 1], a0, a1, a2);
            sv6 S0 = transform_twist(X_sc, sv6(vec3(), a0)), S1 = transform_twist(X_sc, sv6(vec3(), a1)), S2 = transform_twist(X_sc, sv6(vec3(), a2));
            float qd0 = joint_qd[iqd], qd1 = joint_qd[iqd + 1], qd2 = joint_qd[iqd + 2];
            v_j_s = v_j_s + (S0 * qd0 + S1 * qd1 + S2 * qd2);
            S0.store(joint_S_s + 6 * iqd);
            S1.store(joint_S_s + 6 * (iqd + 1));
            S2.store(joint_S_s + 6 * (iqd + 2));
            c_app_ang += cross(a0, a1) * (qd0 * qd1);
            c_app_ang += cross(a0, a2) * (qd0 * qd2);
            c_app_ang += cross(a1, a2) * (qd1 * qd2);
        }
        c_app_s = transform_twist(X_sc, sv6(vec3(), c_app_ang));
        return;
    }
    if (type == JT_BALL) {
        sv6 S0 = transform_twist(X_sc, sv6(vec3(), vec3(1.f, 0.f, 0.f))), S1 = transform_twist(X_sc, sv6(vec3(), vec3(0.f, 1.f, 0.f))),
            S2 = transform_twist(X_sc, sv6(vec3(), vec3(0.f, 0.f, 1.f)));
        S0.store(joint_S_s + 6 * qd_start);
        S1.store(joint_S_s + 6 * (qd_start + 1));
        S2.store(joint_S_s + 6 * (qd_start + 2));
        v_j_s = S0 * joint_qd[qd_start] + S1 * joint_qd[qd_start + 1] + S2 * joint_qd[qd_start + 2];
        return;
    }
    if (type == JT_FIXED) return;
    if (type == JT_FREE || type == JT_DISTANCE) {
        v_j_s = transform_twist(X_sc, sv6::load(joint_qd + qd_start));
        for (int k = 0; k < 6; ++k) {
            sv6 e;
            e.v[k] = 1.0f;
            transform_twist(X_sc, e).store(joint_S_s + 6 * (qd_start + k));
        }
        return;
    }
}

// eval_body_contact with force_in_world_frame = False (semi_implicit/kernels_contact.py:381-556)
inline void eval_body_contact(const nb2_model_desc& m, const float* body_q, const float* body_qd, const nb2_contacts_view& c,
                              float friction_smoothing, float* body_f) {
    int count = c.rigid_contact_count[0];
    for (int tid = 0; tid < c.rigid_contact_max && tid < count; ++tid) {
        float ke = 0.f, kd = 0.f, kf = 0.f, ka = 0.f, mu = 0.f;
        int mat_nonzero = 0;
        float margin_a = c.margin0[tid], margin_b = c.margin1[tid];
        int shape_a = c.shape0[tid], shape_b = c.shape1[tid];
        if (shape_a == shape_b) continue;
        int body_a = -1, body_b = -1;
        if (shape_a >= 0) {
            mat_nonzero += 1;
            ke += m.shape_material_ke[shape_a]; kd += m.shape_material_kd[shape_a]; kf += m.shape_material_kf[shape_a];
            ka += m.shape_material_ka[shape_a]; mu += m.shape_material_mu[shape_a];
            body_a = m.shape_body[shape_a];
        }
        if (shape_b >= 0) {
            mat_nonzero += 1;
            ke += m.shape_material_ke[shape_b]; kd += m.shape_material_kd[shape_b]; kf += m.shape_material_kf[shape_b];
            ka += m.shape_material_ka[shape_b]; mu += m.shape_material_mu[shape_b];
            body_b = m.shape_body[shape_b];
        }
        if (mat_nonzero > 0) {
            ke /= float(mat_nonzero); kd /= float(mat_nonzero); kf /= float(mat_nonzero); ka /= float(mat_nonzero); mu /= float(mat_nonzero);
        }
        vec3 n = -load3(c.normal + 3 * tid);
        vec3 bx_a = load3(c.point0 + 3 * tid), bx_b = load3(c.point1 + 3 * tid);
        vec3 r_a(0.f), r_b(0.f);
        if (body_a >= 0) {
            transform X = transform::load(body_q + 7 * body_a);
            bx_a = transform_point(X, bx_a) - margin_a * n;
            r_a = bx_a - transform_point(X, load3(m.body_com + 3 * body_a));
        }
        if (body_b >= 0) {
            transform X = transform::load(body_q + 7 * body_b);
            bx_b = transform_point(X, bx_b) + margin_b * n;
            r_b = bx_b - transform_point(X, load3(m.body_com + 3 * body_b));
        }
        float d = dot(n, bx_a - bx_b);
        if (d >= ka) continue;
        vec3 bv_a(0.f), bv_b(0.f);
        if (body_a >= 0) bv_a = load3(body_qd + 6 * body_a) + cross(load3(body_qd + 6 * body_a + 3), r_a);
        if (body_b >= 0) bv_b = load3(body_qd + 6 * body_b) + cross(load3(body_qd + 6 * body_b + 3), r_b);
        vec3 v = bv_a - bv_b;
        float vn = dot(n, v);
        vec3 vt = v - n * vn;
        float fn = d * ke;
        float fd = minf(vn, 0.0f) * kd * (d < 0.0f ? 1.0f : 0.0f);  // wp.step(d)
        vec3 ft(0.f);
        if (d < 0.0f) {
            float a = dot(vt, vt);  // wp.norm_huber(vt, delta)
            float vs = (a <= friction_smoothing * friction_smoothing) ? 0.5f * a : friction_smoothing * (std::sqrt(a) - 0.5f * friction_smoothing);
            if (vs > 0.0f) {
                vec3 fr = vt / vs;
                ft = fr * minf(kf * vs, -mu * (fn + fd));
            }
        }
        vec3 f_total = n * (fn + fd) + ft;
        if (body_a >= 0) atomic_sub(body_f, body_a, spatial(f_total, cross(r_a, f_total)));
        if (body_b >= 0) atomic_add(body_f, body_b, spatial(f_total, cross(r_b, f_total)));
    }
}

inline void fs_init(const nb2_model_desc& m, FsScratch& s) {
    const size_t B = m.body_count, D = m.joint_dof_count;
    s.body_q_com.assign(B * 7, 0.f); s.body_qd_fk.assign(B * 6, 0.f); s.body_solve_origin.assign(B * 3, 0.f);
    s.body_I_s.assign(B * 36, 0.f); s.body_v_s.assign(B * 6, 0.f); s.body_a_s.assign(B * 6, 0.f); s.body_f_s.assign(B * 6, 0.f);
    s.body_f_ext.assign(B * 6, 0.f); s.body_ft_s.assign(B * 6, 0.f);
    s.joint_S_s.assign(D * 6, 0.f); s.joint_qd_in.assign(D, 0.f); s.joint_qd_out.assign(D, 0.f); s.joint_f_internal.assign(D, 0.f);
    s.joint_tau.assign(D, 0.f); s.joint_qdd.assign(D, 0.f);
    size_t Js = 0, Ms = 0, Hs = 0;
    for (int a = 0; a < m.articulation_count; ++a) {  // _compute_articulation_indices (solver_featherstone.py:290-359)
        int j0 = m.articulation_start[a], j1 = m.articulation_start[a + 1];
        int nj = j1 - j0, nd = m.joint_qd_start[j1] - m.joint_qd_start[j0];
        s.J_start.push_back(int(Js)); s.M_start.push_back(int(Ms)); s.H_start.push_back(int(Hs));
        Js += size_t(6) * nj * nd; Ms += size_t(36) * nj * nj; Hs += size_t(nd) * nd;
    }
    s.J.assign(Js, 0.f); s.M.assign(Ms, 0.f); s.P.assign(Js, 0.f); s.H.assign(Hs, 0.f); s.L.assign(Hs, 0.f);
    s.init = true;
}

// joint_armature_effective (solver_featherstone.py:269-281): dofs of a joint whose child body is kinematic get 1e10
inline float armature_effective(const nb2_model_desc& m, int j0, int j1, int dof) {
    for (int j = j0; j < j1; ++j)
        if (dof >= m.joint_qd_start[j] && dof < m.joint_qd_start[j + 1])
            return (m.body_flags[m.joint_child[j]] & BODY_KINEMATIC) ? 1.0e10f : m.joint_armature[dof];
    return m.joint_armature[dof];
}

inline void featherstone_step(FsScratch& s, const nb2_model_desc& m, const nb2_featherstone_params& p, const nb2_state_view& sin,
                              const nb2_state_view& sout, const nb2_control_view& ctl, const nb2_contacts_view* contacts, float dt) {
    if (!s.init) fs_init(m, s);
    const int A = m.articulation_count, J = m.joint_count, B = m.body_count;
    auto art_end = [&](int a) { return m.articulation_start[a + 1]; };
    // ---- eval_rigid_fk (kernels.py:687-728) -> state_in.body_q, body_q_com
    for (int a = 0; a < A; ++a)
        for (int i = m.articulation_start[a]; i < art_end(a); ++i) {
            int parent = m.joint_parent[i], child = m.joint_child[i];
            transform X_wpj = transform::load(m.joint_X_p + 7 * i);
            if (parent >= 0) X_wpj = transform::load(sin.body_q + 7 * parent) * X_wpj;
            transform X_j = jcalc_transform(m, m.joint_type[i], m.joint_qd_start[i], m.joint_dof_dim[2 * i], m.joint_dof_dim[2 * i + 1],
                                            sin.joint_q, m.joint_q_start[i]);
            transform X_wc = (X_wpj * X_j) * transform_inverse(transform::load(m.joint_X_c + 7 * i));
            transform X_sm = X_wc * transform(load3(m.body_com + 3 * child), quat_identity());
            X_wc.store(sin.body_q + 7 * child);
            X_sm.store(s.body_q_com.data() + 7 * child);
        }
    // the pre-step poses the descendant FREE / DISTANCE correction integrates from: state_in.body_q as eval_rigid_fk left it, copied
    // because a step in place overwrites it (solver_featherstone.py:481, 514-516)
    bool any_descendant = false;
    for (int j = 0; j < J; ++j) any_descendant = any_descendant || descendant_free_distance(m, j);
    if (any_descendant) s.body_q_prev.assign(sin.body_q, sin.body_q + size_t(B) * 7);
    // ---- body_f_ext = body_f (+ FREE/DISTANCE joint_f as COM wrenches, kernels.py:893-921)
    std::memcpy(s.body_f_ext.data(), sin.body_f, size_t(B) * 6 * sizeof(float));
    for (int j = 0; j < J; ++j) {
        int t = m.joint_type[j];
        if (t != JT_FREE && t != JT_DISTANCE) continue;
        int qd0 = m.joint_qd_start[j];
        atomic_add(s.body_f_ext.data(), m.joint_child[j],
                   spatial(vec3(ctl.joint_f[qd0], ctl.joint_f[qd0 + 1], ctl.joint_f[qd0 + 2]),
                           vec3(ctl.joint_f[qd0 + 3], ctl.joint_f[qd0 + 4], ctl.joint_f[qd0 + 5])));
    }
    // ---- public -> internal qd / joint_f (kernels.py:924-975, 1069-1088)
    for (int j = 0; j < J; ++j) {
        int qd0 = m.joint_qd_start[j], qd1 = m.joint_qd_start[j + 1], t = m.joint_type[j];
        if (t != JT_FREE && t != JT_DISTANCE) {
            for (int i = qd0; i < qd1; ++i) { s.joint_qd_in[i] = sin.joint_qd[i]; s.joint_f_internal[i] = ctl.joint_f[i]; }
            continue;
        }
        for (int i = qd0; i < qd1; ++i) s.joint_f_internal[i] = 0.0f;
        int parent = m.joint_parent[j], child = m.joint_child[j];
        transform X_wpj = transform::load(m.joint_X_p + 7 * j);
        if (parent >= 0) X_wpj = transform::load(sin.body_q + 7 * parent) * X_wpj;
        vec3 x_child_com = transform_point(transform::load(sin.body_q + 7 * child), load3(m.body_com + 3 * child));
        vec3 r = quat_rotate_inv(X_wpj.q, x_child_com - X_wpj.p);
        vec3 v_com(sin.joint_qd[qd0], sin.joint_qd[qd0 + 1], sin.joint_qd[qd0 + 2]);
        vec3 omega(sin.joint_qd[qd0 + 3], sin.joint_qd[qd0 + 4], sin.joint_qd[qd0 + 5]);
        vec3 v_int = v_com - cross(omega, r);
        s.joint_qd_in[qd0] = v_int.x; s.joint_qd_in[qd0 + 1] = v_int.y; s.joint_qd_in[qd0 + 2] = v_int.z;
        s.joint_qd_in[qd0 + 3] = omega.x; s.joint_qd_in[qd0 + 4] = omega.y; s.joint_qd_in[qd0 + 5] = omega.z;
    }
    // ---- eval_rigid_id (kernels.py:1241-1317, compute_link_velocity :764-865)
    std::fill(s.body_f_s.begin(), s.body_f_s.end(), 0.f);
    for (int a = 0; a < A; ++a) {
        int start = m.articulation_start[a], end = art_end(a);
        vec3 solve_origin;
        if (start < end) {
            int rt = m.joint_type[start];
            if (rt == JT_FREE || rt == JT_DISTANCE) solve_origin = load3(s.body_q_com.data() + 7 * m.joint_child[start]);
        }
        for (int i = start; i < end; ++i) {
            int type = m.joint_type[i], child = m.joint_child[i], parent = m.joint_parent[i];
            transform X_wpj = transform::load(m.joint_X_p + 7 * i);
            if (parent >= 0) X_wpj = transform::load(sin.body_q + 7 * parent) * X_wpj;
            transform X_wpj_s(X_wpj.p - solve_origin, X_wpj.q);
            sv6 v_j_s, c_app_s;
            jcalc_motion(m, type, sin.joint_q, m.joint_dof_dim[2 * i], m.joint_dof_dim[2 * i + 1], X_wpj_s, s.joint_qd_in.data(),
                         m.joint_q_start[i], m.joint_qd_start[i], s.joint_S_s.data(), v_j_s, c_app_s);
            sv6 v_parent_s, a_parent_s;
            if (parent >= 0) {
                v_parent_s = sv6::load(s.body_v_s.data() + 6 * parent);
                a_parent_s = sv6::load(s.body_a_s.data() + 6 * parent);
            }
            sv6 v_s = v_parent_s + v_j_s;
            sv6 a_s = a_parent_s + spatial_cross(v_s, v_j_s) + c_app_s;
            transform X_sm = transform::load(s.body_q_com.data() + 7 * child);
            vec3 x_com_s = X_sm.p - solve_origin;
            store3(s.body_solve_origin.data() + 3 * child, solve_origin);
            mat66 I_m;  // compute_spatial_inertia (kernels.py:21-40)
            float mass = m.body_mass[child];
            I_m.m[0][0] = I_m.m[1][1] = I_m.m[2][2] = mass;
            for (int r = 0; r < 3; ++r)
                for (int cc = 0; cc < 3; ++cc) I_m.m[3 + r][3 + cc] = m.body_inertia[9 * child + 3 * r + cc];
            int world_idx = m.body_world[child];
            if (world_idx < 0) world_idx += m.gravity_count;
            vec3 f_g = mass * load3(m.gravity + 3 * world_idx);
            sv6 f_g_s(f_g, cross(x_com_s, f_g));
            mat66 I_s = transform_spatial_inertia(transform(x_com_s, X_sm.q), I_m);
            sv6 f_b_s = mul66v(I_s, a_s) + spatial_cross_dual(v_s, mul66v(I_s, v_s));
            vec3 omega_world = v_s.bot();
            vec3 v_com_world = v_s.top() + cross(omega_world, x_com_s);
            sv6(v_com_world, omega_world).store(s.body_qd_fk.data() + 6 * child);
            v_s.store(s.body_v_s.data() + 6 * child);
            a_s.store(s.body_a_s.data() + 6 * child);
            (f_b_s - f_g_s).store(s.body_f_s.data() + 6 * child);
            for (int r = 0; r < 6; ++r)
                for (int cc = 0; cc < 6; ++cc) s.body_I_s[36 * child + 6 * r + cc] = I_s.m[r][cc];
        }
    }
    // ---- penalty contacts (solver_featherstone.py:650-680)
    if (contacts && contacts->rigid_contact_max)
        eval_body_contact(m, sin.body_q, s.body_qd_fk.data(), *contacts, p.friction_smoothing, s.body_f_ext.data());
    for (int b = 0; b < B; ++b)  // zero_kinematic_body_forces
        if (m.body_flags[b] & BODY_KINEMATIC)
            for (int k = 0; k < 6; ++k) s.body_f_ext[6 * b + k] = 0.f;
    // ---- eval_rigid_tau (kernels.py:1320-1418) + jcalc_tau (:383-461)
    std::fill(s.body_ft_s.begin(), s.body_ft_s.end(), 0.f);
    for (int a = 0; a < A; ++a) {
        int start = m.articulation_start[a], end = art_end(a);
        for (int i = end - 1; i >= start; --i) {
            int type = m.joint_type[i], parent = m.joint_parent[i], child = m.joint_child[i];
            int dof_start = m.joint_qd_start[i], coord_start = m.joint_q_start[i], tq_start = m.joint_target_q_start[i];
            int lin = m.joint_dof_dim[2 * i], ang = m.joint_dof_dim[2 * i + 1];
            sv6 f_b_s = sv6::load(s.body_f_s.data() + 6 * child), f_t_s = sv6::load(s.body_ft_s.data() + 6 * child);
            sv6 fe = sv6::load(s.body_f_ext.data() + 6 * child);
            vec3 x_com_s = load3(s.body_q_com.data() + 7 * child) - load3(s.body_solve_origin.data() + 3 * child);
            sv6 f_ext = -sv6(fe.top(), fe.bot() + cross(x_com_s, fe.top()));
            f_ext.store(s.body_f_ext.data() + 6 * child);
            sv6 f_s = f_b_s + f_t_s + f_ext;
            float* tau = s.joint_tau.data();
            const float* S = s.joint_S_s.data();
            const float* jqd = s.joint_qd_in.data();
            const float* jf = s.joint_f_internal.data();
            if (type == JT_BALL) {
                for (int k = 0; k < 3; ++k) {
                    int j = dof_start + k;
                    float passive_f = -m.joint_damping[j] * jqd[j];
                    tau[j] = -dot6(sv6::load(S + 6 * j), f_s) + jf[j] + passive_f;
                }
            } else if (type == JT_FREE || type == JT_DISTANCE) {
                for (int k = 0; k < 6; ++k) tau[dof_start + k] = -dot6(sv6::load(S + 6 * (dof_start + k)), f_s) + jf[dof_start + k];
            } else if (type == JT_PRISMATIC || type == JT_REVOLUTE || type == JT_D6) {
                for (int k = 0; k < lin + ang; ++k) {
                    int j = dof_start + k;
                    float drive_f = joint_force(sin.joint_q[coord_start + k], jqd[j], ctl.joint_target_q[tq_start + k], ctl.joint_target_qd[j],
                                                m.joint_target_ke[j], m.joint_target_kd[j], m.joint_limit_lower[j], m.joint_limit_upper[j],
                                                m.joint_limit_ke[j], m.joint_limit_kd[j], m.joint_damping[j]);
                    tau[j] = -dot6(sv6::load(S + 6 * j), f_s) + drive_f + jf[j];
                }
            }
            if (parent >= 0) (sv6::load(s.body_ft_s.data() + 6 * parent) + f_s).store(s.body_ft_s.data() + 6 * parent);
        }
    }
    // ---- State.body_parent_f when requested (solver_featherstone.py:691-697, 741-758; compute_body_parent_f kernels.py:2371-2416):
    // the wrench the inbound joint transmits = the RNEA backward-pass sum, moved from the solve origin to the body's COM
    if (sout.body_parent_f) {
        std::fill(sout.body_parent_f, sout.body_parent_f + size_t(B) * 6, 0.f);
        if (A > 0)
            for (int b = 0; b < B; ++b) {
                sv6 f_s = sv6::load(s.body_f_s.data() + 6 * b) + sv6::load(s.body_ft_s.data() + 6 * b) + sv6::load(s.body_f_ext.data() + 6 * b);
                vec3 f_lin = f_s.top(), f_ang_at_origin = f_s.bot();
                vec3 r_com = load3(s.body_q_com.data() + 7 * b) - load3(s.body_solve_origin.data() + 3 * b);
                vec3 f_ang_at_com = f_ang_at_origin - cross(r_com, f_lin);
                sv6(f_lin, f_ang_at_com).store(sout.body_parent_f + 6 * b);
            }
    }
    // ---- mass matrix: J, M, P = M J, H = J^T P, L = chol(H + diag(armature)) (solver_featherstone.py:767-921)
    if (s.mass_matrix_dirty || s.step % (p.update_mass_matrix_interval > 0 ? p.update_mass_matrix_interval : 1) == 0) {
        s.mass_matrix_dirty = false;
        for (int a = 0; a < A; ++a) {
            int j0 = m.articulation_start[a], j1 = art_end(a), nj = j1 - j0;
            int d0 = m.joint_qd_start[j0], nd = m.joint_qd_start[j1] - d0;
            float* Jm = s.J.data() + s.J_start[a];
            float* Mm = s.M.data() + s.M_start[a];
            float* Pm = s.P.data() + s.J_start[a];
            float* Hm = s.H.data() + s.H_start[a];
            float* Lm = s.L.data() + s.H_start[a];
            for (int i = 0; i < nj; ++i) {  // eval_rigid_jacobian (kernels.py:1422-1463)
                int j = j0 + i;
                while (j != -1) {
                    int ds = m.joint_qd_start[j], dc = m.joint_qd_start[j + 1] - ds;
                    for (int dof = 0; dof < dc; ++dof)
                        for (int k = 0; k < 6; ++k) Jm[(i * 6 + k) * nd + (ds - d0) + dof] = s.joint_S_s[6 * (ds + dof) + k];
                    j = m.joint_ancestor[j];
                }
            }
            int stride = nj * 6;  // spatial_mass (kernels.py:1466-1480): NB indexes body_I_s by JOINT index
            for (int l = 0; l < nj; ++l)
                for (int i = 0; i < 6; ++i)
                    for (int jj = 0; jj < 6; ++jj) Mm[(l * 6 + i) * stride + l * 6 + jj] = s.body_I_s[36 * (j0 + l) + 6 * i + jj];
            for (int i = 0; i < stride; ++i)  // dense_gemm P = M J (kernels.py:1504-1538)
                for (int jj = 0; jj < nd; ++jj) {
                    float sum = 0.0f;
                    for (int k = 0; k < stride; ++k) sum += Mm[i * stride + k] * Jm[k * nd + jj];
                    Pm[i * nd + jj] = sum;
                }
            for (int i = 0; i < nd; ++i)  // H = J^T P
                for (int jj = 0; jj < nd; ++jj) {
                    float sum = 0.0f;
                    for (int k = 0; k < stride; ++k) sum += Jm[k * nd + i] * Pm[k * nd + jj];
                    Hm[i * nd + jj] = sum;
                }
            for (int jn = 0; jn < nd; ++jn) {  // dense_cholesky (kernels.py:1690-1719)
                // joint_armature_effective (solver_featherstone.py:269-281): 1e10 on the dofs of joints that drive a kinematic body
                float sv = Hm[jn * nd + jn] + armature_effective(m, j0, j1, d0 + jn);
                for (int k = 0; k < jn; ++k) {
                    float r = Lm[jn * nd + k];
                    sv -= r * r;
                }
                sv = std::sqrt(sv);
                float invS = 1.0f / sv;
                Lm[jn * nd + jn] = sv;
                for (int i = jn + 1; i < nd; ++i) {
                    float t = Hm[i * nd + jn];
                    for (int k = 0; k < jn; ++k) t -= Lm[i * nd + k] * Lm[jn * nd + k];
                    Lm[i * nd + jn] = t * invS;
                }
            }
        }
    }
    // ---- dense_subs: qdd = (L L^T)^-1 tau (kernels.py:1754-1781)
    std::fill(s.joint_qdd.begin(), s.joint_qdd.end(), 0.f);
    for (int a = 0; a < A; ++a) {
        int j0 = m.articulation_start[a], j1 = art_end(a);
        int d0 = m.joint_qd_start[j0], n = m.joint_qd_start[j1] - d0;
        const float* Lm = s.L.data() + s.H_start[a];
        float* x = s.joint_qdd.data() + d0;
        const float* b = s.joint_tau.data() + d0;
        for (int i = 0; i < n; ++i) {
            float t = b[i];
            for (int j = 0; j < i; ++j) t -= Lm[i * n + j] * x[j];
            x[i] = t / Lm[i * n + i];
        }
        for (int i = n - 1; i >= 0; --i) {
            float t = x[i];
            for (int j = i + 1; j < n; ++j) t -= Lm[j * n + i] * x[j];
            x[i] = t / Lm[i * n + i];
        }
    }
    // ---- zero_kinematic_joint_qdd (kernels.py:1933-1948)
    for (int j = 0; j < J; ++j)
        if (m.body_flags[m.joint_child[j]] & BODY_KINEMATIC)
            for (int i = m.joint_qd_start[j]; i < m.joint_qd_start[j + 1]; ++i) s.joint_qdd[i] = 0.0f;
    // ---- integrate_generalized_joints (kernels.py:1849-1893, jcalc_integrate :464-630)
    for (int j = 0; j < J; ++j) {
        int type = m.joint_type[j], parent = m.joint_parent[j], child = m.joint_child[j];
        int cs = m.joint_q_start[j], ds = m.joint_qd_start[j];
        const float* q = sin.joint_q;
        const float* qd = s.joint_qd_in.data();
        const float* qdd = s.joint_qdd.data();
        float* qn = sout.joint_q;
        float* qdn = s.joint_qd_out.data();
        if (type == JT_FIXED) continue;
        if (type == JT_PRISMATIC || type == JT_REVOLUTE) {
            float qd_new = qd[ds] + qdd[ds] * dt;
            qdn[ds] = qd_new;
            qn[cs] = q[cs] + qd_new * dt;
        } else if (type == JT_BALL) {
            vec3 w_new = vec3(qd[ds], qd[ds + 1], qd[ds + 2]) + vec3(qdd[ds], qdd[ds + 1], qdd[ds + 2]) * dt;
            quat r(q[cs], q[cs + 1], q[cs + 2], q[cs + 3]);
            quat drdt = quat(w_new, 0.0f) * r * 0.5f;
            quat rn = normalize(r + drdt * dt);
            qn[cs] = rn.x; qn[cs + 1] = rn.y; qn[cs + 2] = rn.z; qn[cs + 3] = rn.w;
            qdn[ds] = w_new.x; qdn[ds + 1] = w_new.y; qdn[ds + 2] = w_new.z;
        } else if (type == JT_FREE || type == JT_DISTANCE) {
            if (parent < 0) {
                vec3 a_parent(qdd[ds], qdd[ds + 1], qdd[ds + 2]), alpha(qdd[ds + 3], qdd[ds + 4], qdd[ds + 5]);
                vec3 v_parent(qd[ds], qd[ds + 1], qd[ds + 2]), omega(qd[ds + 3], qd[ds + 4], qd[ds + 5]);
                vec3 pp(q[cs], q[cs + 1], q[cs + 2]);
                quat r(q[cs + 3], q[cs + 4], q[cs + 5], q[cs + 6]);
                vec3 r_com_joint = transform_point(transform_inverse(transform::load(m.joint_X_c + 7 * j)), load3(m.body_com + 3 * child));
                vec3 x_com = pp + quat_rotate(r, r_com_joint);
                vec3 v_com = v_parent + cross(omega, x_com);
                vec3 a_com = a_parent + cross(alpha, x_com) + cross(omega, v_com);
                vec3 omega_new = omega + alpha * dt;
                vec3 v_com_new = v_com + a_com * dt;
                quat drdt = quat(omega_new, 0.0f) * r * 0.5f;
                quat r_new = normalize(r + drdt * dt);
                vec3 x_com_new = x_com + v_com_new * dt;
                vec3 p_new = x_com_new - quat_rotate(r_new, r_com_joint);
                vec3 v_parent_new = v_com_new - cross(omega_new, x_com_new);
                qn[cs] = p_new.x; qn[cs + 1] = p_new.y; qn[cs + 2] = p_new.z;
                qn[cs + 3] = r_new.x; qn[cs + 4] = r_new.y; qn[cs + 5] = r_new.z; qn[cs + 6] = r_new.w;
                qdn[ds] = v_parent_new.x; qdn[ds + 1] = v_parent_new.y; qdn[ds + 2] = v_parent_new.z;
                qdn[ds + 3] = omega_new.x; qdn[ds + 4] = omega_new.y; qdn[ds + 5] = omega_new.z;
            } else {
                vec3 w_s = vec3(qd[ds + 3], qd[ds + 4], qd[ds + 5]) + vec3(qdd[ds + 3], qdd[ds + 4], qdd[ds + 5]) * dt;
                vec3 v_s = vec3(qd[ds], qd[ds + 1], qd[ds + 2]) + vec3(qdd[ds], qdd[ds + 1], qdd[ds + 2]) * dt;
                vec3 p_s(q[cs], q[cs + 1], q[cs + 2]);
                vec3 dpdt = v_s + cross(w_s, p_s);
                quat r_s(q[cs + 3], q[cs + 4], q[cs + 5], q[cs + 6]);
                quat drdt = quat(w_s, 0.0f) * r_s * 0.5f;
                vec3 pn = p_s + dpdt * dt;
                quat rn = normalize(r_s + drdt * dt);
                qn[cs] = pn.x; qn[cs + 1] = pn.y; qn[cs + 2] = pn.z; qn[cs + 3] = rn.x; qn[cs + 4] = rn.y; qn[cs + 5] = rn.z; qn[cs + 6] = rn.w;
                qdn[ds] = v_s.x; qdn[ds + 1] = v_s.y; qdn[ds + 2] = v_s.z; qdn[ds + 3] = w_s.x; qdn[ds + 4] = w_s.y; qdn[ds + 5] = w_s.z;
            }
        } else if (type == JT_D6) {
            int n = m.joint_dof_dim[2 * j] + m.joint_dof_dim[2 * j + 1];
            for (int k = 0; k < n; ++k) {
                float qd_new = qd[ds + k] + qdd[ds + k] * dt;
                qdn[ds + k] = qd_new;
                qn[cs + k] = q[cs + k] + qd_new * dt;
            }
        }
    }
    // ---- copy_kinematic_joint_state (kernels.py:1951-1976): prescribed joint state passes through the solve
    for (int j = 0; j < J; ++j)
        if (m.body_flags[m.joint_child[j]] & BODY_KINEMATIC) {
            for (int i = m.joint_q_start[j]; i < m.joint_q_start[j + 1]; ++i) sout.joint_q[i] = sin.joint_q[i];
            for (int i = m.joint_qd_start[j]; i < m.joint_qd_start[j + 1]; ++i) s.joint_qd_out[i] = s.joint_qd_in[i];
        }
    // ---- eval_fk_with_velocity_conversion (kernels.py:1987-2149) -> state_out.body_q / body_qd, joints [start, end) of one articulation
    auto fk_with_velocity_conversion = [&](int start, int end) {
        for (int i = start; i < end; ++i) {
            int parent = m.joint_parent[i], child = m.joint_child[i], type = m.joint_type[i];
            int qs = m.joint_q_start[i], qds = m.joint_qd_start[i];
            int lin = m.joint_dof_dim[2 * i], ang = m.joint_dof_dim[2 * i + 1];
            const float* jq = sout.joint_q;
            const float* jqd = s.joint_qd_out.data();
            transform X_j = jcalc_transform(m, type, qds, lin, ang, jq, qs);
            vec3 vj_lin, vj_ang;
            auto axis = [&](int k) { return load3(m.joint_axis + 3 * k); };
            if (type == JT_PRISMATIC) vj_lin = axis(qds) * jqd[qds];
            if (type == JT_REVOLUTE) vj_ang = axis(qds) * jqd[qds];
            if (type == JT_BALL) vj_ang = vec3(jqd[qds], jqd[qds + 1], jqd[qds + 2]);
            if (type == JT_FREE || type == JT_DISTANCE) {
                vj_lin = vec3(jqd[qds], jqd[qds + 1], jqd[qds + 2]);
                vj_ang = vec3(jqd[qds + 3], jqd[qds + 4], jqd[qds + 5]);
            }
            if (type == JT_D6) {
                for (int k = 0; k < 3; ++k)
                    if (lin > k) vj_lin += axis(qds + k) * jqd[qds + k];
                int iq = qs + lin, iqd = qds + lin;
                if (ang == 1) vj_ang = jqd[iqd] * axis(iqd);
                if (ang == 2) {
                    quat rot;
                    compute_2d_rotational_dofs(axis(iqd), axis(iqd + 1), jq[iq], jq[iq + 1], jqd[iqd], jqd[iqd + 1], rot, vj_ang);
                }
                if (ang == 3) {
                    quat rot;
                    compute_3d_rotational_dofs(axis(iqd), axis(iqd + 1), axis(iqd + 2), jq[iq], jq[iq + 1], jq[iq + 2], jqd[iqd], jqd[iqd + 1],
                                               jqd[iqd + 2], rot, vj_ang);
                }
            }
            transform X_wpj = transform::load(m.joint_X_p + 7 * i);
            transform X_wp;
            if (parent >= 0) {
                X_wp = transform::load(sout.body_q + 7 * parent);
                X_wpj = X_wp * X_wpj;
            }
            transform X_wcj = X_wpj * X_j;
            transform X_wc = X_wcj * transform_inverse(transform::load(m.joint_X_c + 7 * i));
            vec3 x_child_origin = X_wc.p;
            vec3 v_parent_origin, w_parent;
            if (parent >= 0) {
                spatial v_wp = spatial::load(sout.body_qd + 6 * parent);
                w_parent = v_wp.bot;
                v_parent_origin = velocity_at_point(v_wp, x_child_origin - transform_point(X_wp, load3(m.body_com + 3 * parent)));
            }
            vec3 linear_joint_world = transform_vector(X_wpj, vj_lin);
            vec3 angular_joint_world = transform_vector(X_wpj, vj_ang);
            vec3 linear_joint_origin;
            if (type == JT_FREE || type == JT_DISTANCE) {
                sv6 v_j_world = transform_twist(X_wpj, sv6(vj_lin, vj_ang));
                linear_joint_origin = cross(v_j_world.bot(), x_child_origin) + v_j_world.top();
                angular_joint_world = v_j_world.bot();
            } else {
                linear_joint_origin = linear_joint_world + cross(angular_joint_world, x_child_origin - X_wcj.p);
            }
            vec3 v_o = v_parent_origin + linear_joint_origin, w_o = w_parent + angular_joint_world;
            X_wc.store(sout.body_q + 7 * child);
            // origin_twist_to_com_twist (sim/articulation.py)
            vec3 v_com = cross(w_o, transform_vector(X_wc, load3(m.body_com + 3 * child))) + v_o;
            spatial(v_com, w_o).store(sout.body_qd + 6 * child);
        }
    };
    for (int a = 0; a < A; ++a) fk_with_velocity_conversion(m.articulation_start[a], art_end(a));
    if (any_descendant) {
        // correct_free_distance_body_pose_from_world_twist (kernels.py:1914-1930, integrate_body_pose_from_com_twist :1896-1911):
        // a descendant FREE / DISTANCE child moves by its world COM twist from its pre-step pose
        for (int j = 0; j < J; ++j) {
            if (!descendant_free_distance(m, j)) continue;
            int child = m.joint_child[j];
            transform X_wb = transform::load(s.body_q_prev.data() + 7 * child);
            vec3 com = load3(m.body_com + 3 * child);
            vec3 x_com = transform_point(X_wb, com);
            spatial qd = spatial::load(sout.body_qd + 6 * child);
            quat drdt = quat(qd.bot, 0.0f) * X_wb.q * 0.5f;
            quat q_new = normalize(X_wb.q + drdt * dt);
            vec3 x_com_new = x_com + qd.top * dt;
            transform(x_com_new - quat_rotate(q_new, com), q_new).store(sout.body_q + 7 * child);
        }
        // reconstruct_free_distance_joint_q_from_body_pose (kernels.py:978-1012)
        for (int j = 0; j < J; ++j) {
            if (!descendant_free_distance(m, j)) continue;
            int parent = m.joint_parent[j], child = m.joint_child[j];
            transform X_wpj = transform::load(sout.body_q + 7 * parent) * transform::load(m.joint_X_p + 7 * j);
            transform X_wcj = transform::load(sout.body_q + 7 * child) * transform::load(m.joint_X_c + 7 * j);
            vec3 x_err_c = quat_rotate_inv(X_wpj.q, X_wcj.p - X_wpj.p);
            quat q_pc = quat_inverse(X_wpj.q) * X_wcj.q;
            transform(x_err_c, q_pc).store(sout.joint_q + m.joint_q_start[j]);
        }
        // eval_fk_with_velocity_conversion_from_joint_starts (kernels.py:2221-2265, 2332-2368): each articulation again from its
        // first such joint
        for (int a = 0; a < A; ++a)
            for (int i = m.articulation_start[a]; i < art_end(a); ++i)
                if (descendant_free_distance(m, i)) {
                    fk_with_velocity_conversion(i, art_end(a));
                    break;
                }
    }
    // ---- internal -> public qd (kernels.py:1015-1066)
    for (int j = 0; j < J; ++j) {
        int qd0 = m.joint_qd_start[j], qd1 = m.joint_qd_start[j + 1], t = m.joint_type[j];
        if (t != JT_FREE && t != JT_DISTANCE) {
            for (int i = qd0; i < qd1; ++i) sout.joint_qd[i] = s.joint_qd_out[i];
            continue;
        }
        int parent = m.joint_parent[j], child = m.joint_child[j];
        transform X_wpj = transform::load(m.joint_X_p + 7 * j);
        if (parent >= 0) X_wpj = transform::load(sout.body_q + 7 * parent) * X_wpj;
        vec3 x_child_com = transform_point(transform::load(sout.body_q + 7 * child), load3(m.body_com + 3 * child));
        vec3 r = quat_rotate_inv(X_wpj.q, x_child_com - X_wpj.p);
        vec3 v_int(s.joint_qd_out[qd0], s.joint_qd_out[qd0 + 1], s.joint_qd_out[qd0 + 2]);
        vec3 omega(s.joint_qd_out[qd0 + 3], s.joint_qd_out[qd0 + 4], s.joint_qd_out[qd0 + 5]);
        vec3 v_com = v_int + cross(omega, r);
        sout.joint_qd[qd0] = v_com.x; sout.joint_qd[qd0 + 1] = v_com.y; sout.joint_qd[qd0 + 2] = v_com.z;
        sout.joint_qd[qd0 + 3] = omega.x; sout.joint_qd[qd0 + 4] = omega.y; sout.joint_qd[qd0 + 5] = omega.z;
    }
    s.step += 1;
}

// ---- public newton.eval_fk (sim/articulation.py:237-424 eval_single_articulation_fk; launch :420-475 with the optional ----
// articulation_mask / articulation_indices).  joint_qd in the PUBLIC convention (FREE/DISTANCE linear dofs = child COM velocity).
// body_flag_filter (:421): only bodies whose flags intersect the filter are written (BodyFlags.ALL = DYNAMIC | KINEMATIC = 3).
inline void eval_articulation_fk(const nb2_model_desc& m, const float* joint_q, const float* joint_qd, float* body_q, float* body_qd,
                                 const uint8_t* articulation_mask = nullptr, const int* articulation_indices = nullptr, int index_count = 0,
                                 int body_flag_filter = 3) {
    const int dim = articulation_indices ? index_count : m.articulation_count;
    for (int tid = 0; tid < dim; ++tid) {
        const int a = articulation_indices ? articulation_indices[tid] : tid;
        if (a < 0 || a >= m.articulation_count) continue;        // :462-463 bounds check
        if (articulation_mask && !articulation_mask[a]) continue;  // :466-468
        for (int i = m.articulation_start[a]; i < m.articulation_start[a + 1]; ++i) {
            if (m.joint_articulation[i] == -1) continue;
            int parent = m.joint_parent[i], child = m.joint_child[i], type = m.joint_type[i];
            int qs = m.joint_q_start[i], qds = m.joint_qd_start[i];
            int lin = m.joint_dof_dim[2 * i], ang = m.joint_dof_dim[2 * i + 1];
            transform X_j = jcalc_transform(m, type, qds, lin, ang, joint_q, qs);
            vec3 vj_lin, vj_ang;
            auto axis = [&](int k) { return load3(m.joint_axis + 3 * k); };
            if (type == JT_PRISMATIC) vj_lin = axis(qds) * joint_qd[qds];
            if (type == JT_REVOLUTE) vj_ang = axis(qds) * joint_qd[qds];
            if (type == JT_BALL) vj_ang = vec3(joint_qd[qds], joint_qd[qds + 1], joint_qd[qds + 2]);
            if (type == JT_FREE || type == JT_DISTANCE) {
                vj_lin = vec3(joint_qd[qds], joint_qd[qds + 1], joint_qd[qds + 2]);
                vj_ang = vec3(joint_qd[qds + 3], joint_qd[qds + 4], joint_qd[qds + 5]);
            }
            if (type == JT_D6) {
                for (int k = 0; k < 3; ++k)
                    if (lin > k) vj_lin += axis(qds + k) * joint_qd[qds + k];
                int iq = qs + lin, iqd = qds + lin;
                if (ang == 1) vj_ang = joint_qd[iqd] * axis(iqd);
                if (ang == 2) {
                    quat rot;
                    compute_2d_rotational_dofs(axis(iqd), axis(iqd + 1), joint_q[iq], joint_q[iq + 1], joint_qd[iqd], joint_qd[iqd + 1], rot, vj_ang);
                }
                if (ang == 3) {
                    quat rot;
                    compute_3d_rotational_dofs(axis(iqd), axis(iqd + 1), axis(iqd + 2), joint_q[iq], joint_q[iq + 1], joint_q[iq + 2],
                                               joint_qd[iqd], joint_qd[iqd + 1], joint_qd[iqd + 2], rot, vj_ang);
                }
            }
            transform X_wpj = transform::load(m.joint_X_p + 7 * i);
            transform X_wp;
            if (parent >= 0) {
                X_wp = transform::load(body_q + 7 * parent);
                X_wpj = X_wp * X_wpj;
            }
            transform X_wcj = X_wpj * X_j;
            transform X_wc = X_wcj * transform_inverse(transform::load(m.joint_X_c + 7 * i));
            vec3 x_child_origin = X_wc.p;
            vec3 v_parent_origin, w_parent;
            if (parent >= 0) {
                spatial v_wp = spatial::load(body_qd + 6 * parent);
                w_parent = v_wp.bot;
                v_parent_origin = velocity_at_point(v_wp, x_child_origin - transform_point(X_wp, load3(m.body_com + 3 * parent)));
            }
            vec3 linear_joint_world = transform_vector(X_wpj, vj_lin);
            vec3 angular_joint_world = transform_vector(X_wpj, vj_ang);
            vec3 linear_joint_origin;
            if (type == JT_FREE || type == JT_DISTANCE)  // com_twist_to_origin_twist
                linear_joint_origin = linear_joint_world - cross(angular_joint_world, transform_vector(X_wc, load3(m.body_com + 3 * child)));
            else
                linear_joint_origin = linear_joint_world + cross(angular_joint_world, x_child_origin - X_wcj.p);
            vec3 v_o = v_parent_origin + linear_joint_origin, w_o = w_parent + angular_joint_world;
            if ((m.body_flags[child] & body_flag_filter) == 0) continue;  // keeps its values; descendants read them (sim/articulation.py:421)
            X_wc.store(body_q + 7 * child);
            vec3 v_com = cross(w_o, transform_vector(X_wc, load3(m.body_com + 3 * child))) + v_o;  // origin_twist_to_com_twist
            spatial(v_com, w_o).store(body_qd + 6 * child);
        }
    }
}

// wp.quat_twist_angle_signed(axis, q): signed rotation angle of q's twist about `axis`.  Warp built-in (warp-lang >= 1.16,
// not vendored): restated as 2*atan2(q.xyz . axis, q.w), range (-2 pi, 2 pi].  The unfolded range is pinned by the
// reference's own test - newton/tests/test_kinematics.py:95-111 expects eval_ik(eval_fk(+-4.0 rad)) == +-4.0 to 1e-6,
// which a fold into (-pi, pi] would break; operation order inside the built-in remains unpinned at the ulp level.
inline float quat_twist_angle_signed(vec3 axis, quat q) {
    float proj = dot(vec3(q.x, q.y, q.z), axis);
    return 2.0f * atan2_w(proj, q.w);
}

// invert_2d_rotational_dofs / invert_3d_rotational_dofs (sim/articulation.py:85-126, 177-236): joint angles and rates of a D6 joint
// with two / three angular axes from the relative orientation and the angular-velocity error
inline void invert_2d_rotational_dofs(vec3 axis_0, vec3 axis_1, quat q_p, quat q_c, vec3 w_err, float* angles2, float* vel2) {
    quat q_off = quat_from_matrix(matrix_from_cols(axis_0, axis_1, cross(axis_0, axis_1)));
    quat q_pc = quat_inverse(q_off) * quat_inverse(q_p) * q_c * q_off;
    vec3 angles = quat_decompose(q_pc);
    vec3 local_0 = quat_rotate(q_off, vec3(1.f, 0.f, 0.f)), local_1 = quat_rotate(q_off, vec3(0.f, 1.f, 0.f)),
         local_2 = quat_rotate(q_off, vec3(0.f, 0.f, 1.f));
    vec3 a0 = local_0;
    quat q_0 = quat_from_axis_angle(a0, angles.x);
    vec3 a1 = quat_rotate(q_0, local_1);
    quat q_1 = quat_from_axis_angle(a1, angles.y);
    vec3 a2 = quat_rotate(q_1 * q_0, local_2);
    vec3 w_err_p = quat_rotate_inv(q_p, w_err);
    vec3 c12 = cross(a1, a2), c02 = cross(a0, a2);
    angles2[0] = angles.x;
    angles2[1] = angles.y;
    vel2[0] = dot(w_err_p, c12) / dot(a0, c12);
    vel2[1] = dot(w_err_p, c02) / dot(a1, c02);
}
inline void invert_3d_rotational_dofs(vec3 axis_0, vec3 axis_1, vec3 axis_2, quat q_p, quat q_c, vec3 w_err, float* angles3, float* vel3) {
    vec3 axis_2_rh = cross(axis_0, axis_1);
    float s = 1.0f;
    if (dot(axis_2_rh, axis_2) < 0.0f) s = -1.0f;  // left-handed user triple: third angle / rate change sign
    quat q_off = quat_from_matrix(matrix_from_cols(axis_0, axis_1, axis_2_rh));
    quat q_pc = quat_inverse(q_off) * quat_inverse(q_p) * q_c * q_off;
    vec3 angles = quat_decompose(q_pc);
    vec3 local_0 = quat_rotate(q_off, vec3(1.f, 0.f, 0.f)), local_1 = quat_rotate(q_off, vec3(0.f, 1.f, 0.f)),
         local_2 = quat_rotate(q_off, vec3(0.f, 0.f, 1.f));
    vec3 a0 = local_0;
    quat q_0 = quat_from_axis_angle(a0, angles.x);
    vec3 a1 = quat_rotate(q_0, local_1);
    quat q_1 = quat_from_axis_angle(a1, angles.y);
    vec3 a2 = quat_rotate(q_1 * q_0, local_2);
    vec3 w_err_p = quat_rotate_inv(q_p, w_err);
    vec3 c12 = cross(a1, a2), c02 = cross(a0, a2), c01 = cross(a0, a1);
    angles3[0] = angles.x;
    angles3[1] = angles.y;
    angles3[2] = s * angles.z;
    vel3[0] = dot(w_err_p, c12) / dot(a0, c12);
    vel3[1] = dot(w_err_p, c02) / dot(a1, c02);
    vel3[2] = s * (dot(w_err_p, c01) / dot(a2, c01));
}

// ---- public newton.eval_ik (sim/articulation.py:640-932 eval_articulation_ik; one joint per thread, no mask) ---------------
inline int eval_articulation_ik(const nb2_model_desc& m, const float* body_q, const float* body_qd, float* joint_q, float* joint_qd) {
    int unsupported = 0;
    for (int a = 0; a < m.articulation_count; ++a)
        for (int j = m.articulation_start[a]; j < m.articulation_start[a + 1]; ++j) {
            const int parent = m.joint_parent[j], child = m.joint_child[j], type = m.joint_type[j];
            transform X_pj = transform::load(m.joint_X_p + 7 * j), X_cj = transform::load(m.joint_X_c + 7 * j);
            vec3 w_p, v_p;
            spatial v_wp;
            transform X_wpj = X_pj, X_wp;
            if (parent >= 0) {
                X_wp = transform::load(body_q + 7 * parent);
                X_wpj = X_wp * X_pj;
                v_wp = spatial::load(body_qd + 6 * parent);
                w_p = v_wp.bot;
                v_p = velocity_at_point(v_wp, X_wpj.p - transform_point(X_wp, load3(m.body_com + 3 * parent)));
            }
            transform X_wc = transform::load(body_q + 7 * child);
            transform X_wcj = X_wc * X_cj;
            spatial v_wc = spatial::load(body_qd + 6 * child);
            vec3 w_c = v_wc.bot;
            vec3 v_c = velocity_at_point(v_wc, X_wcj.p - transform_point(X_wc, load3(m.body_com + 3 * child)));
            vec3 x_err = X_wcj.p - X_wpj.p, v_err = v_c - v_p, w_err = w_c - w_p;
            quat q_p = X_wpj.q, q_c = X_wcj.q;
            int q_start = m.joint_q_start[j], qd_start = m.joint_qd_start[j];
            int lin = m.joint_dof_dim[2 * j], ang = m.joint_dof_dim[2 * j + 1];
            auto axis = [&](int k) { return load3(m.joint_axis + 3 * k); };
            if (type == JT_PRISMATIC) {
                vec3 axis_p = quat_rotate(q_p, axis(qd_start));
                joint_q[q_start] = dot(x_err, axis_p);
                joint_qd[qd_start] = dot(v_err, axis_p);
            } else if (type == JT_REVOLUTE) {
                quat q_pc = quat_inverse(q_p) * q_c;
                vec3 ax = axis(qd_start);
                joint_q[q_start] = quat_twist_angle_signed(ax, q_pc);
                joint_qd[qd_start] = dot(w_err, transform_vector(X_wpj, ax));
            } else if (type == JT_BALL) {
                quat q_pc = quat_inverse(q_p) * q_c;
                joint_q[q_start] = q_pc.x; joint_q[q_start + 1] = q_pc.y; joint_q[q_start + 2] = q_pc.z; joint_q[q_start + 3] = q_pc.w;
                vec3 ang_vel = transform_vector(transform_inverse(X_wpj), w_err);
                joint_qd[qd_start] = ang_vel.x; joint_qd[qd_start + 1] = ang_vel.y; joint_qd[qd_start + 2] = ang_vel.z;
            } else if (type == JT_FREE || type == JT_DISTANCE) {
                quat q_pc = quat_inverse(q_p) * q_c;
                vec3 x_err_c = quat_rotate_inv(q_p, x_err);
                vec3 x_child_com_world = transform_point(X_wc, load3(m.body_com + 3 * child));
                vec3 v_com_err = v_wc.top;
                if (parent >= 0)
                    v_com_err = v_com_err - velocity_at_point(v_wp, x_child_com_world - transform_point(X_wp, load3(m.body_com + 3 * parent)));
                vec3 v_err_c = quat_rotate_inv(q_p, v_com_err), w_err_c = quat_rotate_inv(q_p, w_err);
                joint_q[q_start] = x_err_c.x; joint_q[q_start + 1] = x_err_c.y; joint_q[q_start + 2] = x_err_c.z;
                joint_q[q_start + 3] = q_pc.x; joint_q[q_start + 4] = q_pc.y; joint_q[q_start + 5] = q_pc.z; joint_q[q_start + 6] = q_pc.w;
                joint_qd[qd_start] = v_err_c.x; joint_qd[qd_start + 1] = v_err_c.y; joint_qd[qd_start + 2] = v_err_c.z;
                joint_qd[qd_start + 3] = w_err_c.x; joint_qd[qd_start + 4] = w_err_c.y; joint_qd[qd_start + 5] = w_err_c.z;
            } else if (type == JT_D6) {
                vec3 x_err_c = quat_rotate_inv(q_p, x_err), v_err_c = quat_rotate_inv(q_p, v_err);
                for (int k = 0; k < 3; ++k)
                    if (lin > k) {
                        joint_q[q_start + k] = dot(x_err_c, axis(qd_start + k));
                        joint_qd[qd_start + k] = dot(v_err_c, axis(qd_start + k));
                    }
                if (ang == 1) {
                    quat q_pc = quat_inverse(q_p) * q_c;
                    vec3 ax = axis(qd_start + lin);
                    joint_q[q_start + lin] = quat_twist_angle_signed(ax, q_pc);
                    joint_qd[qd_start + lin] = dot(w_err, transform_vector(X_wpj, ax));
                }
                if (ang == 2)
                    invert_2d_rotational_dofs(axis(qd_start + lin), axis(qd_start + lin + 1), q_p, q_c, w_err, joint_q + q_start + lin,
                                              joint_qd + qd_start + lin);
                if (ang == 3)
                    invert_3d_rotational_dofs(axis(qd_start + lin), axis(qd_start + lin + 1), axis(qd_start + lin + 2), q_p, q_c, w_err,
                                              joint_q + q_start + lin, joint_qd + qd_start + lin);
            }
        }
    return unsupported;
}

}  // namespace orc

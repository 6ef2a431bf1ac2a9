// oracle_dynamics.h - TEST INFRASTRUCTURE ONLY.
// CPU restatement of the reference's articulation dynamics queries, one function per reference function, run serially in
// articulation order exactly as the reference's one-thread-per-articulation / per-body / per-joint kernels execute them:
//   newton.eval_jacobian                  sim/articulation.py:934-1248
//   newton.eval_mass_matrix               sim/articulation.py:1251-1376, 1593-1690
//   newton.eval_inverse_dynamics_passive  sim/inverse_dynamics.py:18-485 (+ featherstone/kernels.py:21-40, 925-975, 1092-1418)
//   newton.eval_inverse_dynamics_force    sim/articulation.py:1379-1590
// The Warp built-ins and the Featherstone helpers (jcalc_motion, transform_spatial_inertia, joint_force,
// transform_2d/3d_rotational_axes) are the ones oracle_featherstone.h already pins.  `art_end` is Model.articulation_end.
#pragma once
#include <algorithm>
#include <vector>

#include "oracle_featherstone.h"

namespace orc {

// write_free_distance_motion_subspace (sim/articulation.py:934-969)
inline void write_free_distance_motion_subspace(const transform& X_pa_world, vec3 x_child_com_world, int qd_start, float* joint_S_s) {
    vec3 ax = transform_vector(X_pa_world, vec3(1.f, 0.f, 0.f));
    vec3 ay = transform_vector(X_pa_world, vec3(0.f, 1.f, 0.f));
    vec3 az = transform_vector(X_pa_world, vec3(0.f, 0.f, 1.f));
    sv6(ax, vec3()).store(joint_S_s + 6 * (qd_start + 0));
    sv6(ay, vec3()).store(joint_S_s + 6 * (qd_start + 1));
    sv6(az, vec3()).store(joint_S_s + 6 * (qd_start + 2));
    sv6(-cross(ax, x_child_com_world), ax).store(joint_S_s + 6 * (qd_start + 3));
    sv6(-cross(ay, x_child_com_world), ay).store(joint_S_s + 6 * (qd_start + 4));
    sv6(-cross(az, x_child_com_world), az).store(joint_S_s + 6 * (qd_start + 5));
}

// jcalc_motion_subspace (:972-1069); ROD writes nothing
inline void jcalc_motion_subspace(const nb2_model_desc& m, int type, const float* joint_q, int lin, int ang, const transform& X_pa_world,
                                  const transform& X_wc, vec3 body_com_child, int q_start, int qd_start, float* joint_S_s) {
    auto axis = [&](int i) { return load3(m.joint_axis + 3 * i); };
    auto put = [&](int dof, const sv6& S) { S.store(joint_S_s + 6 * dof); };
    if (type == JT_PRISMATIC) {
        put(qd_start, transform_twist(X_pa_world, sv6(axis(qd_start), vec3())));
    } else if (type == JT_REVOLUTE) {
        put(qd_start, transform_twist(X_pa_world, sv6(vec3(), axis(qd_start))));
    } else if (type == JT_D6) {
        for (int k = 0; k < 3; ++k)
            if (lin > k) put(qd_start + k, transform_twist(X_pa_world, sv6(axis(qd_start + k), vec3())));
        int iqd = qd_start + lin, iq = q_start + lin;
        if (ang == 1) put(iqd, transform_twist(X_pa_world, sv6(vec3(), axis(iqd))));
        if (ang == 2) {
            vec3 a0, a1;
            transform_2d_rotational_axes(axis(iqd), axis(iqd + 1), joint_q[iq], a0, a1);
            put(iqd, transform_twist(X_pa_world, sv6(vec3(), a0)));
            put(iqd + 1, transform_twist(X_pa_world, sv6(vec3(), a1)));
        }
        if (ang == 3) {
            vec3 a0, a1, a2;
            transform_3d_rotational_axes(axis(iqd), axis(iqd + 1), axis(iqd + 2), joint_q[iq], joint_q[iq + 1], a0, a1, a2);
            put(iqd, transform_twist(X_pa_world, sv6(vec3(), a0)));
            put(iqd + 1, transform_twist(X_pa_world, sv6(vec3(), a1)));
            put(iqd + 2, transform_twist(X_pa_world, sv6(vec3(), a2)));
        }
    } else if (type == JT_BALL) {
        put(qd_start, transform_twist(X_pa_world, sv6(vec3(), vec3(1.f, 0.f, 0.f))));
        put(qd_start + 1, transform_twist(X_pa_world, sv6(vec3(), vec3(0.f, 1.f, 0.f))));
        put(qd_start + 2, transform_twist(X_pa_world, sv6(vec3(), vec3(0.f, 0.f, 1.f))));
    } else if (type == JT_FREE || type == JT_DISTANCE) {
        write_free_distance_motion_subspace(X_pa_world, transform_point(X_wc, body_com_child), qd_start, joint_S_s);
    }
}

// eval_articulation_jacobian (:1072-1168) after the J.zero_() of eval_jacobian (:1213); joint_S_s starts zero (:1217)
inline void eval_jacobian(const nb2_model_desc& m, const int* art_end, const uint8_t* mask, const float* joint_q, const float* body_q,
                          float* J, int max_links, int max_dofs) {
    const int A = m.articulation_count, rows = 6 * max_links;
    std::fill(J, J + size_t(A) * rows * max_dofs, 0.0f);
    std::vector<float> joint_S_s(size_t(m.joint_dof_count) * 6, 0.0f);
    for (int a = 0; a < A; ++a) {
        if (mask && !mask[a]) continue;
        const int js = m.articulation_start[a], je = art_end[a], nj = je - js, ad0 = m.joint_qd_start[js];
        for (int i = 0; i < nj; ++i) {
            int j = js + i, parent = m.joint_parent[j];
            transform X_wpj = transform::load(m.joint_X_p + 7 * j);
            if (parent >= 0) X_wpj = transform::load(body_q + 7 * parent) * X_wpj;
            int child = m.joint_child[j];
            jcalc_motion_subspace(m, m.joint_type[j], joint_q, m.joint_dof_dim[2 * j], m.joint_dof_dim[2 * j + 1], X_wpj,
                                  transform::load(body_q + 7 * child), load3(m.body_com + 3 * child), m.joint_q_start[j],
                                  m.joint_qd_start[j], joint_S_s.data());
        }
        for (int i = 0; i < nj; ++i) {
            int j = js + i, child = m.joint_child[j];
            vec3 x_com_world = transform_point(transform::load(body_q + 7 * child), load3(m.body_com + 3 * child));
            while (j != -1) {
                int d0 = m.joint_qd_start[j], dc = m.joint_qd_start[j + 1] - d0;
                for (int dof = 0; dof < dc; ++dof) {
                    int col = (d0 - ad0) + dof;
                    sv6 S = sv6::load(joint_S_s.data() + 6 * (d0 + dof));
                    sv6 S_com(cross(S.bot(), x_com_world) + S.top(), S.bot());  // velocity_at_point
                    for (int k = 0; k < 6; ++k) J[(size_t(a) * rows + i * 6 + k) * max_dofs + col] = S_com.v[k];
                }
                j = m.joint_ancestor[j];
            }
        }
    }
}

// compute_body_spatial_inertia (:1283-1315)
inline void compute_body_spatial_inertia(const nb2_model_desc& m, const float* body_q, std::vector<mat66>& body_I_s) {
    body_I_s.assign(size_t(m.body_count), mat66());
    for (int b = 0; b < m.body_count; ++b) {
        quat q = transform::load(body_q + 7 * b).q;
        mat33 R = matrix_from_cols(quat_rotate(q, vec3(1.f, 0.f, 0.f)), quat_rotate(q, vec3(0.f, 1.f, 0.f)), quat_rotate(q, vec3(0.f, 0.f, 1.f)));
        const float* Il = m.body_inertia + 9 * b;
        mat33 I_local(Il[0], Il[1], Il[2], Il[3], Il[4], Il[5], Il[6], Il[7], Il[8]);
        mat33 I_world = (R * I_local) * transpose(R);
        float mass = m.body_mass[b];
        mat66& I = body_I_s[b];
        I.m[0][0] = I.m[1][1] = I.m[2][2] = mass;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) I.m[3 + r][3 + c] = I_world.m[r][c];
    }
}

// eval_articulation_mass_matrix (:1318-1376): every (k, l) term, zeros included, as the reference sums them
inline void eval_articulation_mass_matrix(const nb2_model_desc& m, const int* art_end, const uint8_t* mask, const std::vector<mat66>& body_I_s,
                                          const float* J, float* H, int max_links, int max_dofs) {
    const int rows = 6 * max_links;
    for (int a = 0; a < m.articulation_count; ++a) {
        if (mask && !mask[a]) continue;
        const int js = m.articulation_start[a], je = art_end[a];
        const int nd = m.joint_qd_start[je] - m.joint_qd_start[js];
        const float* Ja = J + size_t(a) * rows * max_dofs;
        float* Ha = H + size_t(a) * max_dofs * max_dofs;
        for (int link = 0; link < je - js; ++link) {
            const mat66& I_s = body_I_s[m.joint_child[js + link]];
            const int r0 = link * 6;
            for (int di = 0; di < nd; ++di)
                for (int dj = 0; dj < nd; ++dj) {
                    float sum_val = 0.0f;
                    for (int k = 0; k < 6; ++k)
                        for (int l = 0; l < 6; ++l) {
                            float J_ik = Ja[(r0 + k) * max_dofs + di], J_jl = Ja[(r0 + l) * max_dofs + dj];
                            sum_val += J_ik * I_s.m[k][l] * J_jl;
                        }
                    Ha[di * max_dofs + dj] = Ha[di * max_dofs + dj] + sum_val;
                }
        }
    }
}

// newton.eval_mass_matrix (:1593-1690); J == nullptr: the Jacobian is computed first (with the mask)
inline void eval_mass_matrix(const nb2_model_desc& m, const int* art_end, const uint8_t* mask, const float* joint_q, const float* body_q,
                             const float* J, float* H, int max_links, int max_dofs) {
    std::fill(H, H + size_t(m.articulation_count) * max_dofs * max_dofs, 0.0f);
    std::vector<mat66> body_I_s;
    compute_body_spatial_inertia(m, body_q, body_I_s);
    std::vector<float> Jown;
    if (!J) {
        Jown.assign(size_t(m.articulation_count) * 6 * max_links * max_dofs, 0.0f);
        eval_jacobian(m, art_end, mask, joint_q, body_q, Jown.data(), max_links, max_dofs);
        J = Jown.data();
    }
    eval_articulation_mass_matrix(m, art_end, mask, body_I_s, J, H, max_links, max_dofs);
}

// _rnea_compensation_pass (sim/inverse_dynamics.py:113-308).  joint_qd_public: the pass's joint_qd (zeros for g), gravity: the
// pass's gravity array (model.gravity for g, zeros for C qd).
inline void rnea_compensation_pass(const nb2_model_desc& m, const int* art_end, const uint8_t* mask, const float* body_q, const float* joint_q,
                                   const float* joint_qd_public, const float* gravity, float* tau_out) {
    const int B = m.body_count, Jn = m.joint_count, A = m.articulation_count;
    std::vector<float> body_ft_s(size_t(B) * 6, 0.0f), body_q_com(size_t(B) * 7, 0.0f), joint_qd_internal(size_t(m.joint_dof_count), 0.0f);
    std::vector<float> body_solve_origin(size_t(B) * 3, 0.0f), joint_S_s(size_t(m.joint_dof_count) * 6, 0.0f);
    std::vector<float> body_v_s(size_t(B) * 6, 0.0f), body_a_s(size_t(B) * 6, 0.0f), body_f_s(size_t(B) * 6, 0.0f);
    std::fill(tau_out, tau_out + m.joint_dof_count, 0.0f);
    // compute_spatial_inertia (featherstone/kernels.py:21-40)
    std::vector<mat66> body_I_m{size_t(B)};
    for (int b = 0; b < B; ++b) {
        float mass = m.body_mass[b];
        body_I_m[b].m[0][0] = body_I_m[b].m[1][1] = body_I_m[b].m[2][2] = mass;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) body_I_m[b].m[3 + r][3 + c] = m.body_inertia[9 * b + 3 * r + c];
    }
    // _compute_body_q_com_kernel (inverse_dynamics.py:18-28)
    for (int b = 0; b < B; ++b)
        (transform::load(body_q + 7 * b) * transform(load3(m.body_com + 3 * b), quat_identity())).store(body_q_com.data() + 7 * b);
    // convert_free_distance_joint_qd_public_to_internal (featherstone/kernels.py:924-975)
    for (int j = 0; j < Jn; ++j) {
        int qd0 = m.joint_qd_start[j], qd1 = m.joint_qd_start[j + 1], t = m.joint_type[j];
        if (t != JT_FREE && t != JT_DISTANCE) {
            for (int i = qd0; i < qd1; ++i) joint_qd_internal[i] = joint_qd_public[i];
            continue;
        }
        int parent = m.joint_parent[j], child = m.joint_child[j];
        transform X_wpj = transform::load(m.joint_X_p + 7 * j);
        if (parent >= 0) X_wpj = transform::load(body_q + 7 * parent) * X_wpj;
        vec3 x_child_com = transform_point(transform::load(body_q + 7 * child), load3(m.body_com + 3 * child));
        vec3 r = quat_rotate_inv(X_wpj.q, x_child_com - X_wpj.p);
        vec3 v_com(joint_qd_public[qd0], joint_qd_public[qd0 + 1], joint_qd_public[qd0 + 2]);
        vec3 omega(joint_qd_public[qd0 + 3], joint_qd_public[qd0 + 4], joint_qd_public[qd0 + 5]);
        vec3 v_int = v_com - cross(omega, r);
        joint_qd_internal[qd0] = v_int.x; joint_qd_internal[qd0 + 1] = v_int.y; joint_qd_internal[qd0 + 2] = v_int.z;
        joint_qd_internal[qd0 + 3] = omega.x; joint_qd_internal[qd0 + 4] = omega.y; joint_qd_internal[qd0 + 5] = omega.z;
    }
    // eval_rigid_id (:1241-1317, compute_link_velocity :764-865) with the mask
    std::vector<mat66> body_I_s{size_t(B)};
    for (int a = 0; a < A; ++a) {
        if (mask && !mask[a]) continue;
        int start = m.articulation_start[a], end = art_end[a];
        vec3 solve_origin;
        if (start < end) {
            int rt = m.joint_type[start];
            if (rt == JT_FREE || rt == JT_DISTANCE) solve_origin = load3(body_q_com.data() + 7 * m.joint_child[start]);
        }
        for (int i = start; i < end; ++i) {
            int type = m.joint_type[i], child = m.joint_child[i], parent = m.joint_parent[i];
            transform X_wpj = transform::load(m.joint_X_p + 7 * i);
            if (parent >= 0) X_wpj = transform::load(body_q + 7 * parent) * X_wpj;
            transform X_wpj_s(X_wpj.p - solve_origin, X_wpj.q);
            sv6 v_j_s, c_app_s;
            jcalc_motion(m, type, joint_q, m.joint_dof_dim[2 * i], m.joint_dof_dim[2 * i + 1], X_wpj_s, joint_qd_internal.data(),
                         m.joint_q_start[i], m.joint_qd_start[i], joint_S_s.data(), v_j_s, c_app_s);
            sv6 v_parent_s, a_parent_s;
            if (parent >= 0) {
                v_parent_s = sv6::load(body_v_s.data() + 6 * parent);
                a_parent_s = sv6::load(body_a_s.data() + 6 * parent);
            }
            sv6 v_s = v_parent_s + v_j_s;
            sv6 a_s = a_parent_s + spatial_cross(v_s, v_j_s) + c_app_s;
            transform X_sm = transform::load(body_q_com.data() + 7 * child);
            vec3 x_com_s = X_sm.p - solve_origin;
            store3(body_solve_origin.data() + 3 * child, solve_origin);
            float mass = m.body_mass[child];
            int world_idx = m.body_world[child];
            if (world_idx < 0) world_idx += m.gravity_count;
            vec3 f_g = mass * load3(gravity + 3 * world_idx);
            sv6 f_g_s(f_g, cross(x_com_s, f_g));
            body_I_s[child] = transform_spatial_inertia(transform(x_com_s, X_sm.q), body_I_m[child]);
            sv6 f_b_s = mul66v(body_I_s[child], a_s) + spatial_cross_dual(v_s, mul66v(body_I_s[child], v_s));
            v_s.store(body_v_s.data() + 6 * child);
            a_s.store(body_a_s.data() + 6 * child);
            (f_b_s - f_g_s).store(body_f_s.data() + 6 * child);
        }
    }
    // eval_rigid_tau (:1320-1418) + jcalc_tau (:383-461) with every gain, target, limit gain, damping, joint_f and body_f_ext zero.
    // With body_f_ext = 0 the external wrench is f_ext = -(0, 0 + x_com_s x 0) = (-0, ..., -0), and x + (-0) == x for every x, so
    // f_s = f_b_s + f_t_s bit for bit.
    for (int a = 0; a < A; ++a) {
        if (mask && !mask[a]) continue;
        int start = m.articulation_start[a], end = art_end[a];
        for (int i = end - 1; i >= start; --i) {
            int type = m.joint_type[i], parent = m.joint_parent[i], child = m.joint_child[i];
            int dof_start = m.joint_qd_start[i], coord_start = m.joint_q_start[i];
            int lin = m.joint_dof_dim[2 * i], ang = m.joint_dof_dim[2 * i + 1];
            sv6 f_s = sv6::load(body_f_s.data() + 6 * child) + sv6::load(body_ft_s.data() + 6 * child);
            const float* S = joint_S_s.data();
            const float* jqd = joint_qd_internal.data();
            if (type == JT_BALL) {
                for (int k = 0; k < 3; ++k) {
                    int j = dof_start + k;
                    float passive_f = -0.0f * jqd[j];  // -joint_damping * qd
                    tau_out[j] = -dot6(sv6::load(S + 6 * j), f_s) + 0.0f + passive_f;
                }
            } else if (type == JT_FREE || type == JT_DISTANCE) {
                for (int k = 0; k < 6; ++k) tau_out[dof_start + k] = -dot6(sv6::load(S + 6 * (dof_start + k)), f_s) + 0.0f;
            } else if (type == JT_PRISMATIC || type == JT_REVOLUTE || type == JT_D6) {
                for (int k = 0; k < lin + ang; ++k) {
                    int j = dof_start + k;
                    float drive_f = joint_force(joint_q[coord_start + k], jqd[j], 0.f, 0.f, 0.f, 0.f, m.joint_limit_lower[j], m.joint_limit_upper[j],
                                                0.f, 0.f, 0.f);
                    tau_out[j] = -dot6(sv6::load(S + 6 * j), f_s) + drive_f + 0.0f;
                }
            }
            if (parent >= 0) (sv6::load(body_ft_s.data() + 6 * parent) + f_s).store(body_ft_s.data() + 6 * parent);
        }
    }
    // convert_free_distance_joint_f_internal_to_public (featherstone/kernels.py:1092-1237).  With a mask, joints outside every
    // articulation (joint_articulation == -1; the reference would index the mask with -1) keep the 0 of tau_out.zero_().
    for (int j = 0; j < Jn; ++j) {
        if (mask) {
            int ja = m.joint_articulation[j];
            if (ja < 0 || !mask[ja]) continue;
        }
        int qd0 = m.joint_qd_start[j], qd1 = m.joint_qd_start[j + 1], t = m.joint_type[j];
        float* f = tau_out;
        if (t == JT_FREE || t == JT_DISTANCE) {
            int parent = m.joint_parent[j], child = m.joint_child[j];
            transform X_wpj = transform::load(m.joint_X_p + 7 * j);
            if (parent >= 0) X_wpj = transform::load(body_q + 7 * parent) * X_wpj;
            quat q_p = X_wpj.q;
            vec3 r = quat_rotate_inv(q_p, load3(body_q_com.data() + 7 * child) - X_wpj.p);
            vec3 v(joint_qd_public[qd0], joint_qd_public[qd0 + 1], joint_qd_public[qd0 + 2]);
            vec3 w(joint_qd_public[qd0 + 3], joint_qd_public[qd0 + 4], joint_qd_public[qd0 + 5]);
            float mass = m.body_mass[child];
            vec3 bc = mass * cross(w, v);
            f[qd0] = f[qd0] + bc.x; f[qd0 + 1] = f[qd0 + 1] + bc.y; f[qd0 + 2] = f[qd0 + 2] + bc.z;
            vec3 shift = cross(r, vec3(f[qd0], f[qd0 + 1], f[qd0 + 2]));
            f[qd0 + 3] = f[qd0 + 3] - shift.x; f[qd0 + 4] = f[qd0 + 4] - shift.y; f[qd0 + 5] = f[qd0 + 5] - shift.z;
            vec3 ac = mass * cross(r, cross(w, v));
            f[qd0 + 3] = f[qd0 + 3] + ac.x; f[qd0 + 4] = f[qd0 + 4] + ac.y; f[qd0 + 5] = f[qd0 + 5] + ac.z;
            vec3 fl = quat_rotate(q_p, vec3(f[qd0], f[qd0 + 1], f[qd0 + 2]));
            vec3 fa = quat_rotate(q_p, vec3(f[qd0 + 3], f[qd0 + 4], f[qd0 + 5]));
            f[qd0] = fl.x; f[qd0 + 1] = fl.y; f[qd0 + 2] = fl.z; f[qd0 + 3] = fa.x; f[qd0 + 4] = fa.y; f[qd0 + 5] = fa.z;
        }
        for (int i = qd0; i < qd1; ++i) f[i] = -f[i];
    }
}

// newton.eval_inverse_dynamics_passive (sim/inverse_dynamics.py:364-485)
inline void eval_inverse_dynamics_passive(const nb2_model_desc& m, const int* art_end, const uint8_t* mask, const float* body_q, const float* joint_q,
                                          const float* joint_qd, float* mass_matrix, float* gravity_force, float* coriolis_force, int max_links,
                                          int max_dofs) {
    if (mass_matrix) eval_mass_matrix(m, art_end, mask, joint_q, body_q, nullptr, mass_matrix, max_links, max_dofs);
    std::vector<float> zeros_dof(size_t(m.joint_dof_count), 0.0f), zero_gravity(size_t(m.gravity_count) * 3, 0.0f);
    if (gravity_force) rnea_compensation_pass(m, art_end, mask, body_q, joint_q, zeros_dof.data(), m.gravity, gravity_force);
    if (coriolis_force) rnea_compensation_pass(m, art_end, mask, body_q, joint_q, joint_qd, zero_gravity.data(), coriolis_force);
}

// eval_articulation_inverse_dynamics_force_kernel (sim/articulation.py:1379-1468)
inline void eval_inverse_dynamics_force(const nb2_model_desc& m, const int* art_end, const uint8_t* mask, const float* body_q, const float* mass_matrix,
                                        const float* joint_qdd, const float* coriolis_force, const float* gravity_force, float* tau, int max_dofs) {
    for (int a = 0; a < m.articulation_count; ++a) {
        int js = m.articulation_start[a], je = art_end[a];
        int dof_start = m.joint_qd_start[js], dof_end = m.joint_qd_start[je], dof_count = dof_end - dof_start;
        int gap_end = m.joint_qd_start[m.articulation_start[a + 1]];
        if (mask && !mask[a]) {
            for (int k = dof_start; k < gap_end; ++k) tau[k] = 0.0f;
            continue;
        }
        const float* Ha = mass_matrix + size_t(a) * max_dofs * max_dofs;
        for (int i = 0; i < dof_count; ++i) {
            float sum_val = 0.0f;
            for (int j = 0; j < dof_count; ++j) sum_val += Ha[i * max_dofs + j] * joint_qdd[dof_start + j];
            tau[dof_start + i] = sum_val;
        }
        for (int ji = js; ji < je; ++ji) {
            int jt = m.joint_type[ji];
            if (jt != JT_FREE && jt != JT_DISTANCE) continue;
            int jd = m.joint_qd_start[ji], parent = m.joint_parent[ji];
            transform X_wpj = transform::load(m.joint_X_p + 7 * ji);
            if (parent >= 0) X_wpj = transform::load(body_q + 7 * parent) * X_wpj;
            vec3 fl = quat_rotate(X_wpj.q, vec3(tau[jd], tau[jd + 1], tau[jd + 2]));
            vec3 fa = quat_rotate(X_wpj.q, vec3(tau[jd + 3], tau[jd + 4], tau[jd + 5]));
            tau[jd] = fl.x; tau[jd + 1] = fl.y; tau[jd + 2] = fl.z; tau[jd + 3] = fa.x; tau[jd + 4] = fa.y; tau[jd + 5] = fa.z;
        }
        for (int i = 0; i < dof_count; ++i) tau[dof_start + i] = tau[dof_start + i] + coriolis_force[dof_start + i] + gravity_force[dof_start + i];
        for (int k = dof_end; k < gap_end; ++k) tau[k] = 0.0f;
    }
}

}  // namespace orc

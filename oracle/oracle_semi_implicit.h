// oracle_semi_implicit.h - TEST INFRASTRUCTURE ONLY.
// CPU restatement of the reference SolverSemiImplicit.step for rigid bodies (solvers/semi_implicit/solver_semi_implicit.py:124-217):
// eval_body_joints (kernels_body.py:54-520) run serially in joint order, then eval_body_contact (kernels_contact.py:381-556, the
// existing restatement in oracle_featherstone.h) in contact order, then integrate_bodies (solvers/solver.py:112-170, oracle_xpbd.h).
// Serial execution fixes the order of the reference's float atomics, as on its CPU device.
#pragma once
#include <vector>

#include "../include/newton_b200.h"
#include "oracle_featherstone.h"
#include "oracle_math.h"
#include "oracle_xpbd.h"

namespace orc {
namespace si {

// wp.acos clamps its argument to [-1, 1] (warp/native/builtin.h: acosf(min(max(x, -1), 1))).  The reference relies on it: r_err.w
// of a product of unit quaternions can round above 1.  acos_w (oracle_math.h) does not clamp and keeps its callers' bits.
inline float acos_clamped(float x) { return acos_w(minf(maxf(x, -1.0f), 1.0f)); }

// kernels_body.py:54-520, restated line for line (assignments that overwrite included), for every joint in index order
inline void eval_body_joints(const nb2_model_desc& m, const float* body_q, const float* body_qd, const nb2_control_view& ctl,
                             float joint_attach_ke, float joint_attach_kd, float* body_f) {
    const float* joint_f = ctl.joint_f;
    const float* joint_target_q = ctl.joint_target_q;
    const float* joint_target_qd = ctl.joint_target_qd;
    auto axis = [&](int i) { return load3(m.joint_axis + 3 * i); };
    for (int tid = 0; tid < m.joint_count; ++tid) {
        const int type = m.joint_type[tid];
        const int c_child = m.joint_child[tid];
        const int c_parent = m.joint_parent[tid];
        if (!m.joint_enabled[tid]) continue;
        const int qd_start = m.joint_qd_start[tid];
        const int target_q_start = m.joint_target_q_start[tid];
        if (type == JT_FREE || type == JT_DISTANCE) {
            spatial wrench(vec3(joint_f[qd_start + 0], joint_f[qd_start + 1], joint_f[qd_start + 2]),
                           vec3(joint_f[qd_start + 3], joint_f[qd_start + 4], joint_f[qd_start + 5]));
            atomic_add(body_f, c_child, wrench);
            continue;
        }
        const transform X_pj = transform::load(m.joint_X_p + 7 * tid);
        const transform X_cj = transform::load(m.joint_X_c + 7 * tid);
        transform X_wp = X_pj;
        vec3 r_p, w_p, v_p;
        if (c_parent >= 0) {
            X_wp = transform::load(body_q + 7 * c_parent) * X_wp;
            r_p = X_wp.p - transform_point(transform::load(body_q + 7 * c_parent), load3(m.body_com + 3 * c_parent));
            spatial twist_p = spatial::load(body_qd + 6 * c_parent);
            w_p = twist_p.bot;
            v_p = twist_p.top + cross(w_p, r_p);
        }
        const transform X_wc = transform::load(body_q + 7 * c_child) * X_cj;
        const vec3 r_c = X_wc.p - transform_point(transform::load(body_q + 7 * c_child), load3(m.body_com + 3 * c_child));
        spatial twist_c = spatial::load(body_qd + 6 * c_child);
        const vec3 w_c = twist_c.bot;
        const vec3 v_c = twist_c.top + cross(w_c, r_c);
        const int lin_axis_count = m.joint_dof_dim[2 * tid + 0];
        const int ang_axis_count = m.joint_dof_dim[2 * tid + 1];
        const vec3 x_p = X_wp.p, x_c = X_wc.p;
        const quat q_p = X_wp.q, q_c = X_wc.q;
        const vec3 x_err = x_c - x_p;
        const quat r_err = quat_inverse(q_p) * q_c;
        const vec3 v_err = v_c - v_p;
        const vec3 w_err = w_c - w_p;
        vec3 t_total, f_total;
        const float angular_damping_scale = 0.01f;
        auto jforce = [&](float q, float qd, int iq, int i) {
            return joint_force(q, qd, joint_target_q[iq], joint_target_qd[i], m.joint_target_ke[i], m.joint_target_kd[i],
                               m.joint_limit_lower[i], m.joint_limit_upper[i], m.joint_limit_ke[i], m.joint_limit_kd[i], m.joint_damping[i]);
        };
        if (type == JT_FIXED) {
            vec3 ang_err = normalize(vec3(r_err.x, r_err.y, r_err.z)) * acos_clamped(r_err.w) * 2.0f;
            f_total += x_err * joint_attach_ke + v_err * joint_attach_kd;
            t_total += transform_vector(X_wp, ang_err) * joint_attach_ke + w_err * joint_attach_kd * angular_damping_scale;
        }
        if (type == JT_PRISMATIC) {
            vec3 ax = axis(qd_start);
            vec3 axis_p = transform_vector(X_wp, ax);
            float q = dot(x_err, axis_p);
            float qd = dot(v_err, axis_p);
            f_total = axis_p * (-joint_f[qd_start] - jforce(q, qd, target_q_start, qd_start));
            vec3 ang_err = normalize(vec3(r_err.x, r_err.y, r_err.z)) * acos_clamped(r_err.w) * 2.0f;
            f_total += (x_err - q * axis_p) * joint_attach_ke + (v_err - qd * axis_p) * joint_attach_kd;
            t_total += transform_vector(X_wp, ang_err) * joint_attach_ke + w_err * joint_attach_kd * angular_damping_scale;
        }
        if (type == JT_REVOLUTE) {
            vec3 ax = axis(qd_start);
            vec3 axis_p = transform_vector(X_wp, ax);
            vec3 axis_c = transform_vector(X_wc, ax);
            float q = quat_twist_angle_signed(ax, r_err);
            float qd = dot(w_err, axis_p);
            t_total = axis_p * (-joint_f[qd_start] - jforce(q, qd, target_q_start, qd_start));
            vec3 swing_err = cross(axis_p, axis_c);
            f_total += x_err * joint_attach_ke + v_err * joint_attach_kd;
            t_total += swing_err * joint_attach_ke + (w_err - qd * axis_p) * joint_attach_kd * angular_damping_scale;
        }
        if (type == JT_BALL) {  // the reference also forms ang_err here and never uses it
            f_total += x_err * joint_attach_ke + v_err * joint_attach_kd;
            vec3 axis_0 = transform_vector(X_wp, axis(qd_start + 0));
            vec3 axis_1 = transform_vector(X_wp, axis(qd_start + 1));
            vec3 axis_2 = transform_vector(X_wp, axis(qd_start + 2));
            t_total += axis_0 * (-joint_f[qd_start + 0] + m.joint_damping[qd_start + 0] * dot(axis_0, w_err));
            t_total += axis_1 * (-joint_f[qd_start + 1] + m.joint_damping[qd_start + 1] * dot(axis_1, w_err));
            t_total += axis_2 * (-joint_f[qd_start + 2] + m.joint_damping[qd_start + 2] * dot(axis_2, w_err));
        }
        if (type == JT_D6) {
            vec3 pos(0.0f), vel(0.0f);
            if (lin_axis_count >= 1) {
                vec3 axis_0 = transform_vector(X_wp, axis(qd_start + 0));
                float q0 = dot(x_err, axis_0), qd0 = dot(v_err, axis_0);
                f_total += axis_0 * (-joint_f[qd_start] - jforce(q0, qd0, target_q_start + 0, qd_start + 0));
                pos += q0 * axis_0;
                vel += qd0 * axis_0;
            }
            if (lin_axis_count >= 2) {
                vec3 axis_1 = transform_vector(X_wp, axis(qd_start + 1));
                float q1 = dot(x_err, axis_1), qd1 = dot(v_err, axis_1);
                f_total += axis_1 * (-joint_f[qd_start + 1] - jforce(q1, qd1, target_q_start + 1, qd_start + 1));
                pos += q1 * axis_1;
                vel += qd1 * axis_1;
            }
            if (lin_axis_count == 3) {
                vec3 axis_2 = transform_vector(X_wp, axis(qd_start + 2));
                float q2 = dot(x_err, axis_2), qd2 = dot(v_err, axis_2);
                f_total += axis_2 * (-joint_f[qd_start + 2] - jforce(q2, qd2, target_q_start + 2, qd_start + 2));
                pos += q2 * axis_2;
                vel += qd2 * axis_2;
            }
            f_total += (x_err - pos) * joint_attach_ke + (v_err - vel) * joint_attach_kd;
            if (ang_axis_count == 0) {
                vec3 ang_err = normalize(vec3(r_err.x, r_err.y, r_err.z)) * acos_clamped(r_err.w) * 2.0f;
                t_total += transform_vector(X_wp, ang_err) * joint_attach_ke + w_err * joint_attach_kd * angular_damping_scale;
            }
            const int i_0 = lin_axis_count + qd_start + 0, i_1 = lin_axis_count + qd_start + 1, i_2 = lin_axis_count + qd_start + 2;
            const int i_0_q = lin_axis_count + target_q_start + 0, i_1_q = lin_axis_count + target_q_start + 1,
                      i_2_q = lin_axis_count + target_q_start + 2;
            const int qdi_start = qd_start + lin_axis_count;
            if (ang_axis_count == 1) {
                vec3 ax = axis(i_0);
                vec3 axis_p = transform_vector(X_wp, ax);
                vec3 axis_c = transform_vector(X_wc, ax);
                float q = quat_twist_angle_signed(ax, r_err);
                float qd = dot(w_err, axis_p);
                t_total = axis_p * (-joint_f[qdi_start] - jforce(q, qd, i_0_q, i_0));
                vec3 swing_err = cross(axis_p, axis_c);
                t_total += swing_err * joint_attach_ke + (w_err - qd * axis_p) * joint_attach_kd * angular_damping_scale;
            }
            if (ang_axis_count == 2 || ang_axis_count == 3) {
                quat q_pc = quat_inverse(q_p) * q_c;
                vec3 angles = quat_decompose(q_pc);
                vec3 orig_axis_0 = axis(i_0), orig_axis_1 = axis(i_1);
                vec3 orig_axis_2 = ang_axis_count == 2 ? cross(orig_axis_0, orig_axis_1) : axis(i_2);
                vec3 axis_0 = orig_axis_0;
                quat q_0 = quat_from_axis_angle(axis_0, angles[0]);
                vec3 axis_1 = quat_rotate(q_0, orig_axis_1);
                quat q_1 = quat_from_axis_angle(axis_1, angles[1]);
                vec3 axis_2 = quat_rotate(q_1 * q_0, orig_axis_2);
                axis_0 = transform_vector(X_wp, axis_0);
                axis_1 = transform_vector(X_wp, axis_1);
                axis_2 = transform_vector(X_wp, axis_2);
                t_total += axis_0 * (-joint_f[qdi_start] - jforce(angles[0], dot(axis_0, w_err), i_0_q, i_0));
                t_total += axis_1 * (-joint_f[qdi_start + 1] - jforce(angles[1], dot(axis_1, w_err), i_1_q, i_1));
                if (ang_axis_count == 2)  // last axis (fixed): target 0, limits (0, 0), limit gains 0
                    t_total += axis_2 * -joint_force(angles[2], dot(axis_2, w_err), 0.0f, 0.0f, joint_attach_ke,
                                                     joint_attach_kd * angular_damping_scale, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f);
                else
                    t_total += axis_2 * (-joint_f[qdi_start + 2] - jforce(angles[2], dot(axis_2, w_err), i_2_q, i_2));
            }
        }
        // every other type (ROD) reaches here with zero f_total / t_total
        if (c_parent >= 0) atomic_add(body_f, c_parent, spatial(f_total, t_total + cross(r_p, f_total)));
        atomic_sub(body_f, c_child, spatial(f_total, t_total + cross(r_c, f_total)));
    }
}

// SolverSemiImplicit.step, rigid-body part (solver_semi_implicit.py:150-217)
inline void step(const nb2_model_desc& m, const nb2_semi_implicit_params& p, const nb2_state_view& in, const nb2_state_view& out,
                 const nb2_control_view& ctl, const nb2_contacts_view* contacts, float dt) {
    if (m.body_count == 0) return;
    // :166-169: with joints and a joint_f array the forces accumulate into a clone; otherwise into state_in.body_f itself
    std::vector<float> clone;
    float* body_f = in.body_f;
    if (m.joint_count > 0 && ctl.joint_f != nullptr) {
        clone.assign(in.body_f, in.body_f + 6 * size_t(m.body_count));
        body_f = clone.data();
    }
    if (m.joint_count > 0) eval_body_joints(m, in.body_q, in.body_qd, ctl, p.joint_attach_ke, p.joint_attach_kd, body_f);
    if (contacts != nullptr && contacts->rigid_contact_max > 0)
        eval_body_contact(m, in.body_q, in.body_qd, *contacts, p.friction_smoothing, body_f);
    integrate_bodies(m, in.body_q, in.body_qd, body_f, p.angular_damping, dt, out.body_q, out.body_qd);
}

}  // namespace si
}  // namespace orc

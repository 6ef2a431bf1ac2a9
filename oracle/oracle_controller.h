// oracle_controller.h - TEST INFRASTRUCTURE ONLY.  CPU restatement of the reference's joint-impedance step
// (controllers/impl/joint_impedance/): each Warp kernel is a serial loop over (robot, dof), run in the reference's launch order
// with the reference's padded [robot_count, max_dofs] intermediates: the gathers, _pd_term_kernel, _add_term_kernel (qdd),
// _mass_matrix_multiply_kernel, _add_term_kernel (gravity, then Coriolis), _scatter_dof_kernel.  Compiled with
// -ffp-contract=off, so every fp32 operation rounds as written.
#pragma once
#include <cstdint>
#include <vector>

#include "../include/newton_b200.h"

namespace orc {
namespace ji {

// _gather_dof_flat_kernel (model_based.py): the internal state's joint_q / joint_qd, flat over all controlled dofs
inline void gather_state(const nb2_joint_impedance_desc& p) {
    int total = 0;
    for (int r = 0; r < p.robot_count; ++r) total += p.dofs_per_robot[r];
    for (int k = 0; k < total; ++k) {
        p.state_joint_q[k] = p.joint_q[p.joint_q_idx[k]];
        p.state_joint_qd[k] = p.joint_qd[p.joint_qd_idx[k]];
    }
}

// ControllerJointImpedanceModelFree.step (model_free.py) with the caller's mass_matrix / gravity_force / coriolis_force
inline void step(const nb2_joint_impedance_desc& p) {
    const int R = p.robot_count, D = p.max_dofs;
    const size_t RD = size_t(R) * D;
    std::vector<float> q(RD), qd(RD), q_des(RD), qd_des(RD), qdd(RD), grav(RD), cor(RD), tau(RD), acc(RD);
    auto gather = [&](const float* src, const int32_t* idx, std::vector<float>& dst) {  // _gather_dof_kernel
        for (int r = 0; r < R; ++r)
            for (int i = 0; i < p.dofs_per_robot[r]; ++i) dst[size_t(r) * D + i] = src[idx[p.dof_offsets[r] + i]];
    };
    auto add = [&](const std::vector<float>& term, std::vector<float>& out) {  // _add_term_kernel
        for (int r = 0; r < R; ++r)
            for (int i = 0; i < p.dofs_per_robot[r]; ++i) out[size_t(r) * D + i] = out[size_t(r) * D + i] + term[size_t(r) * D + i];
    };
    gather(p.joint_q, p.joint_q_idx, q);
    gather(p.joint_qd, p.joint_qd_idx, qd);
    gather(p.joint_q_des, p.joint_q_des_idx, q_des);
    gather(p.joint_qd_des, p.joint_qd_des_idx, qd_des);
    if (p.has_qdd) gather(p.joint_qdd, p.joint_qdd_idx, qdd);
    if (p.use_gravity) gather(p.gravity_force, p.gravity_force_idx, grav);
    if (p.use_coriolis) gather(p.coriolis_force, p.coriolis_force_idx, cor);
    std::vector<float>& work = p.use_inertia ? acc : tau;
    for (int r = 0; r < R; ++r)  // _pd_term_kernel
        for (int i = 0; i < p.dofs_per_robot[r]; ++i) {
            const size_t k = size_t(r) * D + i;
            work[k] = p.stiffness[k] * (q_des[k] - q[k]) + p.damping[k] * (qd_des[k] - qd[k]);
        }
    if (p.has_qdd) add(qdd, work);
    if (p.use_inertia)  // _mass_matrix_multiply_kernel: M[robot, dof, col], summed from +0 in column order
        for (int r = 0; r < R; ++r)
            for (int i = 0; i < p.dofs_per_robot[r]; ++i) {
                float s = 0.0f;
                for (int c = 0; c < p.dofs_per_robot[r]; ++c) s = s + p.mass_matrix[(size_t(r) * D + i) * D + c] * acc[size_t(r) * D + c];
                tau[size_t(r) * D + i] = s;
            }
    if (p.use_gravity) add(grav, tau);
    if (p.use_coriolis) add(cor, tau);
    for (int r = 0; r < R; ++r)  // _scatter_dof_kernel
        for (int i = 0; i < p.dofs_per_robot[r]; ++i) p.joint_f[p.joint_f_idx[p.dof_offsets[r] + i]] = tau[size_t(r) * D + i];
}

}  // namespace ji
}  // namespace orc

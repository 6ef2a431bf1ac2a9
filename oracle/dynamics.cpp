// dynamics.cpp - TEST INFRASTRUCTURE ONLY.  C exports of oracle_dynamics.h, the CPU checker of newton_b200.eval_jacobian /
// eval_mass_matrix / eval_inverse_dynamics_*.
#include "oracle_dynamics.h"

using namespace orc;

extern "C" {

void orc_eval_jacobian(const nb2_model_desc* m, const int* art_end, const uint8_t* mask, const float* joint_q, const float* body_q, float* J,
                       int max_links, int max_dofs) {
    eval_jacobian(*m, art_end, mask, joint_q, body_q, J, max_links, max_dofs);
}

void orc_eval_mass_matrix(const nb2_model_desc* m, const int* art_end, const uint8_t* mask, const float* joint_q, const float* body_q,
                          const float* J, float* H, int max_links, int max_dofs) {
    eval_mass_matrix(*m, art_end, mask, joint_q, body_q, J, H, max_links, max_dofs);
}

void orc_eval_inverse_dynamics_passive(const nb2_model_desc* m, const int* art_end, const uint8_t* mask, const float* body_q,
                                       const float* joint_q, const float* joint_qd, float* mass_matrix, float* gravity_force,
                                       float* coriolis_force, int max_links, int max_dofs) {
    eval_inverse_dynamics_passive(*m, art_end, mask, body_q, joint_q, joint_qd, mass_matrix, gravity_force, coriolis_force, max_links, max_dofs);
}

void orc_eval_inverse_dynamics_force(const nb2_model_desc* m, const int* art_end, const uint8_t* mask, const float* body_q,
                                     const float* mass_matrix, const float* joint_qdd, const float* coriolis_force, const float* gravity_force,
                                     float* joint_f, int max_dofs) {
    eval_inverse_dynamics_force(*m, art_end, mask, body_q, mass_matrix, joint_qdd, coriolis_force, gravity_force, joint_f, max_dofs);
}
}

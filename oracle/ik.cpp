// ik.cpp - TEST INFRASTRUCTURE ONLY.  C exports of oracle_ik.h, the CPU checker of newton_b200.ik.  The entries take the
// arguments of nb2_ik_solve / nb2_ik_sample / nb2_ik_select without the stream, on host arrays.
#include <cstring>

#include "oracle_ik.h"

using namespace orc;

extern "C" {

void orc_ik_solve(const nb2_ik_desc* d, const float* joint_q_in, float* joint_q, float* joint_q_out, float* residuals, float* costs,
                  float* lambda_values, float* jacobian, int32_t iterations, float step_size, int32_t write_lambda, uint32_t* seed_state) {
    const size_t n = size_t(d->n_batch) * d->model.joint_coord_count;
    std::vector<float> q(joint_q_in, joint_q_in + n);  // the expanded buffer (IKSolver._sample + in-place LM)
    std::vector<float> J(size_t(d->n_batch) * d->n_residuals * d->model.joint_dof_count);
    if (iterations == 0 && jacobian) std::memcpy(J.data(), jacobian, J.size() * sizeof(float));
    IkOracle o(*d);
    o.run(q.data(), residuals, costs, lambda_values, J.data(), iterations, step_size, write_lambda != 0);
    std::memcpy(joint_q, q.data(), n * sizeof(float));
    if (joint_q_out) std::memcpy(joint_q_out, q.data(), n * sizeof(float));
    if (jacobian) std::memcpy(jacobian, J.data(), J.size() * sizeof(float));
    if (seed_state) seed_state[0] += 1u;
}

void orc_ik_sample(int32_t sampler, int32_t n_problems, int32_t n_seeds, int32_t n_coords, const float* joint_q_in, const float* lower,
                   const float* upper, const int32_t* bounded, const float* basis, float noise_std, const uint32_t* seed_state, float* out) {
    ik_sample(sampler, n_problems, n_seeds, n_coords, joint_q_in, lower, upper, bounded, basis, noise_std, seed_state, out);
}

void orc_ik_select(int32_t n_problems, int32_t n_seeds, int32_t n_coords, const float* costs, const float* q, int32_t* best, float* out) {
    ik_select(n_problems, n_seeds, n_coords, costs, q, best, out);
}
}

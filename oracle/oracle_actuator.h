// oracle_actuator.h - TEST INFRASTRUCTURE ONLY.  CPU restatement of the reference's actuator kernels (newton.actuators,
// actuators/), each one a serial loop in thread-id order, run in the reference's launch order with the reference's
// intermediate arrays: _delay_read_kernel, the controller kernel, one kernel per clamp (computed -> applied, then in place),
// _scatter_add_kernel, the PID state copy, _delay_buffer_state_kernel.  Compiled with -ffp-contract=off.  min / max / clamp
// are Warp's: min(a, b) = a < b ? a : b, max(a, b) = a > b ? a : b, clamp(x, lo, hi) = min(max(lo, x), hi).
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "../include/newton_b200.h"

namespace orc {
namespace act {

inline float wmin(float a, float b) { return a < b ? a : b; }
inline float wmax(float a, float b) { return a > b ? a : b; }
inline float wclamp(float x, float lo, float hi) { return wmin(wmax(lo, x), hi); }

// _interp_1d (clamping_position_based.py:15-36)
inline float interp_1d(float x, const float* xs, const float* ys, int n) {
    if (n <= 0) return 0.0f;
    if (x <= xs[0]) return ys[0];
    if (x >= xs[n - 1]) return ys[n - 1];
    for (int k = 0; k < n - 1; ++k) {
        if (xs[k + 1] >= x) {
            float dx = xs[k + 1] - xs[k];
            if (dx == 0.0f) return ys[k];
            float t = (x - xs[k]) / dx;
            return ys[k] + t * (ys[k + 1] - ys[k]);
        }
    }
    return ys[n - 1];
}

inline void step(const nb2_actuator_step_desc& d) {
    const int N = d.count;
    if (N <= 0) return;
    std::vector<int> seq(N);
    for (int i = 0; i < N; ++i) seq[i] = i;
    // the controller's view of its targets: the control arrays with the actuator's indices, or the delay's outputs with
    // sequential indices
    const float* target_pos = d.target_pos;
    const float* target_vel = d.target_vel;
    const float* feedforward = d.feedforward;
    const int* tpos_idx = d.target_pos_indices;
    const int* tvel_idx = d.indices;
    std::vector<float> out_pos(N), out_vel(N), out_act(N);
    const int depth = d.buf_depth;
    if (depth > 0) {  // _delay_read_kernel (delay.py:57-93)
        for (int i = 0; i < N; ++i) {
            int n = d.num_pushes_in[i];
            if (n == 0 || d.delay_steps[i] == 0) {
                out_pos[i] = d.target_pos[d.target_pos_indices[i]];
                out_vel[i] = d.target_vel[d.indices[i]];
                float a = 0.0f;
                if (d.feedforward) a = d.feedforward[d.indices[i]];
                out_act[i] = a;
            } else {
                int write_idx = d.write_idx_in[0];
                int lag = d.delay_steps[i] - 1 < n - 1 ? d.delay_steps[i] - 1 : n - 1;
                int read_idx = (write_idx - lag + depth) % depth;
                out_pos[i] = d.buf_pos_in[size_t(read_idx) * N + i];
                out_vel[i] = d.buf_vel_in[size_t(read_idx) * N + i];
                out_act[i] = d.buf_act_in[size_t(read_idx) * N + i];
            }
        }
        target_pos = out_pos.data();
        target_vel = out_vel.data();
        feedforward = out_act.data();
        tpos_idx = seq.data();
        tvel_idx = seq.data();
    }
    std::vector<float> computed(N), next_integral(N), applied(N);
    for (int i = 0; i < N; ++i) {
        float position_error = target_pos[tpos_idx[i]] - d.positions[d.pos_indices[i]];
        float velocity_error = target_vel[tvel_idx[i]] - d.velocities[d.indices[i]];
        float const_e = 0.0f;
        if (d.const_effort) const_e = d.const_effort[i];
        float ff = 0.0f;
        if (feedforward) ff = feedforward[tvel_idx[i]];
        if (d.controller == NB2_ACT_PID) {  // _pid_effort_kernel (controller_pid.py:15-59)
            float integral = d.integral_in[i] + position_error * d.dt;
            integral = wclamp(integral, -d.integral_max[i], d.integral_max[i]);
            computed[i] = const_e + ff + d.kp[i] * position_error + d.ki[i] * integral + d.kd[i] * velocity_error;
            next_integral[i] = integral;
        } else {  // _pd_effort_kernel (controller_pd.py:13-48)
            computed[i] = const_e + ff + d.kp[i] * position_error + d.kd[i] * velocity_error;
        }
    }
    const float* src = computed.data();
    for (int c = 0; c < d.clamp_count; ++c) {
        const nb2_actuator_clamp& k = d.clamps[c];
        if (k.kind == NB2_CLAMP_MAX_EFFORT) {  // _box_clamp_kernel (clamping_max_effort.py:14-22)
            for (int i = 0; i < N; ++i) applied[i] = wclamp(src[i], -k.p0[i], k.p0[i]);
        } else if (k.kind == NB2_CLAMP_DC_MOTOR) {
            std::vector<float> corner(N);  // _compute_corner_velocity_kernel (clamping_dc_motor.py:14-29)
            for (int i = 0; i < N; ++i) {
                float sat = k.p0[i], vel_lim = k.p1[i], max_e = k.p2[i];
                corner[i] = sat > 0.0f ? vel_lim * (1.0f + max_e / sat) : vel_lim;
            }
            for (int i = 0; i < N; ++i) {  // _clamp_dc_motor_kernel (:32-58)
                float sat = k.p0[i], vel_lim = k.p1[i], max_e = k.p2[i];
                float vel = wclamp(d.velocities[d.indices[i]], -corner[i], corner[i]);
                float effort_max = wmin(sat * (1.0f - vel / vel_lim), max_e);
                float effort_min = wmax(sat * (-1.0f - vel / vel_lim), -max_e);
                applied[i] = wclamp(src[i], effort_min, effort_max);
            }
        } else {  // _position_based_clamp_kernel (clamping_position_based.py:39-53)
            for (int i = 0; i < N; ++i) {
                float limit = interp_1d(d.positions[d.pos_indices[i]], k.p0, k.p1, k.lookup_size);
                applied[i] = wclamp(src[i], -limit, limit);
            }
        }
        src = applied.data();
    }
    for (int i = 0; i < N; ++i) {  // _scatter_add_kernel (actuator.py:17-30)
        int idx = d.effort_indices[i];
        d.output[idx] = d.output[idx] + src[i];
        if (d.computed_output) d.computed_output[idx] = d.computed_output[idx] + computed[i];
    }
    if (d.controller == NB2_ACT_PID) std::memcpy(d.integral_out, next_integral.data(), sizeof(float) * N);  // update_state: wp.copy
    if (depth > 0) {  // _delay_buffer_state_kernel (delay.py:12-54)
        for (int i = 0; i < N; ++i) {
            int copy_idx = d.write_idx_in[0];
            int write_idx = (copy_idx + 1) % depth;
            d.buf_pos_out[size_t(copy_idx) * N + i] = d.buf_pos_in[size_t(copy_idx) * N + i];
            d.buf_vel_out[size_t(copy_idx) * N + i] = d.buf_vel_in[size_t(copy_idx) * N + i];
            d.buf_act_out[size_t(copy_idx) * N + i] = d.buf_act_in[size_t(copy_idx) * N + i];
            d.buf_pos_out[size_t(write_idx) * N + i] = d.target_pos[d.target_pos_indices[i]];
            d.buf_vel_out[size_t(write_idx) * N + i] = d.target_vel[d.indices[i]];
            float act = 0.0f;
            if (d.feedforward) act = d.feedforward[d.indices[i]];
            d.buf_act_out[size_t(write_idx) * N + i] = act;
            int np = d.num_pushes_in[i] + 1;
            d.num_pushes_out[i] = np < depth ? np : depth;
            if (i == 0) d.write_idx_out[0] = write_idx;
        }
    }
}

// Delay.State.reset (delay.py:146-168, _delay_masked_reset_kernel :96-112) and ControllerPID.State.reset (_masked_zero_1d).
inline void reset(int N, int depth, const uint8_t* mask, float* bp, float* bv, float* ba, int* num_pushes, int* write_idx, float* integral) {
    for (int i = 0; i < N; ++i) {
        if (mask && !mask[i]) continue;
        if (bp)
            for (int r = 0; r < depth; ++r) bp[size_t(r) * N + i] = bv[size_t(r) * N + i] = ba[size_t(r) * N + i] = 0.0f;
        if (num_pushes) num_pushes[i] = 0;
        if (integral) integral[i] = 0.0f;
    }
    if (!mask && write_idx) write_idx[0] = depth - 1;
}

// ArticulationView.get_actuator_parameter / set_actuator_parameter (_gather_1d_kernel / the masked scatter), 4-byte words.
inline void param_copy(bool gather, const int* map, int entries, int dofs_per_world, const uint8_t* world_mask, const uint32_t* src,
                       uint32_t* dst) {
    for (int k = 0; k < entries; ++k) {
        int j = map[k];
        if (gather) {
            dst[k] = j >= 0 ? src[j] : 0u;
        } else if (j >= 0 && (!world_mask || world_mask[k / dofs_per_world])) {
            dst[j] = src[k];
        }
    }
}

}  // namespace act
}  // namespace orc

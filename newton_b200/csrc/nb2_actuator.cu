// nb2_actuator.cu - actuators: delay -> PD / PID -> clamp chain -> scatter-add, one thread per actuator (reference
// newton.actuators, actuators/).
//
// The reference steps one actuator group with five or more launches (_delay_read_kernel, the controller kernel, one kernel per
// clamp, _scatter_add_kernel, _delay_buffer_state_kernel and, for PID, a copy of the integral).  actuator_step_kernel does all
// of it in one pass per actuator: each launch of the reference touches only element i of its per-actuator arrays (and the
// shared write_idx / lookup tables), so fusing them changes no value.  The PID integral goes straight to the next state.
// Strict fp32 (-fmad=false) in the reference's operation order; min / max / clamp are Warp's (`a < b ? a : b`,
// `a > b ? a : b`, `min(max(lo, x), hi)`), which decides what NaN and infinite parameters produce.
//
// Duplicate effort indices make the reference's scatter a race.  A group whose effort indices repeat (found on the host at
// construction) writes its efforts to scratch, and actuator_scatter_kernel adds them, one thread per distinct target, in
// ascending actuator index: the reference's serial (CPU) result.  Nothing here allocates or synchronises.
#include "nb2_internal.cuh"

namespace nb2 {
namespace {

__device__ __forceinline__ float wmin(float a, float b) { return a < b ? a : b; }
__device__ __forceinline__ float wmax(float a, float b) { return a > b ? a : b; }
__device__ __forceinline__ float wclamp(float x, float lo, float hi) { return wmin(wmax(lo, x), hi); }

// _interp_1d (clamping_position_based.py:15-36)
__device__ __forceinline__ float interp_1d(float x, const float* xs, const float* ys, int n) {
    if (n <= 0) return 0.0f;
    if (x <= xs[0]) return ys[0];
    if (x >= xs[n - 1]) return ys[n - 1];
    for (int k = 0; k < n - 1; ++k) {
        if (xs[k + 1] >= x) {
            const float dx = xs[k + 1] - xs[k];
            if (dx == 0.0f) return ys[k];
            const float t = (x - xs[k]) / dx;
            return ys[k] + t * (ys[k + 1] - ys[k]);
        }
    }
    return ys[n - 1];
}

template <int CTRL, bool DELAY>
__global__ void __launch_bounds__(256) actuator_step_kernel(const nb2_actuator_step_desc D) {
    extern __shared__ float s_lut[];  // per position-based clamp: positions[K] then efforts[K]
    {
        int off = 0;
        for (int c = 0; c < D.clamp_count; ++c) {
            if (D.clamps[c].kind != NB2_CLAMP_POSITION_BASED) continue;
            const int n = D.clamps[c].lookup_size;
            for (int k = threadIdx.x; k < n; k += blockDim.x) {
                s_lut[off + k] = D.clamps[c].p0[k];
                s_lut[off + n + k] = D.clamps[c].p1[k];
            }
            off += 2 * n;
        }
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int N = D.count;
    if (i >= N) return;
    const int vel_idx = D.indices[i];
    const int pos_idx = D.pos_indices[i];
    const float cur_tp = D.target_pos[D.target_pos_indices[i]];
    const float cur_tv = D.target_vel[vel_idx];
    const float cur_ff = D.feedforward ? D.feedforward[vel_idx] : 0.0f;

    // 1. delay read (_delay_read_kernel, delay.py:57-93)
    float tp = cur_tp, tv = cur_tv, ff = cur_ff;
    int write_idx = 0, pushes = 0;
    if (DELAY) {
        write_idx = *D.write_idx_in;
        pushes = D.num_pushes_in[i];
        const int delay = D.delay_steps[i];
        if (!(pushes == 0 || delay == 0)) {
            const int lag = min(delay - 1, pushes - 1);
            const size_t r = size_t((write_idx - lag + D.buf_depth) % D.buf_depth) * N + i;
            tp = D.buf_pos_in[r];
            tv = D.buf_vel_in[r];
            ff = D.buf_act_in[r];
        }
    }

    // 2. controller (_pd_effort_kernel, controller_pd.py:13-48; _pid_effort_kernel, controller_pid.py:15-59)
    const float pe = tp - D.positions[pos_idx];
    const float ve = tv - D.velocities[vel_idx];
    const float ce = D.const_effort ? D.const_effort[i] : 0.0f;
    float computed;
    if (CTRL == NB2_ACT_PID) {
        float integral = D.integral_in[i] + pe * D.dt;
        const float imax = D.integral_max[i];
        integral = wclamp(integral, -imax, imax);
        computed = (((ce + ff) + D.kp[i] * pe) + D.ki[i] * integral) + D.kd[i] * ve;
        D.integral_out[i] = integral;
    } else {
        computed = ((ce + ff) + D.kp[i] * pe) + D.kd[i] * ve;
    }

    // 3. clamp chain, in order
    float applied = computed;
    int off = 0;
    for (int c = 0; c < D.clamp_count; ++c) {
        const nb2_actuator_clamp& C = D.clamps[c];
        if (C.kind == NB2_CLAMP_MAX_EFFORT) {  // _box_clamp_kernel (clamping_max_effort.py:14-22)
            const float m = C.p0[i];
            applied = wclamp(applied, -m, m);
        } else if (C.kind == NB2_CLAMP_DC_MOTOR) {  // _compute_corner_velocity_kernel + _clamp_dc_motor_kernel (clamping_dc_motor.py:14-58)
            const float sat = C.p0[i], vel_lim = C.p1[i], max_e = C.p2[i];
            const float corner = sat > 0.0f ? vel_lim * (1.0f + max_e / sat) : vel_lim;
            const float vel = wclamp(D.velocities[vel_idx], -corner, corner);
            const float e_max = wmin(sat * (1.0f - vel / vel_lim), max_e);
            const float e_min = wmax(sat * (-1.0f - vel / vel_lim), -max_e);
            applied = wclamp(applied, e_min, e_max);
        } else {  // _position_based_clamp_kernel (clamping_position_based.py:39-53)
            const int n = C.lookup_size;
            const float limit = interp_1d(D.positions[pos_idx], s_lut + off, s_lut + off + n, n);
            applied = wclamp(applied, -limit, limit);
            off += 2 * n;
        }
    }

    // 4. scatter-add (_scatter_add_kernel, actuator.py:17-30)
    if (D.dup_target_count > 0) {
        D.scratch[i] = applied;
        D.scratch[N + i] = computed;
    } else {
        const int e = D.effort_indices[i];
        D.output[e] = D.output[e] + applied;
        if (D.computed_output) D.computed_output[e] = D.computed_output[e] + computed;
    }

    // 5. delay write (_delay_buffer_state_kernel, delay.py:12-54)
    if (DELAY) {
        const int depth = D.buf_depth;
        const int next = (write_idx + 1) % depth;
        const size_t cp = size_t(write_idx) * N + i, wr = size_t(next) * N + i;
        D.buf_pos_out[cp] = D.buf_pos_in[cp];
        D.buf_vel_out[cp] = D.buf_vel_in[cp];
        D.buf_act_out[cp] = D.buf_act_in[cp];
        D.buf_pos_out[wr] = cur_tp;
        D.buf_vel_out[wr] = cur_tv;
        D.buf_act_out[wr] = cur_ff;
        D.num_pushes_out[i] = min(pushes + 1, depth);
        if (i == 0) *D.write_idx_out = next;
    }
}

// The scatter of a group with duplicate effort indices: one thread per distinct target, its actuators in ascending index.
__global__ void __launch_bounds__(256) actuator_scatter_kernel(const nb2_actuator_step_desc D) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= D.dup_target_count) return;
    const int e = D.dup_target[t], k0 = D.dup_start[t], k1 = D.dup_start[t + 1];
    float o = D.output[e];
    for (int k = k0; k < k1; ++k) o = o + D.scratch[D.dup_actuator[k]];
    D.output[e] = o;
    if (D.computed_output) {
        float c = D.computed_output[e];
        for (int k = k0; k < k1; ++k) c = c + D.scratch[D.count + D.dup_actuator[k]];
        D.computed_output[e] = c;
    }
}

__global__ void __launch_bounds__(256) actuator_reset_kernel(int N, int depth, const uint8_t* __restrict__ mask, float* bp, float* bv,
                                                             float* ba, int* num_pushes, int* write_idx, float* integral) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!mask && i == 0 && write_idx) *write_idx = depth - 1;
    if (i >= N || (mask && !mask[i])) return;
    if (bp) {
        for (int r = 0; r < depth; ++r) {
            bp[size_t(r) * N + i] = 0.0f;
            bv[size_t(r) * N + i] = 0.0f;
            ba[size_t(r) * N + i] = 0.0f;
        }
    }
    if (num_pushes) num_pushes[i] = 0;
    if (integral) integral[i] = 0.0f;
}

template <typename T>
__global__ void __launch_bounds__(256) actuator_param_gather_kernel(const int* __restrict__ map, int entries, const T* __restrict__ param,
                                                                    T* __restrict__ values) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= entries) return;
    const int j = map[k];
    values[k] = j >= 0 ? param[j] : T(0);
}

template <typename T>
__global__ void __launch_bounds__(256) actuator_param_scatter_kernel(const int* __restrict__ map, int entries, int dofs_per_world,
                                                                     const uint8_t* __restrict__ world_mask, const T* __restrict__ values,
                                                                     T* __restrict__ param) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= entries) return;
    const int j = map[k];
    if (j < 0 || (world_mask && !world_mask[k / dofs_per_world])) return;
    param[j] = values[k];
}

int blocks(int n) { return (n + 255) / 256; }

}  // namespace

nb2_status launch_actuator_step(const nb2_actuator_step_desc& D, cudaStream_t s) {
    size_t smem = 0;
    for (int c = 0; c < D.clamp_count; ++c)
        if (D.clamps[c].kind == NB2_CLAMP_POSITION_BASED) smem += 2 * size_t(D.clamps[c].lookup_size) * sizeof(float);
    if (D.count > 0) {
        const dim3 g(blocks(D.count)), b(256);
        const bool delay = D.buf_depth > 0;
        if (D.controller == NB2_ACT_PID)
            delay ? actuator_step_kernel<NB2_ACT_PID, true><<<g, b, smem, s>>>(D) : actuator_step_kernel<NB2_ACT_PID, false><<<g, b, smem, s>>>(D);
        else
            delay ? actuator_step_kernel<NB2_ACT_PD, true><<<g, b, smem, s>>>(D) : actuator_step_kernel<NB2_ACT_PD, false><<<g, b, smem, s>>>(D);
        count_launch();
        if (D.dup_target_count > 0) {
            actuator_scatter_kernel<<<blocks(D.dup_target_count), 256, 0, s>>>(D);
            count_launch();
        }
    }
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_actuator_reset(int N, int depth, const uint8_t* mask, float* bp, float* bv, float* ba, int* num_pushes, int* write_idx,
                                 float* integral, cudaStream_t s) {
    actuator_reset_kernel<<<blocks(N > 0 ? N : 1), 256, 0, s>>>(N, depth, mask, bp, bv, ba, num_pushes, write_idx, integral);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_actuator_param(bool gather, const int* map, int entries, int dofs_per_world, const uint8_t* world_mask,
                                 const void* src, void* dst, bool is_int, cudaStream_t s) {
    if (entries <= 0) return NB2_OK;
    if (gather) {
        if (is_int)
            actuator_param_gather_kernel<int><<<blocks(entries), 256, 0, s>>>(map, entries, (const int*)src, (int*)dst);
        else
            actuator_param_gather_kernel<float><<<blocks(entries), 256, 0, s>>>(map, entries, (const float*)src, (float*)dst);
    } else {
        if (is_int)
            actuator_param_scatter_kernel<int><<<blocks(entries), 256, 0, s>>>(map, entries, dofs_per_world, world_mask, (const int*)src, (int*)dst);
        else
            actuator_param_scatter_kernel<float><<<blocks(entries), 256, 0, s>>>(map, entries, dofs_per_world, world_mask, (const float*)src,
                                                                                 (float*)dst);
    }
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

}  // namespace nb2

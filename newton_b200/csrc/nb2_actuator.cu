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
#include "nb2_math.cuh"

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

// The stages of one actuator step that every controller shares: the delay read, the clamp chain, the scatter (or the scratch of
// a group with duplicate effort indices) and the delay write.
struct DelayRead {
    float tp, tv, ff;          // the (possibly delayed) targets and feedforward
    float cur_tp, cur_tv, cur_ff;  // this step's commands, which the delay buffers
    int write_idx, pushes;
};

// _delay_read_kernel (delay.py:57-93)
template <bool DELAY>
__device__ __forceinline__ DelayRead delay_read(const nb2_actuator_step_desc& D, int i, int vel_idx) {
    DelayRead r;
    r.cur_tp = D.target_pos[D.target_pos_indices[i]];
    r.cur_tv = D.target_vel[vel_idx];
    r.cur_ff = D.feedforward ? D.feedforward[vel_idx] : 0.0f;
    r.tp = r.cur_tp, r.tv = r.cur_tv, r.ff = r.cur_ff;
    r.write_idx = 0, r.pushes = 0;
    if (DELAY) {
        r.write_idx = *D.write_idx_in;
        r.pushes = D.num_pushes_in[i];
        const int delay = D.delay_steps[i];
        if (!(r.pushes == 0 || delay == 0)) {
            const int lag = min(delay - 1, r.pushes - 1);
            const size_t k = size_t((r.write_idx - lag + D.buf_depth) % D.buf_depth) * D.count + i;
            r.tp = D.buf_pos_in[k];
            r.tv = D.buf_vel_in[k];
            r.ff = D.buf_act_in[k];
        }
    }
    return r;
}

// the clamp chain, in order; s_lut holds the position-based tables (positions[K] then efforts[K] per table)
__device__ __forceinline__ float clamp_chain(const nb2_actuator_step_desc& D, int i, int vel_idx, int pos_idx, float computed,
                                             const float* s_lut) {
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
    return applied;
}

// scatter-add (_scatter_add_kernel, actuator.py:17-30), or the scratch that actuator_scatter_kernel adds in order
__device__ __forceinline__ void emit_effort(const nb2_actuator_step_desc& D, int i, float applied, float computed) {
    if (D.dup_target_count > 0) {
        D.scratch[i] = applied;
        D.scratch[D.count + i] = computed;
    } else {
        const int e = D.effort_indices[i];
        D.output[e] = D.output[e] + applied;
        if (D.computed_output) D.computed_output[e] = D.computed_output[e] + computed;
    }
}

// _delay_buffer_state_kernel (delay.py:12-54)
__device__ __forceinline__ void delay_write(const nb2_actuator_step_desc& D, int i, const DelayRead& r) {
    const int depth = D.buf_depth, N = D.count;
    const int next = (r.write_idx + 1) % depth;
    const size_t cp = size_t(r.write_idx) * N + i, wr = size_t(next) * N + i;
    D.buf_pos_out[cp] = D.buf_pos_in[cp];
    D.buf_vel_out[cp] = D.buf_vel_in[cp];
    D.buf_act_out[cp] = D.buf_act_in[cp];
    D.buf_pos_out[wr] = r.cur_tp;
    D.buf_vel_out[wr] = r.cur_tv;
    D.buf_act_out[wr] = r.cur_ff;
    D.num_pushes_out[i] = min(r.pushes + 1, depth);
    if (i == 0) *D.write_idx_out = next;
}

// the position-based lookup tables of the group into shared memory (every thread of the CTA takes part)
__device__ __forceinline__ void stage_luts(const nb2_actuator_step_desc& D, float* s_lut) {
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

template <int CTRL, bool DELAY>
__global__ void __launch_bounds__(256) actuator_step_kernel(const nb2_actuator_step_desc D) {
    extern __shared__ float s_lut[];  // per position-based clamp: positions[K] then efforts[K]
    stage_luts(D, s_lut);
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D.count) return;
    const int vel_idx = D.indices[i];
    const int pos_idx = D.pos_indices[i];

    // 1. delay read
    const DelayRead r = delay_read<DELAY>(D, i, vel_idx);

    // 2. controller (_pd_effort_kernel, controller_pd.py:13-48; _pid_effort_kernel, controller_pid.py:15-59)
    const float pe = r.tp - D.positions[pos_idx];
    const float ve = r.tv - D.velocities[vel_idx];
    const float ce = D.const_effort ? D.const_effort[i] : 0.0f;
    float computed;
    if (CTRL == NB2_ACT_PID) {
        float integral = D.integral_in[i] + pe * D.dt;
        const float imax = D.integral_max[i];
        integral = wclamp(integral, -imax, imax);
        computed = (((ce + r.ff) + D.kp[i] * pe) + D.ki[i] * integral) + D.kd[i] * ve;
        D.integral_out[i] = integral;
    } else {
        computed = ((ce + r.ff) + D.kp[i] * pe) + D.kd[i] * ve;
    }

    // 3. clamp chain, 4. scatter-add, 5. delay write
    emit_effort(D, i, clamp_chain(D, i, vel_idx, pos_idx, computed, s_lut), computed);
    if (DELAY) delay_write(D, i, r);
}

// ---------------------------------------------------------------------------------------------- learned actuator networks
__device__ __forceinline__ float activate(int kind, float a, float alpha) {
    switch (kind) {
        case NB2_NET_RELU: return relu_w(a);
        case NB2_NET_ELU: return elu_w(a, alpha);
        case NB2_NET_TANH: return tanh_w(a);
        case NB2_NET_SIGMOID: return sigmoid_w(a);
        case NB2_NET_SOFTSIGN: return softsign_w(a);
        default: return a;
    }
}

// acc = w[0] x[0]; acc = acc + w[k] x[k]: a serial dot product, x strided by `stride` floats (one actuator's column)
__device__ __forceinline__ float dot_serial(const float* __restrict__ w, const float* __restrict__ x, int stride, int n) {
    float acc = w[0] * x[0];
    for (int k = 1; k < n; ++k) acc = acc + w[k] * x[k * stride];
    return acc;
}

__host__ __device__ inline size_t neural_scratch_floats(int kind, const nb2_actuator_network& W) {
    if (kind == NB2_ACT_LSTM) return 4 * size_t(W.widths[1]) * (NB2_NET_TILE + 1);
    int m = 1;
    for (int l = 0; l <= W.layer_count; ++l) m = max(m, W.widths[l]);
    return 2 * size_t(m) * NB2_NET_TILE;
}

// One CTA = NB2_NET_TILE actuators.  Shared memory: the packed weights | the lookup tables | the activation scratch.  Each
// thread owns its actuator's dot products (every lane of a warp reads the same weight: a shared-memory broadcast) and its
// activations live in column t of the scratch ([k][t] layout: conflict-free).  The LSTM state tile ([L, N, H]: the tile's
// rows are one contiguous block per layer) moves through shared memory in coalesced order, padded to TILE + 1.
template <int KIND, bool DELAY>
__global__ void __launch_bounds__(NB2_NET_TILE) actuator_neural_step_kernel(const nb2_actuator_step_desc D, const nb2_actuator_network W) {
    extern __shared__ __align__(16) float smem[];
    const int wpad = (W.weight_count + 3) & ~3;
    float* s_w = smem;
    float* s_lut = smem + wpad;
    int lut = 0;
    for (int c = 0; c < D.clamp_count; ++c)
        if (D.clamps[c].kind == NB2_CLAMP_POSITION_BASED) lut += 2 * D.clamps[c].lookup_size;
    float* s_x = s_lut + lut;
    {
        const float4* src = reinterpret_cast<const float4*>(W.weights);
        float4* dst = reinterpret_cast<float4*>(s_w);
        for (int k = threadIdx.x; k < wpad / 4; k += blockDim.x) dst[k] = src[k];  // the packer pads to whole float4s
    }
    stage_luts(D, s_lut);
    __syncthreads();

    const int N = D.count, t = threadIdx.x, i0 = blockIdx.x * NB2_NET_TILE, i = i0 + t;
    const bool active = i < N;
    int vel_idx = 0, pos_idx = 0;
    DelayRead r{};
    float e = 0.0f, v = 0.0f, net = 0.0f;
    if (active) {
        vel_idx = D.indices[i];
        pos_idx = D.pos_indices[i];
        r = delay_read<DELAY>(D, i, vel_idx);
        e = r.tp - D.positions[pos_idx];
        v = D.velocities[vel_idx];
    }

    if (KIND == NB2_ACT_MLP) {
        if (active) {
            constexpr int T = NB2_NET_TILE;
            float* a = s_x + t;  // two [max width][T] buffers, column t
            float* b = a + neural_scratch_floats(KIND, W) / 2;
            const int K = W.input_count;
            for (int q = 0; q < K; ++q) {
                const int k = W.input_idx[q];
                const float pe = k == 0 ? e : W.state0_in[size_t(k - 1) * N + i];
                const float ve = k == 0 ? v : W.state1_in[size_t(k - 1) * N + i];
                a[(W.vel_first ? K + q : q) * T] = pe * W.pos_scale;
                a[(W.vel_first ? q : K + q) * T] = ve * W.vel_scale;
            }
            const float* w = s_w;
            for (int l = 0; l < W.layer_count; ++l) {
                const int in = W.widths[l], out = W.widths[l + 1];
                const float* bias = W.has_bias[l] ? w + size_t(out) * in : nullptr;
                for (int row = 0; row < out; ++row) {
                    float y = dot_serial(w + size_t(row) * in, a, T, in);
                    if (bias) y = y + bias[row];
                    b[row * T] = activate(W.activation[l], y, W.alpha[l]);
                }
                w += size_t(out) * in + (bias ? out : 0);
                float* tmp = a;
                a = b;
                b = tmp;
            }
            net = a[0];
            // next history: [0] = (e, v), [k] = current[k - 1]
            const int H = W.history_length;
            for (int k = H - 1; k >= 1; --k) {
                W.state0_out[size_t(k) * N + i] = W.state0_in[size_t(k - 1) * N + i];
                W.state1_out[size_t(k) * N + i] = W.state1_in[size_t(k - 1) * N + i];
            }
            W.state0_out[i] = e;
            W.state1_out[i] = v;
        }
    } else {
        constexpr int SP = NB2_NET_TILE + 1;
        const int H = W.widths[1], L = W.layer_count, G = 4 * H;
        const int tile_rows = min(NB2_NET_TILE, N - i0);
        float* sx = s_x;            // the layer's input (the previous layer's new h), [H][SP]
        float* sh = sx + H * SP;    // h of this layer, current state
        float* sc = sh + H * SP;    // c, current then next
        float* sn = sc + H * SP;    // h of this layer, next state
        const float x0 = e * W.pos_scale, x1 = v * W.vel_scale;
        const float* w = s_w;
        const bool bias = W.has_bias[0] != 0;
        for (int l = 0; l < L; ++l) {
            const int in = l == 0 ? 2 : H;
            const size_t base = (size_t(l) * N + i0) * H;
            __syncthreads();  // the previous layer's reads of sh and its stores of sn / sc are done
            for (int q = t; q < tile_rows * H; q += NB2_NET_TILE) {
                const int j = q % H, row = q / H;
                sh[j * SP + row] = W.state0_in[base + q];
                sc[j * SP + row] = W.state1_in[base + q];
            }
            __syncthreads();
            const float* w_ih = w;
            const float* w_hh = w_ih + size_t(G) * in;
            const float* b_ih = w_hh + size_t(G) * H;
            const float* b_hh = b_ih + G;
            if (active) {
                for (int j = 0; j < H; ++j) {
                    float g4[4];
#pragma unroll
                    for (int gate = 0; gate < 4; ++gate) {
                        const int row = gate * H + j;
                        float a1 = l == 0 ? (w_ih[size_t(row) * 2] * x0 + w_ih[size_t(row) * 2 + 1] * x1)
                                          : dot_serial(w_ih + size_t(row) * in, sx + t, SP, in);
                        if (bias) a1 = a1 + b_ih[row];
                        float a2 = dot_serial(w_hh + size_t(row) * H, sh + t, SP, H);
                        if (bias) a2 = a2 + b_hh[row];
                        g4[gate] = a1 + a2;
                    }
                    const float ig = sigmoid_w(g4[0]), fg = sigmoid_w(g4[1]), gg = tanh_w(g4[2]), og = sigmoid_w(g4[3]);
                    const float c = fg * sc[j * SP + t] + ig * gg;
                    sc[j * SP + t] = c;
                    sn[j * SP + t] = og * tanh_w(c);
                }
            }
            __syncthreads();
            for (int q = t; q < tile_rows * H; q += NB2_NET_TILE) {
                const int j = q % H, row = q / H;
                W.state0_out[base + q] = sn[j * SP + row];
                W.state1_out[base + q] = sc[j * SP + row];
            }
            w = b_ih + (bias ? 2 * G : 0);
            float* tmp = sx;  // the new h is the next layer's input; the old input buffer takes the next new h
            sx = sn;
            sn = tmp;
        }
        if (active) {
            net = dot_serial(w, sx + t, SP, H);  // the head reads the top layer's new h (its own column)
            if (W.has_bias[1]) net = net + w[H];
        }
    }

    if (!active) return;
    const float computed = net * W.effort_scale;
    emit_effort(D, i, clamp_chain(D, i, vel_idx, pos_idx, computed, s_lut), computed);
    if (DELAY) delay_write(D, i, r);
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

// element (r, i, j) of two [rows, N, width] arrays, for the masked actuators i
__global__ void __launch_bounds__(256) actuator_network_reset_kernel(int N, int rows, int width, const uint8_t* __restrict__ mask, float* a,
                                                                     float* b) {
    const size_t k = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (k >= size_t(rows) * N * width) return;
    const int i = int((k / width) % N);
    if (mask && !mask[i]) return;
    if (a) a[k] = 0.0f;
    if (b) b[k] = 0.0f;
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

size_t actuator_neural_smem_bytes(const nb2_actuator_step_desc& D) {
    size_t floats = (size_t(D.network->weight_count) + 3) / 4 * 4 + neural_scratch_floats(D.controller, *D.network);
    for (int c = 0; c < D.clamp_count; ++c)
        if (D.clamps[c].kind == NB2_CLAMP_POSITION_BASED) floats += 2 * size_t(D.clamps[c].lookup_size);
    return floats * sizeof(float);
}

template <int KIND, bool DELAY>
nb2_status launch_neural(const nb2_actuator_step_desc& D, size_t smem, cudaStream_t s) {
    auto kernel = actuator_neural_step_kernel<KIND, DELAY>;
    if (smem > 48 * 1024) NB2_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    kernel<<<(D.count + NB2_NET_TILE - 1) / NB2_NET_TILE, NB2_NET_TILE, smem, s>>>(D, *D.network);
    return NB2_OK;
}

}  // namespace

nb2_status launch_actuator_step(const nb2_actuator_step_desc& D, cudaStream_t s) {
    size_t smem = 0;
    for (int c = 0; c < D.clamp_count; ++c)
        if (D.clamps[c].kind == NB2_CLAMP_POSITION_BASED) smem += 2 * size_t(D.clamps[c].lookup_size) * sizeof(float);
    if (D.count > 0) {
        const dim3 g(blocks(D.count)), b(256);
        const bool delay = D.buf_depth > 0;
        if (D.controller == NB2_ACT_MLP || D.controller == NB2_ACT_LSTM) {
            const size_t bytes = actuator_neural_smem_bytes(D);
            if (bytes > NB2_ACTUATOR_SMEM_MAX) {
                set_error("nb2_actuator_step: the network's weights and scratch need " + std::to_string(bytes) +
                          " bytes of shared memory, one CTA holds " + std::to_string(int(NB2_ACTUATOR_SMEM_MAX)));
                return NB2_ERR_CAPACITY;
            }
            if (D.controller == NB2_ACT_MLP)
                delay ? launch_neural<NB2_ACT_MLP, true>(D, bytes, s) : launch_neural<NB2_ACT_MLP, false>(D, bytes, s);
            else
                delay ? launch_neural<NB2_ACT_LSTM, true>(D, bytes, s) : launch_neural<NB2_ACT_LSTM, false>(D, bytes, s);
        } else if (D.controller == NB2_ACT_PID)
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

nb2_status launch_actuator_network_reset(int N, int rows, int width, const uint8_t* mask, float* a, float* b, cudaStream_t s) {
    const size_t total = size_t(rows) * N * width;
    if (total > 0) {
        actuator_network_reset_kernel<<<unsigned((total + 255) / 256), 256, 0, s>>>(N, rows, width, mask, a, b);
        count_launch();
    }
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

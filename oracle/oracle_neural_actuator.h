// oracle_neural_actuator.h - TEST INFRASTRUCTURE ONLY.  CPU restatement of one step of a learned actuator network group
// (ControllerNeuralMLP / ControllerNeuralLSTM with Torch checkpoints), serially in actuator order, under the arithmetic
// contract of include/newton_b200.h (nb2_actuator_network): delay read -> network inputs -> network -> effort scale -> clamp
// chain -> scatter-add in ascending actuator index -> next network state -> delay write.  Compiled with -ffp-contract=off;
// the activations are nb2_math.cuh's double-then-round helpers, the clamps and the delay are oracle_actuator.h's.
#pragma once
#include <vector>

#include "../newton_b200/csrc/nb2_math.cuh"
#include "oracle_actuator.h"

namespace orc {
namespace neural {

inline float activate(int kind, float a, float alpha) {
    switch (kind) {
        case NB2_NET_RELU: return nb2::relu_w(a);
        case NB2_NET_ELU: return nb2::elu_w(a, alpha);
        case NB2_NET_TANH: return nb2::tanh_w(a);
        case NB2_NET_SIGMOID: return nb2::sigmoid_w(a);
        case NB2_NET_SOFTSIGN: return nb2::softsign_w(a);
        default: return a;
    }
}

// acc = w[0] x[0], then acc = acc + w[k] x[k]
inline float dot(const float* w, const float* x, int n) {
    float acc = w[0] * x[0];
    for (int k = 1; k < n; ++k) acc = acc + w[k] * x[k];
    return acc;
}

// the network's raw output for actuator i, given its position error e and velocity v; writes the next state
inline float mlp(const nb2_actuator_network& W, int N, int i, float e, float v) {
    const int K = W.input_count;
    std::vector<float> x(2 * K);
    for (int q = 0; q < K; ++q) {
        const int k = W.input_idx[q];
        const float pe = k == 0 ? e : W.state0_in[size_t(k - 1) * N + i];
        const float ve = k == 0 ? v : W.state1_in[size_t(k - 1) * N + i];
        x[W.vel_first ? K + q : q] = pe * W.pos_scale;
        x[W.vel_first ? q : K + q] = ve * W.vel_scale;
    }
    const float* w = W.weights;
    for (int l = 0; l < W.layer_count; ++l) {
        const int in = W.widths[l], out = W.widths[l + 1];
        std::vector<float> y(out);
        for (int r = 0; r < out; ++r) {
            float a = dot(w + size_t(r) * in, x.data(), in);
            if (W.has_bias[l]) a = a + w[size_t(out) * in + r];
            y[r] = activate(W.activation[l], a, W.alpha[l]);
        }
        w += size_t(out) * in + (W.has_bias[l] ? out : 0);
        x.swap(y);
    }
    for (int t = W.history_length - 1; t >= 1; --t) {  // next[0] = (e, v), next[t] = current[t - 1]
        W.state0_out[size_t(t) * N + i] = W.state0_in[size_t(t - 1) * N + i];
        W.state1_out[size_t(t) * N + i] = W.state1_in[size_t(t - 1) * N + i];
    }
    W.state0_out[i] = e;
    W.state1_out[i] = v;
    return x[0];
}

inline float lstm(const nb2_actuator_network& W, int N, int i, float e, float v) {
    const int H = W.widths[1], L = W.layer_count, G = 4 * H;
    const bool bias = W.has_bias[0] != 0;
    std::vector<float> x = {e * W.pos_scale, v * W.vel_scale}, h(H), hn(H);
    const float* w = W.weights;
    for (int l = 0; l < L; ++l) {
        const int in = l == 0 ? 2 : H;
        const float* w_ih = w;
        const float* w_hh = w_ih + size_t(G) * in;
        const float* b_ih = w_hh + size_t(G) * H;
        const float* b_hh = b_ih + G;
        const size_t base = (size_t(l) * N + i) * H;
        for (int j = 0; j < H; ++j) h[j] = W.state0_in[base + j];
        for (int j = 0; j < H; ++j) {
            float g4[4];
            for (int gate = 0; gate < 4; ++gate) {
                const int r = gate * H + j;
                float a1 = dot(w_ih + size_t(r) * in, x.data(), in);
                if (bias) a1 = a1 + b_ih[r];
                float a2 = dot(w_hh + size_t(r) * H, h.data(), H);
                if (bias) a2 = a2 + b_hh[r];
                g4[gate] = a1 + a2;
            }
            const float ig = nb2::sigmoid_w(g4[0]), fg = nb2::sigmoid_w(g4[1]), gg = nb2::tanh_w(g4[2]), og = nb2::sigmoid_w(g4[3]);
            const float c = fg * W.state1_in[base + j] + ig * gg;
            W.state1_out[base + j] = c;
            hn[j] = og * nb2::tanh_w(c);
            W.state0_out[base + j] = hn[j];
        }
        w = b_ih + (bias ? 2 * G : 0);
        x = hn;
    }
    float y = dot(w, x.data(), H);
    if (W.has_bias[1]) y = y + w[H];
    return y;
}

inline void step(const nb2_actuator_step_desc& d) {
    const int N = d.count;
    if (N <= 0) return;
    const nb2_actuator_network& W = *d.network;
    const int depth = d.buf_depth;
    std::vector<float> computed(N), applied(N);
    for (int i = 0; i < N; ++i) {
        float tp = d.target_pos[d.target_pos_indices[i]];
        if (depth > 0 && d.num_pushes_in[i] != 0 && d.delay_steps[i] != 0) {  // _delay_read_kernel (delay.py:57-93)
            const int n = d.num_pushes_in[i];
            const int lag = d.delay_steps[i] - 1 < n - 1 ? d.delay_steps[i] - 1 : n - 1;
            tp = d.buf_pos_in[size_t((d.write_idx_in[0] - lag + depth) % depth) * N + i];
        }
        const float e = tp - d.positions[d.pos_indices[i]];
        const float v = d.velocities[d.indices[i]];
        const float net = d.controller == NB2_ACT_MLP ? mlp(W, N, i, e, v) : lstm(W, N, i, e, v);
        computed[i] = net * W.effort_scale;
    }
    // the clamp chain, one pass per clamp as in orc::act::step (clamping_*.py)
    const float* src = computed.data();
    for (int c = 0; c < d.clamp_count; ++c) {
        const nb2_actuator_clamp& k = d.clamps[c];
        for (int i = 0; i < N; ++i) {
            if (k.kind == NB2_CLAMP_MAX_EFFORT) {
                applied[i] = act::wclamp(src[i], -k.p0[i], k.p0[i]);
            } else if (k.kind == NB2_CLAMP_DC_MOTOR) {
                const float sat = k.p0[i], vel_lim = k.p1[i], max_e = k.p2[i];
                const float corner = sat > 0.0f ? vel_lim * (1.0f + max_e / sat) : vel_lim;
                const float vel = act::wclamp(d.velocities[d.indices[i]], -corner, corner);
                const float effort_max = act::wmin(sat * (1.0f - vel / vel_lim), max_e);
                const float effort_min = act::wmax(sat * (-1.0f - vel / vel_lim), -max_e);
                applied[i] = act::wclamp(src[i], effort_min, effort_max);
            } else {
                const float limit = act::interp_1d(d.positions[d.pos_indices[i]], k.p0, k.p1, k.lookup_size);
                applied[i] = act::wclamp(src[i], -limit, limit);
            }
        }
        src = applied.data();
    }
    for (int i = 0; i < N; ++i) {  // _scatter_add_kernel, serially: repeated effort indices sum in ascending actuator index
        const int idx = d.effort_indices[i];
        d.output[idx] = d.output[idx] + src[i];
        if (d.computed_output) d.computed_output[idx] = d.computed_output[idx] + computed[i];
    }
    if (depth > 0) {  // _delay_buffer_state_kernel (delay.py:12-54): the delay buffers every command, read or not
        const int copy_idx = d.write_idx_in[0], write_idx = (copy_idx + 1) % depth;
        for (int i = 0; i < N; ++i) {
            const size_t cp = size_t(copy_idx) * N + i, wr = size_t(write_idx) * N + i;
            d.buf_pos_out[cp] = d.buf_pos_in[cp];
            d.buf_vel_out[cp] = d.buf_vel_in[cp];
            d.buf_act_out[cp] = d.buf_act_in[cp];
            d.buf_pos_out[wr] = d.target_pos[d.target_pos_indices[i]];
            d.buf_vel_out[wr] = d.target_vel[d.indices[i]];
            d.buf_act_out[wr] = d.feedforward ? d.feedforward[d.indices[i]] : 0.0f;
            const int np = d.num_pushes_in[i] + 1;
            d.num_pushes_out[i] = np < depth ? np : depth;
        }
        d.write_idx_out[0] = write_idx;
    }
}

// ControllerNeuralMLP.State.reset / ControllerNeuralLSTM.State.reset: element (r, i, j) of two [rows, N, width] arrays
inline void reset(int N, int rows, int width, const uint8_t* mask, float* a, float* b) {
    for (int r = 0; r < rows; ++r)
        for (int i = 0; i < N; ++i) {
            if (mask && !mask[i]) continue;
            for (int j = 0; j < width; ++j) {
                const size_t k = (size_t(r) * N + i) * width + j;
                if (a) a[k] = 0.0f;
                if (b) b[k] = 0.0f;
            }
        }
}

}  // namespace neural
}  // namespace orc

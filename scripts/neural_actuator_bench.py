"""Times the learned actuator networks on 4096 seeded quadrupeds: the 12 leg dofs of scenes.quadruped_actuated_model(4096,
seed=1) (49 152 actuators, ClampingDCMotor, delays of 1-3 steps) driven by one ControllerNeuralMLP (input_idx [0, 1, 2],
6 -> 32 -> 32 -> 32 -> 1, Softsign) or one ControllerNeuralLSTM (2 layers, hidden size 32), both seeded and written to a
temporary directory as .pt2 archives.

Prints one JSON line with, per controller: microseconds per step (CUDA events; eagerly, and replayed from a CUDA graph of 10
steps), launches per step, the fused kernel's device time from torch.profiler in its own run, the same module on cuda:0
driven through the reference's Torch-path sequence (index, stack / cat, forward under inference_mode, scale, state update)
timed the same way, a Featherstone frame of 10 substeps with the network group against the PD group, and the algorithmic
FLOPs and bytes per step with the share of the FP32 or HBM bound (whichever is larger); with the card's name, power limit
and SM clock read in the same run.

    python scripts/neural_actuator_bench.py [--envs 4096] [--iters 200]
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import actuator_bench as AB  # noqa: E402

import newton_b200  # noqa: E402
from newton_b200 import _lib, scenes  # noqa: E402
from newton_b200.actuators import Actuator, ControllerNeuralLSTM, ControllerNeuralMLP  # noqa: E402
from tests import neural_nets as NN  # noqa: E402

FP32_PEAK, HBM_PEAK = 67e12, 3.35e12  # H100 SXM data sheet, dense FP32 and HBM3


def networks(tmp):
    mlp = NN.save(NN.mlp([6, 32, 32, 32, 1], "softsign", seed=1), os.path.join(tmp, "mlp.pt2"),
                  metadata={"input_idx": [0, 1, 2], "effort_scale": 20.0})
    lstm = NN.save(NN.lstm(32, 2, seed=1), os.path.join(tmp, "lstm.pt2"),
                   metadata={"num_layers": 2, "hidden_size": 32, "effort_scale": 20.0}, kind="lstm")
    return {"mlp": (ControllerNeuralMLP, mlp), "lstm": (ControllerNeuralLSTM, lstm)}


def neural_model(envs, cls, path):
    """The actuated quadrupeds with their PD group's controller replaced by the network (same indices, delay and clamps)."""
    model = scenes.quadruped_actuated_model(envs, "cuda:0", seed=1)
    pd = model.actuators[0]
    model.actuators = [Actuator(pd.indices, cls(path), delay=pd.delay, clamping=pd.clamping, pos_indices=pd.pos_indices,
                                target_pos_indices=pd.target_pos_indices)]
    return model


def algorithmic(ctrl, n):
    """FLOPs (multiply and add counted apart) and bytes of one step, from shapes."""
    if isinstance(ctrl, ControllerNeuralMLP):
        w = ctrl.widths
        flops = sum(2 * a * b for a, b in zip(w, w[1:]))
        state = 2 * 2 * ctrl.history_length * 4  # two histories, read and written
    else:
        H, L = ctrl.hidden_size, ctrl.num_layers
        flops = sum(2 * 4 * H * ((2 if k == 0 else H) + H) for k in range(L)) + 2 * H
        state = 2 * 2 * L * H * 4  # h and c, read and written
    other = 4 * 4 + 3 * 4 + 4 * 4 + 3 * 4 * 2 + 3 * 4 + 8  # indices, q / qd / target, clamp params, delay read + write, effort
    return flops * n, (state + other) * n, flops


def fused_numbers(model, iters):
    act = model.actuators[0]
    state, ctl = model.state(), model.control()
    a = [act.state(), act.state()]

    def step():
        act.step(state, ctl, a[0], a[1], 0.001)
        a.reverse()

    us = AB.time_call(step, iters)
    l0 = _lib.kernel_launch_count()
    step()
    torch.cuda.synchronize()
    launches = _lib.kernel_launch_count() - l0

    def ten():
        for _ in range(10):
            step()

    g = AB.graph_of(ten)
    us_graph = AB.time_call(g.replay, max(1, iters // 10)) / 10
    return {"us_per_step": round(us, 2), "us_per_step_graph_replay": round(us_graph, 2), "launches_per_step": launches,
            "kernel_us": AB.kernel_us(step)}


def torch_baseline(model, kind, iters):
    """The reference's _compute_torch sequence for the same module on cuda:0 (no delay or clamps: the network part only)."""
    act = model.actuators[0]
    ctrl = act.controller
    net = ctrl.network.to("cuda:0")
    state, ctl = model.state(), model.control()
    pi, vi, ti = (x.long() for x in (act.pos_indices, act.indices, act.target_pos_indices))
    forces = torch.zeros(act.num_actuators, device="cuda:0")
    if kind == "mlp":
        hist = [torch.zeros(ctrl.history_length, act.num_actuators, device="cuda:0") for _ in range(2)]

        def step():
            e = ctl.joint_target_q[ti] - state.joint_q[pi]
            v = state.joint_qd[vi]
            pos_in = torch.stack([e if i == 0 else hist[0][i - 1] for i in ctrl.input_idx], dim=1)
            vel_in = torch.stack([v if i == 0 else hist[1][i - 1] for i in ctrl.input_idx], dim=1)
            x = torch.cat([pos_in * ctrl.pos_scale, vel_in * ctrl.vel_scale], dim=1)
            with torch.inference_mode():
                y = net(x)
            forces.copy_(y.reshape(-1) * ctrl.effort_scale)
            h0, h1 = hist[0].roll(1, 0), hist[1].roll(1, 0)
            h0[0], h1[0] = e, v
            hist[0].copy_(h0)
            hist[1].copy_(h1)
    else:
        shape = (ctrl.num_layers, act.num_actuators, ctrl.hidden_size)
        hc = [torch.zeros(shape, device="cuda:0"), torch.zeros(shape, device="cuda:0")]

        def step():
            e = ctl.joint_target_q[ti] - state.joint_q[pi]
            v = state.joint_qd[vi]
            x = torch.stack([e * ctrl.pos_scale, v * ctrl.vel_scale], dim=1).unsqueeze(1)
            with torch.inference_mode():
                y, (h, c) = net(x, (hc[0], hc[1]))
            forces.copy_(y.reshape(-1) * ctrl.effort_scale)
            hc[0].copy_(h)
            hc[1].copy_(c)

    out = {"us_per_step": round(AB.time_call(step, iters), 2)}
    try:
        def ten():
            for _ in range(10):
                step()

        g = AB.graph_of(ten)
        out["us_per_step_graph_replay"] = round(AB.time_call(g.replay, max(1, iters // 10)) / 10, 2)
    except Exception as exc:  # noqa: BLE001 - the torch path may not be capturable; report why
        out["us_per_step_graph_replay"] = f"not capturable: {type(exc).__name__}"
        torch.cuda.synchronize()
    return out


def frame_us(model, iters, substeps=10, dt=0.001):
    solver = newton_b200.solvers.SolverFeatherstone(model)
    s, ctl = [model.state(), model.state()], model.control()
    act = model.actuators[0]
    a = [act.state(), act.state()]

    def frame():
        for _ in range(substeps):
            ctl.joint_f.zero_()
            act.step(s[0], ctl, a[0], a[1], dt)
            a.reverse()
            solver.step(s[0], s[1], ctl, None, dt)
            s.reverse()

    g = AB.graph_of(frame)
    return round(AB.time_call(g.replay, iters, warmup=5), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("neural_actuator_bench.py measures on a CUDA device; none is visible")
    out = {"envs": args.envs, "iters": args.iters}
    with tempfile.TemporaryDirectory() as tmp:
        nets = networks(tmp)
        pd_model = scenes.quadruped_actuated_model(args.envs, "cuda:0", seed=1)
        for kind, (cls, path) in nets.items():
            model = neural_model(args.envs, cls, path)
            act = model.actuators[0]
            res = {"actuators": act.num_actuators, "smem_bytes_per_cta": act.controller.smem_bytes()}
            res.update(fused_numbers(model, args.iters))
            flops, nbytes, per = algorithmic(act.controller, act.num_actuators)
            kern = sum(res["kernel_us"].values()) * 1e-6
            t_flop, t_byte = flops / FP32_PEAK, nbytes / HBM_PEAK
            res["algorithmic"] = {"flop_per_actuator_step": per, "flop_per_step": flops, "bytes_per_step": nbytes,
                                  "bound": "fp32" if t_flop >= t_byte else "hbm",
                                  "share_of_bound": round(max(t_flop, t_byte) / kern, 4) if kern > 0 else None}
            res["torch_baseline"] = torch_baseline(model, kind, args.iters)
            frames_n, frames_pd = [], []
            for _ in range(3):  # alternate so both frames see the same clock and load
                frames_n.append(frame_us(model, args.iters // 4))
                frames_pd.append(frame_us(pd_model, args.iters // 4))
            res["featherstone_frame_10_substeps_us"] = {"network": frames_n, "pd": frames_pd}
            out[kind] = res
    out.update(AB.card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()

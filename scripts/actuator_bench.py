"""Times Actuator.step on 4096 seeded quadrupeds (scenes.quadruped_actuated_model(4096, seed=1)): the 12 leg dofs of every
quadruped in one group of PD (or PID) + ClampingDCMotor + Delay with delays of 1-3 steps, 49 152 actuators.

Prints one JSON line with, per controller: microseconds per step (CUDA events; eagerly from Python, and replayed from a CUDA
graph of 10 steps), the library's kernel launches per step, and the device time of the step kernel from torch.profiler; then a
Featherstone frame of 10 substeps replayed from a CUDA graph, with the actuator step inside every substep, against the same
frame of scenes.quadruped_model(4096, seed=1) driven by the solver's built-in PD; with the card's name, power limit and SM
clock read in the same run.

    python scripts/actuator_bench.py [--envs 4096] [--iters 200]
"""

from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import newton_b200  # noqa: E402
from newton_b200 import _lib, scenes  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power, max_sm, sm = (float(x) for x in q.splitlines()[0].split(","))
    except Exception:
        power = max_sm = sm = None
    return {"card": name, "power_limit_w": power, "sm_clock_max_mhz": max_sm, "sm_clock_mhz_at_end": sm}


def time_call(fn, iters, warmup=20):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def graph_of(fn):
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        fn()
    torch.cuda.synchronize()
    return g


def kernel_us(fn, calls=50):
    """Mean device time per call of every CUDA kernel torch.profiler records (a separate profiled run)."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    times = {}
    for e in prof.events():
        m = re.search(r"actuator_\w+_kernel", e.name)
        if e.device_type == torch.autograd.DeviceType.CUDA and m:
            key = m.group(0)
            times[key] = times.get(key, 0.0) + e.device_time / calls
    return {k: round(v, 2) for k, v in times.items()}


def actuator_step_numbers(envs, controller, iters):
    model = scenes.quadruped_actuated_model(envs, "cuda:0", seed=1, controller=controller)
    act = model.actuators[0]
    state, ctl = model.state(), model.control()
    a = [act.state(), act.state()]

    def step():
        act.step(state, ctl, a[0], a[1], 0.001)
        a.reverse()

    us = time_call(step, iters)
    l0 = _lib.kernel_launch_count()
    step()
    torch.cuda.synchronize()
    launches = _lib.kernel_launch_count() - l0

    def ten():
        for _ in range(10):
            step()

    g = graph_of(ten)
    us_graph = time_call(g.replay, max(1, iters // 10)) / 10
    return {"actuators": act.num_actuators, "us_per_step": round(us, 2), "us_per_step_graph_replay": round(us_graph, 2),
            "launches_per_step": launches, "kernel_us": kernel_us(step)}


def frame_us(envs, actuated, iters, substeps=10, dt=0.001):
    model = (scenes.quadruped_actuated_model if actuated else scenes.quadruped_model)(envs, "cuda:0", seed=1)
    solver = newton_b200.solvers.SolverFeatherstone(model)
    s = [model.state(), model.state()]
    ctl = model.control()
    act = model.actuators[0] if actuated else None
    a = [act.state(), act.state()] if actuated else None

    def frame():
        for _ in range(substeps):
            if actuated:
                ctl.joint_f.zero_()
                act.step(s[0], ctl, a[0], a[1], dt)
                a.reverse()
            solver.step(s[0], s[1], ctl, None, dt)
            s.reverse()

    g = graph_of(frame)
    return round(time_call(g.replay, iters, warmup=5), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("actuator_bench.py measures on a CUDA device; none is visible")
    out = {"envs": args.envs, "iters": args.iters}
    for controller in ("pd", "pid"):
        out[controller] = actuator_step_numbers(args.envs, controller, args.iters)
    # alternate the two frames so both see the same clock and load
    builtin, actuated = [], []
    for _ in range(3):
        builtin.append(frame_us(args.envs, False, args.iters // 4))
        actuated.append(frame_us(args.envs, True, args.iters // 4))
    out["featherstone_frame_10_substeps_us"] = {"builtin_pd": builtin, "actuator_pd_dc_motor_delay": actuated}
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()

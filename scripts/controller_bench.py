"""Times the joint-impedance controllers on 4096 robots and prints one JSON line.

Workloads:
  (a) model_based_pandas: 4096 Panda-class arms (scenes.impedance_fleet_builder), ControllerJointImpedance with gravity,
      Coriolis, inertia decoupling and the qdd feedforward on;
  (b) model_free_pandas: the same fleet, ControllerJointImpedanceModelFree fed precomputed M, g and C qd;
  (c) model_based_mixed: 4096 robots cycling Panda / fixed-base ant / 1-link pendulum, all terms on.
For each: microseconds per step (CUDA events; eager from Python, and replayed from a CUDA graph of 10 steps), kernel device time
from torch.profiler in a separate run, and the library's launches per step.  For (a) also the unfused composition of the same
step in this library: eval_fk, eval_inverse_dynamics_passive(mass_matrix, gravity_force, coriolis_force), then a model-free step
(plus the two gathers into the internal state, done with torch index_select).  The card's name and power limit are read in the
same run.

    python scripts/controller_bench.py [--robots 4096] [--iters 200]
"""

from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import newton_b200  # noqa: E402
from newton_b200 import _lib, scenes  # noqa: E402
from newton_b200.controllers import ControllerJointImpedance, ControllerJointImpedanceModelFree  # noqa: E402

DEV = "cuda:0"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power, max_sm = (float(x) for x in q.splitlines()[0].split(","))
    except Exception:
        power = max_sm = None
    return {"card": name, "power_limit_w": power, "sm_clock_max_mhz": max_sm}


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


def graph_us(fn, iters):
    """Microseconds per call of ``fn`` replayed from a CUDA graph of 10 calls."""
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        for _ in range(10):
            fn()
    return time_call(g.replay, max(1, iters // 10), warmup=3) / 10


def kernel_us(fn, calls=50):
    """Mean device time per call of every CUDA kernel torch.profiler records (a separate profiled run)."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    times = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            m = re.search(r"(\w+_kernel)", e.name)
            key = m.group(1) if m else e.name[:60]
            times[key] = times.get(key, 0.0) + e.device_time / calls
    return {k: round(v, 2) for k, v in sorted(times.items(), key=lambda kv: -kv[1])}


def launches(fn):
    fn()
    torch.cuda.synchronize()
    n0 = _lib.kernel_launch_count()
    fn()
    return _lib.kernel_launch_count() - n0


def measure(fn, iters):
    eager = time_call(fn, iters)
    return {"eager_us": round(eager, 2), "graph_us": round(graph_us(fn, iters), 2), "launches_per_step": launches(fn),
            "kernel_us": kernel_us(fn)}


def gains(R, D, rng):
    return (torch.from_numpy(rng.uniform(50.0, 150.0, (R, D)).astype(np.float32)),
            torch.from_numpy(rng.uniform(5.0, 25.0, (R, D)).astype(np.float32)))


def seeded_inputs(ctrl, rng):
    inp, out = ctrl.input(), ctrl.output()
    for name, t in vars(inp).items():
        if t is not None and name not in ("stiffness", "damping", "mass_matrix"):
            t.copy_(torch.from_numpy(rng.uniform(-1.0, 1.0, t.shape).astype(np.float32)))
    return inp, out


def model_based(builder, rng):
    n, R = builder.joint_dof_count, builder.articulation_count
    qd = [*builder.joint_qd_start, n]
    D = max(qd[e] - qd[s] for s, e in zip(builder.articulation_start, builder.articulation_end))
    kp, kd = gains(R, D, rng)
    ctrl = ControllerJointImpedance(builder, default_dof_indices=torch.arange(n, dtype=torch.int32), stiffness=kp, damping=kd,
                                    has_qdd_feedforward=True, device=DEV)
    return ctrl, *seeded_inputs(ctrl, rng)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--robots", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("controller_bench.py measures on a CUDA device; none is visible")
    rng = np.random.default_rng(0)
    R = args.robots
    result = {"robots": R, **card()}

    # (a) model-based Pandas, and the unfused composition of the same step
    pandas = scenes.impedance_fleet_builder(R, ("panda",))
    ctrl, inp, out = model_based(pandas, rng)
    result["model_based_pandas"] = measure(lambda: ctrl.step(inputs=inp, outputs=out), args.iters)

    model, n, D = ctrl.model, pandas.joint_dof_count, ctrl.max_dofs
    state = model.state()
    M = torch.zeros(R, D, D, device=DEV)
    g, c = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    kp, kd = ctrl._stiffness, ctrl._damping  # the same gains, so that both paths compute the same torques
    ident = torch.arange(n, dtype=torch.int32)
    free = ControllerJointImpedanceModelFree(robot_count=R, dofs_per_robot=torch.full((R,), 9, dtype=torch.int32), max_dofs=D,
                                             default_dof_indices=ident, stiffness=kp, damping=kd, has_qdd_feedforward=True, device=DEV)
    finp, fout = free.input(), free.output()
    for name in ("joint_q", "joint_qd", "joint_q_des", "joint_qd_des", "joint_qdd"):
        getattr(finp, name).copy_(getattr(inp, name))
    finp.gravity_force, finp.coriolis_force, finp.mass_matrix = g, c, M
    q_idx = ident.to(DEV).long()

    def unfused():
        torch.index_select(inp.joint_q, 0, q_idx, out=state.joint_q)
        torch.index_select(inp.joint_qd, 0, q_idx, out=state.joint_qd)
        newton_b200.eval_fk(model, state.joint_q, state.joint_qd, state)
        newton_b200.eval_inverse_dynamics_passive(model, state, mass_matrix=M, gravity_force=g, coriolis_force=c)
        free.step(inputs=finp, outputs=fout)

    comp = measure(unfused, args.iters)
    comp["note"] = "launches_per_step counts this library's kernels only; the two torch index_select gathers add 2 more"
    result["model_based_pandas"]["unfused_composition"] = comp
    unfused()
    ctrl.step(inputs=inp, outputs=out)
    torch.cuda.synchronize()
    result["model_based_pandas"]["fused_equals_unfused"] = bool(torch.equal(out.joint_f, fout.joint_f))

    # (b) model-free on the same fleet, caller-supplied terms
    result["model_free_pandas"] = measure(lambda: free.step(inputs=finp, outputs=fout), args.iters)

    # (c) heterogeneous fleet
    mixed = scenes.impedance_fleet_builder(R, ("panda", "ant", "pendulum"))
    mctrl, minp, mout = model_based(mixed, rng)
    result["model_based_mixed"] = measure(lambda: mctrl.step(inputs=minp, outputs=mout), args.iters)
    print(json.dumps(result))


if __name__ == "__main__":
    main()

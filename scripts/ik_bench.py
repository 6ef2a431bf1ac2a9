"""Times newton_b200.ik.IKSolver.step on three workloads and prints one JSON line.

  (a) arm        4096 problems, 1 seed,            24 iterations, position + rotation + limits, weight 10 (example_ik_franka)
  (b) arm        1024 problems x 16 Roberts seeds, 24 iterations, same objectives
  (c) quadruped  4096 problems, 1 seed,            32 iterations, four feet + base rotation + limits

Per workload: us per step eager and replayed from a CUDA graph (CUDA events), the kernels' device time per step (torch.profiler),
launches per step (nb2_kernel_launch_count), solves per second, the final position / rotation errors (median and max), and the
launches upstream would issue for the same configuration, counted from its code (not measured).  Workload (a) is also timed at
8, 16 and 32 lanes per problem.  The card name, power limit and SM clock are read in the same run.  Writes nothing.
"""

from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from newton_b200 import _lib, ik  # noqa: E402
from tests import ik_cases as K  # noqa: E402

DEV = "cuda:0"


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the numbers are still reported; the card fields say why they are missing
        return {"name": torch.cuda.get_device_name(0), "error": str(e)}


def upstream_launches(n_obj: int, iterations: int, n_seeds: int, sampler: bool) -> int:
    """Kernels + memsets + copies of IKSolver.step with IKOptimizerLM in ANALYTIC mode, counted from ik_solver.py:348-403 and
    ik_lm_optimizer.py:509-705 (no joint_dof_mask)."""
    residuals = 2 + 1 + n_obj  # _fk_local, fk_accum, residuals.zero_(), one residual kernel per objective
    per_iter = (1  # compute_costs
                + 1 + 1 + n_obj  # jacobian.zero_(), motion subspace, one Jacobian kernel per objective
                + 1 + 1 + 1  # copy residuals -> residuals_3d, dq_dof.zero_(), _lm_solve_tiled
                + 1 + 1  # _integrate_dq_dof, qd_zero.zero_()
                + residuals + 1 + 1 + 1)  # proposal residuals, compute_costs, _accept_reject, _update_lm_state
    step = 1 + 1  # _pull_seed, sample kernel
    step += 2 + 1  # _impl.reset (two zero_), lambda fill
    step += residuals + iterations * per_iter  # iteration 0's residuals + the iterations
    step += residuals + 1  # closing compute_costs
    step += 1 if n_seeds == 1 else 2  # copy to joint_q_out / select + gather
    return step


def time_step(solver, q, iterations, reps=20):
    torch.cuda.synchronize()
    for _ in range(3):
        solver.step(q, q, iterations=iterations)
    torch.cuda.synchronize()
    c0 = _lib.kernel_launch_count()
    solver.step(q, q, iterations=iterations)
    torch.cuda.synchronize()
    launches = _lib.kernel_launch_count() - c0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        solver.step(q, q, iterations=iterations)
    e1.record()
    torch.cuda.synchronize()
    eager = e0.elapsed_time(e1) * 1000.0 / reps
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        solver.step(q, q, iterations=iterations)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        solver.step(q, q, iterations=iterations)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    graph = e0.elapsed_time(e1) * 1000.0 / reps
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            g.replay()
        torch.cuda.synchronize()
    dev_us = sum(e.device_time_total for e in prof.key_averages() if e.device_time_total > 0 and "ik_" in e.key) / 5.0
    return eager, graph, dev_us, launches


def errors(solver, n_pos: int, has_rot: bool, weights) -> dict:
    r = solver.residuals.detach().cpu().numpy()
    q = solver.costs.detach().cpu().numpy().reshape(solver.n_problems, solver.n_seeds)
    best = np.argmin(q, axis=1) + np.arange(solver.n_problems) * solver.n_seeds  # the selected seed's rows
    r = r[best]
    pos = np.concatenate([np.linalg.norm(r[:, 3 * i:3 * i + 3], axis=1) / weights[i] for i in range(n_pos)])
    out = {"pos_err_median_m": float(np.median(pos)), "pos_err_max_m": float(pos.max())}
    if has_rot:
        rot = np.linalg.norm(r[:, 3 * n_pos:3 * n_pos + 3], axis=1) / weights[n_pos]
        out.update(rot_err_median_rad=float(np.median(rot)), rot_err_max_rad=float(rot.max()))
    return out


def workload(name, make, n, iterations, n_pos, has_rot, weights, **kw):
    model, objs, q = make(DEV, n)
    s = ik.IKSolver(model, n, objs, jacobian_mode="analytic", **kw)
    q0 = q.clone()
    eager, graph, dev_us, launches = time_step(s, q, iterations)
    q.copy_(q0)
    s.reset()
    s.step(q, q, iterations=iterations)
    torch.cuda.synchronize()
    seeds = kw.get("n_seeds", 1)
    res = {"workload": name, "problems": n, "seeds": seeds, "iterations": iterations, "us_per_step_eager": round(eager, 1),
           "us_per_step_graph": round(graph, 1), "kernel_device_us": round(dev_us, 1), "launches_per_step": launches,
           "solves_per_s": round(n / (graph * 1e-6)), "upstream_launches_counted": upstream_launches(len(objs), iterations, seeds,
                                                                                               kw.get("sampler", "none") != "none"),
           "lanes": s._impl._desc.lanes or _default_lanes(model)}
    res.update(errors(s, n_pos, has_rot, weights))
    return res, s, q0


def _default_lanes(model) -> int:
    m = max(int(model.joint_count), int(model.joint_dof_count))
    return 8 if m <= 8 else (16 if m <= 16 else 32)


def main() -> None:
    torch.cuda.init()
    out = {"card": card()}
    arm = lambda d, n: K.arm_problem(d, n, seed=21)  # noqa: E731
    a, s, q0 = workload("a_arm", arm, 4096, 24, 1, True, (10.0, 10.0))
    lanes = {}
    for L in (8, 16, 32):
        s._impl._desc.lanes = L
        q = q0.clone()
        lanes[str(L)] = round(time_step(s, q, 24)[1], 1)
    a["us_per_step_graph_by_lanes"] = lanes
    b, _, _ = workload("b_arm_roberts", arm, 1024, 24, 1, True, (10.0, 10.0), sampler="roberts", n_seeds=16)
    c, _, _ = workload("c_quadruped", lambda d, n: K.quadruped_problem(d, n, seed=22), 4096, 32, 4, True, (1.0, 1.0, 1.0, 1.0, 1.0))
    out["workloads"] = [a, b, c]
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Times SolverSemiImplicit on the GPU: collide + SolverSemiImplicit.step per substep, in two workloads:

  (a) scenes.quadruped_model(4096, seed=1), bases lowered to 0.47 m: 13 bodies / 13 joints per environment, feet in penalty
      contact with the ground;
  (b) scenes.box_stack_model(4096, seed=0): 5 free boxes per environment, no joint springs, heavy box-box contacts.

Substep dt = 1 ms for both.  Nothing pins a stable substep for the quadruped under semi-implicit attachment springs, so it was
chosen with the CPU oracle (oracle.semi_implicit): three quadrupeds stay finite, bases above 0.3 m, for 1 s of simulated time at
1 ms with the default joint_attach_ke = 1e4 / kd = 1e2, from this script's start pose (tests/test_semi_implicit.py::
test_quadruped_stays_up_at_the_benchmark_substep;
0.5 ms and 0.25 ms settle the same way).  1 ms is also the Featherstone quadruped substep, so the two solvers compare directly.

Per workload, one JSON line with:
  - substeps per second replayed from a CUDA graph (one graph of `--graph-substeps` substeps) and eager, from CUDA events;
  - the kernel time of semi_implicit_step_kernel from torch.profiler, in a separate run;
  - launches per substep (the library's launch counter), against the reference's 3 kernels + 1 clone on this path
    (eval_body_joints, eval_body_contact, integrate_bodies, wp.clone(body_f); solver_semi_implicit.py:166-217);
  - algorithmic bytes per environment per step (computed from the shapes below) and the share of 3.35 TB/s they imply at the
    measured kernel time;
  - the card's name, power limit and SM clock, read in the same run.

    python scripts/semi_implicit_bench.py [--envs 4096] [--iters 200]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import newton_b200  # noqa: E402
from newton_b200 import _lib, scenes  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
REFERENCE_LAUNCHES = 4  # eval_body_joints + eval_body_contact + integrate_bodies + the clone of body_f
DT = 1e-3


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout
        power, max_sm, sm = (float(x) for x in q.splitlines()[0].split(","))
    except (OSError, subprocess.SubprocessError, ValueError, IndexError):
        power = max_sm = sm = None
    return {"card": name, "power_limit_w": power, "sm_clock_max_mhz": max_sm, "sm_clock_mhz": sm}


def algorithmic_bytes(model, contacts_per_env):
    """Bytes one step must move per environment: body_q / body_qd read and written, body_f read (4 B floats); the model's per-body
    constants (com, mass, inertia and its inverse, flags, world); per joint its frames, type / parents / dims / starts and the
    per-dof drive parameters and controls; per live contact the fields the penalty force reads from the contact blocks."""
    E = model.world_count
    nb, nj, nd = model.body_count / E, model.joint_count / E, model.joint_dof_count / E
    body = nb * 4 * (7 + 6 + 6 + 7 + 6 + 3 + 1 + 9 + 9 + 1 + 1 + 1)
    joint = nj * 4 * (7 + 7 + 8) + nd * 4 * (3 + 9 + 3)
    contact = contacts_per_env * 4 * 18
    return body + joint + contact


def run(workload, envs, iters, graph_substeps):
    if workload == "quadruped":
        model = scenes.quadruped_model(envs, seed=1)
        model.joint_q.view(envs, -1)[:, 2] = 0.47  # feet on the ground, so that every substep has contacts
        scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    else:
        model = scenes.box_stack_model(envs, seed=0)
    mg = model.to("cuda:0")
    solver, pipe = newton_b200.solvers.SolverSemiImplicit(mg), newton_b200.CollisionPipeline(mg)
    s0, s1, ctrl, contacts = mg.state(), mg.state(), mg.control(), pipe.contacts()
    states = [s0, s1]

    def substep(k):
        a, b = states[k % 2], states[(k + 1) % 2]
        a.clear_forces()
        pipe.collide(a, contacts)
        solver.step(a, b, ctrl, contacts, DT)

    for k in range(50):  # warm-up: module load, first-call scratch, settle onto the ground
        substep(k)
    torch.cuda.synchronize()
    l0 = _lib.kernel_launch_count()
    substep(0)
    substep(1)
    torch.cuda.synchronize()
    launches = (_lib.kernel_launch_count() - l0) / 2
    n_contacts = int(contacts.rigid_contact_count.item())

    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for k in range(iters):
        substep(k)
    end.record()
    torch.cuda.synchronize()
    eager_us = start.elapsed_time(end) * 1e3 / iters

    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            for k in range(graph_substeps):
                substep(k)
    graph.replay()
    torch.cuda.synchronize()
    reps = max(1, iters // graph_substeps)
    start.record()
    for _ in range(reps):
        graph.replay()
    end.record()
    torch.cuda.synchronize()
    graph_us = start.elapsed_time(end) * 1e3 / (reps * graph_substeps)
    finite = bool(torch.isfinite(states[0].body_q).all())

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:  # a profiler run of its own; no trace is written
        for k in range(50):
            substep(k)
        torch.cuda.synchronize()
    kernel_us = [e.device_time for e in prof.events() if "semi_implicit_step_kernel" in e.name]
    k_us = sum(kernel_us) / len(kernel_us) if kernel_us else None
    per_env = algorithmic_bytes(model, n_contacts / envs)
    share = per_env * envs / (k_us * 1e-6) / HBM_BYTES_PER_S if k_us else None
    return {
        "workload": workload, "envs": envs, "dt": DT, "contacts": n_contacts, "finite": finite,
        "substeps_per_s_graph": 1e6 / graph_us, "substep_us_graph": graph_us,
        "substeps_per_s_eager": 1e6 / eager_us, "substep_us_eager": eager_us,
        "semi_implicit_step_kernel_us": k_us, "launches_per_substep": launches, "reference_launches_per_substep": REFERENCE_LAUNCHES,
        "algorithmic_bytes_per_env": per_env, "hbm_share_at_kernel_time": share, **card(),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--graph-substeps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("semi_implicit_bench.py measures the GPU: no CUDA device")
    for w in ("quadruped", "box_stack"):
        print(json.dumps(run(w, args.envs, args.iters, args.graph_substeps)), flush=True)


if __name__ == "__main__":
    main()

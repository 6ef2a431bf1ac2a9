"""Times the ArticulationView calls of an RL-style reset / observe step on the BASELINE quadruped batch (one GPU).

  python scripts/selection_bench.py [envs=4096] [iters=200] [warmup=20]  -> one JSON line on stdout

Per call: CUDA-event time on the launching stream (median of `iters` after 20 warm-up calls, arrays resident in L2 - they are
0.3-1.5 MB, so this is the state an RL loop sees them in), algorithmic bytes (4 B read + 4 B written per selected word, plus
the mask bytes), GB/s.  `reset_step` is the whole masked reset (4 scatters + mask translation + masked FK), `observe_step`
the observation gather for XPBD (eval_ik + an index-gather of the 12 actuated joint angles and rates).
"""

import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import newton_b200  # noqa: E402
from newton_b200 import JointType, scenes  # noqa: E402
from newton_b200.selection import ArticulationView  # noqa: E402


WARMUP = 20


def timed(fn, iters):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return float(np.median(ts))


def main():
    E = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 200
    global WARMUP
    WARMUP = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    model = scenes.quadruped_model(E, device="cuda:0")
    state = model.state()
    view = ArticulationView(model, "quadruped")
    legs = ArticulationView(model, "quadruped", exclude_joint_types=[int(JointType.FREE)], exclude_links=["base"])
    hips = ArticulationView(model, "quadruped", include_joints=["*_HAA"])  # non-contiguous: strided index-gather
    rng = np.random.default_rng(0)
    done = torch.from_numpy(rng.random(E) < 0.1).to("cuda:0")
    root0 = view.get_root_transforms(model).clone()
    rootv0 = view.get_root_velocities(model).clone()
    q0 = view.get_dof_positions(model).clone()
    qd0 = view.get_dof_velocities(model).clone()
    links = view.get_link_transforms(state).clone()
    out = {}

    def record(name, fn, words, mask_bytes=0):
        us = timed(fn, iters)
        nbytes = 8 * words + mask_bytes
        out[name] = {"us": round(us, 2), "bytes": int(nbytes), "GB_per_s": round(nbytes / us * 1e-3, 1)}

    record("set_dof_positions_masked", lambda: view.set_dof_positions(state, q0, mask=done), E * 19, E)
    record("set_dof_velocities_masked", lambda: view.set_dof_velocities(state, qd0, mask=done), E * 18, E)
    record("set_root_transforms_masked", lambda: view.set_root_transforms(state, root0, mask=done), E * 7, E)
    record("set_link_transforms_all", lambda: view.set_attribute("body_q", state, links), E * 13 * 7)
    record("gather_hip_angles_indexed", lambda: hips.get_dof_positions(state), E * 4)
    record("articulation_mask", lambda: view.get_model_articulation_mask(done), 0, 2 * E)
    record("eval_fk_masked", lambda: view.eval_fk(state, mask=done), 0, E * (19 + 18 + 13 * 13) * 4)
    record("eval_fk_all", lambda: newton_b200.eval_fk(model, state.joint_q, state.joint_qd, state), 0, E * (19 + 18 + 13 * 13) * 4)
    record("eval_ik", lambda: newton_b200.eval_ik(model, state, state.joint_q, state.joint_qd), 0, E * (19 + 18 + 13 * 13) * 4)

    def reset_step():
        view.set_root_transforms(state, root0, mask=done)
        view.set_root_velocities(state, rootv0, mask=done)
        view.set_dof_positions(state, q0, mask=done)
        view.set_dof_velocities(state, qd0, mask=done)
        view.eval_fk(state, mask=done)

    def observe_step():
        newton_b200.eval_ik(model, state, state.joint_q, state.joint_qd)
        return (view.get_root_transforms(state), view.get_root_velocities(state), legs.get_dof_positions(state), legs.get_dof_velocities(state),
                hips.get_dof_positions(state))

    record("reset_step", reset_step, E * (7 + 6 + 19 + 18), 4 * E)
    record("observe_step", observe_step, E * 4, 0)
    try:  # the same five calls captured once and replayed (every entry point is capturable: include/newton_b200.h)
        graph = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            reset_step()
            torch.cuda.synchronize()
            with torch.cuda.graph(graph, stream=s):
                reset_step()
        record("reset_step_cuda_graph", graph.replay, E * (7 + 6 + 19 + 18), 4 * E)
    except Exception as e:  # noqa: BLE001
        out["reset_step_cuda_graph"] = {"error": repr(e)[:300]}
    line = {"workload": f"quadruped x{E}, 10% of worlds reset", "calls": out, "launches": newton_b200._lib.kernel_launch_count()}
    print(json.dumps(line))


if __name__ == "__main__":
    main()

"""Times SensorContact.update on 4096 seeded quadrupeds (scenes.quadruped_model(4096, seed=1), bases lowered to z = 0.48 so the
feet stand on the ground) after 20 XPBD substeps and update_contacts.  Two sensors:

  shanks_vs_ground      sensing_bodies="*SHANK", counterpart = the ground plane   (16 384 rows, 1 column)
  all_shapes_vs_bodies  every quadruped shape (as an index list), counterpart_bodies="*"   (53 248 rows, 13 columns)

Prints one JSON line: microseconds per update (CUDA events; eagerly from Python, and replayed from a CUDA graph), kernel launches per update (the library's own count and every kernel
of one update seen by torch.profiler, the radix sort's included), and as a yardstick the time of torch.index_add_ summing the same
per-side forces into the sensor's rows (total_force only; its float atomics make it non-deterministic), with the card's name and
power limit read in the same run.

    python scripts/sensor_bench.py [--envs 4096] [--iters 200]
"""

from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import newton_b200  # noqa: E402
from newton_b200 import _lib, scenes  # noqa: E402
from newton_b200.sensors import SensorContact  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        power = float(q.splitlines()[0])
    except Exception:
        power = None
    return name, power


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


def graph_time(fn, iters):
    """µs per call when the call is captured into a CUDA graph and replayed: no host marshalling between calls."""
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        fn()
    return time_call(g.replay, iters)


def kernels_per_call(fn, calls=20):
    """(library's own launch count, CUDA kernels per call as torch.profiler records them, and their mean device times in µs:
    a separate profiled run of `calls` calls, so the timed loop above runs without the profiler)."""
    torch.cuda.synchronize()
    l0 = _lib.kernel_launch_count()
    fn()
    torch.cuda.synchronize()
    own = _lib.kernel_launch_count() - l0
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    events = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    times = {}
    for e in events:
        m = re.search(r"(\w*Kernel\w*|\w+_kernel)", e.name)
        key = e.name if e.name.startswith("Memset") else (m.group(1) if m else e.name[:60])
        times[key] = times.get(key, 0.0) + e.device_time / calls
    kernels = sum(1 for e in events if not e.name.startswith(("Memset", "Memcpy"))) // calls
    return own, kernels, {k: round(v, 2) for k, v in times.items()}


def quadrupeds(envs):
    model = scenes.quadruped_model(envs, seed=1)
    model.joint_q.view(envs, -1)[:, 2] = 0.48
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    return model.to("cuda:0")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sensor_bench.py measures on a CUDA device; none is visible")
    model = quadrupeds(args.envs)
    shapes = [int(s) for s in np.flatnonzero(model.numpy("shape_world") >= 0)]
    ground = [int(s) for s in np.flatnonzero(model.numpy("shape_world") < 0)]
    sensors = {  # built before the Contacts buffer: they request Contacts.force
        "shanks_vs_ground": SensorContact(model, sensing_bodies="*SHANK", counterpart_shapes=ground),
        "all_shapes_vs_bodies": SensorContact(model, sensing_shapes=shapes, counterpart_bodies="*"),
    }
    pipe = newton_b200.CollisionPipeline(model)
    solver = newton_b200.solvers.SolverXPBD(model, iterations=4)
    s0, s1, ctrl, contacts = model.state(), model.state(), model.control(), pipe.contacts()
    for _ in range(20):
        s0.clear_forces()
        pipe.collide(s0, contacts)
        solver.step(s0, s1, ctrl, contacts, 0.005)
        s0, s1 = s1, s0
    solver.update_contacts(contacts)
    torch.cuda.synchronize()
    n = int(contacts.rigid_contact_count.item())
    out = {"envs": args.envs, "iters": args.iters, "contacts": n, "rigid_contact_max": contacts.rigid_contact_max, "configs": {}}
    state = types.SimpleNamespace(body_q=s0.body_q)
    for name, sensor in sensors.items():
        fn = lambda sensor=sensor: sensor.update(state, contacts)  # noqa: E731
        us = time_call(fn, args.iters)
        us_graph = graph_time(fn, args.iters)
        own, kernels, kernel_us = kernels_per_call(fn)
        # yardstick: the same per-side forces summed into the rows with torch.index_add_ (float atomics)
        s0_, s1_ = contacts.rigid_contact_shape0[:n].long(), contacts.rigid_contact_shape1[:n].long()
        f = contacts.force[:n, :3]
        rows = sensor._sensing_shape_to_row.long()
        R = len(sensor.sensing_indices)
        idx = torch.cat([rows[s0_], rows[s1_]])
        vals = torch.cat([f, -f])
        keep = idx >= 0  # unsensed sides
        idx, vals = idx[keep], vals[keep]
        acc = torch.zeros(R, 3, device="cuda:0")

        def index_add():
            acc.zero_()
            acc.index_add_(0, idx, vals)

        us_ia = time_call(index_add, args.iters)
        index_add()
        sensor.update(state, contacts)
        torch.cuda.synchronize()
        rel = float((acc - sensor.total_force).abs().max() / sensor.total_force.abs().max().clamp(min=1e-30))
        out["configs"][name] = {
            "rows": R, "cols": sensor._max_cols, "us_per_update": round(us, 2), "us_per_update_graph_replay": round(us_graph, 2), "own_launches_per_update": own,
            "kernels_per_update": kernels, "kernel_us": kernel_us, "index_add_total_force_us": round(us_ia, 2), "index_add_max_rel_diff": rel,
        }
    name, power = card()
    out["card"] = name
    out["power_limit_w"] = power
    print(json.dumps(out))


if __name__ == "__main__":
    main()

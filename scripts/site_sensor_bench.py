"""Times SensorFrameTransform.update and SensorIMU.update on 4096 seeded quadrupeds (scenes.quadruped_model(4096, seed=1), bases
lowered to z = 0.48 so the feet stand on the ground) after 20 XPBD substeps; body_qdd is (qd_out - qd_in) / dt of the last substep.
Every quadruped carries a base IMU site and four foot sites (``sites=5``); a second copy of the scene carries 16 sites per
quadruped (``sites=16``, the same bodies, so the same state).  Three workloads:

  feet_in_base   SensorFrameTransform, the four feet of every quadruped relative to its base site      (16 384 outputs)
  base_imu       SensorIMU at the base site                                                          (4 096 sensors)
  sites16        SensorFrameTransform, all 16 sites of every quadruped relative to its base site     (65 536 outputs)

Prints one JSON line: µs per update (CUDA events; eagerly from Python, and replayed from a CUDA graph), the kernel's device time
from torch.profiler in a separate run, the library's launch count and the reference's (counted from its code: two launches per
frame update, one per IMU update), the algorithmic bytes per update (every byte the kernel issues, no reuse counted) and the share of
3.35 TB/s they imply at the profiled kernel time; as a yardstick the same math written as a torch composition over the same tensors,
its time and its largest difference from the kernel; the collide kernel's device time per substep with and without the five sites
per quadruped; and the card's name and power limit, read in the same run.

    python scripts/site_sensor_bench.py [--envs 4096] [--iters 200]
"""

from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import newton_b200  # noqa: E402
from newton_b200 import _lib, scenes  # noqa: E402
from newton_b200.sensors import SensorFrameTransform, SensorIMU  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sensor_bench import card, graph_time, time_call  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM 80 GB HBM3 peak
FRAME_BYTES = 2 * 4 + 2 * (4 + 28 + 28) + 28  # two ids; per side shape_body, shape_transform, body_q; the output transform
IMU_BYTES = 4 + 4 + 28 + 4 + 12 + 12 + 16 + 12 + 24 + 24  # site, shape_body, shape_transform, body_world, gravity, body_com,
#                                                           body_q rotation, angular body_qd, body_qdd, both outputs


def quadrupeds(envs, sites):
    model = scenes.quadruped_model(envs, seed=1, sites=sites)
    model.joint_q.view(envs, -1)[:, 2] = 0.48
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    model.request_state_attributes("body_qdd")
    return model.to("cuda:0")


def kernel_us(fn, calls=20, match=None):
    """Mean device time per call of the CUDA kernels whose name contains `match` (all kernels when None), from torch.profiler."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    events = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memset", "Memcpy"))]
    picked = [e for e in events if match is None or match in e.name]
    return sum(e.device_time for e in picked) / calls, len(picked) // calls


# ---------------------------------------------------------------------------------------------------------- torch yardstick
def _qmul(a, b):
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + bw * ax + ay * bz - by * az, aw * by + bw * ay + az * bx - bz * ax,
                        aw * bz + bw * az + ax * by - bx * ay, aw * bw - ax * bx - ay * by - az * bz], -1)


def _qrot(q, v, sign=1.0):
    x, y, z, w = q.unbind(-1)
    vx, vy, vz = v.unbind(-1)
    c = 2.0 * w * w - 1.0
    d = 2.0 * (x * vx + y * vy + z * vz)
    return torch.stack([vx * c + x * d + sign * (y * vz - z * vy) * w * 2.0, vy * c + y * d + sign * (z * vx - x * vz) * w * 2.0,
                        vz * c + z * d + sign * (x * vy - y * vx) * w * 2.0], -1)


def _conj(q):
    return torch.cat([-q[..., :3], q[..., 3:]], -1)


def _world(model, body_q, s):
    b = model.shape_body[s].long()
    xs = model.shape_transform[s]
    xb = body_q[b.clamp(min=0)]
    x = torch.cat([_qrot(xb[:, 3:], xs[:, :3]) + xb[:, :3], _qmul(xb[:, 3:], xs[:, 3:])], -1)
    return torch.where((b >= 0)[:, None], x, xs)


def torch_frame(model, body_q, shapes, refs):
    xo, xr = _world(model, body_q, shapes), _world(model, body_q, refs)
    qi = _conj(xr[:, 3:])
    p_inv = -_qrot(qi, xr[:, :3])
    return torch.cat([_qrot(qi, xo[:, :3]) + p_inv, _qmul(qi, xo[:, 3:])], -1)


def torch_imu(model, state, sites):
    b = model.shape_body[sites].long()  # every bench site sits on a body
    xs = model.shape_transform[sites]
    g = model.gravity[model.body_world[b].long()]
    qb = state.body_q[b, 3:]
    r = _qrot(qb, xs[:, :3] - model.body_com[b])
    w, acc = state.body_qd[b, 3:], state.body_qdd[b]
    a = ((acc[:, :3] - g) + torch.linalg.cross(acc[:, 3:], r)) + torch.linalg.cross(w, torch.linalg.cross(w, r))
    q = _qmul(qb, xs[:, 3:])
    return _qrot(q, a, -1.0), _qrot(q, w, -1.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("site_sensor_bench.py measures on a CUDA device; none is visible")
    dt = 0.005
    plain, m5, m16 = quadrupeds(args.envs, 0), quadrupeds(args.envs, 5), quadrupeds(args.envs, 16)

    # collide kernel time per substep, without and with the five sites per quadruped (same state: sites move no body)
    collide = {}
    for name, model in (("no_sites", plain), ("five_sites", m5)):
        pipe = newton_b200.CollisionPipeline(model)
        state, contacts = model.state(), pipe.contacts()
        collide[name] = round(kernel_us(lambda pipe=pipe, state=state, contacts=contacts: pipe.collide(state, contacts), match="collide")[0], 2)

    pipe = newton_b200.CollisionPipeline(m5)
    solver = newton_b200.solvers.SolverXPBD(m5, iterations=4)
    s0, s1, ctrl, contacts = m5.state(), m5.state(), m5.control(), pipe.contacts()
    for _ in range(20):
        s0.clear_forces()
        pipe.collide(s0, contacts)
        solver.step(s0, s1, ctrl, contacts, dt)
        s1.body_qdd.copy_((s1.body_qd - s0.body_qd) / dt)
        s0, s1 = s1, s0
    torch.cuda.synchronize()
    state = s0

    def tables(model, names):
        labels = model.shape_label
        imu = [i for i, label in enumerate(labels) if label == "quadruped/imu"]
        picked = [i for i, label in enumerate(labels) if names(label)]
        per = len(picked) // len(imu)
        return imu, picked, [s for s in imu for _ in range(per)]

    imu5, feet, feet_refs = tables(m5, lambda label: label.endswith("_foot"))
    _, all16, all16_refs = tables(m16, lambda label: label.startswith("quadruped/") and label.count("/") == 1)
    idx = {k: torch.tensor(v, device="cuda:0") for k, v in (("feet", feet), ("feet_refs", feet_refs), ("imu5", imu5), ("all16", all16),
                                                              ("all16_refs", all16_refs))}
    workloads = {
        "feet_in_base": (SensorFrameTransform(m5, feet, feet_refs), FRAME_BYTES, 2,
                         lambda: torch_frame(m5, state.body_q, idx["feet"], idx["feet_refs"])),
        "base_imu": (SensorIMU(m5, imu5), IMU_BYTES, 1, lambda: torch_imu(m5, state, idx["imu5"])),
        "sites16": (SensorFrameTransform(m16, all16, all16_refs), FRAME_BYTES, 2,
                    lambda: torch_frame(m16, state.body_q, idx["all16"], idx["all16_refs"])),
    }
    out = {"envs": args.envs, "iters": args.iters, "workloads": {}, "collide_kernel_us_per_substep": collide}
    for name, (sensor, per_output, ref_launches, fn_yard) in workloads.items():
        fn = lambda sensor=sensor: sensor.update(state)  # noqa: E731
        us = time_call(fn, args.iters)
        us_graph = graph_time(fn, args.iters)
        l0 = _lib.kernel_launch_count()
        fn()
        torch.cuda.synchronize()
        own = _lib.kernel_launch_count() - l0
        k_us, k_count = kernel_us(fn)
        n = len(sensor.sensor_sites_arr) if isinstance(sensor, SensorIMU) else int(sensor.transforms.shape[0])
        nbytes = n * per_output
        # yardstick: the same math as a torch composition over the same tensors (index tensors built outside the timed call)
        probe = fn_yard()
        probe = probe if isinstance(probe, tuple) else (probe,)
        got = (sensor.accelerometer, sensor.gyroscope) if isinstance(sensor, SensorIMU) else (sensor.transforms,)
        diff = max(float((g - t).abs().max()) for g, t in zip(got, probe))
        us_yard = time_call(fn_yard, args.iters)
        y_us, y_count = kernel_us(fn_yard)
        out["workloads"][name] = {
            "outputs": n, "us_per_update": round(us, 2), "us_per_update_graph_replay": round(us_graph, 2), "kernel_us": round(k_us, 2),
            "kernels_per_update": k_count, "own_launches_per_update": own, "reference_launches_per_update": ref_launches,
            "algorithmic_bytes": nbytes, "hbm_share_at_kernel_time": round(nbytes / (k_us * 1e-6) / HBM_BYTES_PER_S, 4),
            "torch_us_per_update": round(us_yard, 2), "torch_kernel_us": round(y_us, 2), "torch_kernels_per_update": y_count,
            "torch_max_abs_diff": diff,
        }
    name, power = card()
    out["card"] = name
    out["power_limit_w"] = power
    print(json.dumps(out))


if __name__ == "__main__":
    main()

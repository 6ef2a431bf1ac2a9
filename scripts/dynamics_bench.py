"""Times the articulation dynamics queries on the bench batch: 4096 quadrupeds built like bench.py's scene (default_rng(1)),
body poses from eval_fk.  Prints one JSON line: microseconds and launches per call of eval_jacobian, eval_mass_matrix,
eval_inverse_dynamics_passive (M only, and M + g + C qd), eval_inverse_dynamics_force, the bytes each call must move (computed
from the shapes), their share of the H100 SXM's 3.35 TB/s HBM3 figure, and the torch.einsum H = J^T I J a user would write
without eval_mass_matrix as a same-process baseline, with the card's name and power limit read in the same run.

    python scripts/dynamics_bench.py [--envs 4096] [--iters 200]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import newton_b200  # noqa: E402
from newton_b200 import _lib, scenes  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


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
    l0 = _lib.kernel_launch_count()
    fn()
    launches = _lib.kernel_launch_count() - l0
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters, launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dynamics_bench.py measures on a CUDA device; none is visible")
    model = scenes.quadruped_model(args.envs, seed=1).to("cuda:0")
    state = model.state()
    state.joint_qd = torch.tensor(np.random.default_rng(1).normal(0.0, 0.5, model.joint_dof_count), dtype=torch.float32, device="cuda:0")
    newton_b200.eval_fk(model, state.joint_q, state.joint_qd, state)
    A, L, D = model.articulation_count, model.max_joints_per_articulation, model.max_dofs_per_articulation
    nb, nd, nq = model.body_count, model.joint_dof_count, model.joint_coord_count
    J = torch.empty(A, 6 * L, D, device="cuda:0")
    H = torch.empty(A, D, D, device="cuda:0")
    g, c, tau = (torch.empty(nd, device="cuda:0") for _ in range(3))
    qdd = torch.randn(nd, device="cuda:0")

    # algorithmic bytes: model rows every kernel must read per body / joint (pose, COM, mass, inertia; joint header words) +
    # state inputs + outputs, 4-byte words
    body_in = nb * (7 + 3 + 1 + 9) * 4
    joint_hdr = model.joint_count * (1 + 1 + 1 + 1 + 1 + 2 + 7) * 4 + nd * 3 * 4
    f32 = 4
    bytes_ = {
        "eval_jacobian": body_in + joint_hdr + nq * f32 + J.numel() * f32,
        "eval_mass_matrix": body_in + joint_hdr + nq * f32 + H.numel() * f32,
        "eval_inverse_dynamics_passive_M": body_in + joint_hdr + nq * f32 + H.numel() * f32,
        "eval_inverse_dynamics_passive_all": body_in + joint_hdr + (nq + nd) * f32 + H.numel() * f32 + 2 * nd * f32,
        "eval_inverse_dynamics_force": nb * 7 * f32 + joint_hdr + H.numel() * f32 + 4 * nd * f32,
    }
    calls = {
        "eval_jacobian": lambda: newton_b200.eval_jacobian(model, state, J=J),
        "eval_mass_matrix": lambda: newton_b200.eval_mass_matrix(model, state, H=H),
        "eval_inverse_dynamics_passive_M": lambda: newton_b200.eval_inverse_dynamics_passive(model, state, mass_matrix=H),
        "eval_inverse_dynamics_passive_all": lambda: newton_b200.eval_inverse_dynamics_passive(model, state, mass_matrix=H, gravity_force=g,
                                                                                               coriolis_force=c),
        "eval_inverse_dynamics_force": lambda: newton_b200.eval_inverse_dynamics_force(model, state, mass_matrix=H, joint_qdd=qdd,
                                                                                       coriolis_force=c, gravity_force=g, joint_f=tau),
    }
    out = {"envs": args.envs, "articulation": {"links": L, "dofs": D}, "iters": args.iters, "calls": {}}
    for name, fn in calls.items():
        us, launches = time_call(fn, args.iters)
        out["calls"][name] = {"us_per_call": round(us, 2), "launches_per_call": launches, "bytes": int(bytes_[name]),
                              "hbm_share": round(bytes_[name] / (us * 1e-6) / HBM_BYTES_PER_S, 4)}

    # baseline a user would write without eval_mass_matrix: H = sum_links J_i^T I_i J_i with torch.einsum over this library's J
    newton_b200.eval_jacobian(model, state, J=J)
    links = model.joint_child.view(A, L).long()
    bq = state.body_q[links]  # [A, L, 7]
    qx, qy, qz, qw = bq[..., 3], bq[..., 4], bq[..., 5], bq[..., 6]
    R = torch.stack([1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw),
                     2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw),
                     2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)], -1).view(A, L, 3, 3)
    Iw = R @ model.body_inertia[links] @ R.transpose(-1, -2)
    I6 = torch.zeros(A, L, 6, 6, device="cuda:0")
    I6[..., :3, :3] = model.body_mass[links][..., None, None] * torch.eye(3, device="cuda:0")
    I6[..., 3:, 3:] = Iw
    Jl = J.view(A, L, 6, D)

    def einsum_H():
        return torch.einsum("alki,alkm,almj->aij", Jl, I6, Jl)

    us_e, _ = time_call(einsum_H, args.iters)
    newton_b200.eval_mass_matrix(model, state, H=H)
    He = einsum_H()
    torch.cuda.synchronize()
    rel = float((He - H).abs().max() / H.abs().max())
    out["einsum_baseline"] = {"us_per_call": round(us_e, 2), "max_rel_diff_vs_eval_mass_matrix": rel, "agrees_1e-5": rel < 1e-5}
    name, power = card()
    out["card"] = name
    out["power_limit_w"] = power
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Models and solver set-ups shared by tests/test_ik.py (CPU oracle) and tests/test_gpu_ik.py (CUDA parity).

The small models restate the builders of the reference's newton/tests/test_ik.py; the arm and the quadruped come from
newton_b200.scenes.  Every case is a function ``(device) -> (model, objectives, q0)`` that builds fresh tensors on ``device``.
"""

from __future__ import annotations

import numpy as np
import torch

import newton_b200 as nb
from newton_b200 import ik, scenes
from newton_b200.utils import xform as X


def two_link_planar(device="cpu"):
    b = nb.ModelBuilder()
    l1 = b.add_link(xform=X.transform((0.5, 0.0, 0.0)), mass=1.0)
    j1 = b.add_joint_revolute(-1, l1, parent_xform=X.transform((0.0, 0.0, 0.0)), child_xform=X.transform((-0.5, 0.0, 0.0)), axis=(0.0, 0.0, 1.0))
    l2 = b.add_link(xform=X.transform((1.5, 0.0, 0.0)), mass=1.0)
    j2 = b.add_joint_revolute(l1, l2, parent_xform=X.transform((0.5, 0.0, 0.0)), child_xform=X.transform((-0.5, 0.0, 0.0)), axis=(0.0, 0.0, 1.0))
    b.add_articulation([j1, j2])
    m = b.finalize(device="cpu")
    return m.to(device) if str(device) != "cpu" else m


def free_revolute(device="cpu"):
    """A FREE root carrying one revolute link (the reference's free + revolute convergence case)."""
    b = nb.ModelBuilder()
    base = b.add_link(xform=X.transform((0.0, 0.0, 0.5)), mass=1.0, inertia=np.eye(3) * 0.1, com=(0.05, 0.02, 0.0))
    j0 = b.add_joint_free(base)
    arm = b.add_link(xform=X.transform((0.5, 0.0, 0.5)), mass=1.0, inertia=np.eye(3) * 0.1)
    j1 = b.add_joint_revolute(base, arm, parent_xform=X.transform((0.25, 0.0, 0.0)), child_xform=X.transform((-0.25, 0.0, 0.0)),
                              axis=(0.0, 1.0, 0.0))
    b.add_articulation([j0, j1])
    m = b.finalize(device="cpu")
    return m.to(device) if str(device) != "cpu" else m


def d6_six_axis(device="cpu"):
    """One D6 joint with three linear and three angular axes driving a single body."""
    b = nb.ModelBuilder()
    link = b.add_link(mass=1.0, inertia=np.eye(3) * 0.1)
    cfg = nb.JointDofConfig
    j = b.add_joint_d6(-1, link, linear_axes=[cfg(axis=a) for a in ((1, 0, 0), (0, 1, 0), (0, 0, 1))],
                       angular_axes=[cfg(axis=a) for a in ((1, 0, 0), (0, 1, 0), (0, 0, 1))], child_xform=X.transform((0.1, 0.0, 0.0)))
    b.add_articulation([j])
    m = b.finalize(device="cpu")
    return m.to(device) if str(device) != "cpu" else m


def descendant_chain(device="cpu", kind="free"):
    """Revolute root, then a FREE (or DISTANCE) joint, then a revolute: quaternion joints below the root."""
    b = nb.ModelBuilder()
    l0 = b.add_link(mass=1.0, inertia=np.eye(3) * 0.1)
    j0 = b.add_joint_revolute(-1, l0, parent_xform=X.transform((0.0, 0.0, 0.5)), axis=(0.0, 0.0, 1.0))
    l1 = b.add_link(xform=X.transform((0.4, 0.0, 0.5)), mass=1.0, inertia=np.eye(3) * 0.1, com=(0.0, 0.03, 0.0))
    if kind == "free":
        j1 = b.add_joint_free(l1, parent=l0, parent_xform=X.transform((0.4, 0.0, 0.0)))
    else:
        j1 = b.add_joint_distance(l0, l1, parent_xform=X.transform((0.4, 0.0, 0.0)), min_distance=-1.0, max_distance=1.0)
    l2 = b.add_link(xform=X.transform((0.8, 0.0, 0.5)), mass=1.0, inertia=np.eye(3) * 0.1)
    j2 = b.add_joint_revolute(l1, l2, parent_xform=X.transform((0.4, 0.0, 0.0)), axis=(0.0, 1.0, 0.0))
    b.add_articulation([j0, j1, j2])
    m = b.finalize(device="cpu")
    return m.to(device) if str(device) != "cpu" else m


def tensor(a, device):
    return torch.as_tensor(np.asarray(a, dtype=np.float32)).to(device)


def start_q(model, n: int) -> torch.Tensor:
    return model.joint_q.detach().cpu().reshape(1, -1).repeat(n, 1).contiguous()


def random_arm_targets(n: int, seed: int):
    """Reachable hand poses of the arm: FK (the oracle's residual pass with zero targets) of joint configurations drawn inside the
    joint ranges.  Returns (positions [n, 3], rotations [n, 4] xyzw, the configurations)."""
    import oracle.ik as oik

    model = scenes.panda_arm_model()
    rng = np.random.default_rng(seed)
    lo, hi = model.numpy("joint_limit_lower"), model.numpy("joint_limit_upper")
    q = (lo + (hi - lo) * rng.uniform(0.15, 0.85, size=(n, len(lo)))).astype(np.float32)
    pos = ik.IKObjectivePosition(7, (0.0, 0.0, 0.0), np.zeros((n, 3), np.float32))
    rot = ik.IKObjectiveRotation(7, (0.0, 0.0, 0.0, 1.0), np.tile(np.float32([0, 0, 0, 1]), (n, 1)), canonicalize_quat_err=False)
    s = ik.IKSolver(model, n, [pos, rot], jacobian_mode="analytic")
    qt = torch.from_numpy(q)
    with oik.host():
        s._impl.compute_costs(qt)
    r = s.residuals.numpy().astype(np.float64)
    p = -r[:, :3]
    aa = r[:, 3:6]
    ang = np.linalg.norm(aa, axis=1, keepdims=True)
    axis = np.where(ang > 1e-12, aa / np.maximum(ang, 1e-300), 0.0)
    quat = np.concatenate([axis * np.sin(0.5 * ang), np.cos(0.5 * ang)], axis=1)
    return p.astype(np.float32), quat.astype(np.float32), q


def arm_problem(device, n: int, seed: int = 0, weight: float = 10.0, limits: bool = True):
    """The example_ik_franka setting: hand position + rotation (+ joint limits), every weight `weight`."""
    model = scenes.panda_arm_model(device)
    p, qr, _ = random_arm_targets(n, seed)
    objs = [ik.IKObjectivePosition(7, (0.0, 0.0, 0.0), tensor(p, device), weight=weight),
            ik.IKObjectiveRotation(7, (0.0, 0.0, 0.0, 1.0), tensor(qr, device), weight=weight)]
    if limits:
        objs.append(ik.IKObjectiveJointLimit(model.joint_limit_lower, model.joint_limit_upper, weight=weight))
    return model, objs, start_q(model, n).to(device)


QUAD_FEET = (3, 6, 9, 12)  # shank bodies of scenes.quadruped_builder()
FOOT = (0.0, 0.0, -0.25)


def quadruped_problem(device, n: int, seed: int = 0):
    """Foot placement for one quadruped: four foot positions, the base orientation and the joint limits; targets are the
    feet / base of randomly perturbed stances."""
    import oracle.ik as oik

    b = scenes.quadruped_builder()
    model = b.finalize(device="cpu")
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    rng = np.random.default_rng(seed)
    q = model.joint_q.numpy().astype(np.float64).reshape(1, -1).repeat(n, 0)
    q[:, 7:] += rng.normal(0.0, 0.25, size=(n, q.shape[1] - 7))
    q[:, :3] += rng.normal(0.0, 0.05, size=(n, 3))
    q = q.astype(np.float32)
    objs = [ik.IKObjectivePosition(f, FOOT, np.zeros((n, 3), np.float32)) for f in QUAD_FEET]
    s = ik.IKSolver(model, n, objs, jacobian_mode="analytic")
    with oik.host():
        s._impl.compute_costs(torch.from_numpy(q))
    feet = -s.residuals.numpy().reshape(n, 4, 3)
    base_rot = q[:, 3:7]
    m = model.to(device) if str(device) != "cpu" else model
    objs = [ik.IKObjectivePosition(f, FOOT, tensor(feet[:, i], device)) for i, f in enumerate(QUAD_FEET)]
    objs.append(ik.IKObjectiveRotation(0, (0.0, 0.0, 0.0, 1.0), tensor(base_rot, device)))
    objs.append(ik.IKObjectiveJointLimit(m.joint_limit_lower, m.joint_limit_upper, weight=0.1))
    return m, objs, start_q(m, n).to(device)


def planar_problem(device, n: int = 3):
    m = two_link_planar(device)
    tgt = tensor([[1.5, 1.0, 0.0], [0.5, 1.2, 0.0], [-1.0, 1.0, 0.0], [1.2, -1.1, 0.0]][:n], device)
    q0 = tensor([[0.1, 0.2]] * n, device)
    return m, [ik.IKObjectivePosition(1, (0.5, 0.0, 0.0), tgt)], q0


def free_revolute_problem(device, n: int = 2):
    m = free_revolute(device)
    tgt = tensor([[0.9, 0.3, 0.7], [0.2, -0.4, 1.1]][:n], device)
    return m, [ik.IKObjectivePosition(1, (0.25, 0.0, 0.0), tgt)], start_q(m, n).to(device)


def d6_problem(device, n: int = 2):
    m = d6_six_axis(device)
    tgt = tensor([[0.3, -0.2, 0.5], [-0.4, 0.1, 0.2]][:n], device)
    rq = [X.quat_from_axis_angle((0.0, 0.0, 1.0), 0.7), X.quat_from_axis_angle((1.0, 1.0, 0.0), -0.5)]
    rot = tensor(np.asarray(rq[:n], dtype=np.float32) / np.linalg.norm(np.asarray(rq[:n]), axis=1, keepdims=True), device)
    return m, [ik.IKObjectivePosition(0, (0.0, 0.0, 0.0), tgt), ik.IKObjectiveRotation(0, (0.0, 0.0, 0.0, 1.0), rot)], start_q(m, n).to(device)


def descendant_problem(device, kind="free", n: int = 2):
    m = descendant_chain(device, kind)
    tgt = tensor([[0.6, 0.5, 0.6], [0.9, -0.3, 0.4]][:n], device)
    rq = np.asarray([X.quat_from_axis_angle((0.0, 0.0, 1.0), 0.4), X.quat_from_axis_angle((0.0, 1.0, 0.0), 0.3)][:n], dtype=np.float32)
    return m, [ik.IKObjectivePosition(2, (0.2, 0.0, 0.0), tgt), ik.IKObjectiveRotation(2, (0.0, 0.0, 0.0, 1.0), tensor(rq, device))], \
        start_q(m, n).to(device)


def position_error(model_cpu, objectives, q) -> np.ndarray:
    """|target - p| of the first objective (a position objective) at configurations q (oracle FK)."""
    import oracle.ik as oik

    o = objectives[0]
    n = q.shape[0]
    pos = ik.IKObjectivePosition(o.link_index, o.link_offset, o.target_positions.detach().cpu().clone())
    s = ik.IKSolver(model_cpu, n, [pos], jacobian_mode="mixed")
    with oik.host():
        s._impl.compute_costs(q.detach().cpu().contiguous())
    return np.linalg.norm(s.residuals.numpy(), axis=1)


def rotation_error(r_rows: np.ndarray, weight: float) -> np.ndarray:
    return np.linalg.norm(r_rows, axis=1) / weight


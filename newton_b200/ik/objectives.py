"""IK objectives (reference ``newton.ik`` objectives, ``sim/ik/ik_objectives.py``).

The objectives are descriptions: the fused LM kernel (``csrc/nb2_ik.cu``) evaluates their residual rows and analytic Jacobian
columns, in list order, from the tables the solver builds at construction.  Per-problem targets are float32 tensors on the model's
device; the ``set_target_*`` calls are device writes, so they can run beside or inside a captured CUDA graph.
"""

from __future__ import annotations

from enum import Enum

import numpy as np
import torch


class IKJacobianType(Enum):
    """Backend used for the Jacobian (reference ``IKJacobianType``).  This library builds ``ANALYTIC`` and ``MIXED``; ``AUTODIFF``
    needs differentiable kernels, which it does not have."""

    AUTODIFF = "autodiff"
    ANALYTIC = "analytic"
    MIXED = "mixed"


def _vec_targets(a, width: int, name: str) -> torch.Tensor:
    t = a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a, dtype=np.float32))
    if t.dtype != torch.float32:
        raise ValueError(f"{name}: expected float32 values, got {t.dtype}")
    t = t.reshape(-1, width)
    return t if t.is_contiguous() else t.contiguous()


class IKObjective:
    """Base class of the built-in objectives.  Each contributes :meth:`residual_dim` consecutive residual rows; user subclasses are
    not evaluated by this library (their residuals would be Warp kernels) and the solver refuses them."""

    def __init__(self) -> None:
        self.total_residuals = None
        self.residual_offset = None
        self.n_batch = None
        self.device = None

    def set_batch_layout(self, total_residuals: int, residual_offset: int, n_batch: int) -> None:
        """Register this objective's rows inside the optimizer's residual vector."""
        self.total_residuals = total_residuals
        self.residual_offset = residual_offset
        self.n_batch = n_batch

    def _require_batch_layout(self) -> None:
        if self.total_residuals is None or self.residual_offset is None or self.n_batch is None:
            raise RuntimeError(f"Batch layout not assigned for {type(self).__name__}; call set_batch_layout() first")

    def residual_dim(self) -> int:
        raise NotImplementedError

    def supports_analytic(self) -> bool:
        return False

    def bind_device(self, device) -> None:
        self.device = torch.device(device)


class IKObjectivePosition(IKObjective):
    """Match the world position of the point ``link_offset`` (link frame) of body ``link_index``: residual
    ``weight * (target - p)``, Jacobian ``-weight * (v + w x p)`` over the link's ancestor dofs.

    ``target_positions``: ``[problem_count, 3]`` float32 tensor (or array-like, copied to the model's device)."""

    def __init__(self, link_index: int, link_offset, target_positions, weight: float = 1.0) -> None:
        super().__init__()
        self.link_index = int(link_index)
        self.link_offset = tuple(float(x) for x in link_offset)
        self.target_positions = _vec_targets(target_positions, 3, "target_positions")
        self.weight = float(weight)

    def bind_device(self, device) -> None:
        super().bind_device(device)
        t = self.target_positions
        if not isinstance(t, torch.Tensor) or t.device != self.device:
            if isinstance(t, torch.Tensor) and t.device.type != "cpu":
                raise ValueError(f"target_positions live on {t.device}, the model is on {self.device}")
            self.target_positions = t.to(self.device)

    def supports_analytic(self) -> bool:
        return True

    def residual_dim(self) -> int:
        return 3

    def set_target_position(self, problem_idx: int, new_position) -> None:
        """Replace the target of one base problem (three device fills, no host synchronisation)."""
        self._require_batch_layout()
        for c in range(3):
            self.target_positions[problem_idx, c].fill_(float(new_position[c]))

    def set_target_positions(self, new_positions) -> None:
        """Replace every target: a device-to-device copy of ``new_positions`` ``[problem_count, 3]``."""
        self._require_batch_layout()
        expected = self.target_positions.shape[0]
        if new_positions.shape[0] != expected:
            raise ValueError(f"Expected {expected} target positions, got {new_positions.shape[0]}")
        self.target_positions.copy_(new_positions.reshape(expected, 3))


class IKObjectiveRotation(IKObjective):
    """Match the world orientation ``body_rot * link_offset_rotation`` of body ``link_index``: residual ``weight`` times the
    axis-angle of ``actual * target^-1`` (flipped onto the short arc with ``canonicalize_quat_err``), Jacobian ``weight * w``.
    Quaternions are ``(x, y, z, w)``; ``target_rotations`` is ``[problem_count, 4]``."""

    def __init__(self, link_index: int, link_offset_rotation, target_rotations, canonicalize_quat_err: bool = True,
                 weight: float = 1.0) -> None:
        super().__init__()
        self.link_index = int(link_index)
        self.link_offset_rotation = tuple(float(x) for x in link_offset_rotation)
        self.target_rotations = _vec_targets(target_rotations, 4, "target_rotations")
        self.canonicalize_quat_err = bool(canonicalize_quat_err)
        self.weight = float(weight)

    def bind_device(self, device) -> None:
        super().bind_device(device)
        t = self.target_rotations
        if t.device != self.device:
            if t.device.type != "cpu":
                raise ValueError(f"target_rotations live on {t.device}, the model is on {self.device}")
            self.target_rotations = t.to(self.device)

    def supports_analytic(self) -> bool:
        return True

    def residual_dim(self) -> int:
        return 3

    def set_target_rotation(self, problem_idx: int, new_rotation) -> None:
        """Replace the target of one base problem (four device fills, no host synchronisation)."""
        self._require_batch_layout()
        for c in range(4):
            self.target_rotations[problem_idx, c].fill_(float(new_rotation[c]))

    def set_target_rotations(self, new_rotations) -> None:
        """Replace every target: a device-to-device copy of ``new_rotations`` ``[problem_count, 4]``."""
        self._require_batch_layout()
        expected = self.target_rotations.shape[0]
        if new_rotations.shape[0] != expected:
            raise ValueError(f"Expected {expected} target rotations, got {new_rotations.shape[0]}")
        self.target_rotations.copy_(new_rotations.reshape(expected, 4))


class IKObjectiveJointLimit(IKObjective):
    """One row per dof: ``weight * (max(0, q - upper) + max(0, lower - q))``, with gradient ``+-weight`` at and beyond a bound.
    Dof k of joint j reads coordinate ``joint_q_start[j] + k`` (upstream's ``dof_to_coord``, also for quaternion joints); a range
    wider than 9.9e5 is treated as unlimited."""

    def __init__(self, joint_limit_lower, joint_limit_upper, weight: float = 0.1) -> None:
        super().__init__()
        self.joint_limit_lower = _vec_targets(joint_limit_lower, 1, "joint_limit_lower").reshape(-1)
        self.joint_limit_upper = _vec_targets(joint_limit_upper, 1, "joint_limit_upper").reshape(-1)
        self.weight = float(weight)
        self.n_dofs = int(self.joint_limit_lower.shape[0])

    def bind_device(self, device) -> None:
        super().bind_device(device)
        for name in ("joint_limit_lower", "joint_limit_upper"):
            t = getattr(self, name)
            if t.device != self.device:
                if t.device.type != "cpu":
                    raise ValueError(f"{name} lives on {t.device}, the model is on {self.device}")
                setattr(self, name, t.to(self.device))

    def supports_analytic(self) -> bool:
        return True

    def residual_dim(self) -> int:
        return self.n_dofs

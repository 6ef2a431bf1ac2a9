"""Batched inverse kinematics (reference ``newton.ik``): Levenberg-Marquardt over position, rotation and joint-limit objectives,
with multi-seed sampling, on one fused CUDA kernel per solve (``csrc/nb2_ik.cu``)."""

from .objectives import IKJacobianType, IKObjective, IKObjectiveJointLimit, IKObjectivePosition, IKObjectiveRotation
from .solver import IKOptimizer, IKOptimizerLM, IKSampler, IKSolver

__all__ = [
    "IKJacobianType",
    "IKObjective",
    "IKObjectiveJointLimit",
    "IKObjectivePosition",
    "IKObjectiveRotation",
    "IKOptimizer",
    "IKOptimizerLM",
    "IKSampler",
    "IKSolver",
]

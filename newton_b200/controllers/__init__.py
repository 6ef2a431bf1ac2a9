"""Controllers (reference ``newton.controllers``): joint-space impedance control of a batch of robots, one fused CUDA launch per
step (``csrc/nb2_dynamics.cu``)."""

from .controller import ControllerBase
from .joint_impedance import ControllerJointImpedance, ControllerJointImpedanceModelFree

__all__ = ["ControllerBase", "ControllerJointImpedance", "ControllerJointImpedanceModelFree"]

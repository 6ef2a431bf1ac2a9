"""Actuators (reference ``newton.actuators``): PD / PID control laws and learned MLP / LSTM actuator networks, command delay
and effort clamping composed into an :class:`Actuator`, stepped on the GPU by one fused kernel per actuator group.  ``ModelBuilder.add_actuator`` groups
compatible actuators into ``Model.actuators`` at ``finalize``."""

from .actuator import Actuator
from .components import (
    Clamping,
    ClampingDCMotor,
    ClampingMaxEffort,
    ClampingPositionBased,
    Controller,
    ControllerPD,
    ControllerPID,
    Delay,
)
from .neural import ControllerNeuralLSTM, ControllerNeuralMLP, load_metadata

__all__ = [
    "Actuator",
    "Clamping",
    "ClampingDCMotor",
    "ClampingMaxEffort",
    "ClampingPositionBased",
    "Controller",
    "ControllerNeuralLSTM",
    "ControllerNeuralMLP",
    "ControllerPD",
    "ControllerPID",
    "Delay",
    "load_metadata",
]

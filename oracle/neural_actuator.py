"""CPU oracle of the learned actuator networks - TEST INFRASTRUCTURE ONLY.

``liboracle_neural_actuator.so`` (``oracle/neural_actuator.cpp`` + ``oracle_neural_actuator.h``, compiled with the flags of
``oracle/Makefile``) restates one step of a ``ControllerNeuralMLP`` / ``ControllerNeuralLSTM`` group serially, under the
arithmetic contract of ``include/newton_b200.h``.  :func:`host` runs the product's own host code (checkpoint loading, network
extraction and packing, descriptor construction and checks) on CPU tensors; network launches go to this oracle and every
other actuator launch to :mod:`oracle.actuator`.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import os
import subprocess

from . import actuator as _act
from .dynamics import _CXXFLAGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle_neural_actuator.so")
_SOURCES = ("neural_actuator.cpp", "oracle_neural_actuator.h", "oracle_actuator.h")
_LIB = None


def build(force: bool = False) -> str:
    """Compile ``liboracle_neural_actuator.so`` with g++ (``-ffp-contract=off``: every fp32 operation rounds as written)."""
    deps = [os.path.join(_HERE, f) for f in _SOURCES] + [os.path.join(_HERE, "..", "include", "newton_b200.h"),
                                                         os.path.join(_HERE, "..", "newton_b200", "csrc", "nb2_math.cuh")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(p) > os.path.getmtime(_SO) for p in deps):
        cxx = os.environ.get("CXX", "g++")
        subprocess.run([cxx, *_CXXFLAGS, "-shared", "-o", _SO, os.path.join(_HERE, "neural_actuator.cpp")], check=True,
                       capture_output=True)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        build()
        _LIB = C.CDLL(_SO)
        P = C.c_void_p
        _LIB.orc_neural_actuator_step.argtypes = [P]
        _LIB.orc_neural_actuator_step.restype = None
        _LIB.orc_neural_actuator_reset.argtypes = [C.c_int32, C.c_int32, C.c_int32, P, P, P]
        _LIB.orc_neural_actuator_reset.restype = None
    return _LIB


def _backend(name, *args):
    from newton_b200 import _abi

    if name == "step" and args[0]._obj.controller in (_abi.ACT_MLP, _abi.ACT_LSTM):
        lib().orc_neural_actuator_step(args[0])
    elif name == "network_reset":
        lib().orc_neural_actuator_reset(*args)
    else:
        _act._backend(name, *args)


@contextlib.contextmanager
def host():
    """Within the block, actuator launches on CPU tensors run on the oracles (the product's single launch point,
    ``newton_b200.actuators.actuator._call``, is wrapped for the block's duration)."""
    from newton_b200.actuators import actuator as A

    product = A._call

    def call(name, device, *args):
        if str(device).startswith("cuda"):
            product(name, device, *args)
        else:
            _backend(name, *args)

    A._call = call
    try:
        yield
    finally:
        A._call = product


def step(actuator, sim_state, sim_control, current_act_state=None, next_act_state=None, dt=None) -> None:
    """``Actuator.step`` on the CPU: same arguments, same checks, outputs written in place."""
    if str(actuator.device) != "cpu":
        raise ValueError("the oracle runs on CPU tensors only")
    with host():
        actuator.step(sim_state, sim_control, current_act_state, next_act_state, dt)


def reset(state, mask=None) -> None:
    """``<state>.reset(mask)`` on the CPU for an ``Actuator.State`` or a network controller's state."""
    with host():
        state.reset(mask)

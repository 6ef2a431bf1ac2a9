"""CPU oracle of the inverse-kinematics solver - TEST INFRASTRUCTURE ONLY.

``liboracle_ik.so`` (``oracle/ik.cpp`` + ``oracle_ik.h``, compiled with the flags of ``oracle/Makefile``) restates the reference's
IK kernels serially, in launch order.  :func:`host` runs the product's own host code (``newton_b200.ik``: validation, objective
tables, the descriptor, the launch sequence of ``IKSolver.step``) on CPU tensors, with only the launches replaced by the oracle.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import os
import subprocess

from .dynamics import _CXXFLAGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle_ik.so")
_SOURCES = ("ik.cpp", "oracle_ik.h", "oracle_dynamics.h", "oracle_featherstone.h", "oracle_xpbd.h", "oracle_math.h")
_LIB = None


def build(force: bool = False) -> str:
    """Compile ``liboracle_ik.so`` with g++ (``-ffp-contract=off``: every fp32 operation rounds as written)."""
    deps = [os.path.join(_HERE, f) for f in _SOURCES] + [os.path.join(_HERE, "..", "include", "newton_b200.h")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(p) > os.path.getmtime(_SO) for p in deps):
        cxx = os.environ.get("CXX", "g++")
        subprocess.run([cxx, *_CXXFLAGS, "-shared", "-o", _SO, os.path.join(_HERE, "ik.cpp")], check=True, capture_output=True)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        _LIB = C.CDLL(_SO)
        P = C.c_void_p
        _LIB.orc_ik_solve.argtypes = [P, P, P, P, P, P, P, P, C.c_int32, C.c_float, C.c_int32, P]
        _LIB.orc_ik_solve.restype = None
        _LIB.orc_ik_sample.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, P, P, P, P, P, C.c_float, P, P]
        _LIB.orc_ik_sample.restype = None
        _LIB.orc_ik_select.argtypes = [C.c_int32, C.c_int32, C.c_int32, P, P, P, P]
        _LIB.orc_ik_select.restype = None
    return _LIB


@contextlib.contextmanager
def host():
    """Within the block, IK launches on CPU tensors run on the oracle: the product's single launch point
    (``newton_b200.ik.solver._call``, which raises for a CPU device) is wrapped for the block's duration."""
    from newton_b200.ik import solver as S

    product = S._call

    def call(name, device, *args):
        if str(device).startswith("cuda"):
            product(name, device, *args)
        else:
            getattr(lib(), f"orc_ik_{name}")(*args)

    S._call = call
    try:
        yield
    finally:
        S._call = product


def step(solver, joint_q_in, joint_q_out, iterations: int = 50, step_size: float = 1.0) -> None:
    """``IKSolver.step`` on the CPU: same arguments, same checks, outputs written in place."""
    if str(solver.device) != "cpu":
        raise ValueError("the oracle runs on CPU tensors only")
    with host():
        solver.step(joint_q_in, joint_q_out, iterations=iterations, step_size=step_size)

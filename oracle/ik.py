"""CPU oracle of the inverse-kinematics solver - TEST INFRASTRUCTURE ONLY.

``oracle/ik.cpp`` + ``oracle_ik.h`` restate the reference's IK kernels serially, in launch order.  :func:`host` runs the product's
own host code (``newton_b200.ik``: validation, objective tables, the descriptor, the launch sequence of ``IKSolver.step``) on CPU
tensors, with only the launches replaced by the oracle.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import functools

from . import build, lib  # noqa: F401  (each module.build is oracle.build: they share one library)


@functools.cache
def _lib():
    L = lib()
    P = C.c_void_p
    L.orc_ik_solve.argtypes = [P, P, P, P, P, P, P, P, C.c_int32, C.c_float, C.c_int32, P]
    L.orc_ik_solve.restype = None
    L.orc_ik_sample.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, P, P, P, P, P, C.c_float, P, P]
    L.orc_ik_sample.restype = None
    L.orc_ik_select.argtypes = [C.c_int32, C.c_int32, C.c_int32, P, P, P, P]
    L.orc_ik_select.restype = None
    return L


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
            getattr(_lib(), f"orc_ik_{name}")(*args)

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

"""CPU oracle of the articulation dynamics queries - TEST INFRASTRUCTURE ONLY.

``oracle/dynamics.cpp`` + ``oracle_dynamics.h`` restate the reference's ``newton.eval_jacobian`` / ``eval_mass_matrix`` /
``eval_inverse_dynamics_passive`` / ``eval_inverse_dynamics_force`` serially, one function per reference function.  The wrappers
take the reference's call signatures and work on CPU models and tensors; outputs are float32 tensors.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from newton_b200 import _abi

from . import build, lib  # noqa: F401  (each module.build is oracle.build: they share one library)


def _check_cpu(model):
    if str(model.device) != "cpu":
        raise ValueError("the oracle runs on CPU tensors only")


def _f32(a):
    return np.ascontiguousarray(a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a), dtype=np.float32)


def _common(model, mask):
    _check_cpu(model)
    d = _abi.model_desc(model)
    art_end = np.ascontiguousarray(model.numpy("articulation_end"), dtype=np.int32)
    m = None if mask is None else np.ascontiguousarray(np.asarray(mask.cpu() if hasattr(mask, "cpu") else mask), dtype=np.uint8)
    return d, art_end, m


def _p(a):
    return C.c_void_p(None if a is None else a.ctypes.data)


def eval_jacobian(model, state, J=None, joint_S_s=None, mask=None):
    """newton.eval_jacobian: J [articulation_count, 6 max_links, max_dofs] (None without articulations)."""
    if model.articulation_count == 0:
        return None
    d, art_end, m = _common(model, mask)
    L, D = int(model.max_joints_per_articulation), int(model.max_dofs_per_articulation)
    out = np.zeros((model.articulation_count, 6 * L, D), dtype=np.float32)
    bq, jq = _f32(state.body_q), _f32(state.joint_q)
    lib().orc_eval_jacobian(C.byref(d), _p(art_end), _p(m), _p(jq), _p(bq), _p(out), C.c_int(L), C.c_int(D))
    return torch.from_numpy(out)


def eval_mass_matrix(model, state, H=None, J=None, body_I_s=None, joint_S_s=None, mask=None):
    """newton.eval_mass_matrix: H [articulation_count, max_dofs, max_dofs]; `J` (optional) is read instead of being computed."""
    if model.articulation_count == 0:
        return None
    d, art_end, m = _common(model, mask)
    L, D = int(model.max_joints_per_articulation), int(model.max_dofs_per_articulation)
    out = np.zeros((model.articulation_count, D, D), dtype=np.float32)
    bq, jq = _f32(state.body_q), _f32(state.joint_q)
    Jn = None if J is None else _f32(J)
    lib().orc_eval_mass_matrix(C.byref(d), _p(art_end), _p(m), _p(jq), _p(bq), _p(Jn), _p(out), C.c_int(L), C.c_int(D))
    return torch.from_numpy(out)


def eval_inverse_dynamics_passive(model, state, *, mass_matrix=False, gravity_force=False, coriolis_force=False, mask=None):
    """newton.eval_inverse_dynamics_passive; pass True for each wanted output.  Returns (M, g, C qd), None where not requested."""
    d, art_end, m = _common(model, mask)
    L, D, nd = int(model.max_joints_per_articulation), int(model.max_dofs_per_articulation), int(model.joint_dof_count)
    M = np.zeros((model.articulation_count, D, D), dtype=np.float32) if mass_matrix else None
    g = np.zeros(nd, dtype=np.float32) if gravity_force else None
    c = np.zeros(nd, dtype=np.float32) if coriolis_force else None
    if model.articulation_count:
        bq, jq, jqd = _f32(state.body_q), _f32(state.joint_q), _f32(state.joint_qd)
        lib().orc_eval_inverse_dynamics_passive(C.byref(d), _p(art_end), _p(m), _p(bq), _p(jq), _p(jqd), _p(M), _p(g), _p(c), C.c_int(L),
                                                C.c_int(D))
    return tuple(None if x is None else torch.from_numpy(x) for x in (M, g, c))


def eval_inverse_dynamics_force(model, state, *, mass_matrix, joint_qdd, coriolis_force, gravity_force, joint_f=None, mask=None):
    """newton.eval_inverse_dynamics_force: returns joint_f (a copy of the given `joint_f`, or zeros, updated like the reference)."""
    d, art_end, m = _common(model, mask)
    D = int(model.max_dofs_per_articulation)
    tau = np.zeros(int(model.joint_dof_count), dtype=np.float32) if joint_f is None else _f32(joint_f).copy()
    if model.articulation_count:
        lib().orc_eval_inverse_dynamics_force(C.byref(d), _p(art_end), _p(m), _p(_f32(state.body_q)), _p(_f32(mass_matrix)),
                                              _p(_f32(joint_qdd)), _p(_f32(coriolis_force)), _p(_f32(gravity_force)), _p(tau), C.c_int(D))
    return torch.from_numpy(tau)

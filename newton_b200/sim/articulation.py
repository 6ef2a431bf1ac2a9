"""Forward kinematics joint_q -> body_q: ``newton.eval_fk``.

Mirrors ``eval_single_articulation_fk`` of the reference (``newton/_src/sim/articulation.py:237-432``):
``X_wc = X_wp * X_pj * X_j(q) * X_cj^-1`` walked in joint order, body twists reported as COM twists.
Called once before the simulation loop by the examples (``example_basic_urdf.py:87``) and on resets.

Runs the FK kernels of the native library through ``nb2_eval_fk`` / ``nb2_eval_fk_masked`` (one warp per articulation;
SURVEY.md §8(f) first "next" row).  CUDA models only, like every call of this package: a model still on the host raises.
(Scene builders that need initial body poses before ``Model.to(device)`` use ``newton_b200.utils.host_fk`` - input
construction, not this function.)
"""

from __future__ import annotations

import torch


def eval_fk(model, joint_q, joint_qd, state, mask=None, indices=None, body_flag_filter: int = 3) -> None:
    """Write ``state.body_q`` / ``state.body_qd`` from generalized coordinates (reference ``sim/articulation.py:500-574``).

    ``state`` may be the model itself (as in ``newton.eval_fk(model, model.joint_q, model.joint_qd, model)``).
    ``mask`` (bool ``[articulation_count]``) or ``indices`` (int ``[n]``) restrict the update to some articulations;
    bodies of the others keep their values.
    """
    if mask is not None and indices is not None:
        raise ValueError("Cannot specify both mask and indices parameters")
    if state.body_q.is_cuda:
        import ctypes as C

        from .. import _abi, _lib

        nm = _lib.native_model(model)
        jq = joint_q.contiguous()
        jqd = joint_qd.contiguous()
        if mask is not None:
            if mask.dtype != torch.bool or mask.numel() != model.articulation_count:
                raise ValueError(f"Expected Boolean mask with shape ({model.articulation_count},)")
            mask = mask.contiguous()
        if indices is not None:
            indices = torch.as_tensor(indices, dtype=torch.int32, device=state.body_q.device).contiguous()
        dev, nb = model.device, int(model.body_count)
        p_jq = C.c_void_p(_abi.ptr(jq, "f32", dev, int(model.joint_coord_count), "joint_q"))
        p_jqd = C.c_void_p(_abi.ptr(jqd, "f32", dev, int(model.joint_dof_count), "joint_qd"))
        p_bq = C.c_void_p(_abi.ptr(state.body_q, "f32", dev, 7 * nb, "state.body_q"))
        p_bqd = C.c_void_p(_abi.ptr(state.body_qd, "f32", dev, 6 * nb, "state.body_qd"))
        with torch.cuda.device(nm.device_index):
            if mask is None and indices is None and int(body_flag_filter) == 3:  # BodyFlags.ALL
                st = _lib.lib().nb2_eval_fk(nm.handle, p_jq, p_jqd, p_bq, p_bqd, _lib.current_stream_ptr(model))
            else:
                st = _lib.lib().nb2_eval_fk_masked(
                    nm.handle, p_jq, p_jqd, p_bq, p_bqd, C.c_void_p(None if mask is None else mask.data_ptr()),
                    C.c_void_p(None if indices is None else indices.data_ptr()), 0 if indices is None else indices.numel(),
                    int(body_flag_filter), _lib.current_stream_ptr(model))
            _lib.check(st, "nb2_eval_fk")
        return
    from .. import _lib

    raise _lib.Nb2Error(
        "newton_b200.eval_fk runs on CUDA devices only (no CPU path). Scene builders that need initial body poses on the host "
        "use newton_b200.utils.host_fk.host_fk; CPU checks use oracle.eval_fk (test infrastructure)."
    )


def eval_ik(model, state, joint_q, joint_qd) -> None:
    """``newton.eval_ik`` (reference ``sim/articulation.py:883-932``): ``state.body_q`` / ``body_qd`` -> generalized
    ``joint_q`` / ``joint_qd`` for every articulated joint, through ``nb2_eval_ik`` (one thread per joint).  CUDA models only;
    like every simulation call of this package there is no CPU path (the oracle under ``oracle/`` is the CPU checker)."""
    import ctypes as C

    from .. import _abi, _lib

    nm = _lib.native_model(model)  # raises for CPU models
    with torch.cuda.device(nm.device_index):
        _lib.check(
            _lib.lib().nb2_eval_ik(
                nm.handle, C.c_void_p(_abi.ptr(state.body_q, "f32", model.device, 7 * int(model.body_count), "state.body_q")),
                C.c_void_p(_abi.ptr(state.body_qd, "f32", model.device, 6 * int(model.body_count), "state.body_qd")),
                C.c_void_p(_abi.ptr(joint_q, "f32", model.device, int(model.joint_coord_count), "joint_q")),
                C.c_void_p(_abi.ptr(joint_qd, "f32", model.device, int(model.joint_dof_count), "joint_qd")),
                _lib.current_stream_ptr(model)),
            "nb2_eval_ik",
        )


# ---- articulation dynamics queries: newton.eval_jacobian / eval_mass_matrix / eval_inverse_dynamics_passive / _force -------------
# The kernels (csrc/nb2_dynamics.cu) run one warp per articulation and keep every intermediate in shared memory, so a call is one
# launch with no allocation and no host synchronisation once its outputs exist.  Argument checks happen before the CUDA-only
# check, with the reference's messages.


def _has_rod(model) -> bool:
    cached = getattr(model, "_nb2_has_rod", None)
    if cached is None:
        from .enums import JointType

        cached = bool((model.numpy("joint_type") == int(JointType.ROD)).any()) if int(model.joint_count) else False
        model._nb2_has_rod = cached
    return cached


def _check_shape(name, array, expected):
    if array is not None and tuple(array.shape) != tuple(expected):
        raise ValueError(f"{name} has shape {tuple(array.shape)}, expected {tuple(expected)}.")


def _native_call(model, what):
    from .. import _lib

    if not torch.device(model.device).type == "cuda":
        raise _lib.Nb2Error(f"newton_b200.{what} runs on CUDA devices only (no CPU path); CPU checks use oracle.dynamics "
                            "(test infrastructure).")
    return _lib.native_model(model)


def _mask_ptr(mask, model):
    import ctypes as C

    from .. import _abi

    return C.c_void_p(_abi.ptr(mask, "bool", model.device, int(model.articulation_count), "mask"))


def _jacobian_shape(model):
    return (int(model.articulation_count), 6 * int(model.max_joints_per_articulation), int(model.max_dofs_per_articulation))


def _mass_matrix_shape(model):
    return (int(model.articulation_count), int(model.max_dofs_per_articulation), int(model.max_dofs_per_articulation))


def eval_jacobian(model, state, J=None, joint_S_s=None, mask=None):
    """Spatial Jacobian of every articulation (reference ``newton.eval_jacobian``, ``sim/articulation.py:1171-1248``).

    Returns ``J`` of shape ``(articulation_count, 6 * max_joints_per_articulation, max_dofs_per_articulation)`` with
    ``J[a, 6 i : 6 i + 6] @ joint_qd == state.body_qd[link]`` for the child of the articulation's i-th joint (COM-referenced world
    twists), or ``None`` when the model has no articulations.  ``J`` is allocated when omitted; every entry is written, padding and
    masked-out articulations (``mask``, bool ``[articulation_count]``) as 0.  ``joint_S_s`` is accepted for calls written
    against the reference, where it is a temporary; the kernel keeps the motion subspaces in shared memory and never writes it.
    Reads ``state.body_q`` and ``state.joint_q``.
    """
    if int(model.articulation_count) == 0:
        return None
    _check_shape("J", J, _jacobian_shape(model))
    _check_shape("mask", mask, (int(model.articulation_count),))
    nm = _native_call(model, "eval_jacobian")
    import ctypes as C

    from .. import _abi, _lib

    if J is None:
        J = torch.empty(_jacobian_shape(model), dtype=torch.float32, device=model.device)
    dev = model.device
    with torch.cuda.device(nm.device_index):
        _lib.check(_lib.lib().nb2_eval_jacobian(
            nm.handle, C.c_void_p(_abi.ptr(state.body_q, "f32", dev, 7 * int(model.body_count), "state.body_q")),
            C.c_void_p(_abi.ptr(state.joint_q, "f32", dev, int(model.joint_coord_count), "state.joint_q")),
            C.c_void_p(_abi.ptr(J, "f32", dev, J.numel(), "J")), int(model.max_joints_per_articulation), int(model.max_dofs_per_articulation),
            _mask_ptr(mask, model), _lib.current_stream_ptr(model)), "nb2_eval_jacobian")
    return J


def eval_mass_matrix(model, state, H=None, J=None, body_I_s=None, joint_S_s=None, mask=None):
    """Generalized mass matrix ``H = J^T M J`` of every articulation (reference ``newton.eval_mass_matrix``,
    ``sim/articulation.py:1593-1690``), consistent with the kinetic energy of the COM-referenced body twists.

    Returns ``H`` of shape ``(articulation_count, max_dofs_per_articulation, max_dofs_per_articulation)`` (allocated when omitted;
    padding and masked-out articulations are 0), or ``None`` without articulations.  With ``J`` given, that Jacobian is read
    instead of being formed; without it the Jacobian lives in shared memory only.  ``body_I_s`` and ``joint_S_s`` are accepted
    for calls written against the reference, where they are temporaries; they are never written.
    """
    if int(model.articulation_count) == 0:
        return None
    _check_shape("H", H, _mass_matrix_shape(model))
    _check_shape("J", J, _jacobian_shape(model))
    _check_shape("mask", mask, (int(model.articulation_count),))
    nm = _native_call(model, "eval_mass_matrix")
    import ctypes as C

    from .. import _abi, _lib

    if H is None:
        H = torch.empty(_mass_matrix_shape(model), dtype=torch.float32, device=model.device)
    dev = model.device
    with torch.cuda.device(nm.device_index):
        _lib.check(_lib.lib().nb2_eval_mass_matrix(
            nm.handle, C.c_void_p(_abi.ptr(state.body_q, "f32", dev, 7 * int(model.body_count), "state.body_q")),
            C.c_void_p(_abi.ptr(state.joint_q, "f32", dev, int(model.joint_coord_count), "state.joint_q")),
            C.c_void_p(None if J is None else _abi.ptr(J, "f32", dev, J.numel(), "J")),
            C.c_void_p(_abi.ptr(H, "f32", dev, H.numel(), "H")), int(model.max_joints_per_articulation),
            int(model.max_dofs_per_articulation), _mask_ptr(mask, model), _lib.current_stream_ptr(model)), "nb2_eval_mass_matrix")
    return H


def eval_inverse_dynamics_passive(model, state, *, mass_matrix=None, gravity_force=None, coriolis_force=None, mask=None) -> None:
    """Passive inverse-dynamics terms (reference ``newton.eval_inverse_dynamics_passive``, ``sim/inverse_dynamics.py:364-485``).

    Each non-``None`` output is computed, all in one launch: ``mass_matrix`` <- ``M(q)`` (as :func:`eval_mass_matrix`),
    ``gravity_force`` <- ``g(q) = dU/dq`` and ``coriolis_force`` <- ``C(q, qd) qd``, following ``tau = M qdd + C qd + g``.  The
    two force terms come from two separate RNEA passes (joint_qd = 0 under ``model.gravity``; ``state.joint_qd`` under zero
    gravity).  ``state.body_q`` must already reflect ``state.joint_q`` (call :func:`eval_fk` first).  Entries of articulations
    that ``mask`` leaves out are 0.  Loop-closure joints play no part; ROD joints are refused.
    """
    if _has_rod(model):
        raise ValueError("eval_inverse_dynamics_passive() does not support JointType.ROD joints.")
    if mass_matrix is None and gravity_force is None and coriolis_force is None:
        raise ValueError("At least one inverse-dynamics output must be provided.")
    _check_shape("mass_matrix", mass_matrix, _mass_matrix_shape(model))
    for name, array in (("gravity_force", gravity_force), ("coriolis_force", coriolis_force)):
        _check_shape(name, array, (int(model.joint_dof_count),))
    _check_shape("mask", mask, (int(model.articulation_count),))
    if int(model.articulation_count) == 0:
        return
    nm = _native_call(model, "eval_inverse_dynamics_passive")
    import ctypes as C

    from .. import _abi, _lib

    dev, nd = model.device, int(model.joint_dof_count)

    def out(a, name):
        return C.c_void_p(None if a is None else _abi.ptr(a, "f32", dev, a.numel(), name))

    with torch.cuda.device(nm.device_index):
        _lib.check(_lib.lib().nb2_eval_inverse_dynamics_passive(
            nm.handle, C.c_void_p(_abi.ptr(state.body_q, "f32", dev, 7 * int(model.body_count), "state.body_q")),
            C.c_void_p(_abi.ptr(state.joint_q, "f32", dev, int(model.joint_coord_count), "state.joint_q")),
            C.c_void_p(_abi.ptr(state.joint_qd, "f32", dev, nd, "state.joint_qd")), out(mass_matrix, "mass_matrix"),
            out(gravity_force, "gravity_force"), out(coriolis_force, "coriolis_force"), int(model.max_dofs_per_articulation),
            _mask_ptr(mask, model), _lib.current_stream_ptr(model)), "nb2_eval_inverse_dynamics_passive")


def eval_inverse_dynamics_force(model, state, *, mass_matrix, joint_qdd, coriolis_force, gravity_force, joint_f, mask=None) -> None:
    """``joint_f = M(q) qdd + C(q, qd) qd + g(q)`` (reference ``newton.eval_inverse_dynamics_force``,
    ``sim/articulation.py:1471-1590``), in the ``Control.joint_f`` convention: the ``M qdd`` part of every FREE/DISTANCE joint is
    rotated from its parent frame into the world frame with ``state.body_q``.  Dofs of articulations that ``mask`` leaves out and
    loop-closure dofs after an articulation's tree are set to 0.  ROD joints are refused.
    """
    if _has_rod(model):
        raise ValueError("eval_inverse_dynamics_force() does not support JointType.ROD joints.")
    if int(model.articulation_count) == 0:
        return
    _check_shape("mass_matrix", mass_matrix, _mass_matrix_shape(model))
    for name, array in (("joint_qdd", joint_qdd), ("coriolis_force", coriolis_force), ("gravity_force", gravity_force),
                        ("joint_f", joint_f)):
        _check_shape(name, array, (int(model.joint_dof_count),))
    _check_shape("mask", mask, (int(model.articulation_count),))
    nm = _native_call(model, "eval_inverse_dynamics_force")
    import ctypes as C

    from .. import _abi, _lib

    dev, nd = model.device, int(model.joint_dof_count)

    def arg(a, name):
        return C.c_void_p(_abi.ptr(a, "f32", dev, a.numel(), name))

    with torch.cuda.device(nm.device_index):
        _lib.check(_lib.lib().nb2_eval_inverse_dynamics_force(
            nm.handle, C.c_void_p(_abi.ptr(state.body_q, "f32", dev, 7 * int(model.body_count), "state.body_q")),
            arg(mass_matrix, "mass_matrix"), arg(joint_qdd, "joint_qdd"), arg(coriolis_force, "coriolis_force"),
            arg(gravity_force, "gravity_force"), arg(joint_f, "joint_f"), int(model.max_dofs_per_articulation), _mask_ptr(mask, model),
            _lib.current_stream_ptr(model)), "nb2_eval_inverse_dynamics_force")

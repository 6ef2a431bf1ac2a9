"""Joint-space impedance controllers (reference ``newton.controllers.ControllerJointImpedance`` /
``ControllerJointImpedanceModelFree``, ``controllers/impl/joint_impedance/``)::

    tau = [M(q) if use_inertia_decoupling else I] . (qdd_des + Kp (q_des - q) + Kd (qd_des - qd))
          + [C(q, qd) qd if use_coriolis_compensation else 0] + [g(q) if use_gravity_compensation else 0]

Flat simulation arrays in, a flat torque array out.  Robot r's controller dof i reads every input through its index table at
``dof_offsets[r] + i`` and writes ``joint_f[joint_f_idx[dof_offsets[r] + i]]``; gains are ``(robot_count, max_dofs)``.  One
:meth:`step` is one kernel launch (``nb2_joint_impedance_step``, one warp per robot): gather, forward kinematics and the
dynamics terms (model-based controller), the law and the scatter.  It allocates nothing and does not synchronise.
"""

from __future__ import annotations

import ctypes as C
from typing import Any

import numpy as np
import torch

from .. import _abi
from ..sim.builder import ModelBuilder
from ..sim.enums import JointType
from .controller import ControllerBase

_INDEX_DTYPES = (torch.uint32, torch.int32, torch.int64)


def _launch(controller, desc) -> None:
    """``nb2_joint_impedance_step`` on the controller's device and current stream: the one place the controllers launch."""
    from .. import _lib

    if controller.device.type != "cuda":
        raise _lib.Nb2Error(f"controllers run on CUDA devices only (got {controller.device}); there is no CPU path")
    if controller._model is not None:
        desc.model = _lib.native_model(controller._model).handle.value
    stream = C.c_void_p(torch.cuda.current_stream(controller.device).cuda_stream)
    _lib.check(_lib.lib().nb2_joint_impedance_step(C.byref(desc), stream), "nb2_joint_impedance_step")


def _device(device) -> torch.device:
    if device is None:
        device = "cuda" if torch.cuda.is_available() else "cpu"
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return device


def _host_indices(idx) -> np.ndarray:
    return np.asarray(idx.detach().cpu().numpy(), dtype=np.int64).reshape(-1)


def _check_index_type(idx, name: str) -> None:
    if not isinstance(idx, torch.Tensor) or idx.dtype not in _INDEX_DTYPES:
        what = f"{type(idx).__name__} of {idx.dtype}" if isinstance(idx, torch.Tensor) else type(idx).__name__
        raise TypeError(f"Port '{name}': idx must be a uint32, int32 or int64 tensor or None, got {what}.")


class _Port:
    """One index table: int32 values checked on the host (moved to the controller's device by ``to``), and its largest index."""

    def __init__(self, idx, default: _Port | None, name: str, total: int):
        if idx is None:
            self.host, self.max = default.host, default.max
            return
        _check_index_type(idx, name)
        if idx.numel() != total:
            raise ValueError(f"Port '{name}': indices must be the same size as default_dof_indices: {idx.numel()} != {total}.")
        host = _host_indices(idx)
        if host.size and (host.min() < 0 or host.max() > np.iinfo(np.int32).max):
            raise ValueError(f"Port '{name}': indices must lie in [0, 2^31)")
        self.host = host.astype(np.int32)
        self.max = int(host.max()) if host.size else -1

    def to(self, device) -> _Port:
        self.idx = torch.from_numpy(self.host).to(device)
        return self


class _JointImpedance(ControllerBase):
    """What the two controllers share: index tables, gains, the input / output structs and the fused step."""

    _model = None  # ControllerJointImpedance: its own Model (dynamics terms come from it)
    _DYNAMICS_PORTS: tuple = ()  # model-free: the caller-supplied dynamics inputs

    def _setup(self, *, robot_count, dofs, max_dofs, default_dof_indices, stiffness, damping, use_gravity_compensation,
               use_coriolis_compensation, use_inertia_decoupling, has_qdd_feedforward, ports: dict, device, requires_grad):
        if requires_grad:
            raise NotImplementedError(f"{type(self).__name__}(requires_grad=True): the controller kernel is not differentiable")
        self._device = device
        self._requires_grad = False
        self._robot_count = int(robot_count)
        self._max_dofs = int(max_dofs)
        self._use_gravity = bool(use_gravity_compensation)
        self._use_coriolis = bool(use_coriolis_compensation)
        self._use_inertia = bool(use_inertia_decoupling)
        self._has_qdd = bool(has_qdd_feedforward)
        total = int(dofs.sum())
        self._total_dofs = total
        if default_dof_indices.numel() != total:
            raise ValueError(f"default_dof_indices length {default_dof_indices.numel()} must equal sum(dofs_per_robot) = {total}.")
        default = _Port(default_dof_indices, None, "default_dof_indices", total)
        ports = {name: _Port(idx, default, name, total) for name, idx in ports.items()}
        if len(ports["joint_f"].host) != len(np.unique(ports["joint_f"].host)):
            raise ValueError("joint_f output indices must be unique — two robots cannot scatter torques to the same simulation DOF slot.")
        self._stiffness = self._baked_gain(stiffness, "stiffness")
        self._damping = self._baked_gain(damping, "damping")
        # every refusal is above this line: device work starts here
        self._ports = {name: port.to(device) for name, port in ports.items()}
        self._stiffness = None if self._stiffness is None else self._stiffness.to(device, copy=True).contiguous()
        self._damping = None if self._damping is None else self._damping.to(device, copy=True).contiguous()
        offsets = np.zeros(robot_count, dtype=np.int32)
        offsets[1:] = np.cumsum(dofs[:-1])
        self._dofs_per_robot = torch.from_numpy(dofs.astype(np.int32)).to(device)
        self._dof_offsets = torch.from_numpy(offsets).to(device)
        self._cache = _abi.DescCache()

    def _baked_gain(self, value, name):
        if value is None:
            return None
        if not isinstance(value, torch.Tensor):
            raise TypeError(f"Port '{name}': must be a float32 tensor of shape (robot_count, max_dofs) or None; got {type(value).__name__}.")
        expected = (self._robot_count, self._max_dofs)
        if tuple(value.shape) != expected:
            raise ValueError(f"Port '{name}': baked array shape {tuple(value.shape)} must equal (robot_count, max_dofs) = {expected}.")
        if value.dtype != torch.float32:
            raise TypeError(f"Port '{name}': baked array dtype must be float32, got {value.dtype}.")
        return value.detach()

    # ------------------------------------------------------------------ reference properties
    @property
    def robot_count(self) -> int:
        return self._robot_count

    @property
    def max_dofs(self) -> int:
        return self._max_dofs

    @property
    def device(self) -> torch.device:
        return self._device

    @property
    def requires_grad(self) -> bool:
        return self._requires_grad

    def is_graphable(self) -> bool:
        return True

    # ------------------------------------------------------------------ structs
    def _live_ports(self) -> list[str]:
        """Input fields a step reads, in the descriptor's order."""
        names = ["joint_q", "joint_qd", "joint_q_des", "joint_qd_des"]
        if self._has_qdd:
            names.append("joint_qdd")
        for name, on in zip(self._DYNAMICS_PORTS, (self._use_gravity, self._use_coriolis, self._use_inertia)):
            if on:
                names.append(name)
        if self._stiffness is None:
            names.append("stiffness")
        if self._damping is None:
            names.append("damping")
        return names

    def _need(self, name: str) -> int:
        """Elements the input ``name`` must at least have."""
        if name in ("stiffness", "damping"):
            return self._robot_count * self._max_dofs
        if name == "mass_matrix":
            return self._robot_count * self._max_dofs * self._max_dofs
        return self._ports[name].max + 1

    def input(self):
        inputs = self.Inputs()
        for name in self.Inputs.__annotations__:
            setattr(inputs, name, None)
        shapes = {"stiffness": (self._robot_count, self._max_dofs), "mass_matrix": (self._robot_count, self._max_dofs, self._max_dofs)}
        shapes["damping"] = shapes["stiffness"]
        for name in self._live_ports():
            setattr(inputs, name, torch.zeros(shapes.get(name, (self._need(name),)), dtype=torch.float32, device=self._device))
        return inputs

    def output(self):
        outputs = self.Outputs()
        outputs.joint_f = torch.zeros(self._ports["joint_f"].max + 1, dtype=torch.float32, device=self._device)
        return outputs

    # ------------------------------------------------------------------ step
    def _desc(self, inputs, outputs) -> _abi.JointImpedanceDesc:
        """The ``nb2_joint_impedance_step`` descriptor; every live array's dtype, device, contiguity and size is checked here."""
        d = _abi.JointImpedanceDesc()
        d.robot_count, d.max_dofs = self._robot_count, self._max_dofs
        d.use_gravity, d.use_coriolis, d.use_inertia, d.has_qdd = self._use_gravity, self._use_coriolis, self._use_inertia, self._has_qdd
        d.dofs_per_robot, d.dof_offsets = self._dofs_per_robot.data_ptr(), self._dof_offsets.data_ptr()
        for name, port in self._ports.items():
            setattr(d, name + "_idx", port.idx.data_ptr())
        read = []
        for name in self._live_ports():
            a = getattr(inputs, name, None)
            if not isinstance(a, torch.Tensor):
                raise TypeError(f"inputs.{name}: expected a float32 tensor, got {type(a).__name__}")
            if name in ("stiffness", "damping", "mass_matrix"):
                shape = (self._robot_count, self._max_dofs) + ((self._max_dofs,) if name == "mass_matrix" else ())
                if tuple(a.shape) != shape:
                    raise ValueError(f"inputs.{name}: shape {tuple(a.shape)} must equal {shape}")
            self._check_live(a, name)
            setattr(d, name, a.data_ptr())
            read.append(a)
        if self._stiffness is not None:
            d.stiffness = self._stiffness.data_ptr()
        if self._damping is not None:
            d.damping = self._damping.data_ptr()
        f = outputs.joint_f
        if not isinstance(f, torch.Tensor):
            raise TypeError(f"outputs.joint_f: expected a float32 tensor, got {type(f).__name__}")
        self._check_live(f, "joint_f", output=True)
        if any(f.untyped_storage().data_ptr() == a.untyped_storage().data_ptr() for a in read):
            raise ValueError("outputs.joint_f must not share storage with an input array")
        d.joint_f = f.data_ptr()
        if self._model is not None:
            s = self._state
            d.state_joint_q, d.state_joint_qd = s.joint_q.data_ptr(), s.joint_qd.data_ptr()
            d.state_body_q, d.state_body_qd = s.body_q.data_ptr(), s.body_qd.data_ptr()
        return d

    def _check_live(self, a, name: str, output: bool = False) -> None:
        label = ("outputs." if output else "inputs.") + name
        need = self._ports["joint_f"].max + 1 if output else self._need(name)
        if a.numel() < need:
            raise ValueError(f"{label}: {a.numel()} elements, its index map needs at least {need}")
        _abi.ptr(a, "f32", self._device, need, label)  # dtype, device and contiguity

    def step(self, *, inputs, outputs, dt: Any = None) -> None:
        """One control step: writes the torques of every controlled dof to ``outputs.joint_f``.  ``dt`` is unused (accepted for
        API compatibility).  The descriptor is built and checked once per combination of arrays (``_abi.DescCache``)."""
        arrays = tuple(getattr(inputs, n, None) for n in self._live_ports()) + (getattr(outputs, "joint_f", None),)
        if not all(isinstance(a, torch.Tensor) for a in arrays):
            desc = self._desc(inputs, outputs)  # raises the precise error
        else:
            desc = self._cache.get(arrays, lambda: self._desc(inputs, outputs))
        _launch(self, desc)


class ControllerJointImpedanceModelFree(_JointImpedance):
    """Joint-space impedance controller with caller-supplied dynamics (mass matrix, gravity and Coriolis forces).

    Robots may have different dof counts (``dofs_per_robot``); buffers are padded to ``max_dofs`` and padding is never written.

    Args:
        robot_count: number of robots.
        dofs_per_robot: integer tensor ``(robot_count,)``.
        max_dofs: padded width, at least ``max(dofs_per_robot)``.
        default_dof_indices: ``uint32`` / ``int32`` / ``int64`` tensor of length ``sum(dofs_per_robot)``: robot 0's flat indices,
            then robot 1's, ...
        stiffness, damping: baked float32 ``(robot_count, max_dofs)`` gains (copied), or ``None`` to read them from ``inputs``.
        use_gravity_compensation, use_coriolis_compensation, use_inertia_decoupling, has_qdd_feedforward: terms of the law.
        joint_q_idx ... joint_f_idx: per-port overrides of ``default_dof_indices`` (converted to int32 once, here).
        device: torch device of the controller (default: the current CUDA device).
        requires_grad: must be ``False``; the kernel is not differentiable.
    """

    _DYNAMICS_PORTS = ("gravity_force", "coriolis_force", "mass_matrix")

    class Inputs:
        """Input struct of :meth:`ControllerJointImpedanceModelFree.input`; fields of disabled features are ``None``."""

        joint_q: torch.Tensor
        """Current joint positions [m or rad], flat."""
        joint_qd: torch.Tensor
        """Current joint velocities [m/s or rad/s], flat."""
        joint_q_des: torch.Tensor
        """Desired joint positions, flat."""
        joint_qd_des: torch.Tensor
        """Desired joint velocities, flat."""
        joint_qdd: torch.Tensor | None
        """Desired acceleration feedforward, flat; ``has_qdd_feedforward`` only."""
        gravity_force: torch.Tensor | None
        """Gravity generalized forces [N or N m], flat; ``use_gravity_compensation`` only."""
        coriolis_force: torch.Tensor | None
        """Coriolis generalized forces [N or N m], flat; ``use_coriolis_compensation`` only."""
        mass_matrix: torch.Tensor | None
        """Per-robot mass matrices ``(robot_count, max_dofs, max_dofs)``, indexed ``[robot, dof, col]``; ``use_inertia_decoupling``
        only."""
        stiffness: torch.Tensor | None
        """Live Kp ``(robot_count, max_dofs)``; ``None`` when baked."""
        damping: torch.Tensor | None
        """Live Kd ``(robot_count, max_dofs)``; ``None`` when baked."""

    class Outputs:
        """Output struct of :meth:`ControllerJointImpedanceModelFree.output`."""

        joint_f: torch.Tensor
        """Joint torque command [N or N m], flat."""

    def __init__(self, *, robot_count: int, dofs_per_robot, max_dofs: int, default_dof_indices, stiffness, damping,
                 use_gravity_compensation: bool = True, use_coriolis_compensation: bool = True, use_inertia_decoupling: bool = True,
                 has_qdd_feedforward: bool = False, joint_q_idx=None, joint_qd_idx=None, joint_q_des_idx=None, joint_qd_des_idx=None,
                 joint_qdd_idx=None, gravity_force_idx=None, coriolis_force_idx=None, joint_f_idx=None, device: Any = None,
                 requires_grad: bool = False):
        if robot_count < 1:
            raise ValueError(f"robot_count must be >= 1, got {robot_count}.")
        if not isinstance(dofs_per_robot, torch.Tensor) or dofs_per_robot.dtype not in (torch.int32, torch.int64):
            raise TypeError("dofs_per_robot must be an int32 tensor.")
        if dofs_per_robot.numel() != robot_count:
            raise ValueError(f"dofs_per_robot length {dofs_per_robot.numel()} must equal robot_count={robot_count}.")
        if max_dofs < 1:
            raise ValueError(f"max_dofs must be >= 1, got {max_dofs}.")
        _check_index_type(default_dof_indices, "default_dof_indices")
        dofs = _host_indices(dofs_per_robot)
        if dofs.min() < 0 or dofs.max() > max_dofs:
            raise ValueError(f"dofs_per_robot entries must lie in [0, max_dofs={max_dofs}]")
        ports = dict(joint_q=joint_q_idx, joint_qd=joint_qd_idx, joint_q_des=joint_q_des_idx, joint_qd_des=joint_qd_des_idx,
                     joint_qdd=joint_qdd_idx, gravity_force=gravity_force_idx, coriolis_force=coriolis_force_idx, joint_f=joint_f_idx)
        self._setup(robot_count=robot_count, dofs=dofs, max_dofs=max_dofs, default_dof_indices=default_dof_indices, stiffness=stiffness,
                    damping=damping, use_gravity_compensation=use_gravity_compensation,
                    use_coriolis_compensation=use_coriolis_compensation, use_inertia_decoupling=use_inertia_decoupling,
                    has_qdd_feedforward=has_qdd_feedforward, ports=ports, device=_device(device), requires_grad=requires_grad)


class ControllerJointImpedance(_JointImpedance):
    """Joint-space impedance controller whose mass matrix, gravity and Coriolis forces come from its own model.

    The builder's articulations are the robots (they may have different dof counts; buffers are padded to
    ``model.max_dofs_per_articulation``).  Only REVOLUTE, PRISMATIC and FIXED joints are accepted, every joint must belong to
    an articulation and there are no loop-closure joints, so that the articulations tile the model's dofs in order.  Gravity
    is the model's.  Same inputs and outputs as :class:`ControllerJointImpedanceModelFree` without the dynamics fields.

    Args:
        builder: :class:`~newton_b200.ModelBuilder`, finalized here on ``device``.
        default_dof_indices, stiffness, damping, use_*, has_qdd_feedforward, joint_*_idx, device, requires_grad: as for
            :class:`ControllerJointImpedanceModelFree`.
    """

    class Inputs:
        """Input struct of :meth:`ControllerJointImpedance.input`; fields of disabled features are ``None``."""

        joint_q: torch.Tensor
        """Current joint positions [m or rad], flat."""
        joint_qd: torch.Tensor
        """Current joint velocities [m/s or rad/s], flat."""
        joint_q_des: torch.Tensor
        """Desired joint positions, flat."""
        joint_qd_des: torch.Tensor
        """Desired joint velocities, flat."""
        joint_qdd: torch.Tensor | None
        """Desired acceleration feedforward, flat; ``has_qdd_feedforward`` only."""
        stiffness: torch.Tensor | None
        """Live Kp ``(robot_count, max_dofs)``; ``None`` when baked."""
        damping: torch.Tensor | None
        """Live Kd ``(robot_count, max_dofs)``; ``None`` when baked."""

    Outputs = ControllerJointImpedanceModelFree.Outputs

    def __init__(self, builder: ModelBuilder, *, default_dof_indices, stiffness, damping, use_gravity_compensation: bool = True,
                 use_coriolis_compensation: bool = True, use_inertia_decoupling: bool = True, has_qdd_feedforward: bool = False,
                 joint_q_idx=None, joint_qd_idx=None, joint_q_des_idx=None, joint_qd_des_idx=None, joint_qdd_idx=None,
                 joint_f_idx=None, device: Any = None, requires_grad: bool = False):
        if not isinstance(builder, ModelBuilder):
            raise TypeError(f"builder must be a newton_b200.ModelBuilder, got {type(builder).__name__}.")
        _check_index_type(default_dof_indices, "default_dof_indices")
        robot_count = builder.articulation_count
        if robot_count < 1:
            raise ValueError("builder has no articulations.")
        allowed = {int(JointType.REVOLUTE), int(JointType.PRISMATIC), int(JointType.FIXED)}
        unsupported = [(j, JointType(t).name) for j, t in enumerate(builder.joint_type) if t not in allowed]
        if unsupported:
            raise ValueError(f"ControllerJointImpedance only supports 1-DOF joints (Revolute/Prismatic) and "
                             f"zero-DOF fixed joints; found unsupported joint types: {unsupported}")
        starts, ends = list(builder.articulation_start), list(builder.articulation_end)
        if starts[0] != 0 or ends[-1] != builder.joint_count or any(e != s for e, s in zip(ends[:-1], starts[1:])):
            raise ValueError("ControllerJointImpedance needs articulations that cover every joint in order, without loop-closure "
                             "joints (the dynamics terms are read with an identity dof map)")
        if requires_grad:
            raise NotImplementedError("ControllerJointImpedance(requires_grad=True): the controller kernel is not differentiable")
        qd = [*builder.joint_qd_start, builder.joint_dof_count]
        dofs = np.array([qd[e] - qd[s] for s, e in zip(starts, ends)], dtype=np.int64)
        identity = torch.arange(int(dofs.sum()), dtype=torch.int32)
        ports = dict(joint_q=joint_q_idx, joint_qd=joint_qd_idx, joint_q_des=joint_q_des_idx, joint_qd_des=joint_qd_des_idx,
                     joint_qdd=joint_qdd_idx, gravity_force=identity, coriolis_force=identity, joint_f=joint_f_idx)
        device = _device(device)
        self._setup(robot_count=robot_count, dofs=dofs, max_dofs=max(1, int(dofs.max())), default_dof_indices=default_dof_indices,
                    stiffness=stiffness, damping=damping, use_gravity_compensation=use_gravity_compensation,
                    use_coriolis_compensation=use_coriolis_compensation, use_inertia_decoupling=use_inertia_decoupling,
                    has_qdd_feedforward=has_qdd_feedforward, ports=ports, device=device, requires_grad=False)
        self._model = builder.finalize(device=device)
        self._state = self._model.state()
        if device.type == "cuda":
            from .. import _lib

            _lib.native_model(self._model)  # created here so that the first step allocates nothing

    @property
    def model(self):
        """The controller's own :class:`~newton_b200.Model`."""
        return self._model

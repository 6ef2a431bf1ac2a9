"""Composed actuator (reference ``newton.actuators.Actuator``, ``actuators/actuator.py``): delay -> controller -> clamping ->
scatter-add into a control array, stepped by one fused CUDA kernel per call (``csrc/nb2_actuator.cu``)."""

from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch

from .. import _abi
from .components import (
    ClampingDCMotor,
    ClampingMaxEffort,
    ClampingPositionBased,
    Controller,
    ControllerPD,
    ControllerPID,
    Delay,
)
from .neural import NEURAL_CONTROLLERS

def _call(name: str, device, *args) -> None:
    """``nb2_actuator_<name>(*args, stream)`` on ``device``'s current stream: the one place the actuators launch."""
    from .. import _lib

    device = torch.device(device)
    if device.type != "cuda":
        raise _lib.Nb2Error(f"actuators run on CUDA devices only (got {device}); there is no CPU path")
    stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
    _lib.check(getattr(_lib.lib(), f"nb2_actuator_{name}")(*args, stream), f"nb2_actuator_{name}")


def _index_tensor(a, name: str):
    if a is None:
        return None
    if not hasattr(a, "data_ptr"):
        raise TypeError(f"{name}: expected a tensor, got {type(a).__name__}")
    if a.dtype != torch.int32:
        if a.dtype.is_floating_point or a.dtype == torch.bool:
            raise ValueError(f"{name}: expected integer indices, got {a.dtype}")
        a = a.to(torch.int32)
    return a.contiguous()


def _host_max(a) -> int:
    return int(a.max().item()) if a.numel() else -1


class Actuator:
    """Composed actuator: delay -> controller -> clamping, **accumulated** into the output array (``out[idx] += effort``); the
    caller zeroes the output before stepping its actuators.

    One :meth:`step` is one kernel launch (two for a group whose effort indices repeat), allocates nothing and does not
    synchronise, so it can be captured into a CUDA graph together with collision and the solver step.  Effort indices that
    repeat inside one actuator are summed in ascending actuator index, the reference's serial result.
    """

    @dataclass
    class State:
        """Composed state: the delay state (if a delay is present) and the controller state (if stateful)."""

        delay_state: Delay.State | None = None
        controller_state: Controller.State | None = None

        def reset(self, mask=None) -> None:
            """Reset composed state (``mask``: Boolean ``(N,)``, ``True`` entries reset; ``None`` resets all)."""
            for part in (self.delay_state, self.controller_state):
                if part is not None:
                    part.reset(mask)

    def __init__(
        self,
        indices,
        controller: Controller,
        delay: Delay | None = None,
        clamping: list | None = None,
        pos_indices=None,
        target_pos_indices=None,
        effort_indices=None,
        state_pos_attr: str = "joint_q",
        state_vel_attr: str = "joint_qd",
        control_target_pos_attr: str | None = "joint_target_q",
        control_target_vel_attr: str | None = "joint_target_qd",
        control_feedforward_attr: str | None = "joint_act",
        control_output_attr: str = "joint_f",
        control_computed_output_attr: str | None = None,
        requires_grad: bool = False,
    ):
        """Initialize actuator.

        Args:
            indices: dof indices into velocity-shaped arrays (velocities, velocity targets, feedforward, effort output), ``(N,)``.
            controller: :class:`ControllerPD`, :class:`ControllerPID`, :class:`ControllerNeuralMLP` or
                :class:`ControllerNeuralLSTM`.
            delay: optional :class:`Delay`.
            clamping: list of clampings applied in order after the controller.
            pos_indices: indices into coordinate-shaped arrays (``state.joint_q``); default *indices*.
            target_pos_indices: indices into ``control.joint_target_q``; default *pos_indices* when
                ``newton_b200.use_coord_layout_targets`` is ``True``, else *indices*.  The flag is read once, here.
            effort_indices: indices into the output arrays; default *indices*.
            requires_grad: must be ``False``: the actuator kernels are not differentiable.
        """
        if requires_grad:
            raise NotImplementedError("Actuator(requires_grad=True): the actuator kernels are not differentiable")
        indices = _index_tensor(indices, "indices")
        self.indices = indices
        self.pos_indices = _index_tensor(pos_indices, "pos_indices") if pos_indices is not None else indices
        if target_pos_indices is not None:
            self.target_pos_indices = _index_tensor(target_pos_indices, "target_pos_indices")
        else:
            import newton_b200

            self.target_pos_indices = self.pos_indices if newton_b200.use_coord_layout_targets else indices
        self.effort_indices = _index_tensor(effort_indices, "effort_indices") if effort_indices is not None else indices
        for name in ("pos_indices", "target_pos_indices", "effort_indices"):
            if tuple(getattr(self, name).shape) != tuple(indices.shape):
                raise ValueError(f"{name} shape {tuple(getattr(self, name).shape)} must match indices shape {tuple(indices.shape)}")
        self.controller = controller
        self.delay = delay
        self.clamping = list(clamping or [])
        if not isinstance(controller, (ControllerPD, ControllerPID, *NEURAL_CONTROLLERS)):
            raise NotImplementedError(f"{type(controller).__name__}: only ControllerPD, ControllerPID, ControllerNeuralMLP and "
                                      f"ControllerNeuralLSTM are supported")
        for c in self.clamping:
            if not isinstance(c, (ClampingMaxEffort, ClampingDCMotor, ClampingPositionBased)):
                raise NotImplementedError(f"{type(c).__name__}: unsupported clamping")
        if len(self.clamping) > _abi.ACTUATOR_MAX_CLAMPS:
            raise ValueError(f"a clamp chain holds at most {_abi.ACTUATOR_MAX_CLAMPS} clampings, got {len(self.clamping)}")
        self.num_actuators = int(indices.shape[0])
        self.state_pos_attr = state_pos_attr
        self.state_vel_attr = state_vel_attr
        self.control_target_pos_attr = "joint_target_q" if control_target_pos_attr is None else control_target_pos_attr
        self.control_target_vel_attr = "joint_target_qd" if control_target_vel_attr is None else control_target_vel_attr
        self.control_feedforward_attr = control_feedforward_attr
        self.control_output_attr = control_output_attr
        self.control_computed_output_attr = control_computed_output_attr
        self.device = indices.device
        self.requires_grad = False

        for component in (controller, delay, *self.clamping):
            if component is not None:
                component.finalize(self.device, self.num_actuators)
        lookup = sum(c.lookup_size for c in self.clamping if isinstance(c, ClampingPositionBased))
        if lookup > _abi.ACTUATOR_MAX_LOOKUP:
            raise ValueError(f"the lookup tables of one actuator hold at most {_abi.ACTUATOR_MAX_LOOKUP} entries in all")
        if isinstance(controller, NEURAL_CONTROLLERS) and controller.smem_bytes(lookup) > _abi.ACTUATOR_SMEM_MAX:
            from .. import _lib

            raise _lib.Nb2Error(
                f"{type(controller).__name__}('{controller.model_path}'): NB2_ERR_CAPACITY: the fused step stages the network in "
                f"shared memory and needs {controller.smem_bytes(lookup)} bytes per CTA ({4 * controller.weights.numel()} of "
                f"weights, {4 * controller._scratch_floats()} of activation scratch for {_abi.NET_TILE} actuators, "
                f"{8 * lookup} of lookup tables); one CTA holds {_abi.ACTUATOR_SMEM_MAX}")

        # host-side tables, built once: the largest index of each index array (the element counts step() checks) and, for
        # effort indices that repeat, the per-target lists of the ordered second pass
        self._max_index = _host_max(self.indices)
        self._max_pos = _host_max(self.pos_indices)
        self._max_target_pos = _host_max(self.target_pos_indices)
        eff = self.effort_indices.cpu().numpy()
        self._max_effort = int(eff.max()) if eff.size else -1
        if max(_host_max(-self.indices), _host_max(-self.pos_indices), _host_max(-self.target_pos_indices),
               int(-eff.min()) if eff.size else -1) > 0:
            raise ValueError("actuator indices must be non-negative")
        targets, counts = np.unique(eff, return_counts=True)
        self.has_duplicate_effort_indices = bool((counts > 1).any())
        self._dup = None
        self._desc_cache = _abi.DescCache()
        if self.has_duplicate_effort_indices:
            order = np.argsort(eff, kind="stable").astype(np.int32)  # ascending actuator index inside each target
            start = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)  # noqa: E731
            self._dup = (len(targets), t(targets.astype(np.int32)), t(start), t(order),
                         torch.zeros(2 * self.num_actuators, dtype=torch.float32, device=self.device))

    def is_stateful(self) -> bool:
        """True if the delay or the controller keeps state."""
        return self.controller.is_stateful() or self.delay is not None

    def is_graphable(self) -> bool:
        """True if :meth:`step` can be captured in a CUDA graph."""
        return self.controller.is_graphable()

    def state(self) -> Actuator.State | None:
        """A new composed state, or ``None`` for a stateless actuator."""
        n, dev = self.num_actuators, self.device
        delay_state = self.delay.state(n, dev) if self.delay is not None else None
        controller_state = self.controller.state(n, dev) if self.controller.is_stateful() else None
        if delay_state is None and controller_state is None:
            return None
        return Actuator.State(delay_state=delay_state, controller_state=controller_state)

    def _step_desc(self, sim_state, sim_control, current_act_state, next_act_state, dt) -> _abi.ActuatorStepDesc:
        """The ``nb2_actuator_step`` descriptor; every pointer's dtype, device and element count is checked here."""
        if self.is_stateful() and None in (current_act_state, next_act_state):
            raise ValueError("Stateful actuator requires both current_act_state and next_act_state; create them via actuator.state()")
        if self.is_stateful() and current_act_state is next_act_state:
            raise ValueError("current_act_state and next_act_state must be different states (the step reads one and writes the other)")
        pid = isinstance(self.controller, ControllerPID)
        neural = isinstance(self.controller, NEURAL_CONTROLLERS)
        if pid and dt is None:
            raise ValueError("ControllerPID needs dt")
        n, dev, P = self.num_actuators, self.device, _abi.ptr
        d = _abi.ActuatorStepDesc()
        d.count = n
        d.controller = self.controller._KIND if neural else _abi.ACT_PID if pid else _abi.ACT_PD
        d.dt = float(dt) if dt is not None else 0.0
        d.indices = P(self.indices, "i32", dev, n, "indices")
        d.pos_indices = P(self.pos_indices, "i32", dev, n, "pos_indices")
        d.target_pos_indices = P(self.target_pos_indices, "i32", dev, n, "target_pos_indices")
        d.effort_indices = P(self.effort_indices, "i32", dev, n, "effort_indices")
        if n == 0:
            return d
        nv = self._max_index + 1
        d.positions = P(getattr(sim_state, self.state_pos_attr), "f32", dev, self._max_pos + 1, "state." + self.state_pos_attr)
        d.velocities = P(getattr(sim_state, self.state_vel_attr), "f32", dev, nv, "state." + self.state_vel_attr)
        d.target_pos = P(getattr(sim_control, self.control_target_pos_attr), "f32", dev, self._max_target_pos + 1,
                         "control." + self.control_target_pos_attr)
        d.target_vel = P(getattr(sim_control, self.control_target_vel_attr), "f32", dev, nv, "control." + self.control_target_vel_attr)
        if self.control_feedforward_attr:
            d.feedforward = P(getattr(sim_control, self.control_feedforward_attr, None), "f32", dev, nv,
                              "control." + self.control_feedforward_attr)
        d.output = P(getattr(sim_control, self.control_output_attr), "f32", dev, self._max_effort + 1, "control." + self.control_output_attr)
        if self.control_computed_output_attr is not None and self.control_computed_output_attr != self.control_output_attr:
            d.computed_output = P(getattr(sim_control, self.control_computed_output_attr), "f32", dev, self._max_effort + 1,
                                  "control." + self.control_computed_output_attr)
        inputs = {d.positions, d.velocities, d.target_pos, d.target_vel, d.feedforward} - {None}
        if d.output in inputs or (d.computed_output is not None and d.computed_output in inputs):
            raise ValueError("the actuator's output arrays must not be any of its input arrays")
        c = self.controller
        if neural:
            net = c._network_desc(current_act_state.controller_state, next_act_state.controller_state)
            d.network = C.pointer(net)  # the pointer keeps the structure alive with the descriptor
        else:
            d.kp = P(c.kp, "f32", dev, n, "kp")
            d.kd = P(c.kd, "f32", dev, n, "kd")
            d.const_effort = P(c.const_effort, "f32", dev, n, "const_effort")
        if pid:
            d.ki = P(c.ki, "f32", dev, n, "ki")
            d.integral_max = P(c.integral_max, "f32", dev, n, "integral_max")
            d.integral_in = P(current_act_state.controller_state.integral, "f32", dev, n, "current integral")
            d.integral_out = P(next_act_state.controller_state.integral, "f32", dev, n, "next integral")
        if self.delay is not None:
            depth = self.delay.buf_depth
            d.buf_depth = depth
            d.delay_steps = P(self.delay.delay_steps, "i32", dev, n, "delay_steps")
            for side, st in (("in", current_act_state.delay_state), ("out", next_act_state.delay_state)):
                for f in ("pos", "vel", "act"):
                    setattr(d, f"buf_{f}_{side}", P(getattr(st, f"buffer_{f}"), "f32", dev, depth * n, f"buffer_{f}"))
                setattr(d, f"num_pushes_{side}", P(st.num_pushes, "i32", dev, n, "num_pushes"))
                setattr(d, f"write_idx_{side}", P(st.write_idx, "i32", dev, 1, "write_idx"))
            if d.write_idx_in == d.write_idx_out:
                raise ValueError("current_act_state and next_act_state share write_idx storage")
        d.clamp_count = len(self.clamping)
        for k, cl in enumerate(self.clamping):
            e = d.clamps[k]
            if isinstance(cl, ClampingMaxEffort):
                e.kind, e.p0 = _abi.CLAMP_MAX_EFFORT, P(cl.max_effort, "f32", dev, n, "max_effort")
            elif isinstance(cl, ClampingDCMotor):
                e.kind = _abi.CLAMP_DC_MOTOR
                e.p0 = P(cl.saturation_effort, "f32", dev, n, "saturation_effort")
                e.p1 = P(cl.velocity_limit, "f32", dev, n, "velocity_limit")
                e.p2 = P(cl.max_motor_effort, "f32", dev, n, "max_motor_effort")
            else:
                e.kind, e.lookup_size = _abi.CLAMP_POSITION_BASED, cl.lookup_size
                e.p0 = P(cl.lookup_positions, "f32", dev, cl.lookup_size, "lookup_positions")
                e.p1 = P(cl.lookup_efforts, "f32", dev, cl.lookup_size, "lookup_efforts")
        if self._dup is not None:
            T, target, start, order, scratch = self._dup
            d.dup_target_count = T
            d.dup_target, d.dup_start, d.dup_actuator = target.data_ptr(), start.data_ptr(), order.data_ptr()
            d.scratch = scratch.data_ptr()
        return d

    def step(self, sim_state: Any, sim_control: Any, current_act_state: Actuator.State | None = None,
             next_act_state: Actuator.State | None = None, dt: float | None = None) -> None:
        """One control step: delay read, controller, clamping, scatter-add into ``sim_control.<control_output_attr>``, and the
        delay buffers / PID integral of ``next_act_state``.  ``dt`` [s] is required for PID."""
        # A descriptor is built and checked once per combination of arrays (_abi.DescCache).  The ping-pong of two actuator
        # states keeps two entries.
        arrays = self._arrays_read(sim_state, sim_control, current_act_state, next_act_state)
        if not all(a is None or isinstance(a, torch.Tensor) for a in arrays):  # other array types are checked every call
            d = self._step_desc(sim_state, sim_control, current_act_state, next_act_state, dt)
            _call("step", self.device, C.byref(d))
            return
        d = self._desc_cache.get(arrays, lambda: self._step_desc(sim_state, sim_control, current_act_state, next_act_state, dt),
                                 key=(dt, id(current_act_state), id(next_act_state)), keep=(current_act_state, next_act_state))
        _call("step", self.device, C.byref(d))

    def _arrays_read(self, sim_state, sim_control, current_act_state, next_act_state) -> tuple:
        """Every tensor a step descriptor points at, in a fixed order (None where absent)."""
        out = [getattr(sim_state, self.state_pos_attr, None), getattr(sim_state, self.state_vel_attr, None)]
        for name in (self.control_target_pos_attr, self.control_target_vel_attr, self.control_feedforward_attr,
                     self.control_output_attr, self.control_computed_output_attr):
            out.append(getattr(sim_control, name, None) if name else None)
        for component in (self.controller, self.delay, *self.clamping):
            if component is not None:
                out.extend(getattr(component, n) for n in component._ARRAYS)
                if isinstance(component, ClampingPositionBased):
                    out += [component.lookup_positions, component.lookup_efforts]
        if isinstance(self.controller, NEURAL_CONTROLLERS):
            out.append(self.controller.weights)
        for st in (current_act_state, next_act_state):
            ds = st.delay_state if st is not None else None
            cs = st.controller_state if st is not None else None
            out += [getattr(cs, n, None) for n in ("integral", "pos_error_history", "vel_history", "hidden", "cell")] + ([ds.buffer_pos, ds.buffer_vel, ds.buffer_act, ds.num_pushes, ds.write_idx]
                                                       if ds is not None else [None] * 5)
        return tuple(out)

    # ------------------------------------------------------------------ Model.to / Model.shard
    def _rebuilt(self, device, keep=None, dof_offset: int = 0, coord_offset: int = 0) -> Actuator:
        """This actuator on ``device``, restricted to the actuators where ``keep`` (a host Boolean array) is set, with dof
        indices shifted by ``-dof_offset`` and coordinate indices (positions, position targets) by ``-coord_offset``."""
        sel = (lambda a: a) if keep is None else (lambda a: a[torch.from_numpy(keep).to(a.device)])

        def arr(a, off=0):
            return None if a is None else (sel(a) - off).to(device).contiguous()

        def clone(obj):
            out = obj.__class__.__new__(obj.__class__)
            out.__dict__.update(obj.__dict__)
            for name in obj._ARRAYS if hasattr(obj, "_ARRAYS") else ():
                setattr(out, name, arr(getattr(obj, name)))
            return out

        return Actuator(arr(self.indices, dof_offset), clone(self.controller), clone(self.delay) if self.delay is not None else None,
                        [clone(c) for c in self.clamping], pos_indices=arr(self.pos_indices, coord_offset),
                        target_pos_indices=arr(self.target_pos_indices, coord_offset), effort_indices=arr(self.effort_indices, dof_offset),
                        state_pos_attr=self.state_pos_attr, state_vel_attr=self.state_vel_attr,
                        control_target_pos_attr=self.control_target_pos_attr, control_target_vel_attr=self.control_target_vel_attr,
                        control_feedforward_attr=self.control_feedforward_attr, control_output_attr=self.control_output_attr,
                        control_computed_output_attr=self.control_computed_output_attr)

"""Batched inverse kinematics (reference ``newton.ik``: ``IKSolver`` / ``IKOptimizerLM``, ``sim/ik/ik_solver.py``,
``ik_lm_optimizer.py``) on one fused CUDA kernel per solve (``csrc/nb2_ik.cu``).

``IKSolver.step`` with ``sampler="none"`` is a single launch: it runs every LM iteration of every problem and the closing cost
evaluation, and advances the sampler counter on the device.  A sampler adds one launch before it, more than one seed adds the
best-seed selection after it.  Nothing allocates or synchronises the host, so ``step`` can be captured in a CUDA graph.
"""

from __future__ import annotations

import ctypes as C
from collections.abc import Sequence
from enum import Enum
from typing import Any

import numpy as np
import torch

from .. import _abi
from ..sim.enums import JointType
from .objectives import IKJacobianType, IKObjective, IKObjectiveJointLimit, IKObjectivePosition, IKObjectiveRotation

_BUILTIN = (IKObjectivePosition, IKObjectiveRotation, IKObjectiveJointLimit)
MAX_OBJECTIVES = 16  # NB2_IK_MAX_OBJECTIVES


class IKOptimizer(str, Enum):
    LM = "lm"
    LBFGS = "lbfgs"


class IKSampler(str, Enum):
    NONE = "none"
    GAUSS = "gauss"
    ROBERTS = "roberts"
    UNIFORM = "uniform"


_SAMPLER_CODE = {IKSampler.NONE: 0, IKSampler.GAUSS: 1, IKSampler.ROBERTS: 2, IKSampler.UNIFORM: 3}


class IkObjectiveDesc(C.Structure):
    """``nb2_ik_objective``"""

    _fields_ = [("kind", C.c_int32), ("row", C.c_int32), ("link", C.c_int32), ("canonicalize", C.c_int32), ("weight", C.c_float),
                ("offset", C.c_float * 4), ("target", C.c_void_p), ("limit_lower", C.c_void_p), ("limit_upper", C.c_void_p),
                ("affects_dof", C.c_void_p)]


class IkDesc(C.Structure):
    """``nb2_ik_desc``"""

    _fields_ = [("model", _abi.ModelDesc), ("mode", C.c_int32), ("n_batch", C.c_int32), ("n_seeds", C.c_int32), ("n_residuals", C.c_int32),
                ("objective_count", C.c_int32), ("lanes", C.c_int32), ("dof_to_coord", C.c_void_p), ("fk_level", C.c_void_p),
                ("fk_level_count", C.c_int32), ("dof_mask", C.c_void_p), ("lambda_initial", C.c_float), ("lambda_factor", C.c_float),
                ("lambda_min", C.c_float), ("lambda_max", C.c_float), ("rho_min", C.c_float),
                ("objectives", IkObjectiveDesc * MAX_OBJECTIVES)]


def _call(name: str, device, *args) -> None:
    """``nb2_ik_<name>(*args, stream)`` on ``device``'s current stream: the one place the IK solver launches."""
    from .. import _lib

    device = torch.device(device)
    if device.type != "cuda":
        raise _lib.Nb2Error(f"newton_b200.ik runs on CUDA devices only (model.device={device}); there is no CPU path")
    stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
    _lib.check(getattr(_lib.lib(), f"nb2_ik_{name}")(*args, stream), f"nb2_ik_{name}")


def _validate_joint_dof_mask(model, joint_dof_mask) -> None:
    """``_validate_joint_dof_mask`` (ik_lm_optimizer.py:93-118)."""
    if not isinstance(joint_dof_mask, torch.Tensor) or joint_dof_mask.dtype != torch.bool:
        raise ValueError("joint_dof_mask must have dtype torch.bool")
    if joint_dof_mask.ndim != 1 or joint_dof_mask.shape[0] != model.joint_dof_count:
        raise ValueError("joint_dof_mask must have shape [joint_dof_count]")
    if joint_dof_mask.device != torch.device(model.device):
        raise ValueError("joint_dof_mask must be on the model device")
    mask = joint_dof_mask.detach().cpu().numpy()
    joint_type = model.numpy("joint_type")
    qd_start = model.numpy("joint_qd_start")
    for j in range(len(joint_type)):
        if joint_type[j] not in (JointType.BALL, JointType.FREE, JointType.DISTANCE):
            continue
        jm = mask[qd_start[j]:qd_start[j + 1]]
        if jm.any() and not jm.all():
            raise ValueError(
                f"joint_dof_mask partially masks joint {j} ({JointType(int(joint_type[j])).name}): quaternion-integrated joints "
                "must have all of their DOFs masked together"
            )


def _affects_dof(model, link_index: int) -> np.ndarray:
    """The ancestor mask of ``init_buffers`` (ik_objectives.py:290-315): dofs of the joints on the chain from ``link_index`` up."""
    qd_start = model.numpy("joint_qd_start")
    child, parent = model.numpy("joint_child"), model.numpy("joint_parent")
    dof_to_joint = np.empty(int(qd_start[-1]), dtype=np.int32)
    for j in range(len(qd_start) - 1):
        dof_to_joint[qd_start[j]:qd_start[j + 1]] = j
    body_to_joint = np.full(int(model.body_count), -1, np.int32)
    for j in range(int(model.joint_count)):
        if child[j] != -1:
            body_to_joint[child[j]] = j
    ancestors = np.zeros(int(model.joint_count), dtype=bool)
    body = link_index
    while body != -1:
        j = body_to_joint[body]
        if j != -1:
            ancestors[j] = True
        body = parent[j] if j != -1 else -1
    return ancestors[dof_to_joint].astype(np.uint8)


def _fk_levels(model) -> tuple[np.ndarray, int]:
    """Schedule of eval_fk_batched's joint loop (articulation a: joints [articulation_start[a], articulation_end[a]) with
    joint_articulation != -1, in order).  Tree depth when every joint reads a parent pose written by an earlier joint of the
    loop and no body is written twice; otherwise every joint gets its own level (the serial loop)."""
    nj = int(model.joint_count)
    level = np.full(nj, -1, dtype=np.int32)
    starts, ends = model.numpy("articulation_start"), model.articulation_end
    ends = model.numpy("articulation_end") if ends is not None else starts[1:]
    art, parent, child = model.numpy("joint_articulation"), model.numpy("joint_parent"), model.numpy("joint_child")
    order = [j for a in range(int(model.articulation_count)) for j in range(int(starts[a]), int(ends[a])) if art[j] != -1]
    writer: dict[int, int] = {}
    ok = True
    for j in order:
        p = int(parent[j])
        if p >= 0 and p not in writer:
            ok = ok and not any(int(child[k]) == p for k in order)  # read before its writer: only the serial loop reproduces it
        level[j] = 0 if p < 0 or p not in writer else level[writer[p]] + 1
        if int(child[j]) in writer:
            ok = False
        writer[int(child[j])] = j
    if not ok:
        for i, j in enumerate(order):
            level[j] = i
    return level, (int(level.max()) + 1 if len(order) else 0)


class IKOptimizerLM:
    """Levenberg-Marquardt optimizer for a batch of IK rows sharing one model and one objective list (reference
    ``IKOptimizerLM``).  Buffers: ``residuals`` [n_batch, n_residuals], ``jacobian`` [n_batch, n_residuals, n_dofs], ``costs``,
    ``lambda_values`` [n_batch], all float32 on the model's device.

    ``jacobian_mode`` must be ``ANALYTIC`` or ``MIXED``.  ``ANALYTIC`` forms body poses with upstream's two-pass FK, which indexes
    bodies by joint: the model must have ``joint_child[j] == j`` for every joint and as many bodies as joints.
    """

    def __init__(self, model, n_batch: int, objectives: Sequence[IKObjective], lambda_initial: float = 0.1,
                 jacobian_mode: IKJacobianType | str = IKJacobianType.ANALYTIC, lambda_factor: float = 2.0, lambda_min: float = 1e-5,
                 lambda_max: float = 1e10, rho_min: float = 1e-3, *, problem_idx=None, joint_dof_mask=None) -> None:
        if isinstance(jacobian_mode, str):
            jacobian_mode = IKJacobianType(jacobian_mode)
        if jacobian_mode not in (IKJacobianType.ANALYTIC, IKJacobianType.MIXED):
            raise ValueError(f"jacobian_mode {jacobian_mode.value!r} is not supported: newton_b200.ik evaluates the built-in objectives' "
                             "analytic Jacobians ('analytic' or 'mixed'); it has no autodiff")
        for o in objectives:
            if type(o) not in _BUILTIN:
                raise ValueError(f"objective {type(o).__name__} is not supported: newton_b200.ik evaluates IKObjectivePosition, "
                                 "IKObjectiveRotation and IKObjectiveJointLimit only (user objectives would carry Warp kernels)")
        if len(objectives) > MAX_OBJECTIVES:
            raise ValueError(f"at most {MAX_OBJECTIVES} objectives, got {len(objectives)}")
        self.model = model
        self.device = torch.device(model.device)
        self.n_batch = int(n_batch)
        self.n_coords = int(model.joint_coord_count)
        self.n_dofs = int(model.joint_dof_count)
        self.objectives = list(objectives)
        self.jacobian_mode = jacobian_mode
        self.lambda_initial, self.lambda_factor, self.lambda_min = float(lambda_initial), float(lambda_factor), float(lambda_min)
        self.lambda_max, self.rho_min = float(lambda_max), float(rho_min)
        jt = model.numpy("joint_type")
        if (jt == int(JointType.ROD)).any():
            raise ValueError("newton_b200.ik does not support ROD / CABLE joints")
        if jacobian_mode == IKJacobianType.ANALYTIC:
            child = model.numpy("joint_child")
            if int(model.body_count) != int(model.joint_count) or not np.array_equal(child, np.arange(len(child))):
                raise ValueError("jacobian_mode='analytic' forms body poses with a two-pass FK that indexes bodies by joint: it needs "
                                 "joint_child[j] == j for every joint and body_count == joint_count; use jacobian_mode='mixed' "
                                 "for this model")
        if jacobian_mode == IKJacobianType.MIXED and model.articulation_end is not None:
            if not np.array_equal(model.numpy("articulation_end"), model.numpy("articulation_start")[1:]):
                raise ValueError("jacobian_mode='mixed' does not support articulations with loop-closing joints")
        if joint_dof_mask is not None:
            _validate_joint_dof_mask(model, joint_dof_mask)
        self.joint_dof_mask = joint_dof_mask
        self.n_seeds = 1
        if problem_idx is not None:
            pi = np.asarray(problem_idx.detach().cpu().numpy() if isinstance(problem_idx, torch.Tensor) else problem_idx)
            seeds = max(1, self.n_batch // max(1, int(pi.max()) + 1)) if pi.size else 1
            if pi.shape != (self.n_batch,) or not np.array_equal(pi, np.arange(self.n_batch) // seeds):
                raise ValueError("problem_idx must map row i to problem i // n_seeds")
            self.n_seeds = seeds

        offsets, off = [], 0
        for o in self.objectives:
            offsets.append(off)
            off += o.residual_dim()
        self.residual_offsets = offsets
        self.n_residuals = off
        n_problems = self.n_batch // self.n_seeds
        for o, offset in zip(self.objectives, offsets):
            o.set_batch_layout(self.n_residuals, offset, self.n_batch)
            o.bind_device(self.device)
            if isinstance(o, IKObjectiveJointLimit) and o.n_dofs != self.n_dofs:
                raise ValueError(f"IKObjectiveJointLimit has {o.n_dofs} limits, the model has {self.n_dofs} dofs")

        dev = self.device
        f32 = dict(dtype=torch.float32, device=dev)
        self.residuals = torch.zeros((self.n_batch, self.n_residuals), **f32)
        self.jacobian = torch.zeros((self.n_batch, self.n_residuals, self.n_dofs), **f32)
        self.costs = torch.zeros(self.n_batch, **f32)
        self.lambda_values = torch.zeros(self.n_batch, **f32)

        # host-built tables (the reference's init_buffers), kept alive with the descriptor that points at them
        q_start, qd_start, dim = model.numpy("joint_q_start"), model.numpy("joint_qd_start"), model.numpy("joint_dof_dim").reshape(-1, 2)
        d2c = np.full(self.n_dofs, -1, dtype=np.int32)
        for j in range(int(model.joint_count)):
            for k in range(int(dim[j, 0] + dim[j, 1])):
                d2c[qd_start[j] + k] = q_start[j] + k
        self._dof_to_coord = torch.from_numpy(d2c).to(dev)
        self._affects = [torch.from_numpy(_affects_dof(model, o.link_index)).to(dev) if not isinstance(o, IKObjectiveJointLimit) else None
                         for o in self.objectives]
        lv, nlv = _fk_levels(model) if jacobian_mode == IKJacobianType.MIXED else (None, 0)
        self._fk_level = None if lv is None else torch.from_numpy(lv).to(dev)
        self._dof_mask = None if joint_dof_mask is None else joint_dof_mask.to(torch.uint8).contiguous()

        d = IkDesc()
        d.model = _abi.model_desc(model)
        d.mode = 0 if jacobian_mode == IKJacobianType.ANALYTIC else 1
        d.n_batch, d.n_seeds, d.n_residuals, d.objective_count = self.n_batch, self.n_seeds, self.n_residuals, len(self.objectives)
        d.lanes = 0
        nd = self.n_dofs
        d.dof_to_coord = _abi.ptr(self._dof_to_coord, "i32", dev, nd, "dof_to_coord")
        d.fk_level = _abi.ptr(self._fk_level, "i32", dev, int(model.joint_count), "fk_level")
        d.fk_level_count = nlv
        d.dof_mask = _abi.ptr(self._dof_mask, "u8", dev, nd, "joint_dof_mask")
        d.lambda_initial, d.lambda_factor, d.lambda_min, d.lambda_max, d.rho_min = (
            self.lambda_initial, self.lambda_factor, self.lambda_min, self.lambda_max, self.rho_min)
        for i, (o, row) in enumerate(zip(self.objectives, offsets)):
            od = d.objectives[i]
            od.row, od.weight = row, o.weight
            if isinstance(o, IKObjectivePosition):
                od.kind, od.link = 1, o.link_index
                od.offset[:] = (*o.link_offset, 0.0)
                od.target = _abi.ptr(o.target_positions, "f32", dev, 3 * n_problems, "target_positions")
            elif isinstance(o, IKObjectiveRotation):
                od.kind, od.link, od.canonicalize = 2, o.link_index, int(o.canonicalize_quat_err)
                od.offset[:] = o.link_offset_rotation
                od.target = _abi.ptr(o.target_rotations, "f32", dev, 4 * n_problems, "target_rotations")
            else:
                od.kind = 3
                od.limit_lower = _abi.ptr(o.joint_limit_lower, "f32", dev, nd, "joint_limit_lower")
                od.limit_upper = _abi.ptr(o.joint_limit_upper, "f32", dev, nd, "joint_limit_upper")
            if od.kind in (1, 2):
                if not 0 <= o.link_index < int(model.body_count):
                    raise ValueError(f"link_index {o.link_index} is out of range for {int(model.body_count)} bodies")
                od.affects_dof = _abi.ptr(self._affects[i], "u8", dev, nd, "affects_dof")
        self._desc = d

    def _rows(self, a, name: str):
        if not isinstance(a, torch.Tensor) or a.shape != (self.n_batch, self.n_coords):
            raise ValueError(f"{name} has incompatible shape")
        return _abi.ptr(a, "f32", self.device, self.n_batch * self.n_coords, name)

    def _solve(self, joint_q_in, joint_q, joint_q_out, iterations: int, step_size: float, write_lambda: bool, seed_state=None) -> None:
        _call("solve", self.device, C.byref(self._desc), joint_q_in, joint_q, joint_q_out,
              _abi.ptr(self.residuals, "f32", self.device), _abi.ptr(self.costs, "f32", self.device),
              _abi.ptr(self.lambda_values, "f32", self.device), _abi.ptr(self.jacobian, "f32", self.device), C.c_int32(int(iterations)),
              C.c_float(float(step_size)), C.c_int32(1 if write_lambda else 0), seed_state)

    def step(self, joint_q_in, joint_q_out, iterations: int = 10, step_size: float = 1.0) -> None:
        """Run ``iterations`` LM iterations on every row (one launch); ``joint_q_out`` may alias ``joint_q_in``."""
        qi, qo = self._rows(joint_q_in, "joint_q_in"), self._rows(joint_q_out, "joint_q_out")
        self._solve(qi, qo, None, iterations, step_size, True)

    def compute_costs(self, joint_q):
        """Residuals and costs (sum of squares) of ``joint_q`` [n_batch, coords]; returns ``costs``."""
        q = self._rows(joint_q, "joint_q")
        self._solve(q, q, None, 0, 1.0, False)
        return self.costs

    def reset(self) -> None:
        """Clear the LM damping before a new solve."""
        self.lambda_values.zero_()


class IKSolver:
    """Inverse kinematics with optional multi-seed sampling (reference ``newton.ik.IKSolver``).

    Expands ``n_problems`` into ``n_problems * n_seeds`` rows, solves them with :class:`IKOptimizerLM` and keeps the
    lowest-cost seed per problem (the first on ties).  ``optimizer`` must be ``"lm"``; ``jacobian_mode`` ``"analytic"`` or
    ``"mixed"``.  ``joint_dof_mask`` needs ``sampler="none"``.  After :meth:`step`, ``joint_q`` holds the expanded rows, and
    ``residuals`` / ``costs`` / ``lambda_values`` / ``jacobian`` (through the optimizer) those of the last solve.
    """

    def __init__(self, model, n_problems: int, objectives: Sequence[IKObjective], *, optimizer: IKOptimizer | str = IKOptimizer.LM,
                 jacobian_mode: IKJacobianType | str = IKJacobianType.AUTODIFF, sampler: IKSampler | str = IKSampler.NONE,
                 n_seeds: int = 1, noise_std: float = 0.1, rng_seed: int = 12345, lambda_initial: float = 0.1,
                 lambda_factor: float = 2.0, lambda_min: float = 1e-5, lambda_max: float = 1e10, rho_min: float = 1e-3,
                 joint_dof_mask=None, history_len: int = 10, h0_scale: float = 1.0, line_search_alphas=None, wolfe_c1: float = 1e-4,
                 wolfe_c2: float = 0.9) -> None:
        if isinstance(optimizer, str):
            optimizer = IKOptimizer(optimizer)
        if isinstance(jacobian_mode, str):
            jacobian_mode = IKJacobianType(jacobian_mode)
        if isinstance(sampler, str):
            sampler = IKSampler(sampler)
        if n_seeds < 1:
            raise ValueError("n_seeds must be >= 1")
        if sampler is IKSampler.NONE and n_seeds != 1:
            raise ValueError("sampler 'none' requires n_seeds == 1")
        if joint_dof_mask is not None:
            if optimizer is not IKOptimizer.LM:
                raise ValueError("joint_dof_mask is only supported by the LM optimizer")
            if sampler is not IKSampler.NONE:
                raise ValueError("joint_dof_mask requires sampler='none'")
        if optimizer is not IKOptimizer.LM:
            raise ValueError(f"optimizer {optimizer.value!r} is not supported: newton_b200.ik builds the Levenberg-Marquardt optimizer "
                             "('lm') only")
        self.model = model
        self.device = torch.device(model.device)
        self.objectives = objectives
        self.optimizer_type = optimizer
        self.sampler = sampler
        self.n_problems = int(n_problems)
        self.n_seeds = int(n_seeds)
        self.n_expanded = self.n_problems * self.n_seeds
        self.n_coords = int(model.joint_coord_count)
        self.noise_std = float(noise_std)
        self._rng_seed = np.uint32(rng_seed)
        dev = self.device
        self.joint_q_expanded = torch.zeros((self.n_expanded, self.n_coords), dtype=torch.float32, device=dev)
        self.best_indices = torch.zeros(self.n_problems, dtype=torch.int32, device=dev)
        self._seed_state = torch.tensor([int(self._rng_seed)], dtype=torch.int64).to(torch.int32).to(dev)
        self.problem_idx_expanded = torch.repeat_interleave(torch.arange(self.n_problems, dtype=torch.int32), self.n_seeds).to(dev)

        # bound tables of the samplers (ik_solver.py:299-308).  Upstream slices joint_limit_lower[:n_coords], which has only
        # joint_dof_count entries: coordinates at or beyond joint_dof_count are treated as unbounded here.
        nd = int(model.joint_dof_count)
        lower = np.full(self.n_coords, np.inf, dtype=np.float32)
        upper = np.full(self.n_coords, np.inf, dtype=np.float32)
        m = min(nd, self.n_coords)
        lower[:m] = model.numpy("joint_limit_lower")[:m]
        upper[:m] = model.numpy("joint_limit_upper")[:m]
        with np.errstate(invalid="ignore", over="ignore"):
            span = upper - lower
            bounded = (np.isfinite(lower) & np.isfinite(upper) & (np.abs(span) < 1.0e5)).astype(np.int32)
        self.joint_lower = torch.from_numpy(np.where(bounded, lower, 0.0).astype(np.float32)).to(dev)
        self.joint_upper = torch.from_numpy(np.where(bounded, upper, 0.0).astype(np.float32)).to(dev)
        self.joint_bounded = torch.from_numpy(bounded).to(dev)
        self.roberts_basis = (torch.from_numpy(self._compute_roberts_basis(self.n_coords)).to(dev)
                              if sampler is IKSampler.ROBERTS else None)

        self._impl = IKOptimizerLM(model, self.n_expanded, objectives, problem_idx=self.problem_idx_expanded,
                                   lambda_initial=lambda_initial, jacobian_mode=jacobian_mode, lambda_factor=lambda_factor,
                                   lambda_min=lambda_min, lambda_max=lambda_max, rho_min=rho_min, joint_dof_mask=joint_dof_mask)
        self.costs_expanded = self._impl.costs

    def step(self, joint_q_in, joint_q_out, iterations: int = 50, step_size: float = 1.0) -> None:
        """Solve every base problem and write the best seed of each to ``joint_q_out`` (may alias ``joint_q_in``)."""
        shape = (self.n_problems, self.n_coords)
        if not isinstance(joint_q_in, torch.Tensor) or joint_q_in.shape != shape:
            raise ValueError("joint_q_in has incompatible shape")
        if not isinstance(joint_q_out, torch.Tensor) or joint_q_out.shape != shape:
            raise ValueError("joint_q_out has incompatible shape")
        dev, n = self.device, self.n_problems * self.n_coords
        qi = _abi.ptr(joint_q_in, "f32", dev, n, "joint_q_in")
        qo = _abi.ptr(joint_q_out, "f32", dev, n, "joint_q_out")
        qe = _abi.ptr(self.joint_q_expanded, "f32", dev, self.n_expanded * self.n_coords, "joint_q_expanded")
        seed = _abi.ptr(self._seed_state, "i32", dev, 1, "seed_state")
        if self.sampler is IKSampler.NONE:  # one launch: copy-in, LM, closing costs, copy-out, counter advance
            self._impl._solve(qi, qe, None if qo == qe else qo, iterations, step_size, True, seed)
            return
        _call("sample", dev, C.c_int32(_SAMPLER_CODE[self.sampler]), C.c_int32(self.n_problems), C.c_int32(self.n_seeds),
              C.c_int32(self.n_coords), qi, _abi.ptr(self.joint_lower, "f32", dev), _abi.ptr(self.joint_upper, "f32", dev),
              _abi.ptr(self.joint_bounded, "i32", dev), _abi.ptr(self.roberts_basis, "f32", dev), C.c_float(self.noise_std), seed, qe)
        single = self.n_seeds == 1
        self._impl._solve(qe, qe, (None if qo == qe else qo) if single else None, iterations, step_size, True, seed)
        if not single:
            _call("select", dev, C.c_int32(self.n_problems), C.c_int32(self.n_seeds), C.c_int32(self.n_coords),
                  _abi.ptr(self.costs_expanded, "f32", dev), qe, _abi.ptr(self.best_indices, "i32", dev), qo)

    def reset(self) -> None:
        """Reset the optimizer state, the selected seeds and the sampler's counter."""
        self._impl.reset()
        self.best_indices.zero_()
        self._seed_state.fill_(int(np.int32(self._rng_seed.view(np.int32))))

    @property
    def joint_q(self):
        """Expanded joint coordinates of every sampled seed [n_problems * n_seeds, coords]."""
        return self.joint_q_expanded

    @property
    def costs(self):
        """Expanded per-seed costs of the last solve."""
        return self.costs_expanded

    def __getattr__(self, name: str) -> Any:
        if name == "_impl":
            raise AttributeError(name)
        return getattr(self._impl, name)

    @staticmethod
    def _compute_roberts_basis(n_coords: int) -> np.ndarray:
        """Generalised golden ratio of dimension ``n_coords`` (ik_solver.py:502-513), in float64, rounded to float32."""
        x = 1.5
        for _ in range(20):
            f = x ** (n_coords + 1) - x - 1.0
            df = (n_coords + 1) * x**n_coords - 1.0
            x_next = x - f / df
            if abs(x_next - x) < 1.0e-12:
                break
            x = x_next
        basis = 1.0 - 1.0 / x ** (1 + np.arange(n_coords))
        return basis.astype(np.float32)

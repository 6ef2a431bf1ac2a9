"""``SolverFeatherstone`` - drop-in for the reference class
(``newton/_src/solvers/featherstone/solver_featherstone.py:135-1066``).

Same constructor kwargs (``:135-146``) and ``step`` signature (``:461-469``).  One fused CUDA kernel per call
(``newton_b200/csrc/nb2_featherstone.cu``).  ``use_tile_gemm`` / ``fuse_cholesky`` select Warp tile kernels in
the reference.  Here H = J^T M J and its Cholesky factor are always fused (``fuse_cholesky`` is accepted and ignored);
``use_tile_gemm=True`` forms H on the tensor cores (``mma.sync`` m16n8k8, 3xTF32) instead of the ordered FP32 sums - opt-in like
upstream, agrees with the default path to ~1e-6 relative instead of bit for bit.
"""

from __future__ import annotations

import ctypes as C

import torch

from .. import _abi, _lib
from ..sim.enums import ModelFlags
from .solver import SolverBase


class SolverFeatherstone(SolverBase):
    def __init__(self, model, *, angular_damping: float = 0.05, update_mass_matrix_interval: int = 1,
                 friction_smoothing: float = 1.0, use_tile_gemm: bool = False, fuse_cholesky: bool = True,
                 deterministic=None):
        super().__init__(model)
        if getattr(model, "particle_count", 0):
            raise NotImplementedError("particles are outside the hot-path scope")
        self.angular_damping = angular_damping
        self.update_mass_matrix_interval = update_mass_matrix_interval
        self.friction_smoothing = friction_smoothing
        self.use_tile_gemm = use_tile_gemm
        self.fuse_cholesky = fuse_cholesky
        # the mass-matrix schedule and the Cholesky factor the steps in between reuse belong to this solver (solver_featherstone.py:
        # 189-190): a second solver on the same model starts its own count and never reads this one's factor
        self._step = 0
        self._mass_matrix_dirty = False
        self._factor = torch.empty(int(_lib.lib().nb2_featherstone_factor_floats(self._native.handle)), dtype=torch.float32,
                                   device=torch.device("cuda", self._native.device_index))

    def notify_model_changed(self, flags: int) -> None:
        """Reference ``solver_featherstone.py:284-288``: body or dof properties (masses, inertias, kinematic flags, armature)
        enter the mass matrix, so the next step forms it whatever ``update_mass_matrix_interval`` says."""
        super().notify_model_changed(flags)
        if int(flags) & (ModelFlags.BODY_PROPERTIES | ModelFlags.JOINT_DOF_PROPERTIES):
            self._mass_matrix_dirty = True

    def step(self, state_in, state_out, control, contacts, dt: float) -> None:
        """Advance by ``dt`` (reference ``solver_featherstone.py:461-1066``): writes ``state_out.joint_q/joint_qd/
        body_q/body_qd`` (+ ``body_parent_f`` when requested: compute_body_parent_f, featherstone/kernels.py:2371-2416) and, like
        the reference, refreshes ``state_in.body_q`` by forward kinematics."""
        model = self.model
        if control is None:
            control = model.control(clone_variables=False)
        use_contacts = 1 if self._prepare_contacts(contacts) else 0
        form = self._mass_matrix_dirty or self._step % max(int(self.update_mass_matrix_interval), 1) == 0
        p = _abi.FeatherstoneParams(self.angular_damping, int(self.update_mass_matrix_interval), self.friction_smoothing,
                                    1 if self.use_tile_gemm else 0, 1 if form else 0, self._factor.data_ptr())
        st = _lib.lib().nb2_featherstone_step(
            self._native.handle, C.byref(p), C.byref(_abi.state_view(state_in, model)), C.byref(_abi.state_view(state_out, model)),
            C.byref(_abi.control_view(control, model)), use_contacts, C.c_float(dt), _lib.current_stream_ptr(model),
        )
        _lib.check(st, "nb2_featherstone_step")
        if form:
            self._mass_matrix_dirty = False
        self._step += 1

"""CPU oracle - TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import this package.  The product path (``newton_b200``) never does and fails loudly without
its CUDA library.

``liboracle.so`` (built by ``oracle/Makefile`` from every ``oracle/*.cpp``) restates the reference
kernels of SURVEY.md §8(a) on the CPU; this module wraps it behind classes with the reference's own
call signatures (``SolverXPBD.step``, ``CollisionPipeline.collide`` ...) operating on CPU tensors.  The
sub-modules (``oracle.dynamics``, ``oracle.actuator`` ...) wrap the other entry points of the same library.
"""

from __future__ import annotations

import ctypes as C
import glob
import os
import subprocess

import numpy as np
import torch

from newton_b200 import _abi
from newton_b200.sim.model import Contacts

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SO = os.path.join(_HERE, "liboracle.so")
_LIB = None


def build(force: bool = False) -> str:
    """Run ``oracle/Makefile`` when ``liboracle.so`` is missing or older than a file it may compile; make then recompiles
    the objects whose compiler-written dependency lists name a changed file.  Starts no process when the library is current."""
    deps = [os.path.join(_HERE, "Makefile"), os.path.join(_ROOT, "include", "newton_b200.h")]
    for pattern in ("oracle/*.cpp", "oracle/*.h", "newton_b200/csrc/*.cuh"):
        deps += glob.glob(os.path.join(_ROOT, pattern))
    if force or not os.path.exists(_SO) or any(os.path.getmtime(p) > os.path.getmtime(_SO) for p in deps):
        subprocess.run(["make", "-C", _HERE, "-s", "-j", *(["-B"] if force else [])], check=True, capture_output=True)
        os.utime(_SO)  # current now, even when the newer file was a header no object includes and make had nothing to do
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        _LIB = C.CDLL(_SO)
        _LIB.orc_collide.restype = C.c_int
        _LIB.orc_collide_speculative.restype = C.c_int
        _LIB.orc_primitive_pair.restype = C.c_int
        _LIB.orc_convex_pair.restype = C.c_int
        _LIB.orc_version.restype = C.c_char_p
        _LIB.orc_featherstone_new.restype = C.c_void_p
        _LIB.orc_featherstone_free.argtypes = [C.c_void_p]
    return _LIB


def _check_cpu(model):
    if str(model.device) != "cpu":
        raise ValueError("the oracle runs on CPU tensors only")


class CollisionPipeline:
    """Oracle for reference ``CollisionPipeline`` (``sim/collide.py:1104-2207``).

    ``broad_phase="explicit"`` sweeps ``model.shape_contact_pairs``.  ``"nxn"`` / ``"sap"`` generate the candidate pairs at run
    time from the current AABBs (``oracle/broad_phase.py``: restatements of ``_nxn_broadphase_kernel`` and of the SAP project /
    sort / range / sweep kernels with the reference's per-pair filters) and feed them to the same narrow phase;
    ``model.shape_contact_pairs`` is not read.  Pairs of two global (world -1) shapes are dropped in every mode: no body is
    involved, and the product keeps no contact blocks for them."""

    def __init__(self, model, *, broad_phase=None, rigid_contact_max=None, deterministic=True, include_static_kinematic_pairs=True,
                 speculative_config=None, reduce_contacts=False):
        _check_cpu(model)
        if reduce_contacts:  # mesh contacts: only narrow_phase_process_mesh_plane_contacts_kernel (the unreduced variant) is restated
            raise NotImplementedError("the oracle restates the unreduced mesh-plane kernel only (reduce_contacts=False)")
        # speculative contacts (sim/collide.py:1076-1102, 1315-1317): any object with .max_speculative_extension
        self.speculative_config = speculative_config
        if speculative_config is not None:
            v = float(speculative_config.max_speculative_extension)
            if not np.isfinite(v) or v < 0.0:
                raise ValueError(f"max_speculative_extension must be a non-negative finite number, got {v!r}")
        if broad_phase not in (None, "explicit", "nxn", "sap"):
            raise ValueError(f"unknown broad_phase {broad_phase!r}")
        self.model = model
        self.broad_phase = broad_phase or "explicit"
        self.include_static_kinematic_pairs = include_static_kinematic_pairs
        self.deterministic = deterministic
        self._desc = _abi.model_desc(model)
        if self.broad_phase == "explicit":
            pair_count = model.shape_contact_pair_count
        else:
            ns = np.bincount(model.numpy("shape_world")[model.numpy("shape_world") >= 0], minlength=max(1, model.world_count))
            ng = int((model.numpy("shape_world") < 0).sum())
            pair_count = int(sum((n + ng) * (n + ng - 1) // 2 for n in ns))
        st = model.numpy("shape_type")
        mesh_vertices = 0
        if (st == 8).any():  # GeoType.MESH: one contact per vertex and plane (narrow_phase.py:1761-1861)
            mesh_vertices = int(model.numpy("shape_hull_count")[st == 8].sum()) * max(1, int((st == 1).sum()))
        self.rigid_contact_max = int(rigid_contact_max) if rigid_contact_max is not None else max(1000, 5 * pair_count + mesh_vertices)
        self.candidate_count = 0
        self.last_candidates = None

    def contacts(self) -> Contacts:
        return Contacts(self.rigid_contact_max, 0, device="cpu",
                        requested_attributes=self.model._requested_contact_attributes)

    def _candidates(self, state, dt=0.0, max_ext=0.0):
        from . import broad_phase as _bp

        active = self.speculative_config is not None and dt > 0.0 and max_ext > 0.0
        filt = getattr(self.model, "shape_collision_filter_pairs", ())
        if active:  # swept AABBs: compute_shape_velocities + check_aabb_overlap_moving (collide.py:1877-1947)
            lo, hi, disp = shape_aabbs_speculative(self.model, state.body_q, state.body_qd, dt, max_ext)
            if self.broad_phase == "nxn":
                pairs = _bp.nxn_candidate_pairs(self.model, lo, hi, filt, self.include_static_kinematic_pairs, displacement=disp)
            else:
                pairs = _bp.sap_candidate_pairs(self.model, lo, hi, filt, self.include_static_kinematic_pairs, displacement=disp,
                                                sort_axis_displacement_limit=max_ext)
        else:
            lo, hi = shape_aabbs(self.model, state.body_q)
            fn = _bp.nxn_candidate_pairs if self.broad_phase == "nxn" else _bp.sap_candidate_pairs
            pairs = fn(self.model, lo, hi, filt, self.include_static_kinematic_pairs)
        sw = self.model.numpy("shape_world")
        if np.all(sw < 0):  # model built without begin_world(): one implicit world holding everything (builder.py:11276)
            return pairs
        return [p for p in pairs if not (sw[p[0]] < 0 and sw[p[1]] < 0)]

    def collide(self, state, contacts, *, soft_contact_margin=None, dt=None):
        v = _abi.contacts_view(contacts)
        desc = self._desc
        keep = None
        spec_dt, spec_ext = 0.0, 0.0
        if self.speculative_config is not None:  # collide.py:1823-1833
            if dt is None:
                raise ValueError("dt must be provided when speculative contacts are enabled")
            spec_dt = float(dt)
            if not np.isfinite(spec_dt) or spec_dt < 0.0:
                raise ValueError(f"dt must be a non-negative finite number, got {spec_dt!r}")
            spec_ext = float(self.speculative_config.max_speculative_extension)
        if self.broad_phase != "explicit":
            self.last_candidates = self._candidates(state, spec_dt, spec_ext)
            keep = np.ascontiguousarray(np.asarray(self.last_candidates, dtype=np.int32).reshape(-1, 2))
            desc = _abi.ModelDesc.from_buffer_copy(self._desc)
            desc.shape_contact_pairs = keep.ctypes.data if keep.size else None
            desc.shape_pair_count = int(keep.shape[0])
        elif not self.include_static_kinematic_pairs:
            from . import broad_phase as _bp

            m = self.model
            bf = m.numpy("body_flags") if m.body_count else ()
            pairs = [tuple(p) for p in m.numpy("shape_contact_pairs").tolist()
                     if not _bp.is_shape_pair_immovable_filtered(p[0], p[1], m.numpy("shape_body"), bf, False)]
            keep = np.ascontiguousarray(np.asarray(pairs, dtype=np.int32).reshape(-1, 2))
            desc = _abi.ModelDesc.from_buffer_copy(self._desc)
            desc.shape_contact_pairs = keep.ctypes.data if keep.size else None
            desc.shape_pair_count = int(keep.shape[0])
        if self.speculative_config is not None:
            self.candidate_count = lib().orc_collide_speculative(
                C.byref(desc), C.c_void_p(_abi.ptr(state.body_q)), C.c_void_p(_abi.ptr(state.body_qd)), C.c_float(spec_dt),
                C.c_float(spec_ext), C.byref(v), C.c_int(1 if self.deterministic else 0))
        else:
            self.candidate_count = lib().orc_collide(
                C.byref(desc), C.c_void_p(_abi.ptr(state.body_q)), C.byref(v), C.c_int(1 if self.deterministic else 0)
            )
            if self.candidate_count < 0:
                raise NotImplementedError("oracle: mesh-mesh / mesh-convex / mesh-finite-plane pairs (BVH / SDF routes) are not restated")
        del keep


class SolverXPBD:
    """Oracle for reference ``SolverXPBD`` (``solvers/xpbd/solver_xpbd.py:99-862``), rigid-body path."""

    def __init__(self, model, *, iterations=2, soft_body_relaxation=0.9, soft_contact_relaxation=0.9,
                 joint_linear_relaxation=0.7, joint_angular_relaxation=0.4, joint_linear_compliance=0.0,
                 joint_angular_compliance=0.0, rigid_contact_relaxation=0.8, rigid_contact_con_weighting=True,
                 angular_damping=0.0, enable_restitution=False, deterministic=None):
        _check_cpu(model)
        self.model = model
        self._desc = _abi.model_desc(model)
        self.compute_body_velocity_from_position_delta = False  # attribute, solver_xpbd.py:171
        self._args = (iterations, joint_linear_relaxation, joint_angular_relaxation, joint_linear_compliance,
                      joint_angular_compliance, rigid_contact_relaxation, 1 if rigid_contact_con_weighting else 0,
                      angular_damping, 1 if enable_restitution else 0)
        self._contact_impulse = None
        self._last_dt = None

    @property
    def params(self):
        return _abi.XPBDParams(*self._args, 1 if self.compute_body_velocity_from_position_delta else 0)

    def reset(self, state, world_mask=None, flags=None):
        """SolverBase.reset (solvers/solver.py:344-375): no-op for XPBD."""

    def notify_model_changed(self, flags):
        """SolverBase.notify_model_changed (solvers/solver.py:394-429): the kernels read the Model arrays on every step."""
        self._desc = _abi.model_desc(self.model)

    def step(self, state_in, state_out, control, contacts, dt):
        if control is None:
            control = self.model.control(clone_variables=False)
        sv_in, sv_out, cv = _abi.state_view(state_in), _abi.state_view(state_out), _abi.control_view(control)
        imp = None
        if contacts is not None:
            ctv = _abi.contacts_view(contacts)
            ctp = C.byref(ctv)
            if getattr(contacts, "force", None) is not None:
                self._contact_impulse = np.zeros((contacts.rigid_contact_max, 6), dtype=np.float32)
                imp = C.c_void_p(self._contact_impulse.ctypes.data)
        else:
            ctp = None
        p = self.params
        lib().orc_xpbd_step(C.byref(self._desc), C.byref(p), C.byref(sv_in), C.byref(sv_out), C.byref(cv), ctp,
                            C.c_float(dt), imp)
        self._last_dt = dt

    def update_contacts(self, contacts, state=None):
        """``SolverXPBD.update_contacts`` (solver_xpbd.py:864-925)."""
        if getattr(contacts, "force", None) is None:
            raise ValueError("contacts.force is not allocated")
        if self._contact_impulse is None:
            raise ValueError("No contact impulse data available. Call step() before update_contacts().")
        if contacts.rigid_contact_max != self._contact_impulse.shape[0]:
            raise ValueError("Contacts capacity mismatch")
        ctv = _abi.contacts_view(contacts)
        lib().orc_xpbd_update_contacts(C.byref(ctv), C.c_void_p(self._contact_impulse.ctypes.data), C.c_float(self._last_dt))

    def integrate_bodies(self, model, state_in, state_out, dt, angular_damping=0.0):
        sv_in, sv_out = _abi.state_view(state_in), _abi.state_view(state_out)
        lib().orc_integrate_bodies(C.byref(self._desc), C.byref(sv_in), C.byref(sv_out), C.c_float(angular_damping),
                                   C.c_float(dt))


class SolverFeatherstone:
    """Oracle for reference ``SolverFeatherstone`` (``solvers/featherstone/solver_featherstone.py:135-1066``)."""

    def __init__(self, model, *, angular_damping=0.05, update_mass_matrix_interval=1, friction_smoothing=1.0,
                 use_tile_gemm=False, fuse_cholesky=True, deterministic=None):
        _check_cpu(model)
        self.model = model
        self._desc = _abi.model_desc(model)
        self.params = _abi.FeatherstoneParams(angular_damping, update_mass_matrix_interval, friction_smoothing, 0)
        self._h = C.c_void_p(lib().orc_featherstone_new())

    def __del__(self):
        try:
            lib().orc_featherstone_free(self._h)
        except Exception:
            pass

    def reset(self, state, world_mask=None, flags=None):
        """SolverBase.reset (solvers/solver.py:344-375): no-op for Featherstone."""

    def notify_model_changed(self, flags):
        """SolverFeatherstone.notify_model_changed (solver_featherstone.py:284-288): the kernels read the Model arrays on every
        step; BODY_PROPERTIES / JOINT_DOF_PROPERTIES also make the next step form the mass matrix."""
        self._desc = _abi.model_desc(self.model)
        lib().orc_featherstone_notify_changed(self._h, C.c_int(int(flags)))

    def step(self, state_in, state_out, control, contacts, dt):
        if control is None:
            control = self.model.control(clone_variables=False)
        sv_in, sv_out, cv = _abi.state_view(state_in), _abi.state_view(state_out), _abi.control_view(control)
        if contacts is not None:
            ctv = _abi.contacts_view(contacts)
            ctp = C.byref(ctv)
        else:
            ctp = None
        lib().orc_featherstone_step(self._h, C.byref(self._desc), C.byref(self.params), C.byref(sv_in), C.byref(sv_out),
                                    C.byref(cv), ctp, C.c_float(dt))


    def mass_matrix(self, articulation: int = 0):
        """H = J^T M J of one articulation as the last ``step()`` formed it (before the armature goes onto the diagonal): test
        access to the dense stage, used to pin it against the closed forms of ``newton/tests/test_jacobian_mass_matrix.py``."""
        n_max = int(self.model.joint_dof_count)
        out = np.zeros(n_max * n_max, dtype=np.float32)
        L = lib()
        L.orc_featherstone_mass_matrix.restype = C.c_int
        n = L.orc_featherstone_mass_matrix(self._h, C.byref(self._desc), C.c_int(articulation), C.c_void_p(out.ctypes.data),
                                            C.c_int(out.size))
        if n < 0:
            raise RuntimeError("mass_matrix: call step() first / bad articulation index")
        return out[: n * n].reshape(n, n).copy()


class _Shard(C.Structure):
    _fields_ = [("model", C.c_void_p), ("state_0", _abi.StateView), ("state_1", _abi.StateView), ("control", _abi.ControlView),
                ("contacts", _abi.ContactsView), ("featherstone", C.c_void_p)]


class _Loop(C.Structure):
    _fields_ = [("solver", C.c_int32), ("deterministic", C.c_int32), ("substeps", C.c_int32), ("dt", C.c_float), ("xpbd", _abi.XPBDParams),
                ("featherstone", _abi.FeatherstoneParams)]


class FramePool:
    """bench.py's CPU arm: the reference substep loop (clear_forces -> collide -> solver.step -> swap) of many independent
    world shards on a persistent pool of native threads (``orc_pool_*`` in oracle.cpp).  Threads are created here, before any
    timer; :meth:`run_frames` returns the seconds measured inside the library around the parallel region only."""

    def __init__(self, models, make_solver, *, substeps: int, dt: float, threads: int, deterministic: bool = False):
        L = lib()
        L.orc_pool_new.restype = C.c_void_p
        L.orc_pool_free.argtypes = [C.c_void_p]
        L.orc_pool_run_frames.restype = C.c_double
        self.threads = int(threads)
        self._keep = []
        self._shards = (_Shard * len(models))()
        solver0 = None
        for i, m in enumerate(models):
            pipe, solver = CollisionPipeline(m, deterministic=deterministic), make_solver(m)
            s0, s1, ctrl, contacts = m.state(), m.state(), m.control(), pipe.contacts()
            self._keep.append((m, pipe, solver, s0, s1, ctrl, contacts))
            sh = self._shards[i]
            sh.model = C.addressof(solver._desc)
            sh.state_0, sh.state_1 = _abi.state_view(s0), _abi.state_view(s1)
            sh.control, sh.contacts = _abi.control_view(ctrl), _abi.contacts_view(contacts)
            sh.featherstone = solver._h if isinstance(solver, SolverFeatherstone) else None
            solver0 = solver0 or solver
        self._loop = _Loop()
        self._loop.substeps, self._loop.dt = int(substeps), float(dt)
        self._loop.deterministic = 1 if deterministic else 0  # False = the reference default (kernel emission order)
        if isinstance(solver0, SolverFeatherstone):
            self._loop.solver, self._loop.featherstone = 1, solver0.params
        else:
            self._loop.solver, self._loop.xpbd = 0, solver0.params
        self._h = C.c_void_p(L.orc_pool_new(self.threads))

    def run_frames(self, frames: int) -> float:
        self._substeps_done = getattr(self, "_substeps_done", 0) + int(frames) * int(self._loop.substeps)
        return float(lib().orc_pool_run_frames(self._h, self._shards, C.c_int(len(self._shards)), C.byref(self._loop),
                                               C.c_int(int(frames))))

    def current_states(self):
        """The State holding the latest result of every shard (the library swaps its two views after every substep)."""
        odd = getattr(self, "_substeps_done", 0) % 2 == 1
        return [k[4] if odd else k[3] for k in self._keep]

    def contacts(self):
        """The Contacts buffer of every shard (what the last substep's collide produced)."""
        return [k[6] for k in self._keep]

    def close(self):
        if self._h is not None:
            lib().orc_pool_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def primitive_pair(type_a, scale_a, xform_a, type_b, scale_b, xform_b, plane_box_margin=0.0):
    """One analytic collider call: returns (is_analytic, dist[4], pos[4,3], normal[3])."""
    sa = np.asarray(scale_a, dtype=np.float32)
    sb = np.asarray(scale_b, dtype=np.float32)
    xa = np.asarray(xform_a, dtype=np.float32)
    xb = np.asarray(xform_b, dtype=np.float32)
    dist = np.zeros(4, dtype=np.float32)
    pos = np.zeros((4, 3), dtype=np.float32)
    n = np.zeros(3, dtype=np.float32)
    ok = lib().orc_primitive_pair(
        int(type_a), C.c_void_p(sa.ctypes.data), C.c_void_p(xa.ctypes.data), int(type_b), C.c_void_p(sb.ctypes.data),
        C.c_void_p(xb.ctypes.data), C.c_float(plane_box_margin), C.c_void_p(dist.ctypes.data),
        C.c_void_p(pos.ctypes.data), C.c_void_p(n.ctypes.data),
    )
    return bool(ok), dist, pos, n


IMPLS = {"oracle": 0, "product_host": 1}


def convex_pair(type_a, scale_a, xform_a, type_b, scale_b, xform_b, gap_sum=0.2, impl="oracle", margin_a=0.0, margin_b=0.0):
    """GJK/MPR + manifold for one convex pair: returns (count, dist[5], pos[5,3], normal[5,3]).

    ``impl``: "oracle" = oracle_convex.h (the oracle's own restatement), "product_host" = the product's
    nb2_convex.cuh compiled for the host (only for the bit-equality test between the two)."""
    sa = np.asarray(scale_a, dtype=np.float32)
    sb = np.asarray(scale_b, dtype=np.float32)
    xa = np.asarray(xform_a, dtype=np.float32)
    xb = np.asarray(xform_b, dtype=np.float32)
    dist = np.zeros(5, dtype=np.float32)
    pos = np.zeros((5, 3), dtype=np.float32)
    n = np.zeros((5, 3), dtype=np.float32)
    cnt = lib().orc_convex_pair(
        int(type_a), C.c_void_p(sa.ctypes.data), C.c_void_p(xa.ctypes.data), int(type_b), C.c_void_p(sb.ctypes.data),
        C.c_void_p(xb.ctypes.data), C.c_float(gap_sum), C.c_void_p(dist.ctypes.data), C.c_void_p(pos.ctypes.data),
        C.c_void_p(n.ctypes.data), C.c_int(IMPLS[impl]), C.c_float(margin_a), C.c_float(margin_b),
    )
    return cnt, dist, pos, n


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def convex_pair_speculative(type_a, scale_a, xform_a, type_b, scale_b, xform_b, search_gap_sum, base_gap_sum, dt, max_extension, lin_a, ang_a,
                            lin_b, ang_b, impl="oracle"):
    """``convex_pair`` with the speculative writer (write_contact_speculative): the pair sees ``search_gap_sum``, admission uses
    ``base_gap_sum`` + the predictive score from the shapes' velocities (origins = the transforms' positions)."""
    sa, sb, xa, xb = _f32(scale_a), _f32(scale_b), _f32(xform_a), _f32(xform_b)
    spec = _f32(np.concatenate([[base_gap_sum, dt, max_extension], xa[:3], xb[:3], lin_a, lin_b, ang_a, ang_b]))
    dist, pos, n = np.zeros(5, np.float32), np.zeros((5, 3), np.float32), np.zeros((5, 3), np.float32)
    L = lib()
    L.orc_convex_pair_spec.restype = C.c_int
    cnt = L.orc_convex_pair_spec(int(type_a), C.c_void_p(sa.ctypes.data), C.c_void_p(xa.ctypes.data), int(type_b), C.c_void_p(sb.ctypes.data),
                                 C.c_void_p(xb.ctypes.data), C.c_float(search_gap_sum), C.c_void_p(spec.ctypes.data), C.c_void_p(dist.ctypes.data),
                                 C.c_void_p(pos.ctypes.data), C.c_void_p(n.ctypes.data), C.c_int(IMPLS[impl]))
    return cnt, dist, pos, n


def convex_pair_hull(type_a, scale_a, xform_a, hull_a, type_b, scale_b, xform_b, hull_b, gap_sum=0.2, impl="oracle"):
    """``convex_pair`` with CONVEX_MESH operands: ``hull_*`` = unscaled vertices ``[n, 3]`` (None for primitives)."""
    sa, sb, xa, xb = _f32(scale_a), _f32(scale_b), _f32(xform_a), _f32(xform_b)
    ha = None if hull_a is None else _f32(hull_a).reshape(-1, 3)
    hb = None if hull_b is None else _f32(hull_b).reshape(-1, 3)
    dist, pos, n = np.zeros(5, np.float32), np.zeros((5, 3), np.float32), np.zeros((5, 3), np.float32)
    L = lib()
    L.orc_convex_pair_hull.restype = C.c_int
    cnt = L.orc_convex_pair_hull(
        int(type_a), C.c_void_p(sa.ctypes.data), C.c_void_p(xa.ctypes.data), C.c_void_p(None if ha is None else ha.ctypes.data),
        C.c_int(0 if ha is None else ha.shape[0]), int(type_b), C.c_void_p(sb.ctypes.data), C.c_void_p(xb.ctypes.data),
        C.c_void_p(None if hb is None else hb.ctypes.data), C.c_int(0 if hb is None else hb.shape[0]), C.c_float(gap_sum),
        C.c_void_p(dist.ctypes.data), C.c_void_p(pos.ctypes.data), C.c_void_p(n.ctypes.data), C.c_int(IMPLS[impl]))
    return cnt, dist, pos, n


def hull_support_aabb(scale, hull, direction, xform, impl="oracle"):
    """CONVEX_MESH support point in ``direction`` and tight world AABB under ``xform``: returns (support, lower, upper)."""
    s, h, d, x = _f32(scale), _f32(hull).reshape(-1, 3), _f32(direction), _f32(xform)
    out = np.zeros(9, np.float32)
    lib().orc_hull_support_aabb(C.c_void_p(s.ctypes.data), C.c_void_p(h.ctypes.data), C.c_int(h.shape[0]), C.c_void_p(d.ctypes.data),
                                C.c_void_p(x.ctypes.data), C.c_void_p(out.ctypes.data), C.c_int(IMPLS[impl]))
    return out[:3], out[3:6], out[6:]


def mpr_core(type_a, scale_a, type_b, scale_b, pos_b, quat_b, extend=0.0, impl="oracle"):
    """solve_mpr_core in A's frame: returns (collision, point_a, point_b, normal, penetration)."""
    sa, sb, pb, qb = _f32(scale_a), _f32(scale_b), _f32(pos_b), _f32(quat_b)
    out = np.zeros(10, dtype=np.float32)
    hit = lib().orc_mpr_core(int(type_a), C.c_void_p(sa.ctypes.data), int(type_b), C.c_void_p(sb.ctypes.data),
                             C.c_void_p(pb.ctypes.data), C.c_void_p(qb.ctypes.data), C.c_float(extend),
                             C.c_void_p(out.ctypes.data), C.c_int(IMPLS[impl]))
    return hit, out[0:3], out[3:6], out[6:9], float(out[9])


def gjk_core(type_a, scale_a, type_b, scale_b, pos_b, quat_b, extend=0.0, eps=1e-4, impl="oracle"):
    """solve_closest_distance_core in A's frame: returns (separated, point_a, point_b, normal, distance)."""
    sa, sb, pb, qb = _f32(scale_a), _f32(scale_b), _f32(pos_b), _f32(quat_b)
    out = np.zeros(10, dtype=np.float32)
    sep = lib().orc_gjk_core(int(type_a), C.c_void_p(sa.ctypes.data), int(type_b), C.c_void_p(sb.ctypes.data),
                             C.c_void_p(pb.ctypes.data), C.c_void_p(qb.ctypes.data), C.c_float(extend), C.c_float(eps),
                             C.c_void_p(out.ctypes.data), C.c_int(IMPLS[impl]))
    return sep, out[0:3], out[3:6], out[6:9], float(out[9])


def support_map(geo_type, scale, direction, impl="oracle"):
    s, d = _f32(scale), _f32(direction)
    out = np.zeros(3, dtype=np.float32)
    lib().orc_support_map(int(geo_type), C.c_void_p(s.ctypes.data), C.c_void_p(d.ctypes.data), C.c_void_p(out.ctypes.data),
                          C.c_int(IMPLS[impl]))
    return out


def tight_aabb(geo_type, scale, xform, impl="oracle"):
    """compute_tight_aabb_from_support (collision_core.py:454-548): returns (lower, upper)."""
    s, x = _f32(scale), _f32(xform)
    out = np.zeros(6, dtype=np.float32)
    lib().orc_tight_aabb(int(geo_type), C.c_void_p(s.ctypes.data), C.c_void_p(x.ctypes.data), C.c_void_p(out.ctypes.data), C.c_int(IMPLS[impl]))
    return out[:3], out[3:]


def eval_fk(model, joint_q, joint_qd, state, mask=None, indices=None, body_flag_filter=3):
    """newton.eval_fk: writes state.body_q / state.body_qd (state may be the model); optional articulation mask / indices and
    body-flag filter (BodyFlags.ALL = 3; bodies that do not match keep their values)."""
    if mask is not None and indices is not None:
        raise ValueError("Cannot specify both mask and indices parameters")
    d = _abi.model_desc(model)
    if mask is None and indices is None and int(body_flag_filter) == 3:
        lib().orc_eval_fk(C.byref(d), C.c_void_p(_abi.ptr(joint_q)), C.c_void_p(_abi.ptr(joint_qd)),
                          C.c_void_p(_abi.ptr(state.body_q)), C.c_void_p(_abi.ptr(state.body_qd)))
        return
    m = None if mask is None else np.ascontiguousarray(np.asarray(mask.cpu() if hasattr(mask, "cpu") else mask), dtype=np.uint8)
    ix = None if indices is None else np.ascontiguousarray(np.asarray(indices.cpu() if hasattr(indices, "cpu") else indices), dtype=np.int32)
    lib().orc_eval_fk_masked(C.byref(d), C.c_void_p(_abi.ptr(joint_q)), C.c_void_p(_abi.ptr(joint_qd)),
                             C.c_void_p(_abi.ptr(state.body_q)), C.c_void_p(_abi.ptr(state.body_qd)),
                             C.c_void_p(None if m is None else m.ctypes.data), C.c_void_p(None if ix is None else ix.ctypes.data),
                             C.c_int(0 if ix is None else ix.size), C.c_int(int(body_flag_filter)))


def eval_ik(model, state, joint_q, joint_qd):
    """newton.eval_ik: body_q / body_qd -> joint_q / joint_qd (sim/articulation.py:640-932)."""
    d = _abi.model_desc(model)
    lib().orc_eval_ik(C.byref(d), C.c_void_p(_abi.ptr(state.body_q)), C.c_void_p(_abi.ptr(state.body_qd)),
                      C.c_void_p(_abi.ptr(joint_q)), C.c_void_p(_abi.ptr(joint_qd)))


def shape_aabbs_speculative(model, body_q, body_qd, dt, max_extension):
    """compute_shape_aabbs + compute_shape_velocities: (lower, upper, displacement) per shape"""
    d = _abi.model_desc(model)
    lo = np.zeros((model.shape_count, 3), dtype=np.float32)
    hi = np.zeros((model.shape_count, 3), dtype=np.float32)
    disp = np.zeros((model.shape_count, 3), dtype=np.float32)
    lib().orc_shape_aabbs_speculative(C.byref(d), C.c_void_p(_abi.ptr(body_q)), C.c_void_p(_abi.ptr(body_qd)), C.c_float(dt),
                                      C.c_float(max_extension), C.c_void_p(lo.ctypes.data), C.c_void_p(hi.ctypes.data),
                                      C.c_void_p(disp.ctypes.data))
    return lo, hi, disp


def shape_aabbs(model, body_q):
    d = _abi.model_desc(model)
    lo = np.zeros((model.shape_count, 3), dtype=np.float32)
    hi = np.zeros((model.shape_count, 3), dtype=np.float32)
    lib().orc_compute_shape_aabbs(C.byref(d), C.c_void_p(_abi.ptr(body_q)), C.c_void_p(lo.ctypes.data),
                                  C.c_void_p(hi.ctypes.data))
    return lo, hi

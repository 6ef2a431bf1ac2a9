"""Loader for ``libnewton_b200.so`` - the C-ABI library holding every CUDA kernel of the hot path.

There is no CPU fallback: if the library is missing or a call fails, an exception is raised.
"""

from __future__ import annotations

import ctypes as C
import os

from . import _abi

_HERE = os.path.dirname(os.path.abspath(__file__))
# Floating-point mode of the kernels.  "strict" (default): no FMA contraction, correctly rounded inverse trig - the build that
# reproduces the CPU oracle bit for bit.  NB2_FP=fast selects the twin library compiled with nvcc's default contraction: same
# sources, same contact indices / counts on the test scenes, body state within the north-star tolerance (1e-5 relative after 100
# substeps, tests/test_gpu_fast_fp.py).  NB2_LIB overrides both.
FP_MODE = os.environ.get("NB2_FP", "strict").lower()
if FP_MODE not in ("strict", "fast"):
    raise ValueError(f"NB2_FP={FP_MODE!r}: expected 'strict' or 'fast'")
LIB_PATH = os.environ.get("NB2_LIB") or os.path.join(_HERE, "libnewton_b200_fast.so" if FP_MODE == "fast" else "libnewton_b200.so")
_lib = None

STATUS = {0: "NB2_OK", 1: "NB2_ERR_INVALID_ARGUMENT", 2: "NB2_ERR_UNSUPPORTED", 3: "NB2_ERR_CUDA", 4: "NB2_ERR_CAPACITY"}

# every symbol include/newton_b200.h declares
EXPORTED_SYMBOLS = (
    "nb2_model_create", "nb2_model_destroy", "nb2_model_notify_changed", "nb2_model_rigid_contact_max", "nb2_xpbd_plan_info", "nb2_collide_configure", "nb2_collide", "nb2_collide_speculative", "nb2_contacts_match", "nb2_contacts_sort", "nb2_contacts_import",
    "nb2_xpbd_step", "nb2_xpbd_update_contacts", "nb2_integrate_bodies", "nb2_featherstone_factor_floats", "nb2_featherstone_step", "nb2_semi_implicit_step", "nb2_eval_fk", "nb2_eval_ik", "nb2_eval_fk_masked",
    "nb2_eval_jacobian", "nb2_eval_mass_matrix", "nb2_eval_inverse_dynamics_passive", "nb2_eval_inverse_dynamics_force",
    "nb2_sensor_contact_scratch_bytes", "nb2_sensor_contact_update", "nb2_sensor_frame_transform_update", "nb2_sensor_imu_update", "nb2_raycast_refit", "nb2_intersect_ray",
    "nb2_camera_render", "nb2_actuator_step", "nb2_actuator_reset", "nb2_actuator_network_reset", "nb2_actuator_param_gather", "nb2_actuator_param_scatter",
    "nb2_joint_impedance_step",
    "nb2_ik_solve", "nb2_ik_sample", "nb2_ik_select",
    "nb2_view_gather", "nb2_view_scatter", "nb2_view_articulation_mask", "nb2_last_error", "nb2_kernel_launch_count", "nb2_version",
    "nb2_peer_gather_handle_bytes", "nb2_peer_gather_create", "nb2_peer_gather_buffer", "nb2_peer_gather_stride", "nb2_peer_gather_export",
    "nb2_peer_gather_connect", "nb2_peer_gather_push", "nb2_peer_gather_wait", "nb2_peer_gather_destroy",
)


class Nb2Error(RuntimeError):
    pass


def lib():
    """The loaded library (raises if it has not been built: run ``python -m newton_b200.build``)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Nb2Error(
                f"{LIB_PATH} is missing - build it with `python -m newton_b200.build` (nvcc, sm_90a). "
                "newton_b200 has no CPU or PyTorch fallback for the hot path."
            )
        L = C.CDLL(LIB_PATH)
        P = C.c_void_p
        L.nb2_model_create.argtypes = [C.POINTER(_abi.ModelDesc), C.c_int32, C.POINTER(P)]
        L.nb2_model_create.restype = C.c_int
        L.nb2_model_destroy.argtypes = [P]
        L.nb2_model_destroy.restype = None
        L.nb2_model_notify_changed.argtypes = [P, C.POINTER(_abi.ModelDesc), C.c_int32]
        L.nb2_model_notify_changed.restype = C.c_int
        L.nb2_model_rigid_contact_max.argtypes = [P]
        L.nb2_model_rigid_contact_max.restype = C.c_int32
        L.nb2_xpbd_plan_info.argtypes = [P, C.POINTER(C.c_int32)]
        L.nb2_xpbd_plan_info.restype = C.c_int
        L.nb2_collide_configure.argtypes = [P, C.c_int32, C.c_int32, C.c_int32]
        L.nb2_collide_configure.restype = C.c_int
        L.nb2_collide.argtypes = [P, P, C.POINTER(_abi.ContactsView), P]
        L.nb2_collide.restype = C.c_int
        L.nb2_collide_speculative.argtypes = [P, P, P, C.c_float, C.c_float, C.POINTER(_abi.ContactsView), P]
        L.nb2_collide_speculative.restype = C.c_int
        L.nb2_contacts_match.argtypes = [P, P, C.POINTER(_abi.ContactsView), P, C.POINTER(_abi.MatchOptions), P]
        L.nb2_contacts_match.restype = C.c_int
        L.nb2_contacts_sort.argtypes = [P, C.POINTER(_abi.ContactsView), P]
        L.nb2_contacts_sort.restype = C.c_int
        L.nb2_contacts_import.argtypes = [P, C.POINTER(_abi.ContactsView), P]
        L.nb2_contacts_import.restype = C.c_int
        L.nb2_xpbd_step.argtypes = [P, C.POINTER(_abi.XPBDParams), C.POINTER(_abi.StateView), C.POINTER(_abi.StateView),
                                    C.POINTER(_abi.ControlView), C.c_int32, C.c_float, P]
        L.nb2_xpbd_step.restype = C.c_int
        L.nb2_xpbd_update_contacts.argtypes = [P, C.POINTER(_abi.ContactsView), P]
        L.nb2_xpbd_update_contacts.restype = C.c_int
        L.nb2_integrate_bodies.argtypes = [P, C.POINTER(_abi.StateView), C.POINTER(_abi.StateView), C.c_float, C.c_float, P]
        L.nb2_integrate_bodies.restype = C.c_int
        L.nb2_featherstone_factor_floats.argtypes = [P]
        L.nb2_featherstone_factor_floats.restype = C.c_int64
        L.nb2_featherstone_step.argtypes = [P, C.POINTER(_abi.FeatherstoneParams), C.POINTER(_abi.StateView),
                                            C.POINTER(_abi.StateView), C.POINTER(_abi.ControlView), C.c_int32, C.c_float, P]
        L.nb2_featherstone_step.restype = C.c_int
        L.nb2_semi_implicit_step.argtypes = [P, C.POINTER(_abi.SemiImplicitParams), C.POINTER(_abi.StateView),
                                             C.POINTER(_abi.StateView), C.POINTER(_abi.ControlView), C.c_int32, C.c_float, P]
        L.nb2_semi_implicit_step.restype = C.c_int
        L.nb2_eval_fk.argtypes = [P, P, P, P, P, P]
        L.nb2_eval_fk.restype = C.c_int
        L.nb2_eval_ik.argtypes = [P, P, P, P, P, P]
        L.nb2_eval_ik.restype = C.c_int
        L.nb2_eval_fk_masked.argtypes = [P, P, P, P, P, P, P, C.c_int32, C.c_int32, P]
        L.nb2_eval_fk_masked.restype = C.c_int
        L.nb2_eval_jacobian.argtypes = [P, P, P, P, C.c_int32, C.c_int32, P, P]
        L.nb2_eval_jacobian.restype = C.c_int
        L.nb2_eval_mass_matrix.argtypes = [P, P, P, P, P, C.c_int32, C.c_int32, P, P]
        L.nb2_eval_mass_matrix.restype = C.c_int
        L.nb2_eval_inverse_dynamics_passive.argtypes = [P, P, P, P, P, P, P, C.c_int32, P, P]
        L.nb2_eval_inverse_dynamics_passive.restype = C.c_int
        L.nb2_eval_inverse_dynamics_force.argtypes = [P, P, P, P, P, P, P, C.c_int32, P, P]
        L.nb2_eval_inverse_dynamics_force.restype = C.c_int
        L.nb2_sensor_contact_scratch_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_size_t)]
        L.nb2_sensor_contact_scratch_bytes.restype = C.c_int
        L.nb2_sensor_contact_update.argtypes = [C.POINTER(_abi.SensorContactView), C.POINTER(_abi.ContactsView), P, P, C.c_size_t, P]
        L.nb2_sensor_contact_update.restype = C.c_int
        L.nb2_sensor_frame_transform_update.argtypes = [C.POINTER(_abi.SensorFrameTransformView), P, P]
        L.nb2_sensor_frame_transform_update.restype = C.c_int
        L.nb2_sensor_imu_update.argtypes = [C.POINTER(_abi.SensorIMUView), P, P, P, P]
        L.nb2_sensor_imu_update.restype = C.c_int
        L.nb2_raycast_refit.argtypes = [C.POINTER(_abi.RaycastView), P, P]
        L.nb2_raycast_refit.restype = C.c_int
        L.nb2_intersect_ray.argtypes = [C.POINTER(_abi.RaycastView), C.c_int32, P, P, P, C.c_int32, P, P, P, P]
        L.nb2_intersect_ray.restype = C.c_int
        L.nb2_camera_render.argtypes = [C.POINTER(_abi.RaycastView), C.POINTER(_abi.CameraDesc), P]
        L.nb2_camera_render.restype = C.c_int
        L.nb2_actuator_step.argtypes = [C.POINTER(_abi.ActuatorStepDesc), P]
        L.nb2_actuator_step.restype = C.c_int
        L.nb2_actuator_reset.argtypes = [C.c_int32, C.c_int32, P, P, P, P, P, P, P, P]
        L.nb2_actuator_reset.restype = C.c_int
        L.nb2_actuator_network_reset.argtypes = [C.c_int32, C.c_int32, C.c_int32, P, P, P, P]
        L.nb2_actuator_network_reset.restype = C.c_int
        L.nb2_actuator_param_gather.argtypes = [P, C.c_int32, P, P, C.c_int32, P]
        L.nb2_actuator_param_gather.restype = C.c_int
        L.nb2_actuator_param_scatter.argtypes = [P, C.c_int32, C.c_int32, P, P, P, C.c_int32, P]
        L.nb2_actuator_param_scatter.restype = C.c_int
        L.nb2_joint_impedance_step.argtypes = [C.POINTER(_abi.JointImpedanceDesc), P]
        L.nb2_joint_impedance_step.restype = C.c_int
        L.nb2_ik_solve.argtypes = [P, P, P, P, P, P, P, P, C.c_int32, C.c_float, C.c_int32, P, P]
        L.nb2_ik_solve.restype = C.c_int
        L.nb2_ik_sample.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, P, P, P, P, P, C.c_float, P, P, P]
        L.nb2_ik_sample.restype = C.c_int
        L.nb2_ik_select.argtypes = [C.c_int32, C.c_int32, C.c_int32, P, P, P, P, P]
        L.nb2_ik_select.restype = C.c_int
        L.nb2_view_gather.argtypes = [P, C.POINTER(_abi.ViewLayout), P, P]
        L.nb2_view_gather.restype = C.c_int
        L.nb2_view_scatter.argtypes = [P, C.POINTER(_abi.ViewLayout), P, P, C.c_int32, P]
        L.nb2_view_scatter.restype = C.c_int
        L.nb2_view_articulation_mask.argtypes = [P, C.c_int32, P, C.c_int32, C.c_int32, P, C.c_int32, P]
        L.nb2_view_articulation_mask.restype = C.c_int
        L.nb2_peer_gather_handle_bytes.restype = C.c_size_t
        L.nb2_peer_gather_create.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_size_t, C.POINTER(P)]
        L.nb2_peer_gather_create.restype = C.c_int
        L.nb2_peer_gather_buffer.argtypes = [P, C.c_int32]
        L.nb2_peer_gather_buffer.restype = P
        L.nb2_peer_gather_stride.argtypes = [P]
        L.nb2_peer_gather_stride.restype = C.c_size_t
        L.nb2_peer_gather_export.argtypes = [P, P]
        L.nb2_peer_gather_export.restype = C.c_int
        L.nb2_peer_gather_connect.argtypes = [P, P]
        L.nb2_peer_gather_connect.restype = C.c_int
        L.nb2_peer_gather_push.argtypes = [P, P, C.c_size_t, C.c_int32, P]
        L.nb2_peer_gather_push.restype = C.c_int
        L.nb2_peer_gather_wait.argtypes = [P, C.c_int32, P]
        L.nb2_peer_gather_wait.restype = C.c_int
        L.nb2_peer_gather_destroy.argtypes = [P]
        L.nb2_peer_gather_destroy.restype = None
        L.nb2_last_error.restype = C.c_char_p
        L.nb2_kernel_launch_count.restype = C.c_int64
        L.nb2_version.restype = C.c_char_p
        _lib = L
    return _lib


def check(status: int, what: str) -> None:
    if status != 0:
        msg = lib().nb2_last_error().decode()
        if status == 2:
            raise NotImplementedError(f"{what}: {msg}")
        if status == 1:
            raise ValueError(f"{what}: {msg}")
        raise Nb2Error(f"{what}: {STATUS.get(status, status)}: {msg}")


def kernel_launch_count() -> int:
    return int(lib().nb2_kernel_launch_count())


class NativeModel:
    """Owner of one ``nb2_model`` handle; shared by the pipeline and solvers built on the same Model."""

    def __init__(self, model):
        import torch

        dev = torch.device(model.device) if not isinstance(model.device, torch.device) else model.device
        if dev.type != "cuda":
            raise Nb2Error(
                f"newton_b200 solvers run on CUDA devices only (model.device={model.device}); there is no CPU path. "
                "Use oracle/ (test infrastructure) for CPU checks."
            )
        self.model = model
        self.device_index = dev.index if dev.index is not None else torch.cuda.current_device()
        self.desc = _abi.model_desc(model)
        handle = C.c_void_p()
        with torch.cuda.device(self.device_index):
            check(lib().nb2_model_create(C.byref(self.desc), self.device_index, C.byref(handle)), "nb2_model_create")
        self.handle = handle
        self.contact_stamp = 0  # bumped whenever the contact blocks are overwritten (collide / import)
        self.rigid_contact_max = int(lib().nb2_model_rigid_contact_max(handle))

    def configure_broad_phase(self, mode: int, max_pairs_per_world: int, include_static_kinematic_pairs: bool):
        """``nb2_collide_configure``: explicit (0) / nxn (1) / sap (2); re-sizes the contact blocks, hence ``rigid_contact_max``."""
        check(lib().nb2_collide_configure(self.handle, int(mode), int(max_pairs_per_world), 1 if include_static_kinematic_pairs else 0),
              "nb2_collide_configure")
        self.rigid_contact_max = int(lib().nb2_model_rigid_contact_max(self.handle))
        self.contact_stamp += 1  # whatever sat in the old blocks is gone

    def xpbd_plan_info(self) -> dict:
        """What the last XPBD step launch chose (``nb2_xpbd_plan_info``): template mode, cached contacts, contact records, shared bytes."""
        out = (C.c_int32 * 4)()
        check(lib().nb2_xpbd_plan_info(self.handle, out), "nb2_xpbd_plan_info")
        return {"template": bool(out[0]), "contact_cache": int(out[1]), "contact_cap": int(out[2]), "smem_bytes": int(out[3])}

    def notify_model_changed(self, flags: int):
        self.desc = _abi.model_desc(self.model)
        check(lib().nb2_model_notify_changed(self.handle, C.byref(self.desc), int(flags)), "nb2_model_notify_changed")

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                lib().nb2_model_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


def native_model(model) -> NativeModel:
    nm = getattr(model, "_nb2_native", None)
    if nm is None:
        nm = NativeModel(model)
        model._nb2_native = nm
    return nm


def current_stream_ptr(model) -> C.c_void_p:
    import torch

    return C.c_void_p(torch.cuda.current_stream(native_model(model).device_index).cuda_stream)

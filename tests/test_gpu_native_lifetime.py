"""Lifetime of the native library's device memory and current device: a model with grown sort, match and import scratch gives
back every byte when it is dropped, and the frames after a growth equal those of a model sized for the larger pipeline from the
start; a one-rank peer gather round-trips a push; no entry point leaves the caller on the model's device."""

import ctypes as C
import gc

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import _abi, _lib, scenes
from newton_b200.sim.builder import ModelBuilder
from newton_b200.utils import xform as X
from tests.test_mesh_plane import box_mesh

pytestmark = pytest.mark.gpu

ENVS, FRAMES, DT = 64, 4, 1.0 / 240
MATCH = dict(contact_matching="sticky", contact_report=True, deterministic=True, contact_matching_pos_threshold=0.01)
FIELDS = ("shape0", "shape1", "point0", "point1", "offset0", "offset1", "normal", "margin0", "margin1", "tids")


def _quadrupeds(device="cuda:0"):
    m = scenes.quadruped_model(ENVS, seed=1)
    m.joint_q.view(ENVS, -1)[:, 2] = 0.48
    scenes.host_fk(m, m.joint_q, m.joint_qd, m)
    return m.to(device)


def _snapshot(c):
    n = int(c.rigid_contact_count.item())
    out = {name: getattr(c, "rigid_contact_" + name)[:n].cpu().numpy() for name in FIELDS + ("match_index",)}
    out["new"] = c.rigid_contact_new_indices[: int(c.rigid_contact_new_count.item())].cpu().numpy()
    out["broken"] = c.rigid_contact_broken_indices[: int(c.rigid_contact_broken_count.item())].cpu().numpy()
    out["count"] = n
    return out


def _foreign_copy(c):
    """The same contacts in a buffer no pipeline of the model filled: the solver loads it through nb2_contacts_import."""
    d = newton_b200.Contacts(c.rigid_contact_max, 0, device=c.rigid_contact_shape0.device)
    d.rigid_contact_count.copy_(c.rigid_contact_count)
    for name in FIELDS:
        getattr(d, "rigid_contact_" + name).copy_(getattr(c, "rigid_contact_" + name))
    return d


def _run(grow):
    """FRAMES frames of sticky matching with the contact report through a pipeline of twice the model's contact capacity; with
    `grow`, a pipeline of the model's own capacity collides first, so the larger one replaces its sort and match scratch."""
    model = _quadrupeds()
    solver = newton_b200.solvers.SolverXPBD(model, iterations=4)
    s0, s1 = model.state(), model.state()
    if grow:
        small = newton_b200.CollisionPipeline(model, **MATCH)
        small.collide(s0, small.contacts())
    big = newton_b200.CollisionPipeline(model, rigid_contact_max=2 * _lib.native_model(model).rigid_contact_max, **MATCH)
    contacts = big.contacts()
    frames = []
    for _ in range(FRAMES):
        s0.clear_forces()
        big.collide(s0, contacts)
        frames.append(_snapshot(contacts))
        solver.step(s0, s1, None, _foreign_copy(contacts), DT)
        s0, s1 = s1, s0
    frames.append({"body_q": s0.body_q.cpu().numpy()})
    return frames


def _free_bytes():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def test_models_give_back_their_memory_and_grown_scratch_keeps_results(cuda_lib):
    fresh = _run(grow=False)
    assert any((f["match_index"] >= 0).any() for f in fresh[1:-1]), "no contact was matched: the comparison would be vacuous"
    baseline = _free_bytes()
    for _ in range(5):
        grown = _run(grow=True)
        for k, (a, b) in enumerate(zip(grown, fresh)):
            assert a.keys() == b.keys()
            for name in a:
                np.testing.assert_array_equal(a[name], b[name], err_msg=f"frame {k}: {name}")
        del grown
    leaked = baseline - _free_bytes()
    assert leaked <= 2 << 20, f"{leaked} bytes of device memory were not given back"


def test_peer_gather_single_rank_round_trip(cuda_lib):
    L = cuda_lib
    nbytes = 1000
    src = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda:0", generator=torch.Generator(device="cuda:0").manual_seed(5))
    g = C.c_void_p()
    _lib.check(L.nb2_peer_gather_create(0, 0, 1, nbytes, C.byref(g)), "nb2_peer_gather_create")
    try:
        handle = C.create_string_buffer(int(L.nb2_peer_gather_handle_bytes()))
        _lib.check(L.nb2_peer_gather_export(g, handle), "nb2_peer_gather_export")
        _lib.check(L.nb2_peer_gather_connect(g, handle), "nb2_peer_gather_connect")
        stream = torch.cuda.current_stream(0)
        _lib.check(L.nb2_peer_gather_push(g, C.c_void_p(src.data_ptr()), nbytes, 1, C.c_void_p(stream.cuda_stream)), "nb2_peer_gather_push")
        torch.cuda.synchronize(0)
        assert int(L.nb2_peer_gather_stride(g)) >= nbytes

        class _Slot:  # receive slot 1 (sequence 1), rank 0's slice first
            __cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (int(L.nb2_peer_gather_buffer(g, 1)), False),
                                        "version": 3, "strides": None}

        assert torch.equal(torch.as_tensor(_Slot(), device="cuda:0"), src)
    finally:
        L.nb2_peer_gather_destroy(g)


def test_entry_points_restore_the_callers_device(cuda_lib):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    L = cuda_lib
    model = _quadrupeds("cuda:0")
    nm = _lib.native_model(model)
    b = ModelBuilder()
    body = b.add_body(xform=X.transform((0.0, 0.0, 0.5), X.quat_identity()))
    b.add_shape_mesh(body, mesh=box_mesh())
    b.add_ground_plane()
    mesh_nm = _lib.native_model(b.finalize().to("cuda:0"))
    contacts = newton_b200.Contacts(nm.rigid_contact_max, 0, device="cuda:0", contact_matching=True)
    s0, s1, ctrl = model.state(), model.state(), model.control()
    view, sv0, sv1, cv = _abi.contacts_view(contacts, model), _abi.state_view(s0, model), _abi.state_view(s1, model), _abi.control_view(ctrl, model)
    params = newton_b200.solvers.SolverXPBD(model, iterations=4)._params()
    opt = _abi.MatchOptions(0.0005, 0.995, None, 0, 1)
    stream = C.c_void_p(torch.cuda.current_stream(0).cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    calls = {
        "nb2_collide": lambda: L.nb2_collide(nm.handle, p(s0.body_q), C.byref(view), stream),
        "nb2_contacts_sort": lambda: L.nb2_contacts_sort(nm.handle, C.byref(view), stream),
        "nb2_contacts_match": lambda: L.nb2_contacts_match(nm.handle, p(s0.body_q), C.byref(view), p(contacts.rigid_contact_match_index),
                                                           C.byref(opt), stream),
        "nb2_xpbd_step": lambda: L.nb2_xpbd_step(nm.handle, C.byref(params), C.byref(sv0), C.byref(sv1), C.byref(cv), 1, C.c_float(DT), stream),
        "nb2_eval_fk": lambda: L.nb2_eval_fk(nm.handle, p(s0.joint_q), p(s0.joint_qd), p(s1.body_q), p(s1.body_qd), stream),
    }
    torch.cuda.set_device(1)
    try:
        for name, call in calls.items():
            _lib.check(call(), name)
            assert torch.cuda.current_device() == 1, f"{name} left cuda:{torch.cuda.current_device()} current"
        # a call that fails after switching: the mesh-plane pair keeps the model on the explicit broad phase
        assert L.nb2_collide_configure(mesh_nm.handle, 1, 0, 1) == 2  # NB2_ERR_UNSUPPORTED
        assert torch.cuda.current_device() == 1
        torch.cuda.synchronize(0)
    finally:
        torch.cuda.set_device(0)

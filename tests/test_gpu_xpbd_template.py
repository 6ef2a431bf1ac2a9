"""XPBD template mode: when every world's body and joint constants are bit-identical, xpbd_step_kernel keeps one copy of them per
CTA and gives the freed shared memory to the contact-constant cache.  Worlds that differ in a single constant, and models changed
after creation, must take the general layout; both layouts must match the CPU oracle bit for bit.

The small scenes force 8 lanes per world (``NB2_LANES``), so that one CTA holds several worlds and reads the constants of the
others from its first world's copy; at the library's own choice (32 lanes, one world per CTA) the template layout would not be
smaller and is not taken."""

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import _lib, scenes
from newton_b200.sim.enums import ModelFlags
from tests.helpers import canonical_contacts, simulate
from tests.variant_cases import chain_model

pytestmark = pytest.mark.gpu


def _quadrupeds(worlds):
    model = scenes.quadruped_model(worlds, seed=1)
    model.joint_q.view(worlds, -1)[:, 2] = 0.48
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    return model


def _gpu_run(model_cpu, substeps, kw, edit=None):
    model = model_cpu.to("cuda:0")
    if edit is not None:  # a constant changed after the native model exists, then notify_model_changed
        solver = newton_b200.solvers.SolverXPBD(model, **kw)
        edit(model)
        solver.notify_model_changed(int(ModelFlags.ALL))
    state, contacts, counts = simulate(model, newton_b200.CollisionPipeline, newton_b200.solvers.SolverXPBD, substeps=substeps,
                                       dt=0.005, solver_kwargs=kw, record_contacts=True)
    torch.cuda.synchronize()
    return model, state, contacts, counts, _lib.native_model(model).xpbd_plan_info()


def _assert_matches_oracle(oracle, model_cpu, substeps, kw, gpu):
    _, gs, gc, gcounts, _ = gpu
    rs, rc, rcounts = simulate(model_cpu, oracle.CollisionPipeline, oracle.SolverXPBD, substeps=substeps, dt=0.005,
                               solver_kwargs=kw, record_contacts=True)
    assert rcounts == gcounts
    n_ref, cr = canonical_contacts(rc, model_cpu)
    n_gpu, cg = canonical_contacts(gc, model_cpu)
    assert n_ref == n_gpu > 0
    for k in cr:
        np.testing.assert_array_equal(cr[k], cg[k], err_msg=f"contact field {k}")
    np.testing.assert_array_equal(gs.body_q.cpu().numpy(), rs.body_q.numpy())
    np.testing.assert_array_equal(gs.body_qd.cpu().numpy(), rs.body_qd.numpy())


def _max_live_contacts(model, contacts):
    n = min(int(contacts.rigid_contact_count.item()), contacts.rigid_contact_max)
    body_world = model.body_world.cpu().numpy()
    shape_body = model.shape_body.cpu().numpy()
    worlds = []
    for s0, s1 in zip(contacts.rigid_contact_shape0[:n].cpu().numpy(), contacts.rigid_contact_shape1[:n].cpu().numpy()):
        b = shape_body[s0] if shape_body[s0] >= 0 else shape_body[s1]
        worlds.append(body_world[b])
    return int(np.bincount(np.asarray(worlds, dtype=np.int64)).max()) if worlds else 0


def _first_dof(model, joint):
    return int(model.joint_qd_start.cpu()[joint])


@pytest.fixture
def shared_ctas(monkeypatch):
    monkeypatch.setenv("NB2_LANES", "8")


def test_identical_worlds_take_template_mode(oracle_lib, cuda_lib, shared_ctas):
    model = _quadrupeds(4)
    kw = {"iterations": 4}
    gpu = _gpu_run(model, 40, kw)
    assert gpu[4]["template"]
    _assert_matches_oracle(oracle_lib, model, 40, kw, gpu)


def _perturb_inertia(model):
    nb = model.body_count // 4
    model.body_inertia.view(-1, 9)[2 * nb + 3, 4] *= 1.25
    model.body_inv_inertia.view(-1, 9)[2 * nb + 3, 4] /= 1.25


def _perturb_limit(model):
    nj = model.joint_count // 4
    dof = _first_dof(model, 3 * nj + 5)
    upper = float(model.joint_limit_upper[dof])
    model.joint_limit_upper[dof] = 0.9 * upper if np.isfinite(upper) and upper != 0.0 else 1.0


def _perturb_ke(model):
    nj = model.joint_count // 4
    model.joint_target_ke[_first_dof(model, nj + 2)] += 1.0


@pytest.mark.parametrize("perturb", [_perturb_inertia, _perturb_limit, _perturb_ke], ids=["inertia", "limit", "ke"])
def test_one_differing_world_takes_general_layout(oracle_lib, cuda_lib, shared_ctas, perturb):
    """(a) one world differs in one constant at creation: general layout, still bit-exact."""
    model = _quadrupeds(4)
    perturb(model)
    kw = {"iterations": 4}
    gpu = _gpu_run(model, 40, kw)
    assert not gpu[4]["template"]
    _assert_matches_oracle(oracle_lib, model, 40, kw, gpu)


@pytest.mark.parametrize("perturb", [_perturb_inertia, _perturb_limit, _perturb_ke], ids=["inertia", "limit", "ke"])
def test_changed_constant_and_notify_leaves_template_mode(oracle_lib, cuda_lib, shared_ctas, perturb):
    """(b) the same change made after the native model exists, followed by notify_model_changed."""
    model = _quadrupeds(4)
    kw = {"iterations": 4}
    gpu = _gpu_run(model, 40, kw, edit=perturb)
    assert not gpu[4]["template"]
    perturb(model)  # the CPU model gets the same change
    _assert_matches_oracle(oracle_lib, model, 40, kw, gpu)


def test_contacts_beyond_the_cache_in_template_mode(oracle_lib, cuda_lib, shared_ctas):
    """(c) a world with more live contacts than the contact-constant cache: the uncached rows run from global memory."""
    model = scenes.box_stack_model(2, seed=None, n_boxes=12)
    kw = {"iterations": 4}
    gpu = _gpu_run(model, 30, kw)
    plan = gpu[4]
    assert plan["template"]
    assert plan["contact_cache"] < _max_live_contacts(gpu[0], gpu[2])
    _assert_matches_oracle(oracle_lib, model, 30, kw, gpu)


def test_headline_plan_caches_every_live_contact(cuda_lib):
    """(d) 4096 quadrupeds after settling: template mode, and a contact cache that holds every world's live contacts."""
    model = _quadrupeds(4096).to("cuda:0")
    state, contacts, _ = simulate(model, newton_b200.CollisionPipeline, newton_b200.solvers.SolverXPBD, substeps=200, dt=0.005,
                                  solver_kwargs={"iterations": 4}, record_contacts=False)
    torch.cuda.synchronize()
    plan = _lib.native_model(model).xpbd_plan_info()
    live = _max_live_contacts(model, contacts)
    assert plan["template"]
    assert live > 0
    assert plan["contact_cache"] >= live, (plan, live)


def test_one_large_world_keeps_the_general_layout(oracle_lib, cuda_lib):
    """One world of a 600-link chain (about 1 200 contact records): a single world per CTA, where the template copy would only add
    to the plan and overflow shared memory.  The step takes the general layout and still runs, bit-exact."""
    model = chain_model(600, world_count=1)
    kw = {"iterations": 4}
    rs, _, rcounts = simulate(model, oracle_lib.CollisionPipeline, oracle_lib.SolverXPBD, substeps=4, dt=1.0 / 240, solver_kwargs=kw,
                              record_contacts=True)
    model_gpu = model.to("cuda:0")
    gs, _, gcounts = simulate(model_gpu, newton_b200.CollisionPipeline, newton_b200.solvers.SolverXPBD, substeps=4, dt=1.0 / 240,
                              solver_kwargs=kw, record_contacts=True)
    torch.cuda.synchronize()
    plan = _lib.native_model(model_gpu).xpbd_plan_info()
    assert not plan["template"]
    assert plan["contact_cap"] >= 1000 and plan["smem_bytes"] > 0, plan
    assert rcounts == gcounts
    np.testing.assert_array_equal(gs.body_q.cpu().numpy(), rs.body_q.numpy())
    np.testing.assert_array_equal(gs.body_qd.cpu().numpy(), rs.body_qd.numpy())

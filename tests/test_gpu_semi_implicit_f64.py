"""The CUDA solvers on hand-written and generated states, held to the CPU oracle word for word and, for SolverSemiImplicit, to the
independent float64 step of ``tests/f64_semi_implicit.py`` within the rounding bound of ``tests/test_semi_implicit_f64.py``."""

import numpy as np
import pytest
import torch

import newton_b200
from tests import semi_implicit_cases as cases
from tests.helpers import word_diff

pytestmark = pytest.mark.gpu


def _one_sided_solvers(name, oracle_lib):
    from oracle.semi_implicit import SolverSemiImplicit

    if name == "xpbd":
        return (lambda m: oracle_lib.SolverXPBD(m, iterations=4, enable_restitution=True),
                lambda m: newton_b200.solvers.SolverXPBD(m, iterations=4, enable_restitution=True), 1.0 / 240)
    if name == "featherstone":
        return lambda m: oracle_lib.SolverFeatherstone(m), lambda m: newton_b200.solvers.SolverFeatherstone(m), 1.0 / 480
    return lambda m: SolverSemiImplicit(m), lambda m: newton_b200.solvers.SolverSemiImplicit(m), 1.0e-3


@pytest.mark.parametrize("solver_name", ["xpbd", "featherstone", "semi_implicit"])
def test_one_sided_contacts_import(oracle_lib, cuda_lib, solver_name):
    """A Contacts buffer written by hand: contacts against fixed world points (shape id -1 on either side), contacts whose two shape
    ids are equal and static-static pairs, interleaved with ordinary box-ground contacts of three worlds.  Every word of body_q /
    body_qd after each of 10 substeps equals the oracle's, which applies the one-sided contacts with the materials of the one
    shape present."""
    model = cases.one_sided_model(3)
    mg = model.to("cuda:0")
    mk_o, mk_g, dt = _one_sided_solvers(solver_name, oracle_lib)
    oc, gc = cases.one_sided_contacts(model, "cpu"), cases.one_sided_contacts(mg, "cuda:0")
    so, sg = mk_o(model), mk_g(mg)
    o0, o1, g0, g1 = model.state(), model.state(), mg.state(), mg.state()
    for step in range(10):
        o0.clear_forces()
        g0.clear_forces()
        so.step(o0, o1, None, oc, dt)
        sg.step(g0, g1, None, gc, dt)
        torch.cuda.synchronize()
        for name in ("body_q", "body_qd"):
            a, b = getattr(g1, name).cpu().numpy(), getattr(o1, name).numpy()
            assert np.isfinite(b).all()
            assert word_diff(a, b) == 0, f"substep {step}: {name} differs in {word_diff(a, b)} words"
        o0, o1, g0, g1 = o1, o0, g1, g0
    # the one-sided rows matter: the oracle without them (both shape ids -1, a row every solver skips) ends elsewhere for every box
    without = cases.one_sided_contacts(model, "cpu")
    one_sided = (without.rigid_contact_shape0 < 0) != (without.rigid_contact_shape1 < 0)
    assert int(one_sided.sum()) > 0
    without.rigid_contact_shape0[one_sided] = -1
    without.rigid_contact_shape1[one_sided] = -1
    so, w0, w1 = mk_o(model), model.state(), model.state()
    for _ in range(10):
        w0.clear_forces()
        so.step(w0, w1, None, without, dt)
        w0, w1 = w1, w0
    assert (w0.body_qd != o0.body_qd).any(dim=1).all()


def _first_clear(make, count, near, kw):
    """The first ``count`` seeded draws of ``make(seed) -> (model, contacts)`` with no decision within ``near`` of its edge, with
    the solver settings ``kw`` the test steps them with."""
    from tests import f64_semi_implicit as F

    out = []
    for seed in range(40):
        model, contacts = make(seed)
        if F.step(model, model.state(), model.control(), contacts, 0.01, **kw, near=near)["branches"].clear():
            out.append((model, contacts))
        if len(out) == count:
            return out
    raise AssertionError("too few draws clear of the knife edges")


@pytest.mark.parametrize("lanes", [8, 16, 32])
def test_generated_states_against_float64(oracle_lib, cuda_lib, monkeypatch, lanes):
    """The generated joint and contact states of test_semi_implicit_f64.py (50 contacts per environment: two record chunks of 32)
    at each group width: the CUDA step equals the oracle word for word and is within the float64 bound."""
    from oracle.semi_implicit import SolverSemiImplicit
    from tests import f64_semi_implicit as F
    from tests.test_semi_implicit_f64 import NEAR_CONTACTS, compare, contact_scene, joint_scene

    monkeypatch.setenv("NB2_LANES", str(lanes))
    kw = dict(angular_damping=0.1, friction_smoothing=0.5)
    scenes_ = _first_clear(lambda s: (joint_scene(s)[0], None), 2, F.NEAR, kw)
    scenes_ += _first_clear(lambda s: contact_scene(s, per_pair=2), 2, NEAR_CONTACTS, kw)
    for k, (model, contacts) in enumerate(scenes_):
        mg = model.to("cuda:0")
        gc = None
        if contacts is not None:
            gc = type(contacts)(contacts.rigid_contact_max, 0, device="cuda:0", requested_attributes=mg._requested_contact_attributes)
            for name, value in vars(contacts).items():
                if isinstance(value, torch.Tensor) and isinstance(getattr(gc, name, None), torch.Tensor):
                    getattr(gc, name).copy_(value)
        o0, o1, g0, g1 = model.state(), model.state(), mg.state(), mg.state()
        ref = F.step(model, o0, model.control(), contacts, 0.01, **kw, near=F.NEAR if contacts is None else NEAR_CONTACTS)
        assert ref["branches"].clear()
        SolverSemiImplicit(model, **kw).step(o0, o1, model.control(), contacts, 0.01)
        newton_b200.solvers.SolverSemiImplicit(mg, **kw).step(g0, g1, mg.control(), gc, 0.01)
        torch.cuda.synchronize()
        for name in ("body_q", "body_qd"):
            diff = word_diff(getattr(g1, name).cpu().numpy(), getattr(o1, name).numpy())
            assert diff == 0, f"scene {k}: {name} differs in {diff} words"
        assert word_diff(g0.body_f.cpu().numpy(), o0.body_f.numpy()) == 0, f"scene {k}: state_in.body_f"
        compare(g0, g1, ref, body_f=g0.body_f if ref["into_state_in"] else None, label=f"scene {k}: ")


def test_quadrupeds_4096_sampled_against_float64(cuda_lib):
    """4096 quadrupeds on the ground, collide + step for 20 substeps: at every substep a seeded sample of 64 worlds is held to the
    float64 step from the same float32 state_in."""
    from newton_b200 import scenes
    from tests import f64_semi_implicit as F
    from tests.test_semi_implicit_f64 import NEAR_TRAJECTORY, compare

    model = scenes.quadruped_model(4096, seed=1)
    model.joint_q.view(4096, -1)[:, 2] = 0.47
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    mg = model.to("cuda:0")
    worlds = np.random.default_rng(7).choice(4096, 64, replace=False)
    sample = np.isin(mg.body_world.cpu().numpy(), worlds)
    solver, pipe = newton_b200.solvers.SolverSemiImplicit(mg), newton_b200.CollisionPipeline(mg)
    contacts = pipe.contacts()
    s0, s1, ctl = mg.state(), mg.state(), mg.control()
    worst, touched = 0.0, 0
    for k in range(20):
        s0.clear_forces()
        pipe.collide(s0, contacts)
        solver.step(s0, s1, ctl, contacts, 1e-3)
        torch.cuda.synchronize()
        ref = F.step(mg, s0, ctl, contacts, 1e-3, near=NEAR_TRAJECTORY)
        worst = max(worst, compare(s0, s1, ref, label=f"substep {k}: ", bodies=sample))
        touched += int(ref["branches"].counts["contact_penetrating"])
        s0, s1 = s1, s0
    assert touched > 0
    print(f"4096 quadrupeds, 64 sampled worlds: largest ratio {worst:.2f}")

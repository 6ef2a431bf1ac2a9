"""The CPU oracle of SolverSemiImplicit (oracle/oracle_semi_implicit.h) against known answers.

Restated from the reference's semi_implicit rows, with its thresholds: test_physics_verification.py (free fall along +Y, pendulum
period, energy conservation) and test_joint_damping.py::test_semi_implicit_ball_joint_damping_decays_velocity.  The
test_control_force.py, test_kinematic_links.py and test_runtime_gravity.py rows are in test_semi_implicit_reference_rows.py.

In the spirit of the reference but with scenes of their own: projectile motion and momentum conservation, an applied body
force and torque with a kinematic body next to it.  Closed forms the reference does not check: a prismatic spring-damper, exactly
zero motion at rest for every joint type, the state_in.body_f rule of solver_semi_implicit.py:166-169 and the substep of
scripts/semi_implicit_bench.py."""

import math

import numpy as np
import pytest
import torch

from newton_b200.sim.builder import ModelBuilder
from newton_b200.sim.enums import JointType
from newton_b200.utils import xform as X
from tests import semi_implicit_cases as cases


@pytest.fixture(scope="module")
def si():
    import oracle
    import oracle.semi_implicit

    oracle.build()
    return oracle.semi_implicit


def _run(model, solver, steps, dt, before=None, contacts_pipe=None):
    s0, s1 = model.state(), model.state()
    contacts = contacts_pipe.contacts() if contacts_pipe is not None else None
    for i in range(steps):
        s0.clear_forces()
        if before is not None:
            before(s0, i)
        if contacts_pipe is not None:
            contacts_pipe.collide(s0, contacts)
        solver.step(s0, s1, None, contacts, dt)
        s0, s1 = s1, s0
    return s0


def test_free_fall_up_axis_y(si):
    """test_physics_verification.py test_free_fall (semi_implicit row): g = -10 along +Y, h0 = 5, dt = 1 ms, 500 steps."""
    g, h0, dt = -10.0, 5.0, 1e-3
    b = ModelBuilder(up_axis="y", gravity=g)
    body = b.add_body(xform=X.transform((0.0, h0, 0.0)))
    b.add_shape_sphere(body, radius=0.1)
    model = b.finalize()
    solver = si.SolverSemiImplicit(model, angular_damping=0.0)
    s0, s1 = model.state(), model.state()
    for i in range(1, 501):
        s0.clear_forces()
        solver.step(s0, s1, None, None, dt)
        s0, s1 = s1, s0
        if i % 100 == 0:
            t = i * dt
            pos, vel = s0.body_q.numpy()[0, :3], s0.body_qd.numpy()[0, :3]
            assert abs(pos[1] - (h0 + 0.5 * g * t * t)) < max(2.0 * 0.5 * abs(g) * dt * t, 1e-3)
            assert abs(vel[1] - g * t) < max(abs(g) * dt, 1e-3)
            assert abs(pos[0]) < 1e-6 and abs(pos[2]) < 1e-6


def test_projectile_and_momentum(si):
    """test_projectile_motion / test_momentum_conservation (semi_implicit rows): a thrown body follows the parabola; two free
    bodies without gravity keep their total momentum and angular velocity magnitude (angular_damping = 0)."""
    b = ModelBuilder(gravity=-9.81)
    body = b.add_body(xform=X.transform((0.0, 0.0, 1.0)), mass=2.0, inertia=np.eye(3) * 0.1)
    model = b.finalize()
    model.body_qd[0] = torch.tensor([3.0, -1.0, 4.0, 0.0, 0.0, 0.0])
    s = _run(model, si.SolverSemiImplicit(model, angular_damping=0.0), 400, 1e-3)
    t = 0.4
    p = s.body_q.numpy()[0, :3]
    np.testing.assert_allclose(p, [3.0 * t, -1.0 * t, 1.0 + 4.0 * t - 0.5 * 9.81 * t * t], atol=0.5 * 9.81 * 1e-3 * t * 2 + 1e-4)
    del body

    b = ModelBuilder(gravity=0.0)
    for x in (-1.0, 1.0):
        b.add_body(xform=X.transform((x, 0.0, 0.0)), mass=1.5, inertia=np.diag([0.1, 0.2, 0.3]))
    model = b.finalize()
    model.body_qd.copy_(torch.tensor([[1.0, 0.5, 0.0, 0.0, 0.0, 2.0], [-0.5, 0.0, 0.2, 0.0, 0.0, -1.0]]))
    p0 = (model.body_qd[:, :3] * 1.5).sum(0).numpy()
    s = _run(model, si.SolverSemiImplicit(model, angular_damping=0.0), 300, 1e-3)
    np.testing.assert_allclose((s.body_qd[:, :3] * 1.5).sum(0).numpy(), p0, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(s.body_qd[:, 5].numpy(), [2.0, -1.0], rtol=1e-3)


def _pendulum(sphere_radius):
    b = ModelBuilder(up_axis="y", gravity=-10.0)
    link = b.add_link()
    b.add_shape_sphere(link, radius=sphere_radius)
    j = b.add_joint_revolute(-1, link, axis=(0.0, 0.0, 1.0), parent_xform=X.transform((0.0, 0.0, 0.0)),
                             child_xform=X.transform((0.0, 1.0, 0.0)), armature=0.0)
    b.add_articulation([j])
    model = b.finalize()
    model.joint_q[0] = 0.05
    from newton_b200 import scenes

    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    return model


def test_pendulum_period(si):
    """test_pendulum_period (semi_implicit row): sim_dt = 3e-4, sphere radius 0.1, joint_attach_ke = 1e5, joint_attach_kd = 1e1;
    trajectory within 1 % of the small-angle solution over 3.5 periods."""
    model = _pendulum(0.1)
    mass = float(model.body_mass[0])
    I_pivot = float(model.body_inertia[0, 2, 2]) + mass
    T = 2.0 * math.pi * math.sqrt(I_pivot / (mass * 10.0))
    dt = 3e-4
    n = int(3.5 * T / dt)
    solver = si.SolverSemiImplicit(model, angular_damping=0.0, joint_attach_ke=1e5, joint_attach_kd=1e1)
    s0, s1 = model.state(), model.state()
    angles = []
    for _ in range(n):
        s0.clear_forces()
        solver.step(s0, s1, None, None, dt)
        s0, s1 = s1, s0
        bq = s0.body_q.numpy()[0]
        angles.append(float(np.arctan2(bq[0], -bq[1])))
    times = np.arange(1, n + 1) * dt
    err = np.mean(np.abs(np.array(angles) - 0.05 * np.cos(2.0 * math.pi / T * times))) / 0.05
    assert err < 0.01, err


def test_energy_conservation(si):
    """test_energy_conservation (semi_implicit row, same set-up as the period test), 2 s: the kinetic energy reaches < 1 % of |E0|
    (the pendulum turns) and the energy drifts < 0.5 % of |E0| - the reference's two checks.  |E0| is mostly the constant
    -m g L, so the drift is also held to 1 % of the oscillation energy m g L (1 - cos 0.05) itself."""
    model = _pendulum(0.1)
    mass = float(model.body_mass[0])
    I_pivot = float(model.body_inertia[0, 2, 2]) + mass
    dt = 3e-4
    solver = si.SolverSemiImplicit(model, angular_damping=0.0, joint_attach_ke=1e5, joint_attach_kd=1e1)
    s0, s1 = model.state(), model.state()

    def ke_pe(s):
        bq = s.body_q.numpy()[0]
        th = float(np.arctan2(bq[0], -bq[1]))
        w = float(s.body_qd.numpy()[0, 5])
        return 0.5 * I_pivot * w * w, mass * 10.0 * (-math.cos(th))

    ke0, pe0 = ke_pe(s0)
    e0 = ke0 + pe0
    kes, energies = [ke0], [e0]
    for _ in range(int(2.0 / dt)):
        s0.clear_forces()
        solver.step(s0, s1, None, None, dt)
        s0, s1 = s1, s0
        ke, pe = ke_pe(s0)
        kes.append(ke)
        energies.append(ke + pe)
    drift = float(np.max(np.abs(np.array(energies) - e0)))
    assert min(kes[1:]) / abs(e0) < 0.01
    assert drift / abs(e0) < 0.005
    assert drift / (mass * 10.0 * (1.0 - math.cos(0.05))) < 0.01


def test_ball_joint_damping_decays_velocity(si):
    """test_joint_damping.py::test_semi_implicit_ball_joint_damping_decays_velocity: undamped keeps |w|, damping 3 loses > 15 %."""
    def speed(damping, w0):
        b = ModelBuilder(up_axis="y", gravity=0.0)
        body = b.add_link(mass=1.0, inertia=np.eye(3), lock_inertia=True)
        j = b.add_joint_ball(-1, body, damping=damping, armature=0.0)
        b.add_articulation([j])
        model = b.finalize()
        model.joint_qd[0:3] = torch.tensor(w0)
        from newton_b200 import scenes

        scenes.host_fk(model, model.joint_q, model.joint_qd, model)
        s = _run(model, si.SolverSemiImplicit(model, angular_damping=0.0), 8, 0.01)
        return float(np.linalg.norm(s.body_qd.numpy()[0, 3:]))

    for w0 in ((1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0), (0.5, -0.25, 1.0)):
        n0 = float(np.linalg.norm(w0))
        np.testing.assert_allclose(speed(0.0, w0), n0, rtol=1e-5, atol=1e-5)
        assert speed(3.0, w0) < 0.85 * n0


def test_prismatic_spring_damper_closed_form(si):
    """One PRISMATIC joint driven by target_ke / target_kd, no gravity: x'' = -(k x + c x') / m, started at x0 with the spring
    stretched, against the analytic under-damped response."""
    m_, k, c, x0 = 2.0, 50.0, 1.0, 0.05
    b = ModelBuilder(gravity=0.0)
    link = b.add_link(mass=m_, inertia=np.eye(3) * 0.1)
    j = b.add_joint_prismatic(-1, link, axis=(1.0, 0.0, 0.0), target_ke=k, target_kd=c, armature=0.0)
    b.add_articulation([j])
    model = b.finalize()
    model.joint_q[0] = x0
    from newton_b200 import scenes

    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    dt, n = 1e-4, 20000
    s = _run(model, si.SolverSemiImplicit(model, angular_damping=0.0), n, dt)
    t = n * dt
    zeta, wn = c / (2.0 * math.sqrt(k * m_)), math.sqrt(k / m_)
    wd = wn * math.sqrt(1.0 - zeta * zeta)
    x = x0 * math.exp(-zeta * wn * t) * (math.cos(wd * t) + zeta * wn / wd * math.sin(wd * t))
    assert abs(float(s.body_q[0, 0]) - x) < 2e-3 * x0 + 1e-5
    assert abs(float(s.body_q[0, 1])) < 1e-6 and abs(float(s.body_q[0, 2])) < 1e-6


@pytest.mark.parametrize("kind", ["prismatic", "revolute", "ball", "fixed", "d6_lin", "d6_ang1", "d6_ang2", "d6_ang3", "free",
                                  "distance", "rod"])
def test_every_joint_type_at_rest_gives_zero_wrench(si, kind):
    """Aligned joint frames, zero velocity, zero joint_f, targets at the joint position, no gravity: the body stays exactly where
    it is (every joint wrench is exactly zero)."""
    b = ModelBuilder(gravity=0.0)
    parent = b.add_link(xform=X.transform((0.0, 0.0, 1.0)), mass=1.0, inertia=np.eye(3) * 0.1)
    child = b.add_link(xform=X.transform((0.0, 0.0, 0.5)), mass=1.0, inertia=np.eye(3) * 0.1)
    px, cx = X.transform((0.0, 0.0, -0.25)), X.transform((0.0, 0.0, 0.25))
    kw = dict(parent_xform=px, child_xform=cx)
    from newton_b200.sim.builder import JointDofConfig as D

    j0 = b.add_joint_fixed(-1, parent, parent_xform=X.transform((0.0, 0.0, 1.0)))
    if kind == "prismatic":
        j = b.add_joint_prismatic(parent, child, axis=(1.0, 0.0, 0.0), target_ke=10.0, **kw)
    elif kind == "revolute":
        j = b.add_joint_revolute(parent, child, axis=(0.0, 1.0, 0.0), target_ke=10.0, **kw)
    elif kind == "ball":
        j = b.add_joint_ball(parent, child, **kw)
    elif kind == "fixed":
        j = b.add_joint_fixed(parent, child, **kw)
    elif kind == "d6_lin":
        j = b.add_joint_d6(parent, child, linear_axes=[D(axis="x"), D(axis="y"), D(axis="z")], **kw)
    elif kind.startswith("d6_ang"):
        n = int(kind[-1])
        j = b.add_joint_d6(parent, child, angular_axes=[D(axis=a, target_ke=5.0) for a in "xyz"[:n]], **kw)
    elif kind == "free":
        j = b.add_joint_free(child, parent=parent, **kw)
    elif kind == "distance":
        j = b.add_joint_distance(parent, child, **kw)
    else:
        j = b.add_joint(JointType.ROD, parent, child, **kw)
    b.add_articulation([j0, j])
    model = b.finalize()
    model.joint_q.zero_()
    q0 = model.body_q.clone()
    s0, s1 = model.state(), model.state()
    si.SolverSemiImplicit(model, angular_damping=0.0).step(s0, s1, None, None, 1e-3)
    assert torch.equal(s1.body_q, q0), kind
    assert torch.equal(s1.body_qd, torch.zeros_like(s1.body_qd)), kind


def test_body_f_side_effect_rule(si):
    """solver_semi_implicit.py:166-169: a model without joints accumulates the contact forces into state_in.body_f; a model with
    joints works on a copy and leaves state_in.body_f as it was."""
    import oracle

    model = cases.jointless_links_model(2)
    assert model.joint_count == 0
    pipe = oracle.CollisionPipeline(model)
    s0, s1, contacts = model.state(), model.state(), pipe.contacts()
    s0.body_f[:, 0] = 0.25  # an applied force, kept and summed with the contacts
    pipe.collide(s0, contacts)
    assert int(contacts.rigid_contact_count.item()) > 0
    si.SolverSemiImplicit(model).step(s0, s1, None, contacts, 1e-3)
    f = s0.body_f.numpy()
    assert np.all(f[:, 2] > 0.0), "the ground pushes every sphere up: the contact force is in state_in.body_f"
    assert np.all(f[:, 0] == 0.25)

    model = cases.boxes_on_ground_model(1, boxes=2)
    assert model.joint_count > 0
    pipe = oracle.CollisionPipeline(model)
    s0, s1, contacts = model.state(), model.state(), pipe.contacts()
    s0.body_f[:, 1] = -0.5
    pipe.collide(s0, contacts)
    si.SolverSemiImplicit(model).step(s0, s1, None, contacts, 1e-3)
    assert np.all(s0.body_f.numpy()[:, 1] == -0.5) and np.all(s0.body_f.numpy()[:, [0, 2, 3, 4, 5]] == 0.0)
    assert float(s1.body_qd[0, 2]) > -9.81e-3  # the contacts did act, on the copy


def test_applied_body_force_and_kinematic_body(si):
    """test_body_force.py / test_kinematic_links.py (semi_implicit rows): a body force accelerates a free body by f / m (and a
    torque spins it by I^-1 t); a kinematic body ignores forces and passes through unchanged."""
    b = ModelBuilder(gravity=0.0)
    free = b.add_body(mass=2.0, inertia=np.eye(3) * 0.5)
    kin = b.add_body(xform=X.transform((1.0, 0.0, 0.0)), mass=2.0, inertia=np.eye(3) * 0.5, is_kinematic=True)
    model = b.finalize()
    model.body_qd[kin] = torch.tensor([0.3, 0.0, 0.0, 0.0, 0.0, 0.0])

    def push(s, i):
        s.body_f[:] = torch.tensor([4.0, 0.0, 0.0, 0.0, 0.0, 1.0])

    s = _run(model, si.SolverSemiImplicit(model, angular_damping=0.0), 100, 1e-3, before=push)
    np.testing.assert_allclose(s.body_qd.numpy()[free, 0], 4.0 / 2.0 * 0.1, rtol=1e-5)
    np.testing.assert_allclose(s.body_qd.numpy()[free, 5], 1.0 / 0.5 * 0.1, rtol=1e-4)
    np.testing.assert_allclose(s.body_qd.numpy()[kin], [0.3, 0.0, 0.0, 0.0, 0.0, 0.0])
    np.testing.assert_allclose(s.body_q.numpy()[kin, 0], 1.0)  # body_q is prescribed by the user, never integrated


def test_quadruped_stays_up_at_the_benchmark_substep(si):
    """The substep of scripts/semi_implicit_bench.py (1 ms) from the benchmark's start (bases lowered to 0.47 m): three quadrupeds
    stay finite with their bases above the ground for 1 s of simulated time under the default attachment gains."""
    import oracle
    from newton_b200 import scenes

    model = scenes.quadruped_model(3, seed=1)
    model.joint_q.view(3, -1)[:, 2] = 0.47
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    s = _run(model, si.SolverSemiImplicit(model), 1000, 1e-3, contacts_pipe=oracle.CollisionPipeline(model))
    q = s.body_q.numpy().reshape(3, 13, 7)
    assert np.isfinite(q).all()
    assert np.all(q[:, 0, 2] > 0.3)


def test_body_f_rule_follows_control_joint_f(si):
    """solver_semi_implicit.py:167 clones body_f only when the model has joints AND control.joint_f is not None.  A model whose only
    joint is FIXED (no dofs) has an empty joint_f array: forces go to the copy.  With control.joint_f = None they go to
    state_in.body_f."""
    import oracle

    model = cases.fixed_root_and_link_model(1)
    assert model.joint_count == 1 and model.joint_dof_count == 0
    for joint_f_none in (False, True):
        pipe = oracle.CollisionPipeline(model)
        s0, s1, contacts, control = model.state(), model.state(), pipe.contacts(), model.control()
        if joint_f_none:
            control.joint_f = None
        pipe.collide(s0, contacts)
        assert int(contacts.rigid_contact_count.item()) > 0
        si.SolverSemiImplicit(model).step(s0, s1, control, contacts, 1e-3)
        f = s0.body_f.numpy()
        if joint_f_none:  # (the FIXED joint to the world filters the box's own ground contact; the sphere touches it)
            assert f[1, 2] > 0.0, "the ground's push on the sphere is in state_in.body_f"
        else:
            assert np.all(f == 0.0), "forces went to the copy"

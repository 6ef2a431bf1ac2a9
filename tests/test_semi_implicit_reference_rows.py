"""The reference's own ``semi_implicit`` rows of test_control_force.py, test_kinematic_links.py and test_runtime_gravity.py,
restated on the CPU oracle of SolverSemiImplicit (oracle/oracle_semi_implicit.h) with the reference's scenes, step counts and
thresholds.  The control-force rows are the answers that do not come from the oracle itself for the joint_f terms of
eval_body_joints: +joint_f on a FREE joint's child, -joint_f along a D6 joint's linear axes, and the child-side torque
t_total + r_c x f_total of a joint anchored away from the child's COM."""

import numpy as np
import pytest
import torch

from newton_b200 import BodyFlags
from newton_b200.sim.builder import JointDofConfig, ModelBuilder
from newton_b200.sim.enums import ModelFlags
from newton_b200.utils import xform as X

KINEMATIC_TEST_WRENCH = torch.tensor([20.0, -15.0, 10.0, 0.5, -0.4, 0.3])  # test_kinematic_links.py:223


@pytest.fixture(scope="module")
def si():
    import oracle
    import oracle.semi_implicit

    oracle.build()
    return oracle.semi_implicit


def _solver(si, model):
    """The ``semi_implicit`` entry of the reference tests' solver tables: SolverSemiImplicit(model, angular_damping=0.0)."""
    return si.SolverSemiImplicit(model, angular_damping=0.0)


def _quat_rpy(r, p, y):
    """wp.quat_rpy (roll about x, pitch about y, yaw about z)."""
    cy, sy, cr, sr, cp, sp = np.cos(y * 0.5), np.sin(y * 0.5), np.cos(r * 0.5), np.sin(r * 0.5), np.cos(p * 0.5), np.sin(p * 0.5)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


# ---- test_control_force.py:49-87 (test_floating_body_angular_semi_implicit) ---------------------------------------------------
def test_control_force_floating_body_angular(si):
    import oracle

    builder = ModelBuilder(up_axis="y", gravity=(0.0, 0.0, 0.0))
    b = builder.add_body()
    builder.add_shape_box(b)
    builder.joint_q = [1.0, 2.0, 3.0, *_quat_rpy(-1.3, 0.8, 2.4)]
    model = builder.finalize()
    solver = _solver(si, model)
    s0, s1 = model.state(), model.state()
    oracle.eval_fk(model, model.joint_q, model.joint_qd, s0)
    control = model.control()
    control.joint_f.copy_(torch.tensor([0.0, 0.0, 0.0, 0.0, 0.0, 100.0]))
    for _ in range(4):
        solver.step(s0, s1, control, None, 1.0 / 10.0)
        s0, s1 = s1, s0
    qd = s0.body_qd.numpy()[0]
    assert 0.04 < qd[5] < 0.4
    assert np.abs(qd[:5]).max() <= 2e-6


# ---- test_control_force.py:90-139 (test_3d_articulation_semi_implicit) --------------------------------------------------------
def test_control_force_3d_articulation(si):
    import oracle

    builder = ModelBuilder(gravity=(0.0, 0.0, 0.0))
    builder.default_shape_cfg.density = 100.0
    b = builder.add_link()
    builder.add_shape_sphere(b)
    j = builder.add_joint_d6(-1, b, linear_axes=[JointDofConfig(axis=a, armature=0.0) for a in ((1, 0, 0), (0, 1, 0), (0, 0, 1))])
    builder.add_articulation([j])
    model = builder.finalize()
    assert model.joint_dof_count == 3
    for dim in range(3):
        solver = _solver(si, model)
        s0, s1 = model.state(), model.state()
        control = model.control()
        f = np.zeros(3, dtype=np.float32)
        f[dim] = 100.0
        control.joint_f.copy_(torch.from_numpy(f))
        for _ in range(4):
            solver.step(s0, s1, control, None, 1.0 / 10.0)
            s0, s1 = s1, s0
        oracle.eval_ik(model, s0, s0.joint_q, s0.joint_qd)  # maximal coordinates: joint_qd from body_qd
        qd = s0.joint_qd.numpy()
        assert 0.009 < qd[dim] < 0.4
        assert np.abs(np.delete(qd, dim)).max() <= 1e-6


# ---- test_control_force.py:142-198 (test_child_xform_moment_arm_semi_implicit) ------------------------------------------------
def test_control_force_child_xform_moment_arm(si):
    offset_y = 2.0
    builder = ModelBuilder(gravity=(0.0, 0.0, 0.0))
    builder.default_shape_cfg.density = 100.0
    b = builder.add_link()
    builder.add_shape_sphere(b)
    axes = ((1, 0, 0), (0, 1, 0), (0, 0, 1))
    j = builder.add_joint_d6(-1, b, child_xform=X.transform((0.0, offset_y, 0.0)),
                             linear_axes=[JointDofConfig(axis=a, armature=0.0) for a in axes],
                             angular_axes=[JointDofConfig(axis=a, armature=0.0) for a in axes])
    builder.add_articulation([j])
    model = builder.finalize()
    solver = _solver(si, model)
    s0, s1 = model.state(), model.state()
    control = model.control()
    f = np.zeros(model.joint_dof_count, dtype=np.float32)
    f[0] = 100.0  # force along X at the joint anchor, 2 m from the COM
    control.joint_f.copy_(torch.from_numpy(f))
    for _ in range(4):
        solver.step(s0, s1, control, None, 1.0 / 10.0)
        s0, s1 = s1, s0
    qd = s0.body_qd.numpy()[0]
    assert qd[0] > 0.001
    assert qd[5] < -0.001  # cross((0, offset_y, 0), (F, 0, 0)) = (0, 0, -F offset_y)


# ---- test_kinematic_links.py:304-715, semi_implicit rows ------------------------------------------------------------------------
def _contact_defaults(builder):
    builder.default_shape_cfg.ke, builder.default_shape_cfg.kd, builder.default_shape_cfg.kf = 1.0e4, 500.0, 0.5


def _quat_close(qa, qb, min_dot):
    assert abs(float(np.dot(qa, qb))) > min_dot


def test_kinematic_free_base_prescribed_motion(si):
    """:400-481"""
    import oracle

    dt, steps, x0, vx = 1.0 / 240.0, 100, -0.3, 1.0

    def run_once(apply_force):
        builder = ModelBuilder(gravity=(0.0, 0.0, 0.0))
        _contact_defaults(builder)
        kin = builder.add_body(xform=X.transform((-0.3, 0.0, 0.0)), mass=1.0, is_kinematic=True, label="kinematic_free")
        builder.add_shape_box(kin, hx=0.25, hy=0.15, hz=0.15)
        probe = builder.add_body(xform=X.transform((0.45, 0.0, 0.0)), mass=1.0, label="probe")
        builder.add_shape_sphere(probe, radius=0.1)
        model = builder.finalize()
        joint = int(np.flatnonzero(model.numpy("joint_child") == kin)[0])
        qs, qds = int(model.joint_q_start[joint]), int(model.joint_qd_start[joint])
        solver = _solver(si, model)
        pipe = oracle.CollisionPipeline(model)
        contacts = pipe.contacts()
        s0, s1 = model.state(), model.state()
        p0 = s0.body_q.numpy()[probe, :3].copy()
        max_speed = 0.0
        for i in range(steps):
            s0.joint_q[qs : qs + 7] = torch.tensor([x0 + vx * i * dt, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
            s0.joint_qd[qds : qds + 6] = torch.tensor([vx, 0.0, 0.0, 0.0, 0.0, 0.0])
            oracle.eval_fk(model, s0.joint_q, s0.joint_qd, s0, body_flag_filter=int(BodyFlags.KINEMATIC))
            s0.clear_forces()
            if apply_force:
                s0.body_f[kin] = KINEMATIC_TEST_WRENCH
            pipe.collide(s0, contacts)
            solver.step(s0, s1, None, contacts, dt)
            s0, s1 = s1, s0
            max_speed = max(max_speed, float(np.linalg.norm(s0.body_qd.numpy()[probe, :3])))
        q, qd = s0.body_q.numpy(), s0.body_qd.numpy()
        return dict(kin_pos=q[kin, :3].copy(), kin_quat=q[kin, 3:].copy(), kin_qd=qd[kin].copy(), probe_qd=qd[probe].copy(),
                    probe_max_speed=max_speed, probe_displacement=float(np.linalg.norm(q[probe, :3] - p0)))

    free, forced = run_once(False), run_once(True)
    assert free["kin_pos"][0] == pytest.approx(x0 + vx * (steps - 1) * dt, abs=4e-2)
    assert abs(free["kin_pos"][1]) < 2e-2 and abs(free["kin_pos"][2]) < 2e-2 and free["kin_qd"][0] > 2e-1
    np.testing.assert_allclose(forced["kin_pos"], free["kin_pos"], atol=8e-3)
    _quat_close(forced["kin_quat"], free["kin_quat"], 0.9995)
    assert np.linalg.norm(forced["kin_qd"] - free["kin_qd"]) < 4e-1
    assert free["probe_max_speed"] > 3e-2
    assert np.linalg.norm(free["probe_qd"][:3]) > 5e-3 or free["probe_displacement"] > 1e-3


def test_kinematic_revolute_root_pendulum_prescribed_motion(si):
    """:484-575 - a maximal-coordinate solver gets the root's body_q / body_qd prescribed directly."""
    import oracle

    dt, steps, theta0, omega = 1.0 / 240.0, 120, -1.0, 2.0

    def run_once(apply_force):
        builder = ModelBuilder(gravity=(0.0, 0.0, 0.0))
        _contact_defaults(builder)
        root = builder.add_link(mass=1.0, is_kinematic=True, label="kinematic_root")
        pendulum = builder.add_link(mass=1.0, label="pendulum")
        j_root = builder.add_joint_revolute(-1, root, axis=(0.0, 1.0, 0.0), label="kinematic_root_joint")
        j_pend = builder.add_joint_revolute(root, pendulum, axis=(0.0, 1.0, 0.0), parent_xform=X.transform((0.45, 0.0, 0.0)),
                                            child_xform=X.transform((0.0, 0.0, 0.0)), label="pendulum_joint")
        builder.add_articulation([j_root, j_pend])
        builder.add_shape_box(root, xform=X.transform((0.6, 0.0, 0.0)), hx=0.15, hy=0.08, hz=0.08)
        builder.add_shape_sphere(pendulum, xform=X.transform((0.3, 0.0, 0.0)), radius=0.1)
        probe = builder.add_body(xform=X.transform((0.72, 0.0, 0.0)), mass=0.6, label="probe")
        builder.add_shape_sphere(probe, radius=0.1)
        model = builder.finalize()
        solver = _solver(si, model)
        pipe = oracle.CollisionPipeline(model)
        contacts = pipe.contacts()
        s0, s1 = model.state(), model.state()
        p0 = s0.body_q.numpy()[probe, :3].copy()
        max_probe = max_pend = 0.0
        for i in range(steps):
            theta = theta0 + omega * i * dt
            s0.body_q[root] = torch.tensor([0.0, 0.0, 0.0, 0.0, np.sin(theta / 2), 0.0, np.cos(theta / 2)], dtype=torch.float32)
            s0.body_qd[root] = torch.tensor([0.0, 0.0, 0.0, 0.0, omega, 0.0])
            s0.clear_forces()
            if apply_force:
                s0.body_f[root] = KINEMATIC_TEST_WRENCH
            pipe.collide(s0, contacts)
            solver.step(s0, s1, None, contacts, dt)
            s0, s1 = s1, s0
            qd = s0.body_qd.numpy()
            max_probe = max(max_probe, float(np.linalg.norm(qd[probe, :3])))
            max_pend = max(max_pend, float(np.linalg.norm(qd[pendulum])))
        q, qd = s0.body_q.numpy(), s0.body_qd.numpy()
        return dict(root_pos=q[root, :3].copy(), root_quat=q[root, 3:].copy(), root_qd=qd[root].copy(), probe_max_speed=max_probe,
                    pendulum_max_speed=max_pend, probe_displacement=float(np.linalg.norm(q[probe, :3] - p0)))

    free, forced = run_once(False), run_once(True)
    theta_end = theta0 + omega * (steps - 1) * dt
    _quat_close(free["root_quat"], np.array([0.0, np.sin(theta_end / 2), 0.0, np.cos(theta_end / 2)]), 0.99)
    assert np.linalg.norm(free["root_qd"][3:]) > 5e-1
    np.testing.assert_allclose(forced["root_pos"], free["root_pos"], atol=1.5e-2)
    _quat_close(forced["root_quat"], free["root_quat"], 0.995)
    assert np.linalg.norm(forced["root_qd"] - free["root_qd"]) < 8e-1
    assert free["probe_max_speed"] > 2e-2 and free["probe_displacement"] > 1e-2 and free["pendulum_max_speed"] > 2e-2


def test_kinematic_fixed_root_static_force_immune(si):
    """:578-638"""
    import oracle

    dt, steps, probe_vx = 1.0 / 240.0, 140, 3.0

    def run_once(apply_force):
        builder = ModelBuilder(gravity=(0.0, 0.0, 0.0))
        _contact_defaults(builder)
        static = builder.add_link(xform=X.transform((0.0, 0.0, 0.0)), mass=1.0, is_kinematic=True, label="static_root")
        builder.add_articulation([builder.add_joint_fixed(-1, static, label="static_root_joint")])
        builder.add_shape_box(static, hx=0.25, hy=0.25, hz=0.25)
        probe = builder.add_body(xform=X.transform((-1.0, 0.0, 0.0)), mass=1.0, label="probe")
        builder.add_shape_sphere(probe, radius=0.12)
        model = builder.finalize()
        joint = int(np.flatnonzero(model.numpy("joint_child") == probe)[0])
        qds = int(model.joint_qd_start[joint])
        solver = _solver(si, model)
        pipe = oracle.CollisionPipeline(model)
        contacts = pipe.contacts()
        s0, s1 = model.state(), model.state()
        s0.joint_qd[qds : qds + 6] = torch.tensor([probe_vx, 0.0, 0.0, 0.0, 0.0, 0.0])
        oracle.eval_fk(model, s0.joint_q, s0.joint_qd, s0)
        q_init = s0.body_q.numpy()[static].copy()
        for _ in range(steps):
            s0.clear_forces()
            if apply_force:
                s0.body_f[static] = KINEMATIC_TEST_WRENCH
            pipe.collide(s0, contacts)
            solver.step(s0, s1, None, contacts, dt)
            s0, s1 = s1, s0
        q, qd = s0.body_q.numpy(), s0.body_qd.numpy()
        return dict(q_init=q_init, static_pos=q[static, :3].copy(), static_quat=q[static, 3:].copy(), static_qd=qd[static].copy(),
                    probe_pos=q[probe, :3].copy(), probe_qd=qd[probe].copy())

    free, forced = run_once(False), run_once(True)
    np.testing.assert_allclose(free["static_pos"], free["q_init"][:3], atol=2e-3)
    _quat_close(free["static_quat"], free["q_init"][3:], 0.9999)
    assert np.linalg.norm(free["static_qd"]) < 4e-1
    np.testing.assert_allclose(forced["static_pos"], free["static_pos"], atol=2e-3)
    _quat_close(forced["static_quat"], free["static_quat"], 0.9999)
    assert np.linalg.norm(forced["static_qd"] - free["static_qd"]) < 6e-2
    assert free["probe_pos"][0] < 0.25 and abs(free["probe_qd"][0] - probe_vx) > 2.5e-1


def test_kinematic_runtime_toggle(si):
    """:641-715 - body_flags edited at run time + notify_model_changed(BODY_PROPERTIES)."""
    import oracle

    builder = ModelBuilder(gravity=(0.0, 0.0, 0.0))
    body = builder.add_body(xform=X.transform((0.0, 0.0, 0.0)), mass=1.0, is_kinematic=True, label="toggle_body")
    builder.add_shape_sphere(body, radius=0.1)
    model = builder.finalize()
    solver = _solver(si, model)
    pipe = oracle.CollisionPipeline(model)
    contacts = pipe.contacts()
    s0, s1 = model.state(), model.state()

    def phase(s0, s1):
        for _ in range(60):
            s0.clear_forces()
            s0.body_f[body] = torch.tensor([10.0, 0.0, 0.0, 0.0, 0.0, 0.0])
            pipe.collide(s0, contacts)
            solver.step(s0, s1, None, contacts, 1.0 / 240.0)
            s0, s1 = s1, s0
        return s0, s1

    s0, s1 = phase(s0, s1)
    assert np.linalg.norm(s0.body_q.numpy()[body, :3]) < 1e-3
    model.body_flags[body] = int(BodyFlags.DYNAMIC)
    solver.notify_model_changed(ModelFlags.BODY_PROPERTIES)
    s0, s1 = phase(s0, s1)
    assert s0.body_q.numpy()[body, 0] > 0.05
    model.body_flags[body] = int(BodyFlags.KINEMATIC)
    solver.notify_model_changed(ModelFlags.BODY_PROPERTIES)
    before = s0.body_q.numpy()[body, :3].copy()
    s0, s1 = phase(s0, s1)
    assert np.linalg.norm(s0.body_q.numpy()[body, :3] - before) < 1e-3


# ---- test_runtime_gravity.py (body rows, run with this solver) -------------------------------------------------------------------
def _box_world():
    w = ModelBuilder(gravity=(0.0, 0.0, -9.81))
    w.default_shape_cfg.density = 1000.0
    b = w.add_body()
    w.add_shape_box(b, hx=0.5, hy=0.5, hz=0.5)
    return w


def _run(solver, model, s0, s1, n, dt=0.01):
    control = model.control()
    for _ in range(n):
        s0.clear_forces()
        solver.step(s0, s1, control, None, dt)
        s0, s1 = s1, s0
    return s0, s1


def test_runtime_gravity_bodies(si):
    """:124-163 - set_gravity between steps + notify_model_changed(MODEL_PROPERTIES)."""
    model = _box_world().finalize()
    solver = _solver(si, model)
    s0, s1 = _run(solver, model, model.state(), model.state(), 10)
    assert s0.body_qd.numpy()[0, 2] < -0.5
    model.set_gravity((9.81, 0.0, 0.0))
    solver.notify_model_changed(ModelFlags.MODEL_PROPERTIES)
    s0, s1 = _run(solver, model, s0, s1, 20)
    assert s0.body_qd.numpy()[0, 0] > 0.5


def test_per_world_gravity_bodies(si):
    """:266-318 - one gravity per world."""
    main = ModelBuilder(gravity=(0.0, 0.0, -9.81))
    main.replicate(_box_world(), 3)
    model = main.finalize()
    solver = _solver(si, model)
    model.set_gravity((0.0, 0.0, 0.0), world=0)
    model.set_gravity((0.0, 0.0, -4.905), world=1)
    model.set_gravity((0.0, 0.0, -9.81), world=2)
    solver.notify_model_changed(ModelFlags.MODEL_PROPERTIES)
    s0, _ = _run(solver, model, model.state(), model.state(), 10)
    vz = s0.body_qd.numpy()[:, 2]
    assert vz[0] == pytest.approx(0.0, abs=5e-5)
    assert vz[2] < vz[1] < 0.0 and vz[2] < -0.5
    assert vz[1] == pytest.approx(-0.4905, abs=1e-5) and vz[2] == pytest.approx(-0.981, abs=1e-5)


def test_global_gravity_bodies(si):
    """:362-381 - a body of the global world -1 falls with the last gravity entry."""
    builder = ModelBuilder(gravity=(0.0, 0.0, -2.0))
    global_body = builder.add_body(mass=1.0, inertia=np.eye(3))
    builder.begin_world(gravity=(0.0, 0.0, -5.0))
    local_body = builder.add_body(mass=1.0, inertia=np.eye(3))
    builder.end_world()
    model = builder.finalize()
    s_in, s_out = model.state(), model.state()
    _solver(si, model).step(s_in, s_out, model.control(), None, 0.1)
    qd = s_out.body_qd.numpy()
    assert qd[global_body, 2] == pytest.approx(-0.2, abs=1e-6)
    assert qd[local_body, 2] == pytest.approx(-0.5, abs=1e-6)


# ---- test_body_velocity.py:124-372 with the semi_implicit row of :871 (body_qd set directly, tolerance 1e-4) -------------------
# test_semi_implicit.py's test_applied_body_force_and_kinematic_body drives a body whose COM is at its origin; none of these rows
# (a COM away from the body origin, body_qd given at the COM) was covered.
COM_OFFSETS = [(0.5, 0.0, 0.0), (0.0, 0.3, 0.0), (0.0, 0.0, 0.4), (0.2, 0.3, 0.1)]
AXIS_VECTORS = [(0.0, 0.0, 1.0), (0.0, 1.0, 0.0), (1.0, 0.0, 0.0)]
LINEAR_VELOCITIES = [(0.7, 0.0, 0.0), (0.0, 0.7, 0.0), (0.0, 0.0, 0.7)]


def _offset_com_box(com, pos, rot=None):
    """One free box (add_body) at ``pos`` whose COM is moved to ``com`` after its shape is added, without gravity."""
    import oracle

    b = ModelBuilder(gravity=(0.0, 0.0, 0.0))
    body = b.add_body(xform=X.transform(pos, rot) if rot is not None else X.transform(pos))
    b.add_shape_box(body, hx=0.1, hy=0.1, hz=0.1)
    b.body_com[body] = np.asarray(com, dtype=np.float64)
    model = b.finalize()
    s0, s1 = model.state(), model.state()
    oracle.eval_fk(model, model.joint_q, model.joint_qd, s0)
    return model, s0, s1


def _com_world(model, state):
    q = state.body_q.numpy()[0].astype(np.float64)
    from scipy.spatial.transform import Rotation

    return q[:3] + Rotation.from_quat(q[3:]).apply(model.body_com.numpy()[0].astype(np.float64))


def _free_steps(si, model, s0, s1, n, dt, control=None, wrench=None):
    solver = _solver(si, model)
    for _ in range(n):
        solver.step(s0, s1, control, None, dt)
        s0, s1 = s1, s0
        if wrench is not None:  # re-applied for the next step, as the reference does
            s0.body_f.copy_(wrench)
            s1.body_f.copy_(wrench)
    return s0


@pytest.mark.parametrize("com", COM_OFFSETS)
@pytest.mark.parametrize("w", AXIS_VECTORS)
def test_body_velocity_angular_com_stationary(si, com, w):
    """:124-211 - angular velocity alone turns the body about its COM: the COM moves < 1e-4 in 10 steps of 10 ms."""
    model, s0, s1 = _offset_com_box(com, (1.0, 2.0, 3.0))
    s0.body_qd.copy_(torch.tensor([[0.0, 0.0, 0.0, *w]]))
    q0, c0 = s0.body_q.numpy()[0].copy(), _com_world(model, s0)
    s = _free_steps(si, model, s0, s1, 10, 0.01)
    assert np.linalg.norm(_com_world(model, s) - c0) < 1e-4
    assert abs(float(np.dot(q0[3:], s.body_q.numpy()[0, 3:]))) < 0.9999


@pytest.mark.parametrize("com", COM_OFFSETS)
@pytest.mark.parametrize("v", LINEAR_VELOCITIES)
def test_body_velocity_linear_com_moves(si, com, v):
    """:214-287 - linear velocity alone moves the COM by v t, within 1e-4."""
    model, s0, s1 = _offset_com_box(com, (0.0, 0.0, 1.0))
    s0.body_qd.copy_(torch.tensor([[*v, 0.0, 0.0, 0.0]]))
    c0 = _com_world(model, s0)
    s = _free_steps(si, model, s0, s1, 10, 0.01)
    assert np.linalg.norm(_com_world(model, s) - c0 - np.array(v) * 0.1) < 1e-4


@pytest.mark.parametrize("com", COM_OFFSETS)
def test_body_velocity_combined(si, com):
    """:290-371 - (0.1, 0, 0) m/s and (0, 0, 1) rad/s together: the COM moves by v t within 1e-4 and the body turns."""
    model, s0, s1 = _offset_com_box(com, (0.0, 0.0, 1.0))
    s0.body_qd.copy_(torch.tensor([[0.1, 0.0, 0.0, 0.0, 0.0, 1.0]]))
    q0, c0 = s0.body_q.numpy()[0].copy(), _com_world(model, s0)
    s = _free_steps(si, model, s0, s1, 10, 0.01)
    assert np.linalg.norm(_com_world(model, s) - c0 - np.array([0.01, 0.0, 0.0])) < 1e-4
    assert abs(float(np.dot(q0[3:], s.body_q.numpy()[0, 3:]))) < 0.9999


# ---- test_body_force.py:356-528 with the semi_implicit row of :551 (non-zero COM) ------------------------------------------------
def _rotated_offset_com_box(com):
    return _offset_com_box(com, (0.0, 0.0, 1.0), X.quat_from_axis_angle((1.0, 0.0, 0.0), 0.5 * np.pi))


def _apply(model, s0, s1, wrench, use_control):
    w = torch.tensor([wrench], dtype=torch.float32)
    if use_control:
        control = model.control()
        control.joint_f.copy_(w[0])
        return control, None
    s0.body_f.copy_(w)
    s1.body_f.copy_(w)
    return None, w


@pytest.mark.parametrize("use_control", [False, True])
@pytest.mark.parametrize("com", COM_OFFSETS)
@pytest.mark.parametrize("direction", LINEAR_VELOCITIES)
def test_body_force_no_rotation(si, com, direction, use_control):
    """:356-444 - a 10 N force at the COM of a rotated box (body_f or Control.joint_f), 5 steps of 10 ms: no angular velocity
    (< 1e-3) and F / m t along the force within 5 %."""
    model, s0, s1 = _rotated_offset_com_box(com)
    f = np.array(direction) / 0.7 * 10.0
    control, wrench = _apply(model, s0, s1, [*f, 0.0, 0.0, 0.0], use_control)
    s = _free_steps(si, model, s0, s1, 5, 0.01, control, wrench)
    qd = s.body_qd.numpy()[0]
    expected = 10.0 / float(model.body_mass[0]) * 0.05
    assert np.abs(qd[3:]).max() < 1e-3
    assert float(np.dot(f / 10.0, qd[:3])) == pytest.approx(expected, abs=5e-2 * expected)


@pytest.mark.parametrize("use_control", [False, True])
@pytest.mark.parametrize("com", COM_OFFSETS)
def test_body_force_combined_force_torque(si, com, use_control):
    """:447-528 - 10 N along x and 10 Nm about z, 10 steps of 10 ms: v_x = F / m t and w_z = tau / I_zz t within 5 % of (1 + x),
    every other component < 1e-3."""
    model, s0, s1 = _rotated_offset_com_box(com)
    control, wrench = _apply(model, s0, s1, [10.0, 0.0, 0.0, 0.0, 0.0, 10.0], use_control)
    s = _free_steps(si, model, s0, s1, 10, 0.01, control, wrench)
    qd = s.body_qd.numpy()[0]
    v = 10.0 / float(model.body_mass[0]) * 0.1
    w = 10.0 / float(model.body_inertia[0, 2, 2]) * 0.1
    assert qd[0] == pytest.approx(v, abs=5e-2 * (1 + v))
    assert qd[5] == pytest.approx(w, abs=5e-2 * (1 + w))
    assert np.abs(qd[[1, 2, 3, 4]]).max() < 1e-3


# ---- test_rigid_contact.py:28-235 (test_shapes_on_plane), semi_implicit row --------------------------------------------------------
def test_shapes_on_plane(si):
    """Spheres, lying capsules, boxes, upright cylinders and a triangle-mesh cube whose vertices are offset by (1, 0, 0) from its
    origin, at two sizes, dropped from 0.5 m: ke 1e4, kd 1e3, kf 0, gap 0.1; SolverSemiImplicit(angular_damping=0.15,
    friction_smoothing=2.0); 120 frames of 30 substeps at 60 fps.  At the end |v| and |w| < 0.2, positions within 0.25 of the
    resting heights and quaternions within 0.1 of identity.  The mesh goes through CollisionPipeline(reduce_contacts=False), its
    route here (one contact per vertex near the plane)."""
    import oracle
    from newton_b200.geometry.mesh import Mesh

    s = 0.3
    corners = [(-s, -s, -s), (-s, -s, s), (-s, s, s), (-s, s, -s), (s, -s, -s), (s, -s, s), (s, s, s), (s, s, -s),
               (-s, -s, -s), (-s, -s, s), (s, -s, s), (s, -s, -s), (-s, s, -s), (-s, s, s), (s, s, s), (s, s, -s),
               (-s, -s, -s), (-s, s, -s), (s, s, -s), (s, -s, -s), (-s, -s, s), (-s, s, s), (s, s, s), (s, -s, s)]
    vertices = np.array(corners, dtype=np.float32) + np.array([1.0, 0.0, 0.0], dtype=np.float32)
    indices = [0, 1, 2, 0, 2, 3, 4, 6, 5, 4, 7, 6, 8, 10, 9, 8, 11, 10, 12, 13, 14, 12, 14, 15, 16, 17, 18, 16, 18, 19,
               20, 22, 21, 20, 23, 22]
    cube = Mesh(vertices, np.array(indices, dtype=np.int32))
    b = ModelBuilder()
    cfg = b.default_shape_cfg
    cfg.ke, cfg.kd, cfg.kf, cfg.gap = 1e4, 1000.0, 0.0, 0.1
    expected = []
    z_to_y = X.quat_between_vectors((0.0, 0.0, 1.0), (0.0, 1.0, 0.0))
    for i, scale in enumerate((0.5, 1.0)):
        y = 1.5 * i
        body = b.add_body(xform=X.transform((0.0, y, 0.5)))
        b.add_shape_sphere(body, radius=0.1 * scale)
        expected.append((0.0, y, 0.1 * scale))
        body = b.add_body(xform=X.transform((2.0, y, 0.5)))
        b.add_shape_capsule(body, xform=X.transform((0.0, 0.0, 0.0), z_to_y), radius=0.1 * scale, half_height=0.3 * scale)
        expected.append((2.0, y, 0.1 * scale))
        body = b.add_body(xform=X.transform((4.0, y, 0.5)))
        b.add_shape_box(body, hx=0.2 * scale, hy=0.25 * scale, hz=0.3 * scale)
        expected.append((4.0, y, 0.3 * scale))
        body = b.add_body(xform=X.transform((5.0, y, 0.5)))
        b.add_shape_cylinder(body, radius=0.1 * scale, half_height=0.3 * scale)
        expected.append((5.0, y, 0.3 * scale))
        body = b.add_body(xform=X.transform((7.0, y, 0.5)))
        b.add_shape_mesh(body, mesh=cube, scale=(scale, scale, scale))
        expected.append((7.0, y, 0.3 * scale))
    b.add_ground_plane()
    model = b.finalize()
    solver = si.SolverSemiImplicit(model, angular_damping=0.15, friction_smoothing=2.0)
    pipe = oracle.CollisionPipeline(model, reduce_contacts=False)
    contacts = pipe.contacts()
    s0, s1, ctl = model.state(), model.state(), model.control()
    dt = 1.0 / 60.0 / 30
    for _ in range(120 * 30):
        s0.clear_forces()
        pipe.collide(s0, contacts)
        solver.step(s0, s1, ctl, contacts, dt)
        s0, s1 = s1, s0
    q, qd = s0.body_q.numpy(), s0.body_qd.numpy()
    assert np.isfinite(q).all() and np.isfinite(qd).all()
    assert np.abs(qd[:, :3]).max() < 0.2 and np.abs(qd[:, 3:]).max() < 0.2
    np.testing.assert_allclose(q[:, :3], np.array(expected), atol=0.25)
    np.testing.assert_allclose(q[:, 3:], np.tile([0.0, 0.0, 0.0, 1.0], (model.body_count, 1)), atol=1e-1)

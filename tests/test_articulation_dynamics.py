"""Articulation Jacobians, mass matrices and inverse dynamics (newton.eval_jacobian / eval_mass_matrix /
eval_inverse_dynamics_passive / eval_inverse_dynamics_force).

CPU part: the oracle restatement (oracle/oracle_dynamics.h) against the known answers of the reference's own tests
(newton/tests/test_jacobian_mass_matrix.py, test_inverse_dynamics.py): closed forms, J @ qd == body_qd, kinetic energy, gravity
as the gradient of the potential energy, the Coriolis / mass-matrix / free-joint wrench closed forms, and the manipulator-equation
round trip through the oracle's SolverFeatherstone; plus the
host-side argument handling of the product functions.  The scene builders here are shared with
tests/test_gpu_articulation_dynamics.py, which holds the CUDA kernels to the oracle bit for bit.
"""

from __future__ import annotations

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import JointType, ModelBuilder
from newton_b200.utils import xform as X

I3 = np.eye(3)


def _tf(p=(0.0, 0.0, 0.0), axis=(0.0, 0.0, 1.0), angle=0.0):
    return list(X.transform(np.asarray(p, float), X.quat_from_axis_angle(np.asarray(axis, float), angle)))


def _inertia(a, b, c):
    return np.diag([a, b, c])


# ---- scenes ----------------------------------------------------------------------------------------------------------------
def pendulum(b: ModelBuilder, L=1.0, m=2.0):
    """Fixed-base pendulum about z; the link COM sits L along x from the joint."""
    body = b.add_link(xform=_tf((L, 0.0, 0.0)), mass=m, inertia=_inertia(0.1, 0.2, 0.3))
    j = b.add_joint_revolute(-1, body, axis=(0.0, 0.0, 1.0), child_xform=_tf((-L, 0.0, 0.0)))
    b.add_articulation([j])


def slider(b: ModelBuilder):
    """Prismatic joint on a translated, rotated anchor, COM offset in the child."""
    body = b.add_link(mass=1.5, com=(0.1, 0.2, 0.0), inertia=_inertia(0.2, 0.1, 0.3))
    j = b.add_joint_prismatic(-1, body, axis=(1.0, 0.0, 0.0), parent_xform=_tf((0.3, -0.2, 1.0), (0, 1, 0), 0.4))
    b.add_articulation([j])


def double_pendulum(b: ModelBuilder):
    b0 = b.add_link(mass=1.0, com=(0.05, 0.0, 0.02), inertia=_inertia(0.1, 0.12, 0.08))
    b1 = b.add_link(mass=0.7, com=(0.0, 0.03, -0.1), inertia=_inertia(0.05, 0.06, 0.02))
    j0 = b.add_joint_revolute(-1, b0, axis=(0.0, 1.0, 0.0), parent_xform=_tf((0.0, 0.0, 2.0), (1, 0, 0), 0.3),
                              child_xform=_tf((-0.5, 0.0, 0.0)))
    j1 = b.add_joint_revolute(b0, b1, axis=(0.0, 1.0, 0.0), parent_xform=_tf((0.5, 0.0, 0.0), (0, 0, 1), -0.2),
                              child_xform=_tf((-0.4, 0.0, 0.0)))
    b.add_articulation([j0, j1])


def d6_chain(b: ModelBuilder, angular=3, linear=0):
    """D6 root with `angular` angular axes (transported axes; reference :834), then a revolute child."""
    b0 = b.add_link(mass=1.2, com=(0.1, -0.05, 0.2), inertia=_inertia(0.3, 0.2, 0.25))
    b1 = b.add_link(mass=0.4, com=(0.0, 0.0, -0.2), inertia=_inertia(0.02, 0.03, 0.01))
    from newton_b200.sim.builder import JointDofConfig as D

    ang = [D(axis=(1.0, 0.0, 0.0)), D(axis=(0.0, 1.0, 0.0)), D(axis=(0.0, 0.0, 1.0))][:angular]
    lin = [D(axis=(0.0, 0.0, 1.0))][:linear]
    j0 = b.add_joint_d6(-1, b0, linear_axes=lin, angular_axes=ang, parent_xform=_tf((0.0, 0.0, 1.0)))
    j1 = b.add_joint_revolute(b0, b1, axis=(1.0, 0.0, 0.0), parent_xform=_tf((0.2, 0.0, -0.3)))
    b.add_articulation([j0, j1])


def ball_chain(b: ModelBuilder):
    b0 = b.add_link(mass=0.9, com=(0.0, 0.0, -0.3), inertia=_inertia(0.04, 0.05, 0.03))
    b1 = b.add_link(mass=0.5, com=(0.1, 0.0, -0.2), inertia=_inertia(0.02, 0.02, 0.01))
    j0 = b.add_joint_ball(-1, b0, parent_xform=_tf((0.0, 0.0, 1.5), (0, 1, 0), 0.5))
    j1 = b.add_joint_revolute(b0, b1, axis=(0.0, 1.0, 0.0), parent_xform=_tf((0.0, 0.0, -0.6)))
    b.add_articulation([j0, j1])


def free_root(b: ModelBuilder):
    """Floating base with a COM offset and a revolute child under a rotated anchor."""
    b0 = b.add_link(xform=_tf((0.2, -0.1, 1.0), (1, 1, 0), 0.6), mass=3.0, com=(0.05, 0.02, -0.04), inertia=_inertia(0.3, 0.4, 0.5))
    b1 = b.add_link(mass=0.6, com=(0.0, 0.1, 0.0), inertia=_inertia(0.03, 0.01, 0.02))
    j0 = b.add_joint_free(b0)
    j1 = b.add_joint_revolute(b0, b1, axis=(0.0, 0.0, 1.0), parent_xform=_tf((0.3, 0.0, 0.0), (0, 1, 0), 0.7))
    b.add_articulation([j0, j1])


def free_descendant(b: ModelBuilder):
    """A FREE joint below a revolute root whose anchor is rotated: non-root free joints use the parent frame."""
    b0 = b.add_link(mass=1.0, com=(0.0, 0.0, 0.1), inertia=_inertia(0.1, 0.1, 0.1))
    b1 = b.add_link(xform=_tf((0.4, 0.1, 1.2), (0, 0, 1), 0.3), mass=0.8, com=(0.03, -0.02, 0.05), inertia=_inertia(0.02, 0.05, 0.04))
    j0 = b.add_joint_revolute(-1, b0, axis=(0.0, 0.0, 1.0), parent_xform=_tf((0.0, 0.0, 1.0), (1, 0, 0), 0.4))
    j1 = b.add_joint_free(b1, parent=b0, parent_xform=_tf((0.2, 0.0, 0.1), (0, 1, 0), -0.5))
    b.add_articulation([j0, j1])


def loop_closed(b: ModelBuilder):
    """Fixed base + two revolutes, then a loop-closing revolute that is not part of the articulation."""
    b0 = b.add_link(mass=2.0, inertia=I3)
    b1 = b.add_link(mass=2.0, inertia=I3)
    b2 = b.add_link(mass=2.0, inertia=I3)
    one, mone = _tf((1.0, 0.0, 0.0)), _tf((-1.0, 0.0, 0.0))
    j0 = b.add_joint_fixed(-1, b0)
    j1 = b.add_joint_revolute(b0, b1, axis=(0.0, 0.0, 1.0), parent_xform=one, child_xform=mone)
    j2 = b.add_joint_revolute(b1, b2, axis=(0.0, 0.0, 1.0), parent_xform=one, child_xform=mone)
    b.add_articulation([j0, j1, j2])
    b.add_joint_revolute(b0, b2, axis=(0.0, 0.0, 1.0), parent_xform=one, child_xform=mone)


def d6_mixed(b: ModelBuilder):
    """D6 with one linear and two angular axes.  The reference's subspaces turn its angular axes about the joint anchor, not
    about the translated joint frame, so J @ qd differs from body_qd here upstream too; used for the bit-parity checks only."""
    d6_chain(b, angular=2, linear=1)


KINEMATIC_SCENES = {f.__name__: f for f in (pendulum, slider, double_pendulum, d6_chain, ball_chain, free_root, free_descendant, loop_closed)}
SCENES = dict(KINEMATIC_SCENES, d6_mixed=d6_mixed)


def build(*parts, worlds=1, gravity=None, seed=0, noise=0.4):
    """One world per entry of `gravity` (or `worlds` copies), each holding every scene in `parts`; joint_q / joint_qd seeded."""
    b = ModelBuilder()
    gravities = gravity if gravity is not None else [None] * worlds
    for g in gravities:
        b.begin_world(gravity=g)
        for p in parts:
            SCENES[p](b) if isinstance(p, str) else p(b)
        b.end_world()
    model = b.finalize("cpu")
    randomize(model, seed, noise)
    return model


def randomize(model, seed, noise=0.4):
    rng = np.random.default_rng(seed)
    jq = model.joint_q.numpy().astype(np.float64)
    qs, types = model.numpy("joint_q_start"), model.numpy("joint_type")
    for j, t in enumerate(types):
        a, e = qs[j], qs[j + 1]
        if t == JointType.BALL:
            q = rng.normal(size=4)
            jq[a:e] = q / np.linalg.norm(q)
        elif t in (JointType.FREE, JointType.DISTANCE):
            jq[a : a + 3] += rng.normal(0.0, noise, 3)
            q = np.asarray(jq[a + 3 : a + 7]) + rng.normal(0.0, noise, 4)
            jq[a + 3 : a + 7] = q / np.linalg.norm(q)
        else:
            jq[a:e] += rng.normal(0.0, noise, e - a)
    model.joint_q = torch.tensor(jq, dtype=torch.float32)
    model.joint_qd = torch.tensor(rng.normal(0.0, 1.0, int(model.joint_dof_count)), dtype=torch.float32)


def fk_state(oracle, model, joint_qd=None):
    state = model.state()
    state.joint_q = model.joint_q.clone()
    state.joint_qd = (model.joint_qd if joint_qd is None else joint_qd).clone()
    oracle.eval_fk(model, state.joint_q, state.joint_qd, state)
    return state


@pytest.fixture(scope="module")
def od(oracle_lib):
    import oracle.dynamics as od

    od.build()
    return od


def _twists_from_J(model, J, qd):
    """Per-articulation J @ qd as [A, links, 6]."""
    out = []
    qs, starts, ends = model.numpy("joint_qd_start"), model.numpy("articulation_start"), model.numpy("articulation_end")
    for a in range(model.articulation_count):
        d0, d1 = qs[starts[a]], qs[ends[a]]
        v = J[a][:, : d1 - d0].astype(np.float64) @ qd[d0:d1].astype(np.float64)
        out.append(v.reshape(-1, 6))
    return out


def _links(model, a):
    return model.numpy("joint_child")[model.numpy("articulation_start")[a] : model.numpy("articulation_end")[a]]


# ---- Jacobian -----------------------------------------------------------------------------------------------------------------
def test_jacobian_simple_pendulum(od, oracle_lib):
    model = build("pendulum", noise=0.0)
    model.joint_q.zero_()
    J = od.eval_jacobian(model, fk_state(oracle_lib, model)).numpy()
    assert J.shape == (1, 6, 1)
    np.testing.assert_allclose(J[0, :, 0], [0.0, 1.0, 0.0, 0.0, 0.0, 1.0], atol=1e-6)  # z x (L, 0, 0), w = z


def test_prismatic_jacobian(od, oracle_lib):
    model = build("slider", noise=0.0)
    state = fk_state(oracle_lib, model)
    J = od.eval_jacobian(model, state).numpy()
    axis = X.quat_rotate(X.quat_from_axis_angle(np.array([0.0, 1.0, 0.0]), 0.4), np.array([1.0, 0.0, 0.0]))
    np.testing.assert_allclose(J[0, :, 0], [*axis, 0.0, 0.0, 0.0], atol=1e-6)


@pytest.mark.parametrize("scene", sorted(KINEMATIC_SCENES))
def test_jacobian_times_qd_is_body_twist(od, oracle_lib, scene):
    """J_link @ joint_qd == state.body_qd[link] (COM-referenced world twists), free roots and descendants included."""
    model = build(scene, seed=3)
    state = fk_state(oracle_lib, model)
    J = od.eval_jacobian(model, state).numpy()
    bqd = state.body_qd.numpy()
    for a, tw in enumerate(_twists_from_J(model, J, state.joint_qd.numpy())):
        np.testing.assert_allclose(tw, bqd[_links(model, a)], atol=2e-5, rtol=1e-5)


def test_jacobian_finite_difference(od, oracle_lib):
    """Columns of J against central differences of the link COM positions (revolute / prismatic chain)."""
    model = build("double_pendulum", "slider", seed=5)
    state = fk_state(oracle_lib, model)
    J = od.eval_jacobian(model, state).numpy()
    com = model.numpy("body_com").astype(np.float64)
    h = 1e-3

    def coms(q):
        s = model.state()
        oracle_lib.eval_fk(model, torch.tensor(q, dtype=torch.float32), model.joint_qd, s)
        bq = s.body_q.numpy().astype(np.float64)
        return np.array([X.transform_point(bq[i], com[i]) for i in range(model.body_count)])

    q0 = state.joint_q.numpy().astype(np.float64)
    for dof in range(2):  # double pendulum: coords == dofs
        qp, qm = q0.copy(), q0.copy()
        qp[dof] += h
        qm[dof] -= h
        dc = (coms(qp) - coms(qm)) / (2 * h)
        for i, body in enumerate(_links(model, 0)):
            np.testing.assert_allclose(J[0, 6 * i : 6 * i + 3, dof], dc[body], atol=2e-3)


def test_jacobian_multiple_articulations_and_mask(od, oracle_lib):
    model = build("double_pendulum", "free_root", "ball_chain", worlds=2, seed=7)
    state = fk_state(oracle_lib, model)
    J = od.eval_jacobian(model, state).numpy()
    assert J.shape == (6, 6 * model.max_joints_per_articulation, model.max_dofs_per_articulation)
    mask = torch.tensor([True, False, True, False, False, True])
    Jm = od.eval_jacobian(model, state, mask=mask).numpy()
    for a in range(6):
        if mask[a]:
            np.testing.assert_array_equal(Jm[a], J[a])
        else:
            assert not Jm[a].any()
    H = od.eval_mass_matrix(model, state).numpy()
    Hm = od.eval_mass_matrix(model, state, mask=mask).numpy()
    for a in range(6):
        if mask[a]:
            np.testing.assert_array_equal(Hm[a], H[a])
        else:
            assert not Hm[a].any()


# ---- mass matrix ---------------------------------------------------------------------------------------------------------------
def test_fixed_base_pendulum_mass_matrix(od, oracle_lib):
    """H = m L^2 + I_zz (parallel-axis theorem)."""
    model = build("pendulum", seed=1)
    H = od.eval_mass_matrix(model, fk_state(oracle_lib, model)).numpy()
    np.testing.assert_allclose(H[0, 0, 0], 2.0 * 1.0 + 0.3, rtol=1e-5)


def test_floating_base_pendulum_mass_matrix(od, oracle_lib):
    """7 x 7 closed form of a free body at the origin with a revolute pendulum below it (identity poses)."""
    b = ModelBuilder()
    m0, m1, L = 3.0, 2.0, 1.0
    b0 = b.add_link(mass=m0, inertia=_inertia(0.1, 0.2, 0.3))
    b1 = b.add_link(xform=_tf((L, 0.0, 0.0)), mass=m1, inertia=_inertia(0.01, 0.02, 0.03))
    j0 = b.add_joint_free(b0)
    j1 = b.add_joint_revolute(b0, b1, axis=(0.0, 0.0, 1.0), child_xform=_tf((-L, 0.0, 0.0)))
    b.add_articulation([j0, j1])
    model = b.finalize("cpu")
    H = od.eval_mass_matrix(model, fk_state(oracle_lib, model)).numpy()[0].astype(np.float64)
    M = m0 + m1
    E = np.zeros((7, 7))
    E[:3, :3] = M * np.eye(3)
    r = np.array([L, 0.0, 0.0])  # link-1 COM relative to the base COM
    skew = np.array([[0, -r[2], r[1]], [r[2], 0, -r[0]], [-r[1], r[0], 0]])
    E[:3, 3:6] = -m1 * skew
    E[3:6, :3] = m1 * skew
    E[3:6, 3:6] = np.diag([0.1, 0.2, 0.3]) + np.diag([0.01, 0.02, 0.03]) + m1 * (r @ r * np.eye(3) - np.outer(r, r))
    E[1, 6] = E[6, 1] = m1 * L
    E[5, 6] = E[6, 5] = m1 * L * L + 0.03
    E[6, 6] = m1 * L * L + 0.03
    np.testing.assert_allclose(H, E, atol=1e-5)


@pytest.mark.parametrize("scene", sorted(KINEMATIC_SCENES))
def test_mass_matrix_kinetic_energy_symmetry_pd(od, oracle_lib, scene):
    """1/2 qd^T H qd equals the kinetic energy of the COM twists; H is symmetric and positive definite."""
    model = build(scene, seed=11)
    state = fk_state(oracle_lib, model)
    H = od.eval_mass_matrix(model, state).numpy().astype(np.float64)
    bq, bqd = state.body_q.numpy().astype(np.float64), state.body_qd.numpy().astype(np.float64)
    mass, inertia = model.numpy("body_mass"), model.numpy("body_inertia").reshape(-1, 3, 3)
    qs, starts, ends = model.numpy("joint_qd_start"), model.numpy("articulation_start"), model.numpy("articulation_end")
    qd = state.joint_qd.numpy().astype(np.float64)
    for a in range(model.articulation_count):
        d0, d1 = qs[starts[a]], qs[ends[a]]
        Ha = H[a, : d1 - d0, : d1 - d0]
        ke = 0.0
        for body in _links(model, a):
            R = X.quat_to_matrix(bq[body, 3:])
            v, w = bqd[body, :3], bqd[body, 3:]
            ke += 0.5 * mass[body] * v @ v + 0.5 * w @ (R @ inertia[body] @ R.T) @ w
        np.testing.assert_allclose(0.5 * qd[d0:d1] @ Ha @ qd[d0:d1], ke, rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(Ha, Ha.T, rtol=1e-5, atol=1e-6)
        assert np.linalg.eigvalsh(Ha).min() > 0.0
        assert not H[a, d1 - d0 :].any() and not H[a, :, d1 - d0 :].any()


# ---- inverse dynamics -------------------------------------------------------------------------------------------------------------
def _potential(oracle_lib, model, q):
    s = model.state()
    oracle_lib.eval_fk(model, torch.tensor(q, dtype=torch.float32), model.joint_qd, s)
    bq = s.body_q.numpy().astype(np.float64)
    com, mass, world = model.numpy("body_com").astype(np.float64), model.numpy("body_mass"), model.numpy("body_world")
    g = model.numpy("gravity").astype(np.float64)
    return sum(-mass[b] * g[world[b]] @ X.transform_point(bq[b], com[b]) for b in range(model.body_count))


@pytest.mark.parametrize("parts,gravity", [(("double_pendulum",), None), (("slider", "pendulum"), None),
                                           (("double_pendulum", "slider"), [(0, 0, -9.81), (9.81, 0, 0), (0, -4.0, 0)])])
def test_gravity_force_is_potential_gradient(od, oracle_lib, parts, gravity):
    """g(q) = dU/dq for revolute / prismatic chains, one world per gravity axis."""
    model = build(*parts, gravity=gravity, seed=2)
    state = fk_state(oracle_lib, model)
    _, g, _ = od.eval_inverse_dynamics_passive(model, state, gravity_force=True)
    q0, h = state.joint_q.numpy().astype(np.float64), 1e-3
    for dof in range(model.joint_dof_count):
        qp, qm = q0.copy(), q0.copy()
        qp[dof] += h
        qm[dof] -= h
        fd = (_potential(oracle_lib, model, qp) - _potential(oracle_lib, model, qm)) / (2 * h)
        np.testing.assert_allclose(g.numpy()[dof], fd, atol=2e-3, rtol=2e-3)


def test_free_body_gravity_is_world_wrench(od, oracle_lib):
    """A free body under a rotated anchor: g holds m g_world at the COM (world frame), no torque."""
    b = ModelBuilder(gravity=-10.0)
    body = b.add_link(xform=_tf((0.0, 0.0, 1.0), (1, 0, 0), 0.7), mass=2.0, com=(0.1, 0.0, 0.0), inertia=I3 * 0.1)
    b.add_articulation([b.add_joint_free(body, parent_xform=_tf((0.0, 0.0, 0.5), (0, 1, 0), 0.9))])
    model = b.finalize("cpu")
    _, g, _ = od.eval_inverse_dynamics_passive(model, fk_state(oracle_lib, model), gravity_force=True)
    np.testing.assert_allclose(g.numpy(), [0.0, 0.0, 20.0, 0.0, 0.0, 0.0], atol=1e-5)


@pytest.mark.parametrize("scene", sorted(SCENES))
def test_coriolis_zero_at_rest(od, oracle_lib, scene):
    model = build(scene, seed=4)
    state = fk_state(oracle_lib, model, torch.zeros(model.joint_dof_count))
    _, _, c = od.eval_inverse_dynamics_passive(model, state, coriolis_force=True)
    np.testing.assert_allclose(c.numpy(), 0.0, atol=1e-6)


def test_passive_mass_matrix_equals_eval_mass_matrix(od, oracle_lib):
    model = build("double_pendulum", "free_root", "d6_chain", seed=6)
    state = fk_state(oracle_lib, model)
    M, _, _ = od.eval_inverse_dynamics_passive(model, state, mass_matrix=True)
    np.testing.assert_array_equal(M.numpy(), od.eval_mass_matrix(model, state).numpy())


def test_force_hand_crafted_inputs(od, oracle_lib):
    """tau = M qdd + C qd + g on a fixed-base model (no frame rotation involved)."""
    model = build("double_pendulum", seed=8)
    state = fk_state(oracle_lib, model)
    D = model.max_dofs_per_articulation
    M = torch.tensor(np.arange(D * D, dtype=np.float32).reshape(1, D, D) / 7.0)
    qdd, cor, grav = (torch.tensor([1.5, -2.0]), torch.tensor([0.25, 0.5]), torch.tensor([-1.0, 3.0]))
    tau = od.eval_inverse_dynamics_force(model, state, mass_matrix=M, joint_qdd=qdd, coriolis_force=cor, gravity_force=grav)
    expect = M[0].double().numpy() @ qdd.double().numpy() + cor.numpy() + grav.numpy()
    np.testing.assert_allclose(tau.numpy(), expect, rtol=1e-6)


def test_loop_closing_joint_leaves_tau_clean(od, oracle_lib):
    model = build("loop_closed", worlds=1, seed=9)  # the loop joint's dof sits after the tree's
    state = fk_state(oracle_lib, model)
    M, g, c = od.eval_inverse_dynamics_passive(model, state, mass_matrix=True, gravity_force=True, coriolis_force=True)
    qdd = torch.tensor([0.3, -0.7, 1e6])  # large orphan acceleration on the loop dof
    tau = od.eval_inverse_dynamics_force(model, state, mass_matrix=M, joint_qdd=qdd, coriolis_force=c, gravity_force=g)
    assert tau[2] == 0.0
    expect = M[0, :2, :2].double().numpy() @ qdd[:2].double().numpy() + c[:2].numpy() + g[:2].numpy()
    np.testing.assert_allclose(tau[:2].numpy(), expect, rtol=1e-5)


# ---- known answers ported from the reference's test_inverse_dynamics.py --------------------------------------------------------
def _set_state(oracle, model, q, qd):
    model.joint_q = torch.tensor(q, dtype=torch.float32)
    model.joint_qd = torch.tensor(qd, dtype=torch.float32)
    return fk_state(oracle, model)


def _two_revolute_y(com_x=0.0, m=25.0):
    """Fixed-base double pendulum, both joints about world +Y, link length 1, unit inertia (reference :1156, :1821)."""
    b = ModelBuilder(gravity=-10.0)
    half, mhalf = _tf((0.5, 0.0, 0.0)), _tf((-0.5, 0.0, 0.0))
    b1 = b.add_link(mass=m, inertia=I3, com=(com_x, 0.0, 0.0))
    j1 = b.add_joint_revolute(-1, b1, axis=(0.0, 1.0, 0.0), child_xform=mhalf)
    b2 = b.add_link(mass=m, inertia=I3, com=(com_x, 0.0, 0.0))
    j2 = b.add_joint_revolute(b1, b2, axis=(0.0, 1.0, 0.0), parent_xform=half, child_xform=mhalf)
    b.add_articulation([j1, j2])
    return b.finalize("cpu")


@pytest.mark.parametrize("qd", [(1.5, 0.0), (1.5, 1.5)])
def test_coriolis_double_pendulum_closed_form(od, oracle_lib, qd):
    """c1 = -m L1 l2c sin q2 (2 qd1 qd2 + qd2^2), c2 = m L1 l2c sin q2 qd1^2 at q = (0, pi/2) (reference :1156)."""
    model = _two_revolute_y()
    _, _, c = od.eval_inverse_dynamics_passive(model, _set_state(oracle_lib, model, (0.0, np.pi / 2), qd), coriolis_force=True)
    p = 25.0 * 1.0 * 0.5
    np.testing.assert_allclose(c.numpy(), [-p * (2 * qd[0] * qd[1] + qd[1] ** 2), p * qd[0] ** 2], atol=1e-3, rtol=1e-5)


@pytest.mark.parametrize("com_x", [0.0, 0.1])
@pytest.mark.parametrize("q2", [0.0, np.pi / 2, np.pi])
def test_mass_matrix_planar_double_pendulum_closed_form(od, oracle_lib, com_x, q2):
    """M(q) of the planar double pendulum (reference :1821)."""
    model = _two_revolute_y(com_x)
    M, _, _ = od.eval_inverse_dynamics_passive(model, _set_state(oracle_lib, model, (0.7, q2), (0.0, 0.0)), mass_matrix=True)
    m, lc, c2 = 25.0, 0.5 + com_x, np.cos(q2)
    M11 = m * lc**2 + m * (1.0 + lc**2 + 2.0 * lc * c2) + 2.0
    M12 = m * (lc**2 + lc * c2) + 1.0
    M22 = m * lc**2 + 1.0
    np.testing.assert_allclose(M.numpy()[0], [[M11, M12], [M12, M22]], atol=1e-3, rtol=1e-5)


@pytest.mark.parametrize("inertia", [1e-6, 1.0, 100.0])
def test_coriolis_radial_slider_closed_form(od, oracle_lib, inertia):
    """c_theta = 2 m r omega v_r, c_r = -m r omega^2, whatever the link inertias (reference :1261)."""
    b = ModelBuilder(gravity=0.0)
    base = b.add_link(mass=1e-6, inertia=I3 * inertia)
    j0 = b.add_joint_revolute(-1, base, axis=(0.0, 0.0, 1.0))
    slider_body = b.add_link(mass=0.5, inertia=I3 * inertia)
    j1 = b.add_joint_prismatic(base, slider_body, axis=(1.0, 0.0, 0.0))
    b.add_articulation([j0, j1])
    model = b.finalize("cpu")
    omega, v_r, r = 2.0, 0.1, 1.0
    _, _, c = od.eval_inverse_dynamics_passive(model, _set_state(oracle_lib, model, (0.7, r), (omega, v_r)), coriolis_force=True)
    np.testing.assert_allclose(c.numpy(), [2 * 0.5 * r * omega * v_r, -0.5 * r * omega**2], atol=1e-4, rtol=1e-5)


@pytest.mark.parametrize("mass", [0.5, 50.0])
def test_coriolis_anisotropic_gimbal_closed_form(od, oracle_lib, mass):
    """c1 = (Ix - Iz) sin 2q2 qd1 qd2, c2 = -(Ix - Iz) sin 2q2 qd1^2 / 2, independent of mass (reference :1358)."""
    b = ModelBuilder(gravity=0.0)
    inner = b.add_link(mass=mass, inertia=I3)
    j0 = b.add_joint_revolute(-1, inner, axis=(0.0, 0.0, 1.0))
    outer = b.add_link(mass=mass, inertia=_inertia(2.0, 1.5, 1.0))
    j1 = b.add_joint_revolute(inner, outer, axis=(0.0, 1.0, 0.0))
    b.add_articulation([j0, j1])
    model = b.finalize("cpu")
    q2 = np.pi / 4
    _, _, c = od.eval_inverse_dynamics_passive(model, _set_state(oracle_lib, model, (0.0, q2), (1.0, 1.0)), coriolis_force=True)
    np.testing.assert_allclose(c.numpy(), [(2.0 - 1.0) * np.sin(2 * q2), -0.5 * (2.0 - 1.0) * np.sin(2 * q2)], atol=1e-4, rtol=1e-5)


@pytest.mark.parametrize("v_com", [(0.0, 0.0, 0.0), (0.1, -0.2, 0.05)])
def test_coriolis_floating_root_with_com_offset(od, oracle_lib, v_com):
    """Free body, COM offset (0.5, 0.2, -0.3), identity pose: linear bias 0, angular bias omega x (I omega) (reference :1453).
    Exercises the m (w x v) and m r x (w x v) corrections of the internal-to-public conversion."""
    b = ModelBuilder(gravity=0.0)
    body = b.add_link(mass=1.0, inertia=_inertia(2.0, 1.5, 1.0), com=(0.5, 0.2, -0.3))
    b.add_articulation([b.add_joint_free(body)])
    model = b.finalize("cpu")
    omega = np.array([0.3, -0.1, 0.2])
    state = _set_state(oracle_lib, model, (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0), (*v_com, *omega))
    _, _, c = od.eval_inverse_dynamics_passive(model, state, coriolis_force=True)
    np.testing.assert_allclose(c.numpy()[:3], 0.0, atol=1e-5, rtol=1e-5)
    np.testing.assert_allclose(c.numpy()[3:], np.cross(omega, np.diag([2.0, 1.5, 1.0]) @ omega), atol=1e-5, rtol=1e-5)


_QX = X.quat_from_axis_angle(np.array([1.0, 0.0, 0.0]), np.pi / 2)
_I_LOCAL = np.diag([0.3, 0.5, 0.4])
_QDD6 = np.array([0.5, -0.3, 0.7, 0.2, 0.4, -0.6])


def _world_wrench_of_qdd():
    R = X.quat_to_matrix(_QX)
    return np.concatenate([2.0 * (R @ _QDD6[:3]), R @ (_I_LOCAL @ _QDD6[3:])])


def _force_from_mass_matrix(od, model, state):
    M, _, _ = od.eval_inverse_dynamics_passive(model, state, mass_matrix=True)
    nd = model.joint_dof_count
    z = torch.zeros(nd)
    return od.eval_inverse_dynamics_force(model, state, mass_matrix=M, joint_qdd=torch.tensor(_QDD6, dtype=torch.float32), coriolis_force=z,
                                          gravity_force=z)


def test_force_free_root_rotated_parent(od, oracle_lib):
    """A free root under a parent frame turned 90 deg about x: tau = (m R a, R I alpha) in the world frame (reference :2568)."""
    b = ModelBuilder(gravity=0.0)
    link = b.add_link(mass=2.0, inertia=_I_LOCAL)
    j = b.add_joint_free(link, parent_xform=list(X.transform(np.zeros(3), _QX)))
    b.add_articulation([j])
    b.joint_q[b.joint_q_start[j] : b.joint_q_start[j] + 7] = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]
    model = b.finalize("cpu")
    tau = _force_from_mass_matrix(od, model, fk_state(oracle_lib, model, torch.zeros(6)))
    np.testing.assert_allclose(tau.numpy(), _world_wrench_of_qdd(), atol=1e-5, rtol=1e-5)


@pytest.mark.parametrize("kind", ["free", "distance"])
def test_force_non_root_free_joint_rotated_parent(od, oracle_lib, kind):
    """The same wrench for a FREE / DISTANCE joint below a FIXED root (reference :2625)."""
    b = ModelBuilder(gravity=0.0)
    body1 = b.add_link(mass=1.0, inertia=I3)
    body2 = b.add_link(mass=2.0, inertia=_I_LOCAL)
    j0 = b.add_joint_fixed(-1, body1)
    px = list(X.transform(np.zeros(3), _QX))
    if kind == "free":
        j1 = b.add_joint_free(body2, parent=body1, parent_xform=px)
    else:
        j1 = b.add_joint_distance(body1, body2, parent_xform=px, max_distance=-1.0)
    b.add_articulation([j0, j1])
    b.joint_q[b.joint_q_start[j1] : b.joint_q_start[j1] + 7] = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]
    model = b.finalize("cpu")
    tau = _force_from_mass_matrix(od, model, fk_state(oracle_lib, model, torch.zeros(6)))
    np.testing.assert_allclose(tau.numpy(), _world_wrench_of_qdd(), atol=1e-5, rtol=1e-5)


# ---- manipulator-equation round trip (reference :2136-2564, Featherstone column) ----------------------------------------------
ROOT_TYPES = ["fixed", "free", "ball", "d6_revolute", "d6_2lin", "d6_1lin_1ang", "d6_2ang", "d6_ball"]
MASSES = [16.0, 32.0, 8.0, 24.0, 18.0, 12.0, 30.0, 6.0, 20.0, 28.0, 14.0, 22.0, 10.0, 26.0, 34.0, 4.0]
ROUND_TRIP_CASES = [((0.0, 0.0), (0.02, 0.04)), ((0.3, 0.5), (0.5, -0.3)), ((np.pi / 4, -np.pi / 3), (1.0, 1.0)),
                    ((np.pi / 2, np.pi / 2), (-0.7, 0.2))]


def three_link_chains(gravity_on: bool):
    """2 worlds x 8 three-link chains (root of every type in ROOT_TYPES, then a revolute and a prismatic joint), 4 x 2 x 2
    boxes of varying mass, COM offset (0.5, 0.2, -0.3) on every link, joint frames turned 30 deg about y."""
    from newton_b200.sim.builder import JointDofConfig as D

    ax = {"x": (1.0, 0.0, 0.0), "y": (0.0, 1.0, 0.0), "z": (0.0, 0.0, 1.0)}
    jrot = X.quat_from_axis_angle(np.array([0.0, 1.0, 0.0]), np.pi / 6)
    pos_two, neg_two = list(X.transform(np.array([2.0, 0.0, 0.0]), jrot)), list(X.transform(np.array([-2.0, 0.0, 0.0]), jrot))
    root_px = _tf((0.7, -0.4, 0.3))
    d6 = {"d6_revolute": ([], ["z"]), "d6_2lin": (["x", "y"], []), "d6_1lin_1ang": (["x"], ["z"]), "d6_2ang": ([], ["x", "z"]),
          "d6_ball": ([], ["x", "y", "z"])}
    builder = ModelBuilder(gravity=-10.0 if gravity_on else 0.0)
    k = 0
    for _ in range(2):
        builder.begin_world()
        for root in ROOT_TYPES:
            m = MASSES[k]
            k += 1
            inertia = np.diag([m * 8.0 / 12.0, m * 20.0 / 12.0, m * 20.0 / 12.0])
            com = (0.5, 0.2, -0.3)
            l0 = builder.add_link(mass=m, inertia=inertia, com=com)
            if root == "free":
                j0 = builder.add_joint_free(l0, parent_xform=root_px)
            elif root == "ball":
                j0 = builder.add_joint_ball(-1, l0, parent_xform=root_px)
            elif root == "fixed":
                j0 = builder.add_joint_fixed(-1, l0, parent_xform=root_px)
            else:
                lin, ang = d6[root]
                j0 = builder.add_joint_d6(-1, l0, parent_xform=root_px, linear_axes=[D(axis=ax[a]) for a in lin],
                                          angular_axes=[D(axis=ax[a]) for a in ang])
            l1 = builder.add_link(mass=m, inertia=inertia, com=com)
            j1 = builder.add_joint_revolute(l0, l1, axis=(0.0, 0.0, 1.0), parent_xform=pos_two, child_xform=neg_two)
            l2 = builder.add_link(mass=m, inertia=inertia, com=com)
            j2 = builder.add_joint_prismatic(l1, l2, axis=(1.0, 0.0, 0.0), parent_xform=pos_two, child_xform=neg_two)
            builder.add_articulation([j0, j1, j2])
        builder.end_world()
    return builder.finalize("cpu")


def round_trip_vectors(case, velocity_on):
    """joint_q / joint_qd / commanded joint_qdd of three_link_chains for one case (the reference's per-type root state)."""
    (q_int, qdd_int) = ROUND_TRIP_CASES[case]
    qd_int = (0.5, -0.3) if velocity_on else (0.0, 0.0)
    w = (0.3, -0.1, 0.2) if velocity_on else (0.0, 0.0, 0.0)
    al, lin = (0.2, -0.25, 0.3), (0.05, -0.1, 0.15)
    root_q = {"fixed": (), "ball": (0.0, 0.0, 0.0, 1.0), "d6_revolute": (0.0,), "d6_2lin": (0.0, 0.0), "d6_1lin_1ang": (0.0, 0.0),
              "d6_2ang": (0.0, 0.0), "d6_ball": (0.0, 0.0, 0.0), "free": (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)}
    root_qd = {"fixed": (), "ball": w, "d6_revolute": (w[2],), "d6_2lin": (0.0, 0.0), "d6_1lin_1ang": (0.0, w[2]), "d6_2ang": (w[0], w[2]),
               "d6_ball": w, "free": (0.0, 0.0, 0.0, *w)}
    root_qdd = {"fixed": (), "ball": al, "d6_revolute": (al[2],), "d6_2lin": lin[:2], "d6_1lin_1ang": (lin[0], al[2]),
                "d6_2ang": (al[0], al[2]), "d6_ball": al, "free": (*lin, *al)}
    q, qd, qdd = [], [], []
    for root in ROOT_TYPES * 2:
        q += [*root_q[root], *q_int]
        qd += [*root_qd[root], *qd_int]
        qdd += [*root_qdd[root], *qdd_int]
    return (np.asarray(v, dtype=np.float32) for v in (q, qd, qdd))


@pytest.mark.parametrize("gravity_on", [False, True])
@pytest.mark.parametrize("velocity_on", [False, True])
def test_manipulator_equation_round_trip(od, oracle_lib, gravity_on, velocity_on):
    """tau = M qdd + C qd + g, fed to SolverFeatherstone for one 1e-4 s step, gives back the commanded qdd to atol = rtol = 1e-3."""
    model = three_link_chains(gravity_on)
    solver = oracle_lib.SolverFeatherstone(model)
    for case in range(len(ROUND_TRIP_CASES)):
        q, qd, qdd = round_trip_vectors(case, velocity_on)
        state = _set_state(oracle_lib, model, q, qd)
        M, g, c = od.eval_inverse_dynamics_passive(model, state, mass_matrix=True, gravity_force=True, coriolis_force=True)
        tau = od.eval_inverse_dynamics_force(model, state, mass_matrix=M, joint_qdd=torch.tensor(qdd), coriolis_force=c, gravity_force=g)
        control = model.control()
        control.joint_f = tau.clone()
        out = model.state()
        solver.step(state, out, control, None, 1e-4)
        np.testing.assert_allclose((out.joint_qd.numpy() - qd) / 1e-4, qdd, atol=1e-3, rtol=1e-3, err_msg=f"case {case}")


def test_free_joint_below_the_root_is_a_body_wrench_in_the_solver(od, oracle_lib):
    """Why the round trip is run on floating ROOTS only: SolverFeatherstone (like upstream's
    accumulate_free_distance_joint_f_to_body_force, featherstone/kernels.py:894-921) applies a FREE joint's joint_f to the child
    body alone, with no reaction on the parent.  For a FREE joint below a moving parent that wrench also loads the parent's dofs,
    so tau from inverse dynamics does not reproduce qdd there.  Removing that load from the parent's entries - the wrench's
    generalized force through the child's Jacobian rows - makes the step return the commanded qdd."""
    b = ModelBuilder(gravity=0.0)
    SCENES["free_descendant"](b)
    model = b.finalize("cpu")
    randomize(model, 12, 0.3)
    model.joint_qd.zero_()
    state = fk_state(oracle_lib, model)
    qdd = torch.tensor(np.random.default_rng(21).normal(0.0, 1.0, model.joint_dof_count), dtype=torch.float32)
    M, g, c = od.eval_inverse_dynamics_passive(model, state, mass_matrix=True, gravity_force=True, coriolis_force=True)
    tau = od.eval_inverse_dynamics_force(model, state, mass_matrix=M, joint_qdd=qdd, coriolis_force=c, gravity_force=g).numpy()

    def step(joint_f):
        control = model.control()
        control.joint_f = torch.tensor(joint_f, dtype=torch.float32)
        out = model.state()
        oracle_lib.SolverFeatherstone(model).step(state, out, control, None, 1e-4)
        return out.joint_qd.numpy() / 1e-4

    assert np.abs(step(tau) - qdd.numpy()).max() > 0.1  # the parent dof is pushed by the unreacted wrench
    J = od.eval_jacobian(model, state).numpy()[0].astype(np.float64)
    compensated = tau.astype(np.float64)
    compensated[0] -= J[6:12, 0] @ tau[1:7]  # link 1 (the free joint's child), parent column
    np.testing.assert_allclose(step(compensated), qdd.numpy(), atol=1e-3, rtol=1e-3)


# ---- host-side API of the product functions (argument checks run before the CUDA-only check) --------------------------------------
@pytest.fixture(scope="module")
def small():
    return build("double_pendulum", worlds=2, seed=1)


def test_shape_errors(small):
    st = small.state()
    D, nd = small.max_dofs_per_articulation, small.joint_dof_count
    with pytest.raises(ValueError, match="mass_matrix has shape"):
        newton_b200.eval_inverse_dynamics_passive(small, st, mass_matrix=torch.zeros(2, D + 1, D))
    with pytest.raises(ValueError, match="gravity_force has shape"):
        newton_b200.eval_inverse_dynamics_passive(small, st, gravity_force=torch.zeros(nd + 1))
    with pytest.raises(ValueError, match="mask has shape"):
        newton_b200.eval_inverse_dynamics_passive(small, st, coriolis_force=torch.zeros(nd), mask=torch.ones(3, dtype=torch.bool))
    ok = dict(mass_matrix=torch.zeros(2, D, D), joint_qdd=torch.zeros(nd), coriolis_force=torch.zeros(nd), gravity_force=torch.zeros(nd),
              joint_f=torch.zeros(nd))
    for name in ("joint_qdd", "coriolis_force", "gravity_force", "joint_f"):
        bad = dict(ok, **{name: torch.zeros(nd + 2)})
        with pytest.raises(ValueError, match=f"{name} has shape"):
            newton_b200.eval_inverse_dynamics_force(small, st, **bad)
    with pytest.raises(ValueError, match="mass_matrix has shape"):
        newton_b200.eval_inverse_dynamics_force(small, st, **dict(ok, mass_matrix=torch.zeros(1, D, D)))
    with pytest.raises(ValueError, match="J has shape"):
        newton_b200.eval_jacobian(small, st, J=torch.zeros(2, 6, D))
    with pytest.raises(ValueError, match="H has shape"):
        newton_b200.eval_mass_matrix(small, st, H=torch.zeros(2, D, D + 1))


def test_no_outputs_requested_raises(small):
    with pytest.raises(ValueError, match="At least one inverse-dynamics output"):
        newton_b200.eval_inverse_dynamics_passive(small, small.state())


def test_arrays_are_keyword_only(small):
    st, nd, D = small.state(), small.joint_dof_count, small.max_dofs_per_articulation
    with pytest.raises(TypeError):
        newton_b200.eval_inverse_dynamics_passive(small, st, torch.zeros(2, D, D))  # noqa
    with pytest.raises(TypeError):
        newton_b200.eval_inverse_dynamics_force(small, st, torch.zeros(2, D, D), torch.zeros(nd), torch.zeros(nd), torch.zeros(nd),
                                                torch.zeros(nd))


def test_rod_joint_refused(small):
    small._nb2_has_rod = None
    types = small.joint_type.clone()
    small.joint_type[1] = int(JointType.ROD)
    try:
        with pytest.raises(ValueError, match="does not support JointType.ROD"):
            newton_b200.eval_inverse_dynamics_passive(small, small.state(), gravity_force=torch.zeros(small.joint_dof_count))
        small._nb2_has_rod = None
        with pytest.raises(ValueError, match="does not support JointType.ROD"):
            nd = small.joint_dof_count
            newton_b200.eval_inverse_dynamics_force(small, small.state(), mass_matrix=None, joint_qdd=torch.zeros(nd),
                                                    coriolis_force=torch.zeros(nd), gravity_force=torch.zeros(nd), joint_f=torch.zeros(nd))
    finally:
        small.joint_type = types
        small._nb2_has_rod = None


def test_zero_articulations():
    b = ModelBuilder()
    b.add_link(mass=1.0, inertia=I3)
    model = b.finalize("cpu")
    assert model.articulation_count == 0
    st = model.state()
    assert newton_b200.eval_jacobian(model, st) is None
    assert newton_b200.eval_mass_matrix(model, st) is None
    jf = torch.full((model.joint_dof_count,), 7.0)
    newton_b200.eval_inverse_dynamics_force(model, st, mass_matrix=torch.zeros(0, 0, 0), joint_qdd=jf, coriolis_force=jf,
                                            gravity_force=jf, joint_f=jf)
    assert (jf == 7.0).all()
    newton_b200.eval_inverse_dynamics_passive(model, st, gravity_force=torch.zeros(model.joint_dof_count))


def test_cpu_model_has_no_cpu_path(small):
    from newton_b200 import _lib

    with pytest.raises(_lib.Nb2Error, match="CUDA devices only"):
        newton_b200.eval_jacobian(small, small.state())

"""newton_b200.controllers on the CPU oracle path (oracle/controller.py runs the product's host code with only the launch
replaced): the behaviours the reference's joint-impedance tests check, restated as known answers; closed forms of the
model-based terms for a one-link pendulum and a two-link planar arm; and every refusal of the constructors and of step()."""

import math
import os
import re

import numpy as np
import pytest
import torch

import oracle.controller as oc
from newton_b200 import ModelBuilder, scenes
from newton_b200.controllers import ControllerBase, ControllerJointImpedance, ControllerJointImpedanceModelFree

G = 9.81
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_descriptor_matches_header_field_order():
    from newton_b200 import _abi, _lib

    header = open(os.path.join(ROOT, "include", "newton_b200.h")).read()
    body = header.split("typedef struct nb2_joint_impedance_desc {")[1].split("} nb2_joint_impedance_desc;")[0]
    body = re.sub(r"/[*].*?[*]/", "", body, flags=re.S)
    assert re.findall(r"\b([A-Za-z_0-9]+)\s*;", body) == [n for n, _ in _abi.JointImpedanceDesc._fields_]
    assert "nb2_joint_impedance_step" in _lib.EXPORTED_SYMBOLS


def u32(values):
    return torch.tensor(values, dtype=torch.int64).to(torch.uint32)


def mf(dofs=(2,), max_dofs=None, kp=None, kd=None, grav=False, cor=False, inertia=False, qdd=False, **kw):
    dofs = list(dofs)
    R, D = len(dofs), max_dofs or max(dofs)
    gain = lambda v: None if v is None else torch.full((R, D), float(v))  # noqa: E731
    return ControllerJointImpedanceModelFree(
        robot_count=R, dofs_per_robot=torch.tensor(dofs, dtype=torch.int32), max_dofs=D,
        default_dof_indices=kw.pop("default", u32(range(sum(dofs)))), stiffness=gain(kp), damping=gain(kd),
        use_gravity_compensation=grav, use_coriolis_compensation=cor, use_inertia_decoupling=inertia, has_qdd_feedforward=qdd,
        device="cpu", **kw)


def run(ctrl, **fields):
    inp, out = ctrl.input(), ctrl.output()
    for k, v in fields.items():
        getattr(inp, k)[...] = torch.as_tensor(v, dtype=torch.float32)
    oc.step(ctrl, inputs=inp, outputs=out, dt=0.01)
    return out.joint_f


def test_base_class_and_graphable():
    c = mf(kp=1, kd=1)
    assert isinstance(c, ControllerBase) and c.is_graphable()
    assert c.robot_count == 1 and c.max_dofs == 2 and not c.requires_grad


def test_zero_error_gives_zero_torque():
    f = run(mf(kp=100, kd=10), joint_q=[0.3, -0.2], joint_q_des=[0.3, -0.2], joint_qd=[1.0, 2.0], joint_qd_des=[1.0, 2.0])
    assert f.tolist() == [0.0, 0.0]


def test_pure_stiffness_and_pure_damping():
    assert run(mf(kp=10, kd=0), joint_q=[0.5, 0.0], joint_q_des=[1.0, -0.25]).tolist() == [5.0, -2.5]
    assert run(mf(kp=0, kd=4), joint_qd=[1.0, 0.5], joint_qd_des=[0.0, 1.0]).tolist() == [-4.0, 2.0]


def test_robots_are_independent():
    c = mf(dofs=(1, 1), kp=2, kd=0)
    a = run(c, joint_q_des=[1.0, 1.0])
    b = run(c, joint_q_des=[1.0, 7.0])
    assert a[0] == b[0] == 2.0 and b[1] == 14.0


def test_inertia_decoupling_scales_by_m():
    c = mf(kp=1, kd=0, inertia=True)
    f = run(c, joint_q_des=[1.0, 2.0], mass_matrix=[[[2.0, 0.5], [0.5, 3.0]]])
    assert f.tolist() == [2.0 * 1 + 0.5 * 2, 0.5 * 1 + 3.0 * 2]


def test_gravity_and_coriolis_are_added():
    c = mf(kp=1, kd=0, grav=True, cor=True)
    f = run(c, joint_q_des=[1.0, 0.0], gravity_force=[0.5, 0.25], coriolis_force=[0.125, 4.0])
    assert f.tolist() == [1.625, 4.25]


def test_qdd_feedforward_is_added_before_the_m_product():
    c = mf(kp=1, kd=0, inertia=True, qdd=True)
    f = run(c, joint_q_des=[1.0, 0.0], joint_qdd=[1.0, 1.0], mass_matrix=[[[2.0, 0.0], [0.0, 3.0]]])
    assert f.tolist() == [4.0, 3.0]


def test_live_gain_ports():
    c = mf(kp=None, kd=None)
    inp = c.input()
    assert inp.stiffness.shape == (1, 2) and inp.damping.shape == (1, 2)
    f = run(c, joint_q_des=[1.0, 1.0], joint_qd_des=[1.0, 0.0], stiffness=[[3.0, 5.0]], damping=[[7.0, 11.0]])
    assert f.tolist() == [10.0, 5.0]


def test_partial_and_permuted_indices():
    # 2 robots x 2 dofs in a sim of 6 dofs; the position port reads a permuted layout, the output skips slots 0 and 3
    c = mf(dofs=(2, 2), kp=1, kd=0, default=u32([1, 2, 4, 5]), joint_q_des_idx=u32([5, 4, 2, 1]))
    inp, out = c.input(), c.output()
    assert inp.joint_q.numel() == 6 and out.joint_f.numel() == 6
    inp.joint_q_des[:] = torch.tensor([0.0, 10.0, 20.0, 30.0, 40.0, 50.0])
    out.joint_f[:] = -7.0
    oc.step(c, inputs=inp, outputs=out, dt=0.0)
    assert out.joint_f.tolist() == [-7.0, 50.0, 40.0, -7.0, 20.0, 10.0]


def test_heterogeneous_fleet_padding_is_never_scattered():
    c = mf(dofs=(1, 3), max_dofs=3, kp=2, kd=0, inertia=True, grav=True, default=u32([0, 2, 3, 4]))
    inp, out = c.input(), c.output()
    inp.joint_q_des[:] = 1.0
    inp.gravity_force[:] = torch.arange(5, dtype=torch.float32)
    inp.mass_matrix[:] = torch.eye(3) * 2.0
    inp.mass_matrix[0, 0, 1:] = 99.0  # padding columns of robot 0: never read
    out.joint_f[:] = -1.0
    oc.step(c, inputs=inp, outputs=out, dt=0.0)
    assert out.joint_f.tolist() == [4.0, -1.0, 6.0, 7.0, 8.0]
    # independence across a heterogeneous fleet
    inp.joint_q_des[0] = 3.0
    oc.step(c, inputs=inp, outputs=out, dt=0.0)
    assert out.joint_f.tolist() == [12.0, -1.0, 6.0, 7.0, 8.0]


def test_inputs_outputs_fields_and_sizes():
    c = mf(dofs=(2, 1), kp=1, kd=None, default=u32([0, 5, 3]), joint_f_idx=u32([1, 2, 9]), inertia=True)
    inp, out = c.input(), c.output()
    assert set(vars(inp)) == {"joint_q", "joint_qd", "joint_q_des", "joint_qd_des", "joint_qdd", "gravity_force", "coriolis_force",
                              "mass_matrix", "stiffness", "damping"}
    assert inp.joint_q.shape == (6,) and inp.joint_qdd is None and inp.gravity_force is None and inp.coriolis_force is None
    assert inp.mass_matrix.shape == (2, 2, 2) and inp.stiffness is None and inp.damping.shape == (2, 2)
    assert out.joint_f.shape == (10,) and out.joint_f.dtype == torch.float32
    mb = ControllerJointImpedance(scenes.pendulum_link_builder(), default_dof_indices=u32([0]), stiffness=None, damping=None,
                                  has_qdd_feedforward=True, device="cpu")
    inp = mb.input()
    assert set(vars(inp)) == {"joint_q", "joint_qd", "joint_q_des", "joint_qd_des", "joint_qdd", "stiffness", "damping"}
    assert inp.joint_qdd.shape == (1,) and mb.output().joint_f.shape == (1,)


# ---- model-based closed forms ---------------------------------------------------------------------------------------------
def model_based(builder, n, **kw):
    return ControllerJointImpedance(builder, default_dof_indices=torch.arange(n, dtype=torch.int32),
                                    stiffness=torch.zeros(builder.articulation_count, n), damping=torch.zeros(builder.articulation_count, n),
                                    device="cpu", **kw)


def terms(builder, n, q, qd):
    """(M acc with acc = e_k columns, g, C qd) of the model-based controller at (q, qd), each isolated by its flags."""
    g = run(model_based(builder, n, use_coriolis_compensation=False, use_inertia_decoupling=False), joint_q=q, joint_qd=qd)
    c = run(model_based(builder, n, use_gravity_compensation=False, use_inertia_decoupling=False), joint_q=q, joint_qd=qd)
    ctrl = model_based(builder, n, use_gravity_compensation=False, use_coriolis_compensation=False, has_qdd_feedforward=True)
    M = np.stack([run(ctrl, joint_q=q, joint_qd=qd, joint_qdd=np.eye(n)[k]).numpy() for k in range(n)], axis=1)
    return M, g.numpy(), c.numpy()


@pytest.mark.parametrize("q", [0.0, 0.4, -1.1, 2.5])
def test_pendulum_closed_form(q):
    m, l, inertia = 1.5, 0.4, 0.02
    M, g, c = terms(scenes.pendulum_link_builder(m, l, inertia), 1, [q], [0.7])
    np.testing.assert_allclose(g, [m * G * l * math.sin(q)], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(M, [[inertia + m * l * l]], rtol=1e-5)
    np.testing.assert_allclose(c, [0.0], atol=1e-6)


def two_link_builder(m1, m2, l1, lc1, lc2, i1, i2):
    """Planar arm in the x-z plane, joints about -y (q counter-clockwise from +x towards +z, gravity -z)."""
    b = ModelBuilder()
    a = b.add_link(mass=m1, com=(lc1, 0.0, 0.0), inertia=np.eye(3) * i1)
    c = b.add_link(mass=m2, com=(lc2, 0.0, 0.0), inertia=np.eye(3) * i2)
    b.add_joint_revolute(-1, a, axis=(0.0, -1.0, 0.0))
    b.add_joint_revolute(a, c, parent_xform=np.array([l1, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]), axis=(0.0, -1.0, 0.0))
    b.add_articulation([0, 1])
    return b


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_two_link_planar_arm_closed_form(seed):
    m1, m2, l1, lc1, lc2, i1, i2 = 1.2, 0.8, 0.6, 0.3, 0.25, 0.03, 0.02
    rng = np.random.default_rng(seed)
    q, qd = rng.uniform(-2, 2, 2), rng.uniform(-3, 3, 2)
    M, g, c = terms(two_link_builder(m1, m2, l1, lc1, lc2, i1, i2), 2, q, qd)
    c2, s2 = math.cos(q[1]), math.sin(q[1])
    M_ref = np.array([[m1 * lc1**2 + m2 * (l1**2 + lc2**2 + 2 * l1 * lc2 * c2) + i1 + i2, m2 * (lc2**2 + l1 * lc2 * c2) + i2],
                      [m2 * (lc2**2 + l1 * lc2 * c2) + i2, m2 * lc2**2 + i2]])
    h = m2 * l1 * lc2 * s2
    c_ref = [-h * (2 * qd[0] * qd[1] + qd[1] ** 2), h * qd[0] ** 2]
    c12 = math.cos(q[0] + q[1])
    g_ref = [(m1 * lc1 + m2 * l1) * G * math.cos(q[0]) + m2 * lc2 * G * c12, m2 * lc2 * G * c12]
    np.testing.assert_allclose(M, M_ref, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(g, g_ref, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(c, c_ref, rtol=2e-5, atol=2e-5)


def test_model_based_heterogeneous_fleet_matches_the_model_free_law_on_oracle_terms():
    """The model-based step equals the model-free step fed the oracle's own M, g and C qd of each robot (panda, ant, pendulum)."""
    import oracle
    import oracle.dynamics as dyn

    b = scenes.impedance_fleet_builder(3, ("panda", "ant", "pendulum"))
    n = b.joint_dof_count
    rng = np.random.default_rng(3)
    D = 9
    kp, kd = torch.rand(3, D, generator=torch.Generator().manual_seed(0)) * 50, torch.full((3, D), 2.0)
    ctrl = ControllerJointImpedance(b, default_dof_indices=torch.arange(n), stiffness=kp, damping=kd, device="cpu")
    q, qd, qdes = (torch.tensor(rng.uniform(-1, 1, n), dtype=torch.float32) for _ in range(3))
    f = run(ctrl, joint_q=q, joint_qd=qd, joint_q_des=qdes)
    model = b.finalize()
    st = model.state()
    st.joint_q[:], st.joint_qd[:] = q, qd
    oracle.eval_fk(model, st.joint_q, st.joint_qd, st)
    M = dyn.eval_mass_matrix(model, st)
    _, g, c = dyn.eval_inverse_dynamics_passive(model, st, gravity_force=True, coriolis_force=True)
    free = mf(dofs=(9, 8, 1), kp=None, kd=None, grav=True, cor=True, inertia=True)
    f2 = run(free, joint_q=q, joint_qd=qd, joint_q_des=qdes, gravity_force=g, coriolis_force=c, mass_matrix=M, stiffness=kp, damping=kd)
    assert torch.equal(f, f2)
    assert torch.equal(ctrl._state.joint_q, q) and torch.equal(ctrl._state.body_q, st.body_q)


# ---- refusals -------------------------------------------------------------------------------------------------------------
def test_model_free_constructor_refusals():
    with pytest.raises(ValueError, match="robot_count"):
        mf(dofs=(), max_dofs=1, kp=1, kd=1)
    with pytest.raises(TypeError):
        mf(kp=1, kd=1, default=torch.arange(2, dtype=torch.float32))
    with pytest.raises(TypeError):
        mf(kp=1, kd=1, joint_q_idx=[0, 1])
    with pytest.raises(ValueError, match="same size"):
        mf(kp=1, kd=1, joint_qd_idx=u32([0]))
    with pytest.raises(ValueError, match="must equal sum"):
        mf(kp=1, kd=1, default=u32([0, 1, 2]))
    with pytest.raises(ValueError, match="unique"):
        mf(dofs=(1, 1), kp=1, kd=1, joint_f_idx=u32([3, 3]))
    with pytest.raises(ValueError, match="baked array shape"):
        ControllerJointImpedanceModelFree(robot_count=1, dofs_per_robot=torch.tensor([2], dtype=torch.int32), max_dofs=2,
                                          default_dof_indices=u32([0, 1]), stiffness=torch.zeros(2, 1), damping=None, device="cpu")
    with pytest.raises(NotImplementedError):
        mf(kp=1, kd=1, requires_grad=True)


def test_model_based_constructor_refusals():
    with pytest.raises(TypeError):
        ControllerJointImpedance(object(), default_dof_indices=u32([0]), stiffness=None, damping=None, device="cpu")
    with pytest.raises(TypeError):
        ControllerJointImpedance(scenes.pendulum_link_builder(), default_dof_indices=[0], stiffness=None, damping=None, device="cpu")
    with pytest.raises(ValueError, match="no articulations"):
        ControllerJointImpedance(ModelBuilder(), default_dof_indices=u32([]), stiffness=None, damping=None, device="cpu")
    with pytest.raises(ValueError, match="only supports 1-DOF joints"):
        ControllerJointImpedance(scenes.ant_builder(floating=True), default_dof_indices=u32(range(14)), stiffness=None, damping=None,
                                 device="cpu")
    with pytest.raises(ValueError, match="must equal"):
        ControllerJointImpedance(scenes.panda_arm_builder(), default_dof_indices=u32(range(8)), stiffness=None, damping=None, device="cpu")
    loose = scenes.pendulum_link_builder()
    extra = loose.add_link(mass=1.0, inertia=np.eye(3))
    loose.add_joint_revolute(0, extra, axis=(0.0, 1.0, 0.0))  # outside every articulation
    with pytest.raises(ValueError, match="cover every joint"):
        ControllerJointImpedance(loose, default_dof_indices=u32([0, 1]), stiffness=None, damping=None, device="cpu")
    with pytest.raises(NotImplementedError):
        ControllerJointImpedance(scenes.pendulum_link_builder(), default_dof_indices=u32([0]), stiffness=None, damping=None, device="cpu",
                                 requires_grad=True)


def test_step_refusals_happen_before_any_launch(monkeypatch):
    from newton_b200.controllers import joint_impedance as J

    launched = []
    monkeypatch.setattr(J, "_launch", lambda c, d: launched.append(d))
    c = mf(dofs=(2,), kp=None, kd=1, default=u32([0, 3]), grav=True, inertia=True)
    inp, out = c.input(), c.output()
    c.step(inputs=inp, outputs=out, dt=0.0)
    assert len(launched) == 1
    bad = [("joint_q", torch.zeros(3)),                         # too short for its index map (largest index 3)
           ("joint_qd", torch.zeros(4, dtype=torch.float64)),    # wrong dtype
           ("joint_q_des", torch.zeros(8)[::2]),                 # not contiguous
           ("gravity_force", None),                              # enabled term missing
           ("mass_matrix", torch.zeros(1, 2, 3)),                # wrong shape
           ("stiffness", torch.zeros(2, 2))]                     # wrong live gain shape
    for name, value in bad:
        inp2 = c.input()
        setattr(inp2, name, value)
        with pytest.raises((ValueError, TypeError)):
            c.step(inputs=inp2, outputs=out, dt=0.0)
    out2 = c.output()
    out2.joint_f = torch.zeros(3)
    with pytest.raises(ValueError):
        c.step(inputs=inp, outputs=out2, dt=0.0)
    with pytest.raises(ValueError, match="share storage"):
        c.step(inputs=inp, outputs=_out(inp.joint_q), dt=0.0)
    assert len(launched) == 1
    # an input rebound to a tensor too short for its index map, after a cached step
    inp.joint_qd = torch.zeros(2)
    with pytest.raises(ValueError, match="needs at least 4"):
        c.step(inputs=inp, outputs=out, dt=0.0)
    assert len(launched) == 1


def _out(t):
    o = ControllerJointImpedanceModelFree.Outputs()
    o.joint_f = t
    return o


def test_cpu_device_has_no_product_path():
    from newton_b200 import _lib

    c = mf(kp=1, kd=1)
    with pytest.raises(_lib.Nb2Error):
        c.step(inputs=c.input(), outputs=c.output(), dt=0.0)

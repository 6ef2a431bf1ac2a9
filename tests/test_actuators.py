"""Actuators: the host-side construction of newton_b200.actuators (validation, grouping, descriptors, duplicate tables, view
mappings, Model.to / shard) and the CPU oracle of their step (oracle/oracle_actuator.h), pinned by the reference's known
answers (newton/tests/test_actuators.py) restated here.  The same cases run on the GPU against the oracle in
tests/test_gpu_actuators.py."""

import math
import types

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import JointType, ModelBuilder
from newton_b200.actuators import (
    Actuator,
    ClampingDCMotor,
    ClampingMaxEffort,
    ClampingPositionBased,
    ControllerPD,
    ControllerPID,
    Delay,
)


@pytest.fixture(scope="module")
def oact():
    import oracle
    import oracle.actuator as oact

    oracle.build()
    return oact


def f32(v, device="cpu"):
    return torch.tensor(v, dtype=torch.float32, device=device)


def i32(v, device="cpu"):
    return torch.tensor(v, dtype=torch.int32, device=device)


def io(n_q, n_qd, device="cpu", **kw):
    """A state / control pair of plain tensors (``kw`` overrides entries)."""
    st = types.SimpleNamespace(joint_q=torch.zeros(n_q, device=device), joint_qd=torch.zeros(n_qd, device=device))
    ctl = types.SimpleNamespace(joint_target_q=torch.zeros(n_q, device=device), joint_target_qd=torch.zeros(n_qd, device=device),
                                joint_act=torch.zeros(n_qd, device=device), joint_f=torch.zeros(n_qd, device=device))
    for k, v in kw.items():
        setattr(st if k in ("joint_q", "joint_qd") else ctl, k, v)
    return st, ctl


# ---------------------------------------------------------------------------------------------------- controllers
def test_pd_compute(oact):
    kp, kd = [100.0, 200.0, 50.0], [10.0, 20.0, 5.0]
    q, qd, tq, tqd = [0.1, -0.2, 0.3], [1.0, -1.0, 0.5], [0.5, 0.1, -0.3], [0.0, 0.5, 1.0]
    ce, ff = [1.0, -2.0, 0.5], [3.0, 0.0, -1.0]
    a = Actuator(i32([0, 1, 2]), ControllerPD(f32(kp), f32(kd), const_effort=f32(ce)))
    st, ctl = io(3, 3, joint_q=f32(q), joint_qd=f32(qd), joint_target_q=f32(tq), joint_target_qd=f32(tqd), joint_act=f32(ff))
    oact.step(a, st, ctl)
    for i in range(3):
        expect = ce[i] + ff[i] + kp[i] * (tq[i] - q[i]) + kd[i] * (tqd[i] - qd[i])
        assert ctl.joint_f[i].item() == pytest.approx(expect, rel=1e-5)
    # ((const + ff) + kp pe) + kd ve, rounded to float32 after every operation
    f = np.float32
    pe, ve = f(tq[0]) - f(q[0]), f(tqd[0]) - f(qd[0])
    assert ctl.joint_f[0].item() == float(((f(ce[0]) + f(ff[0])) + f(kp[0]) * pe) + f(kd[0]) * ve)


def test_pid_compute_integral_and_anti_windup(oact):
    kp, ki, kd, imax, dt = 10.0, 100.0, 1.0, 0.015, 0.01
    a = Actuator(i32([0]), ControllerPID(f32([kp]), f32([ki]), f32([kd]), f32([imax]), const_effort=f32([0.5])))
    st, ctl = io(1, 1, joint_target_q=f32([1.0]), joint_act=f32([0.25]))
    s0, s1 = a.state(), a.state()
    integral = 0.0
    for _ in range(4):
        ctl.joint_f.zero_()
        oact.step(a, st, ctl, s0, s1, dt)
        integral = min(max(integral + 1.0 * dt, -imax), imax)
        assert s1.controller_state.integral.item() == pytest.approx(integral, rel=1e-6)
        assert ctl.joint_f.item() == pytest.approx(0.5 + 0.25 + kp * 1.0 + ki * integral, rel=1e-5)
        s0, s1 = s1, s0
    assert s0.controller_state.integral.item() == pytest.approx(imax)  # saturated by the anti-windup clamp
    with pytest.raises(ValueError, match="dt"):
        oact.step(a, st, ctl, s0, s1, None)
    with pytest.raises(ValueError, match="different states"):
        oact.step(a, st, ctl, s0, s0, dt)


# ---------------------------------------------------------------------------------------------------- delay
def test_delay_buffer_shape():
    d = Delay(i32([3, 3]), max_delay=3)
    a = Actuator(i32([0, 1]), ControllerPD(f32([1.0, 1.0]), f32([0.0, 0.0])), delay=d)
    s = a.state().delay_state
    assert s.buffer_pos.shape == (3, 2) and s.buffer_vel.shape == (3, 2) and s.buffer_act.shape == (3, 2)
    assert s.num_pushes.tolist() == [0, 0] and s.write_idx.tolist() == [2]
    with pytest.raises(ValueError, match="max_delay"):
        Delay(i32([0]), max_delay=0)


def _delayed(history, k, delay):
    """The target a dof with ``delay`` sees at step ``k`` when ``history[j]`` was written at step j."""
    if k == 0 or delay == 0:
        return history[k]
    return history[k - 1 - min(delay - 1, k - 1)]


def test_delay_latency_and_mixed_zero_delays(oact):
    delays = [0, 1, 3]
    a = Actuator(i32([0, 1, 2]), ControllerPD(f32([1.0] * 3), f32([0.0] * 3)), delay=Delay(i32(delays), max_delay=3))
    st, ctl = io(3, 3)
    s0, s1 = a.state(), a.state()
    history = []
    for k in range(7):
        tgt = float(k + 1)
        history.append(tgt)
        ctl.joint_target_q.fill_(tgt)
        ctl.joint_f.zero_()
        oact.step(a, st, ctl, s0, s1, 0.01)
        s0, s1 = s1, s0
        assert ctl.joint_f.tolist() == [_delayed(history, k, d) for d in delays], k
        assert s0.delay_state.num_pushes.tolist() == [min(k + 1, 3)] * 3


# ---------------------------------------------------------------------------------------------------- clamping
def _clamped(oact, clamp, src, q=0.0, qd=0.0):
    """Step a one-actuator PD whose raw effort is ``src`` (const_effort) through ``clamp``."""
    a = Actuator(i32([0]), ControllerPD(f32([0.0]), f32([0.0]), const_effort=f32([src])), clamping=[clamp])
    st, ctl = io(1, 1, joint_q=f32([q]), joint_qd=f32([qd]))
    oact.step(a, st, ctl)
    return ctl.joint_f.item()


def test_clamping_max_effort(oact):
    for src in (100.0, -80.0, 30.0):
        assert _clamped(oact, ClampingMaxEffort(f32([50.0])), src) == max(min(src, 50.0), -50.0)


def test_clamping_dc_motor_quadrants(oact):
    sat, v_lim, max_f = 100.0, 10.0, 200.0
    for raw in (500.0, -500.0):
        for qd in (0.0, 5.0, 10.0, -5.0, -10.0, 25.0):
            corner = v_lim * (1.0 + max_f / sat)
            v = min(max(qd, -corner), corner)
            expect = max(min(raw, min(sat * (1.0 - v / v_lim), max_f)), max(sat * (-1.0 - v / v_lim), -max_f))
            got = _clamped(oact, ClampingDCMotor(f32([sat]), f32([v_lim]), f32([max_f])), raw, qd=qd)
            assert got == pytest.approx(expect, abs=1e-3), (raw, qd)


def test_clamping_dc_motor_infinite_and_zero_saturation(oact):
    inf = math.inf
    # all-infinite parameters pass the effort through (the corner velocity is NaN, Warp's min / max then ignore it)
    assert _clamped(oact, ClampingDCMotor(f32([inf]), f32([inf]), f32([inf])), 123.0, qd=3.0) == 123.0
    # sat = 0: the corner velocity is velocity_limit and the motor produces nothing
    assert _clamped(oact, ClampingDCMotor(f32([0.0]), f32([5.0]), f32([10.0])), 50.0, qd=1.0) == 0.0


def test_clamping_position_based(oact):
    clamp = lambda: ClampingPositionBased(lookup_positions=(-1.0, 0.0, 1.0), lookup_efforts=(10.0, 30.0, 50.0))  # noqa: E731
    for pos, limit in ((-1.0, 10.0), (0.0, 30.0), (1.0, 50.0), (-0.5, 20.0), (0.5, 40.0), (-3.0, 10.0), (7.0, 50.0)):
        assert _clamped(oact, clamp(), 999.0, q=pos) == pytest.approx(limit, abs=1e-5), pos
        assert _clamped(oact, clamp(), -999.0, q=pos) == pytest.approx(-limit, abs=1e-5), pos
    # at a repeated position the interval ending there wins (with sorted positions the interpolation reaches a zero-width
    # interval only past its end, so the dx == 0 branch is never taken)
    rep = ClampingPositionBased(lookup_positions=(0.0, 0.5, 0.5, 1.0), lookup_efforts=(10.0, 20.0, 40.0, 50.0))
    assert _clamped(oact, rep, 999.0, q=0.5) == 20.0


def test_clamping_position_based_file(oact, tmp_path):
    p = tmp_path / "table.txt"
    p.write_text("# position, effort\n-1.0, 10.0\n\n0.0 30.0\n  # comment\n1.0,50.0\n")
    assert _clamped(oact, ClampingPositionBased(lookup_table_path=str(p)), 999.0, q=0.5) == pytest.approx(40.0)
    bad = tmp_path / "bad.txt"
    bad.write_text("1.0 5.0\n0.0 5.0\n")
    with pytest.raises(ValueError, match="non-decreasing"):
        Actuator(i32([0]), ControllerPD(f32([0.0]), f32([0.0])), clamping=[ClampingPositionBased(lookup_table_path=str(bad))])
    neg = tmp_path / "neg.txt"
    neg.write_text("0.0 -1.0\n")
    with pytest.raises(ValueError, match="non-negative"):
        Actuator(i32([0]), ControllerPD(f32([0.0]), f32([0.0])), clamping=[ClampingPositionBased(lookup_table_path=str(neg))])
    empty = tmp_path / "empty.txt"
    empty.write_text("# nothing\n")
    with pytest.raises(ValueError, match="empty"):
        Actuator(i32([0]), ControllerPD(f32([0.0]), f32([0.0])), clamping=[ClampingPositionBased(lookup_table_path=str(empty))])
    with pytest.raises(ValueError, match="not found"):
        Actuator(i32([0]), ControllerPD(f32([0.0]), f32([0.0])), clamping=[ClampingPositionBased(lookup_table_path=str(tmp_path / "x"))])


def test_clamp_chain_limit():
    with pytest.raises(ValueError, match="at most 8"):
        Actuator(i32([0]), ControllerPD(f32([0.0]), f32([0.0])), clamping=[ClampingMaxEffort(f32([1.0]))] * 9)


# ---------------------------------------------------------------------------------------------------- full pipeline
def two_joint_template(free_root=False):
    t = ModelBuilder()
    joints = []
    parent = -1
    if free_root:
        base = t.add_link()
        joints.append(t.add_joint_free(base))
        parent = base
    la = t.add_link()
    joints.append(t.add_joint_revolute(parent, la, axis="z"))
    lb = t.add_link()
    joints.append(t.add_joint_revolute(la, lb, axis="y"))
    t.add_articulation(joints)
    return t, joints[-2:]


def full_pipeline_model(device="cpu", envs=3):
    kp, kd, sat, v_lim = 50.0, 5.0, 80.0, 20.0
    t, (ja, jb) = two_joint_template()
    dc = {"saturation_effort": sat, "velocity_limit": v_lim, "max_motor_effort": 1e6}
    t.add_actuator(ControllerPD, index=t.joint_qd_start[ja], kp=kp, kd=kd, delay_steps=2, clamping=[(ClampingDCMotor, dc)])
    t.add_actuator(ControllerPD, index=t.joint_qd_start[jb], kp=kp, kd=kd, delay_steps=3, clamping=[(ClampingDCMotor, dc)])
    b = ModelBuilder()
    b.replicate(t, envs)
    return b.finalize(device)


def test_full_pipeline(oact):
    kp, kd, sat, v_lim, qd = 50.0, 5.0, 80.0, 20.0, 2.0
    model = full_pipeline_model()
    assert len(model.actuators) == 1
    act = model.actuators[0]
    n = act.num_actuators
    assert n == 6 and act.delay.delay_steps.tolist() == [2, 3] * 3 and act.delay.buf_depth == 3
    state, control = model.state(), model.control()
    dofs = act.indices.tolist()
    state.joint_qd[dofs] = qd
    s0, s1 = act.state(), act.state()
    history = []
    for k, tgt in enumerate((10.0, 20.0, 30.0, 40.0, 50.0)):
        control.joint_target_q[act.target_pos_indices.long()] = tgt
        history.append(tgt)
        control.joint_f.zero_()
        oact.step(act, state, control, s0, s1, 0.01)
        s0, s1 = s1, s0
        for i, d in enumerate(dofs):
            raw = kp * _delayed(history, k, [2, 3][i % 2]) + kd * (0.0 - qd)
            expect = max(min(raw, min(sat * (1.0 - qd / v_lim), 1e6)), max(sat * (-1.0 - qd / v_lim), -1e6))
            assert control.joint_f[d].item() == pytest.approx(expect, abs=1e-3), (k, i)
    assert s0.delay_state.num_pushes.tolist() == [3] * n


# ---------------------------------------------------------------------------------------------------- builder
def test_builder_programmatic():
    b = ModelBuilder()
    links = [b.add_link() for _ in range(3)]
    joints = [b.add_joint_revolute(-1 if i == 0 else links[i - 1], link, axis="z") for i, link in enumerate(links)]
    b.add_articulation(joints)
    dofs = [b.joint_qd_start[j] for j in joints]
    b.add_actuator(ControllerPD, index=dofs[0], kp=50.0, kd=5.0, const_effort=1.0)
    b.add_actuator(ControllerPID, index=dofs[1], kp=100.0, ki=10.0, kd=20.0,
                   clamping=[(ClampingDCMotor, {"saturation_effort": 80.0, "velocity_limit": 15.0, "max_motor_effort": 200.0})])
    b.add_actuator(ControllerPD, index=dofs[2], kp=150.0, delay_steps=4)
    model = b.finalize()
    assert len(model.actuators) == 3
    pd = next(a for a in model.actuators if isinstance(a.controller, ControllerPD) and a.delay is None)
    pid = next(a for a in model.actuators if isinstance(a.controller, ControllerPID))
    pdd = next(a for a in model.actuators if isinstance(a.controller, ControllerPD) and a.delay is not None)
    assert pd.controller.kp.tolist() == [50.0] and pd.controller.const_effort.tolist() == [1.0] and pd.state() is None
    assert pid.controller.ki.tolist() == [10.0] and pid.controller.integral_max.tolist() == [math.inf]
    assert isinstance(pid.clamping[0], ClampingDCMotor) and pid.clamping[0].max_motor_effort.tolist() == [200.0]
    assert pid.state().controller_state.integral.tolist() == [0.0]
    assert pdd.delay.delay_steps.dtype == torch.int32 and pdd.delay.buf_depth == 4
    assert pdd.state().delay_state.buffer_pos.shape == (4, 1)


def test_builder_free_joint_replicate():
    t, (j1, j2) = two_joint_template(free_root=True)
    t.add_actuator(ControllerPD, index=t.joint_qd_start[j1], kp=100.0, kd=10.0, pos_index=t.joint_q_start[j1], delay_steps=2)
    t.add_actuator(ControllerPD, index=t.joint_qd_start[j2], kp=200.0, kd=20.0, pos_index=t.joint_q_start[j2], delay_steps=3)
    b = ModelBuilder()
    b.replicate(t, 3)
    model = b.finalize()
    assert len(model.actuators) == 1
    act = model.actuators[0]
    assert act.indices.tolist() == [6, 7, 14, 15, 22, 23]
    assert act.pos_indices.tolist() == [7, 8, 16, 17, 25, 26]
    assert act.target_pos_indices.tolist() == act.pos_indices.tolist()  # the model's targets are in the coordinate layout
    assert act.controller.kp.tolist() == [100.0, 200.0] * 3 and act.delay.delay_steps.tolist() == [2, 3] * 3
    assert act.delay.buf_depth == 3 and act.state().delay_state.buffer_pos.shape == (3, 6)


def test_builder_grouping_keys():
    b = ModelBuilder()
    links = [b.add_link() for _ in range(5)]
    for i, link in enumerate(links):
        b.add_joint_revolute(-1, link, axis="z")
    lut = {"lookup_positions": (0.0, 1.0), "lookup_efforts": (1.0, 2.0)}
    b.add_actuator(ControllerPD, index=0, kp=1.0, clamping=[(ClampingPositionBased, lut)])
    b.add_actuator(ControllerPD, index=1, kp=2.0, clamping=[(ClampingPositionBased, lut)])  # same table: same group
    b.add_actuator(ControllerPD, index=2, kp=3.0, clamping=[(ClampingPositionBased, {**lut, "lookup_efforts": (1.0, 3.0)})])
    b.add_actuator(ControllerPD, index=3, kp=4.0, delay_steps=0)  # delay present (0 steps) vs absent: different groups
    b.add_actuator(ControllerPD, index=4, kp=5.0, delay_steps=2)
    model = b.finalize()
    assert sorted(a.num_actuators for a in model.actuators) == [1, 2, 2]


def test_builder_warnings_and_errors():
    b = ModelBuilder()
    b.add_joint_revolute(-1, b.add_link(), axis="z")
    with pytest.warns(UserWarning, match="unrecognized parameter"):
        b.add_actuator(ControllerPD, index=0, kp=1.0, gain=3.0)
    with pytest.raises(TypeError, match="controller_class"):
        b.add_actuator(index=0)
    with pytest.raises(TypeError, match="index"):
        b.add_actuator(ControllerPD)


@pytest.mark.parametrize("cls,args,match", [
    (ControllerPD, {"kp": -1.0}, "kp"), (ControllerPD, {"kd": -1.0}, "kd"),
    (ControllerPID, {"kp": -1.0}, "kp"), (ControllerPID, {"ki": -1.0}, "ki"), (ControllerPID, {"kd": -1.0}, "kd"),
    (ControllerPID, {"integral_max": -1.0}, "integral_max"),
    (ClampingMaxEffort, {"max_effort": -1.0}, "max_effort"),
    (ClampingDCMotor, {"saturation_effort": -1.0}, "saturation_effort"), (ClampingDCMotor, {"velocity_limit": 0.0}, "velocity_limit"),
    (ClampingDCMotor, {"max_motor_effort": -1.0}, "max_motor_effort"),
    (ClampingPositionBased, {}, "requires"), (ClampingPositionBased, {"lookup_table_path": "x", "lookup_positions": (0.0,)}, "not both"),
    (ClampingPositionBased, {"lookup_positions": (0.0,)}, "Both"), (ClampingPositionBased, {"lookup_positions": (), "lookup_efforts": ()}, "empty"),
    (ClampingPositionBased, {"lookup_positions": (0.0, 1.0), "lookup_efforts": (1.0,)}, "length"),
    (ClampingPositionBased, {"lookup_positions": (0.0,), "lookup_efforts": (-1.0,)}, "non-negative"),
    (ClampingPositionBased, {"lookup_positions": (1.0, 0.0), "lookup_efforts": (1.0, 1.0)}, "non-decreasing"),
    (Delay, {}, "delay_steps"), (Delay, {"delay_steps": -1}, "delay_steps"),
])
def test_resolve_arguments_errors(cls, args, match):
    with pytest.raises(ValueError, match=match):
        cls.resolve_arguments(args)


def test_resolve_arguments_defaults():
    assert ControllerPD.resolve_arguments({}) == {"kp": 0.0, "kd": 0.0, "const_effort": 0.0}
    assert ControllerPID.resolve_arguments({}) == {"kp": 0.0, "ki": 0.0, "kd": 0.0, "integral_max": math.inf, "const_effort": 0.0}
    assert ClampingMaxEffort.resolve_arguments({}) == {"max_effort": math.inf}
    assert ClampingDCMotor.resolve_arguments({}) == {"saturation_effort": math.inf, "velocity_limit": math.inf, "max_motor_effort": math.inf}


def test_requires_grad_and_shapes():
    with pytest.raises(NotImplementedError, match="differentiable"):
        Actuator(i32([0]), ControllerPD(f32([1.0]), f32([0.0])), requires_grad=True)
    with pytest.raises(ValueError, match="kp shape"):
        ControllerPD(f32([1.0, 2.0]), f32([0.0]))
    with pytest.raises(ValueError, match="pos_indices shape"):
        Actuator(i32([0]), ControllerPD(f32([1.0]), f32([0.0])), pos_indices=i32([0, 1]))


# ---------------------------------------------------------------------------------------------------- target layouts and names
def test_target_pos_read_from_dof_index(oact):
    a = Actuator(i32([1]), ControllerPD(f32([100.0]), f32([0.0]), const_effort=f32([0.0])), pos_indices=i32([3]), target_pos_indices=i32([1]))
    st, ctl = io(4, 2, joint_q=f32([0.0, 0.0, 0.0, 0.5]), joint_target_q=f32([0.0, 2.0, 0.0, 99.0]),
                 joint_target_qd=torch.zeros(4), joint_act=None, joint_f=torch.zeros(4))
    oact.step(a, st, ctl, None, None, dt=0.01)
    assert ctl.joint_f[1].item() == 150.0


def test_use_coord_layout_targets_flag(monkeypatch):
    ctrl = lambda: ControllerPD(f32([1.0]), f32([0.0]))  # noqa: E731
    assert newton_b200.use_coord_layout_targets is False
    assert Actuator(i32([1]), ctrl(), pos_indices=i32([3])).target_pos_indices.tolist() == [1]
    monkeypatch.setattr(newton_b200, "use_coord_layout_targets", True)
    a = Actuator(i32([1]), ctrl(), pos_indices=i32([3]))
    monkeypatch.setattr(newton_b200, "use_coord_layout_targets", False)
    assert a.target_pos_indices.tolist() == [3]  # read once, at construction


def test_attribute_names(oact):
    ctrl = lambda: ControllerPD(f32([2.0]), f32([0.0]))  # noqa: E731
    a = Actuator(i32([0]), ctrl())
    assert (a.control_target_pos_attr, a.control_target_vel_attr, a.control_feedforward_attr) == ("joint_target_q", "joint_target_qd", "joint_act")
    a = Actuator(i32([0]), ctrl(), control_target_pos_attr=None, control_target_vel_attr=None)
    assert (a.control_target_pos_attr, a.control_target_vel_attr) == ("joint_target_q", "joint_target_qd")
    a = Actuator(i32([0]), ctrl(), state_pos_attr="p", state_vel_attr="v", control_target_pos_attr="tp", control_target_vel_attr="tv",
                 control_feedforward_attr=None, control_output_attr="out", control_computed_output_attr="raw",
                 clamping=[ClampingMaxEffort(f32([1.0]))])
    st = types.SimpleNamespace(p=f32([0.0]), v=f32([0.0]))
    ctl = types.SimpleNamespace(tp=f32([3.0]), tv=f32([0.0]), joint_act=f32([100.0]), out=f32([0.5]), raw=f32([0.0]))
    oact.step(a, st, ctl)
    assert ctl.out.item() == 1.5 and ctl.raw.item() == 6.0  # feedforward skipped; outputs accumulate


# ---------------------------------------------------------------------------------------------------- resets
def _delay_actuator(n=4, depth=3):
    return Actuator(i32(list(range(n))), ControllerPID(f32([1.0] * n), f32([1.0] * n), f32([0.0] * n), f32([math.inf] * n)),
                    delay=Delay(i32([depth] * n), max_delay=depth))


def _fill(oact, a, steps=3):
    st, ctl = io(a.num_actuators, a.num_actuators, joint_target_q=f32(list(range(1, a.num_actuators + 1))))
    s0, s1 = a.state(), a.state()
    for _ in range(steps):
        oact.step(a, st, ctl, s0, s1, 0.1)
        s0, s1 = s1, s0
    return s0


def test_delay_full_and_masked_reset(oact):
    a = _delay_actuator()
    s = _fill(oact, a)
    ds = s.delay_state
    wi = ds.write_idx.item()
    oact.reset(ds, torch.tensor([True, False, True, False]))
    assert ds.write_idx.item() == wi  # a masked reset leaves write_idx alone
    assert ds.num_pushes.tolist() == [0, 3, 0, 3]
    assert (ds.buffer_pos[:, [0, 2]] == 0).all() and (ds.buffer_pos[:, 1] != 0).any()
    oact.reset(ds)
    assert ds.write_idx.item() == 2 and ds.num_pushes.tolist() == [0] * 4 and not ds.buffer_act.any() and not ds.buffer_pos.any()


def test_pid_masked_reset_and_rejections(oact):
    a = _delay_actuator()
    s = _fill(oact, a)
    cs = s.controller_state
    before = cs.integral.clone()
    oact.reset(cs, torch.tensor([False, True, False, True]))
    assert cs.integral.tolist() == [before[0].item(), 0.0, before[2].item(), 0.0]
    for bad, match in ((torch.ones(4, dtype=torch.int32), "Boolean"), (torch.ones(2, 2, dtype=torch.bool), "Boolean"),
                       (torch.ones(3, dtype=torch.bool), "length")):
        with pytest.raises(ValueError, match=match):
            cs.reset(bad)


def test_composed_reset(oact):
    a = _delay_actuator()
    s = _fill(oact, a)
    oact.reset(s, torch.tensor([True, True, False, False]))
    assert s.controller_state.integral[:2].tolist() == [0.0, 0.0] and s.controller_state.integral[2].item() != 0.0
    assert s.delay_state.num_pushes.tolist() == [0, 0, 3, 3]
    oact.reset(s)
    assert not s.controller_state.integral.any() and s.delay_state.write_idx.item() == 2


# ---------------------------------------------------------------------------------------------------- host logic
def test_duplicate_effort_indices_serial_sum(oact):
    eff = [2, 0, 2, 1, 2]
    a = Actuator(i32([0, 1, 2, 3, 4]), ControllerPD(f32([0.0] * 5), f32([0.0] * 5), const_effort=f32([0.1, 0.2, 0.3, 0.4, 0.5])),
                 effort_indices=i32(eff))
    assert a.has_duplicate_effort_indices
    T, target, start, order, _ = a._dup
    assert T == 3 and target.tolist() == [0, 1, 2] and start.tolist() == [0, 1, 2, 5] and order.tolist() == [1, 3, 0, 2, 4]
    st, ctl = io(5, 5, joint_f=f32([1.0, 0.0, 1e8, 0.0, 0.0]))
    oact.step(a, st, ctl)
    f = np.float32
    assert ctl.joint_f[2].item() == float(((f(1e8) + f(0.1)) + f(0.3)) + f(0.5))
    assert not Actuator(i32([0, 1]), ControllerPD(f32([0.0] * 2), f32([0.0] * 2))).has_duplicate_effort_indices


def test_output_must_not_alias_inputs():
    a = Actuator(i32([0]), ControllerPD(f32([1.0]), f32([0.0])), control_output_attr="joint_act")
    st, ctl = io(1, 1)
    with pytest.raises(ValueError, match="output"):
        a._step_desc(st, ctl, None, None, None)


def test_step_checks_element_counts():
    a = Actuator(i32([0, 5]), ControllerPD(f32([1.0, 1.0]), f32([0.0, 0.0])))
    st, ctl = io(3, 3)
    with pytest.raises(ValueError, match="at least 6"):
        a._step_desc(st, ctl, None, None, None)


def test_step_descriptor_cache(oact):
    """Eager steps reuse the checked descriptor while they touch the very same arrays; a replaced array is checked again."""
    a = Actuator(i32([0, 1]), ControllerPD(f32([1.0, 2.0]), f32([0.0, 0.0])), delay=Delay(i32([1, 1]), 1))
    st, ctl = io(2, 2, joint_target_q=f32([1.0, 1.0]))
    s = [a.state(), a.state()]
    for _ in range(4):
        ctl.joint_f.zero_()
        oact.step(a, st, ctl, s[0], s[1])
        s.reverse()
    assert len(a._desc_cache) == 2 and ctl.joint_f.tolist() == [1.0, 2.0]
    ctl.joint_f = torch.zeros(1)
    with pytest.raises(ValueError, match="at least 2"):
        oact.step(a, st, ctl, s[0], s[1])
    a.controller.kp = f32([3.0, 4.0])  # a new parameter tensor is picked up
    ctl.joint_f = torch.zeros(2)
    oact.step(a, st, ctl, s[0], s[1])
    assert ctl.joint_f.tolist() == [3.0, 4.0]


def test_cpu_step_raises():
    a = Actuator(i32([0]), ControllerPD(f32([1.0]), f32([0.0])))
    st, ctl = io(1, 1)
    with pytest.raises(newton_b200._lib.Nb2Error, match="CUDA"):
        a.step(st, ctl)


def test_model_to_round_trip_and_no_actuators():
    model = full_pipeline_model()
    back = model.to("cpu")
    assert len(back.actuators) == 1 and back.actuators[0] is not model.actuators[0]
    a, b = model.actuators[0], back.actuators[0]
    for name in ("indices", "pos_indices", "target_pos_indices", "effort_indices"):
        assert torch.equal(getattr(a, name), getattr(b, name))
    assert torch.equal(a.controller.kp, b.controller.kp) and torch.equal(a.delay.delay_steps, b.delay.delay_steps)
    assert b.controller.kp.data_ptr() != a.controller.kp.data_ptr() and b.delay.buf_depth == 3
    plain = ModelBuilder()
    plain.add_joint_revolute(-1, plain.add_link(), axis="z")
    assert plain.finalize().actuators == [] and plain.finalize().to("cpu").actuators == []


def test_shard_tables():
    t, (j1, j2) = two_joint_template(free_root=True)
    t.add_actuator(ControllerPD, index=t.joint_qd_start[j1], kp=1.0, pos_index=t.joint_q_start[j1],
                   clamping=[(ClampingMaxEffort, {"max_effort": 5.0})])
    t.add_actuator(ControllerPD, index=t.joint_qd_start[j2], kp=2.0, pos_index=t.joint_q_start[j2],
                   clamping=[(ClampingMaxEffort, {"max_effort": 6.0})])
    t.add_actuator(ControllerPID, index=t.joint_qd_start[j2], ki=1.0)
    b = ModelBuilder()
    b.replicate(t, 4)
    model = b.finalize()
    pd = model.actuators[0]
    shard = model.shard(1, 2)
    assert len(shard.actuators) == 2
    s = shard.actuators[0]
    assert s.indices.tolist() == [6, 7, 14, 15] and s.pos_indices.tolist() == [7, 8, 16, 17]
    assert s.target_pos_indices.tolist() == [7, 8, 16, 17] and s.effort_indices.tolist() == [6, 7, 14, 15]
    assert s.controller.kp.tolist() == [1.0, 2.0, 1.0, 2.0] and s.clamping[0].max_effort.tolist() == [5.0, 6.0, 5.0, 6.0]
    assert shard.actuators[1].indices.tolist() == [7, 15]
    assert pd.indices.tolist() == [6, 7, 14, 15, 22, 23, 30, 31]  # the source model is untouched
    # a group whose dofs all sit in other worlds is dropped
    one = ModelBuilder()
    one.replicate(two_joint_template()[0], 2)
    one.add_actuator(ControllerPD, index=0, kp=1.0)
    assert len(one.finalize().shard(1, 2).actuators) == 0


# ---------------------------------------------------------------------------------------------------- ArticulationView
def view_model(arts_per_world, worlds=3, device="cpu"):
    """``worlds`` worlds of ``arts_per_world`` two-revolute arms; the second joint of every arm has a PD actuator."""
    b = ModelBuilder()
    for _ in range(worlds):
        b.begin_world()
        for _ in range(arts_per_world):
            la = b.add_link()
            ja = b.add_joint_revolute(-1, la, axis="z", label="arm/j0")
            lb = b.add_link()
            jb = b.add_joint_revolute(la, lb, axis="z", label="arm/j1")
            b.add_articulation([ja, jb], label="arm")
            b.add_actuator(ControllerPD, index=b.joint_qd_start[jb], kp=10.0 + b.joint_qd_start[jb], kd=1.0)
        b.end_world()
    return b.finalize(device)


@pytest.mark.parametrize("per_world", [1, 2])
@pytest.mark.parametrize("with_mask", [False, True])
def test_actuator_parameter_get_set(oact, per_world, with_mask):
    from newton_b200.selection import ArticulationView

    model = view_model(per_world)
    act = model.actuators[0]
    view = ArticulationView(model, "arm")
    with oact.host():
        kp = view.get_actuator_parameter(act, act.controller, "kp")
        assert kp.shape == (3, 2 * per_world)
        expect = np.zeros((3, 2 * per_world), np.float32)
        expect[:, 1::2] = (10.0 + act.indices.numpy()).reshape(3, per_world)
        np.testing.assert_array_equal(kp.numpy(), expect)
        new = torch.arange(6.0 * per_world).reshape(3, 2 * per_world)
        mask = torch.tensor([True, False, True]) if with_mask else None
        view.set_actuator_parameter(act, act.controller, "kp", new, mask=mask)
        got = view.get_actuator_parameter(act, act.controller, "kp").numpy()
    for w in range(3):
        want = new[w].numpy() if (mask is None or mask[w]) else expect[w]
        np.testing.assert_array_equal(got[w, 1::2], want[1::2])
        assert not got[w, 0::2].any()


def chain_view_model(arts_per_world, worlds=3, device="cpu"):
    """``worlds`` worlds of ``arts_per_world`` three-revolute chains; joints 0 and 2 of every chain have a PD actuator."""
    b = ModelBuilder()
    for _ in range(worlds):
        b.begin_world()
        for _ in range(arts_per_world):
            joints, parent = [], -1
            for k in range(3):
                link = b.add_link()
                joints.append(b.add_joint_revolute(parent, link, axis="z", label=f"chain/j{k}"))
                parent = link
            b.add_articulation(joints, label="chain")
            for j in (joints[0], joints[2]):
                b.add_actuator(ControllerPD, index=b.joint_qd_start[j], kp=100.0 + b.joint_qd_start[j], kd=1.0)
        b.end_world()
    return b.finalize(device)


@pytest.mark.parametrize("per_world", [1, 2])
def test_actuator_parameter_index_selection(oact, per_world):
    """A view without the middle joint selects dofs (0, 2) of each chain: the index-array branch of the dof mapping."""
    from newton_b200.selection import ArticulationView
    from newton_b200.sim.model import AttributeFrequency

    model = chain_view_model(per_world)
    act = model.actuators[0]
    view = ArticulationView(model, "chain", exclude_joints=["j1"])
    assert not view.frequency_layouts[AttributeFrequency.JOINT_DOF].is_contiguous
    dofs = model.joint_qd_start[:-1].numpy().reshape(3, per_world, 3)[:, :, [0, 2]].reshape(3, -1)
    with oact.host():
        np.testing.assert_array_equal(view.get_actuator_parameter(act, act.controller, "kp").numpy(), 100.0 + dofs)
        new = torch.arange(6.0 * per_world).reshape(3, 2 * per_world)
        view.set_actuator_parameter(act, act.controller, "kp", new, mask=torch.tensor([False, True, True]))
        got = view.get_actuator_parameter(act, act.controller, "kp").numpy()
    np.testing.assert_array_equal(got[0], 100.0 + dofs[0])
    np.testing.assert_array_equal(got[1:], new[1:].numpy())
    middle = model.joint_qd_start[:-1].numpy().reshape(3, per_world, 3)[:, :, 1].reshape(-1)
    assert not np.isin(act.indices.numpy(), middle).any()


def test_actuator_parameter_mask_rejections(oact):
    from newton_b200.selection import ArticulationView

    model = view_model(1)
    act = model.actuators[0]
    view = ArticulationView(model, "arm")
    before = act.controller.kp.clone()

    def never(*a):
        raise AssertionError("launched")

    import newton_b200.actuators.actuator as A

    for bad in (torch.ones(2, dtype=torch.bool), torch.ones(3, dtype=torch.int32), torch.ones(3, 1, dtype=torch.bool)):
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(A, "_call", never)
            with pytest.raises(ValueError):
                view.set_actuator_parameter(act, act.controller, "kp", torch.zeros(3, 2), mask=bad)
    assert torch.equal(act.controller.kp, before)


# ---------------------------------------------------------------------------------------------------- Featherstone end to end
def drive_model(world_count=2, device="cpu"):
    """Quadrupeds whose model drive gains are zeroed, each leg dof driven by a ControllerPD with the original gains.
    Joint damping is 0 in the quadruped."""
    from newton_b200 import scenes

    model = scenes.quadruped_model(world_count, seed=1)
    leg = [d for j in range(model.joint_count) if model.joint_type[j].item() == JointType.REVOLUTE
           for d in range(model.joint_qd_start[j].item(), model.joint_qd_start[j + 1].item())]
    coord = [model.joint_q_start[j].item() + (d - model.joint_qd_start[j].item())
             for j in range(model.joint_count) if model.joint_type[j].item() == JointType.REVOLUTE
             for d in range(model.joint_qd_start[j].item(), model.joint_qd_start[j + 1].item())]
    ke, kd = model.joint_target_ke[leg].clone(), model.joint_target_kd[leg].clone()
    act = Actuator(i32(leg), ControllerPD(ke, kd), pos_indices=i32(coord), target_pos_indices=i32(coord))
    driven = model.to("cpu")
    driven.joint_target_ke.zero_()
    driven.joint_target_kd.zero_()
    assert not model.joint_damping.any()
    return (model.to(device), driven.to(device), act._rebuilt(device))


def test_featherstone_builtin_pd_equivalence(oact):
    import oracle

    model, driven, act = drive_model()
    ref, out = model.state(), driven.state()
    ref1, out1 = model.state(), driven.state()
    c_ref, c_out = model.control(), driven.control()
    solver_ref, solver_out = oracle.SolverFeatherstone(model), oracle.SolverFeatherstone(driven)
    for _ in range(200):
        solver_ref.step(ref, ref1, c_ref, None, 0.001)
        c_out.joint_f.zero_()
        oact.step(act, out, c_out)
        solver_out.step(out, out1, c_out, None, 0.001)
        ref, ref1, out, out1 = ref1, ref, out1, out
    np.testing.assert_array_equal(out.joint_q.numpy().view(np.int32), ref.joint_q.numpy().view(np.int32))
    np.testing.assert_array_equal(out.joint_qd.numpy().view(np.int32), ref.joint_qd.numpy().view(np.int32))

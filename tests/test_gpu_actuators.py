"""CUDA Actuator.step against the CPU oracle (oracle/oracle_actuator.h), bit for bit: every float32 word of the output, the
computed output and every array of the next state (integral, the three delay buffers, num_pushes, write_idx) after each of
50 steps, on the hand-written cases of tests/test_actuators.py, seeded random groups over {PD, PID} x {no delay, delay} x
clamp chains of 0-3 (infinite parameters, sat = 0, repeated lookup positions), duplicate effort indices, ball and FREE
joints in both target layouts, a masked reset mid-run and 4096 quadrupeds in the benchmark configuration; the
Featherstone built-in-PD equivalence; parameter access through ArticulationView (slice and index-array dof selections); and
CUDA-graph capture of actuator.step -> SolverFeatherstone.step and eval_ik -> actuator.step -> SolverXPBD.step, whose replays
equal the eager run and the oracle."""

import math
import types

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import ModelBuilder, _lib, scenes
from newton_b200.actuators import (
    Actuator,
    ClampingDCMotor,
    ClampingMaxEffort,
    ClampingPositionBased,
    ControllerPD,
    ControllerPID,
    Delay,
)
from tests import test_actuators as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STATE_ARRAYS = (("controller_state", "integral"), ("delay_state", "buffer_pos"), ("delay_state", "buffer_vel"),
                ("delay_state", "buffer_act"), ("delay_state", "num_pushes"), ("delay_state", "write_idx"))


@pytest.fixture(scope="module")
def oact():
    import oracle
    import oracle.actuator as oact

    oracle.build()
    return oact


def _eq(got, ref, what):
    g, r = got.detach().cpu().contiguous().numpy(), ref.detach().contiguous().numpy()
    assert g.shape == r.shape, what
    np.testing.assert_array_equal(g.view(np.int32), r.view(np.int32), err_msg=what)


def _eq_state(g, r, what):
    if r is None:
        assert g is None
        return
    for part, name in STATE_ARRAYS:
        rp = getattr(r, part)
        if rp is not None:
            _eq(getattr(getattr(g, part), name), getattr(rp, name), f"{what}: {part}.{name}")


def run_pair(oact, act, n_q, n_qd, steps=50, dt=0.01, seed=0, reset_at=None, zero_output=True, scale=1.0, io=None):
    """Step ``act`` (a CPU actuator) on the oracle and its device copy on the GPU with the same seeded inputs; compare after
    every step.  ``io`` (CPU state, control) defaults to random plain tensors of ``n_q`` coordinates and ``n_qd`` dofs."""
    gact = act._rebuilt(DEV)
    rng = np.random.default_rng(seed)
    st, ctl = io if io is not None else T.io(n_q, n_qd)
    outs = [a for a in (act.control_output_attr, act.control_computed_output_attr) if a is not None]
    if io is None:
        for a in outs:
            setattr(ctl, a, torch.zeros(n_qd))
    gst = types.SimpleNamespace(**{k: v.to(DEV) for k, v in vars(st).items() if isinstance(v, torch.Tensor)})
    gctl = types.SimpleNamespace(**{k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in vars(ctl).items()})
    cs, gs = [act.state(), act.state()], [gact.state(), gact.state()]
    launches = []
    for k in range(steps):
        for obj, gobj, names in ((st, gst, (act.state_pos_attr, act.state_vel_attr)),
                                 (ctl, gctl, (act.control_target_pos_attr, act.control_target_vel_attr, act.control_feedforward_attr))):
            for name in names:
                t = getattr(obj, name, None) if name else None
                if t is None:
                    continue
                t.copy_(torch.from_numpy((rng.normal(size=t.shape) * scale).astype(np.float32)))
                getattr(gobj, name).copy_(t)
        if zero_output:
            for a in outs:
                getattr(ctl, a).zero_()
                getattr(gctl, a).zero_()
        oact.step(act, st, ctl, cs[0], cs[1], dt)
        before = _lib.kernel_launch_count()
        gact.step(gst, gctl, gs[0], gs[1], dt)
        launches.append(_lib.kernel_launch_count() - before)
        torch.cuda.synchronize()
        for a in outs:
            _eq(getattr(gctl, a), getattr(ctl, a), f"step {k}: {a}")
        _eq_state(gs[1], cs[1], f"step {k}")
        cs.reverse()
        gs.reverse()
        if reset_at == k:
            mask = torch.from_numpy(rng.random(act.num_actuators) < 0.5)
            oact.reset(cs[0], mask)
            gs[0].reset(mask.to(DEV))
            _eq_state(gs[0], cs[0], "after reset")
    return launches


# ---------------------------------------------------------------------------------------------------- CPU cases on the GPU
def test_hand_written_cases(oact):
    lut = ClampingPositionBased(lookup_positions=(-1.0, 0.0, 0.0, 1.0), lookup_efforts=(10.0, 30.0, 35.0, 50.0))
    cases = [
        Actuator(T.i32([0, 1, 2]), ControllerPD(T.f32([100.0, 200.0, 50.0]), T.f32([10.0, 20.0, 5.0]), T.f32([1.0, -2.0, 0.5]))),
        Actuator(T.i32([0]), ControllerPID(T.f32([10.0]), T.f32([100.0]), T.f32([1.0]), T.f32([0.015]), T.f32([0.5]))),
        Actuator(T.i32([0, 1, 2]), ControllerPD(T.f32([1.0] * 3), T.f32([0.0] * 3)), delay=Delay(T.i32([0, 1, 3]), 3)),
        Actuator(T.i32([0]), ControllerPD(T.f32([30.0]), T.f32([1.0])), clamping=[ClampingMaxEffort(T.f32([50.0]))]),
        Actuator(T.i32([0]), ControllerPD(T.f32([300.0]), T.f32([1.0])), clamping=[ClampingDCMotor(T.f32([100.0]), T.f32([10.0]), T.f32([200.0]))]),
        Actuator(T.i32([0]), ControllerPD(T.f32([300.0]), T.f32([1.0])), clamping=[lut]),
        T._delay_actuator(),
    ]
    for i, act in enumerate(cases):
        run_pair(oact, act, 3 if i != 6 else 4, 3 if i != 6 else 4, seed=i, scale=0.5 if i != 5 else 3.0)


def test_full_pipeline_and_builder_models(oact):
    model = T.full_pipeline_model()
    act = model.actuators[0]
    st, ctl = model.state(), model.control()
    run_pair(oact, act, model.joint_coord_count, model.joint_dof_count, io=(st, ctl))
    assert model.to(DEV).actuators[0].controller.kp.is_cuda


def test_attribute_names_and_target_layouts(oact, monkeypatch):
    # FREE root: pos_index != index; targets in the dof layout (module flag off) and the coordinate layout (flag on)
    t, (j1, j2) = T.two_joint_template(free_root=True)
    b = ModelBuilder()
    b.add_builder(t)
    ball = b.add_link()
    jb = b.add_joint_ball(-1, ball)
    b.add_articulation([jb])
    model = b.finalize()
    dofs = [model.joint_qd_start[j].item() for j in (j1, j2)] + list(range(model.joint_qd_start[jb].item(), model.joint_qd_start[jb].item() + 3))
    coords = [model.joint_q_start[j].item() for j in (j1, j2)] + list(range(model.joint_q_start[jb].item(), model.joint_q_start[jb].item() + 3))
    assert dofs != coords
    for flag in (False, True):
        monkeypatch.setattr(newton_b200, "use_coord_layout_targets", flag)
        act = Actuator(T.i32(dofs), ControllerPID(T.f32([5.0] * 5), T.f32([2.0] * 5), T.f32([1.0] * 5), T.f32([math.inf] * 5)),
                       delay=Delay(T.i32([2, 0, 1, 2, 2]), 2), pos_indices=T.i32(coords), control_computed_output_attr="raw",
                       clamping=[ClampingMaxEffort(T.f32([1.0] * 5))])
        assert act.target_pos_indices.tolist() == (coords if flag else dofs)
        run_pair(oact, act, model.joint_coord_count, model.joint_dof_count, seed=int(flag))


# ---------------------------------------------------------------------------------------------------- random groups
def random_actuator(rng, pid, delay, n_clamps, n=300, n_q=340, n_qd=320, duplicates=False):
    idx = rng.choice(n_qd, n, replace=False).astype(np.int32)
    pos = rng.choice(n_q, n, replace=False).astype(np.int32)
    tpos = rng.choice(n_q, n, replace=False).astype(np.int32)
    eff = rng.integers(0, n_qd // 4, n).astype(np.int32) if duplicates else idx
    f = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))  # noqa: E731

    def with_specials(a, specials):
        a = np.asarray(a, dtype=np.float32)
        a[rng.random(n) < 0.1] = rng.choice(specials)
        return a

    kp, kd = f(rng.uniform(0, 100, n)), f(rng.uniform(0, 10, n))
    ce = f(rng.normal(size=n)) if rng.random() < 0.5 else None
    ctrl = (ControllerPID(kp, f(rng.uniform(0, 50, n)), kd, f(with_specials(rng.uniform(0, 0.05, n), [math.inf, 0.0])), ce)
            if pid else ControllerPD(kp, kd, ce))
    d = Delay(torch.from_numpy(rng.integers(0, 5, n).astype(np.int32)), 4) if delay else None
    clamps = []
    for _ in range(n_clamps):
        kind = rng.integers(0, 3)
        if kind == 0:
            clamps.append(ClampingMaxEffort(f(with_specials(rng.uniform(0, 60, n), [math.inf, 0.0]))))
        elif kind == 1:
            clamps.append(ClampingDCMotor(f(with_specials(rng.uniform(0, 120, n), [math.inf, 0.0])),
                                          f(with_specials(rng.uniform(0.5, 30, n), [math.inf])),
                                          f(with_specials(rng.uniform(0, 80, n), [math.inf, 0.0]))))
        else:
            xs = np.sort(rng.normal(size=12)).astype(np.float32)
            xs[5] = xs[4]  # a repeated position: dx == 0
            clamps.append(ClampingPositionBased(lookup_positions=tuple(xs.tolist()),
                                                lookup_efforts=tuple(rng.uniform(0, 40, 12).astype(np.float32).tolist())))
    return Actuator(torch.from_numpy(idx), ctrl, d, clamps, pos_indices=torch.from_numpy(pos), target_pos_indices=torch.from_numpy(tpos),
                    effort_indices=torch.from_numpy(eff), control_computed_output_attr="raw")


@pytest.mark.parametrize("pid", [False, True])
@pytest.mark.parametrize("delay", [False, True])
@pytest.mark.parametrize("n_clamps", [0, 1, 2, 3])
def test_random_groups(oact, pid, delay, n_clamps):
    rng = np.random.default_rng(100 * pid + 10 * delay + n_clamps)
    act = random_actuator(rng, pid, delay, n_clamps)
    launches = run_pair(oact, act, 340, 320, seed=n_clamps, scale=20.0, reset_at=24 if (pid or delay) else None)
    assert set(launches) == {1}


def test_duplicate_effort_indices_take_the_ordered_pass(oact):
    rng = np.random.default_rng(7)
    act = random_actuator(rng, True, True, 2, duplicates=True)
    assert act.has_duplicate_effort_indices
    launches = run_pair(oact, act, 340, 320, seed=3, scale=20.0, zero_output=False)
    assert set(launches) == {2}


# ---------------------------------------------------------------------------------------------------- bench configuration
@pytest.mark.parametrize("controller", ["pd", "pid"])
def test_quadrupeds_bench_configuration(oact, controller):
    model = scenes.quadruped_actuated_model(4096, seed=1, controller=controller)
    act = model.actuators[0]
    assert act.num_actuators == 4096 * 12 and not act.has_duplicate_effort_indices
    launches = run_pair(oact, act, model.joint_coord_count, model.joint_dof_count, steps=20, scale=0.3, reset_at=9,
                        io=(model.state(), model.control()))
    assert set(launches) == {1}


# ---------------------------------------------------------------------------------------------------- Featherstone
def test_featherstone_builtin_pd_equivalence(cuda_lib):
    model, driven, act = T.drive_model(8, DEV)
    sref, sout = newton_b200.solvers.SolverFeatherstone(model), newton_b200.solvers.SolverFeatherstone(driven)
    ref, ref1, out, out1 = model.state(), model.state(), driven.state(), driven.state()
    c_ref, c_out = model.control(), driven.control()
    for _ in range(200):
        sref.step(ref, ref1, c_ref, None, 0.001)
        c_out.joint_f.zero_()
        act.step(out, c_out)
        sout.step(out, out1, c_out, None, 0.001)
        ref, ref1, out, out1 = ref1, ref, out1, out
    torch.cuda.synchronize()
    assert not torch.equal(ref.joint_q, model.joint_q)
    _eq(out.joint_q, ref.joint_q.cpu(), "joint_q")
    _eq(out.joint_qd, ref.joint_qd.cpu(), "joint_qd")


def _graph_frame(model, act, solver, substeps, dt, ik=False):
    """One frame of ``substeps`` x (joint_f = 0 -> [eval_ik] -> actuator.step -> solver.step); returns (run, final state)."""
    s = [model.state(), model.state()]
    a = [act.state(), act.state()]
    ctl = model.control()

    def frame():
        for _ in range(substeps):
            ctl.joint_f.zero_()
            if ik:
                newton_b200.eval_ik(model, s[0], s[0].joint_q, s[0].joint_qd)
            act.step(s[0], ctl, a[0], a[1], dt)
            solver.step(s[0], s[1], ctl, None, dt)
            s.reverse()
            a.reverse()

    return frame, s, a, ctl


@pytest.mark.parametrize("solver_name", ["featherstone", "xpbd"])
def test_cuda_graph_replay_matches_eager_and_oracle(oact, cuda_lib, solver_name):
    import oracle

    cpu_model = scenes.quadruped_actuated_model(32, seed=1)
    model = cpu_model.to(DEV)
    act = model.actuators[0]
    make = (lambda m: newton_b200.solvers.SolverFeatherstone(m)) if solver_name == "featherstone" else \
        (lambda m: newton_b200.solvers.SolverXPBD(m, iterations=2))
    ik = solver_name == "xpbd"
    frames, substeps, dt = 5, 10, 0.001

    def run(graph):
        frame, s, a, _ = _graph_frame(model, act, make(model), substeps, dt, ik)
        if graph:
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                frame()
            torch.cuda.synchronize()
            for st, fresh in zip(s, (model.state(), model.state())):
                st.assign(fresh)
            for st in a:
                st.reset()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                frame()
            for _ in range(frames):
                g.replay()
        else:
            for _ in range(frames):
                frame()
        torch.cuda.synchronize()
        return s, a

    eager, ea = run(False)
    graph, ga = run(True)
    for name in ("joint_q", "joint_qd", "body_q"):
        _eq(getattr(graph[0], name), getattr(eager[0], name).cpu(), f"graph vs eager: {name}")
    for name in ("buffer_pos", "buffer_vel", "buffer_act", "num_pushes", "write_idx"):
        _eq(getattr(ga[0].delay_state, name), getattr(ea[0].delay_state, name).cpu(), f"graph vs eager: {name}")
    # the same substeps on the oracle: eval_ik, actuator step and solver step on the CPU model
    cact = cpu_model.actuators[0]
    s = [cpu_model.state(), cpu_model.state()]
    a = [cact.state(), cact.state()]
    ctl = cpu_model.control()
    solver = oracle.SolverFeatherstone(cpu_model) if solver_name == "featherstone" else oracle.SolverXPBD(cpu_model, iterations=2)
    for _ in range(frames * substeps):
        ctl.joint_f.zero_()
        if ik:
            oracle.eval_ik(cpu_model, s[0], s[0].joint_q, s[0].joint_qd)
        oact.step(cact, s[0], ctl, a[0], a[1], dt)
        solver.step(s[0], s[1], ctl, None, dt)
        s.reverse()
        a.reverse()
    for name in ("joint_q", "joint_qd", "body_q", "body_qd"):
        _eq(getattr(graph[0], name), getattr(s[0], name), f"graph vs oracle: {name}")
    _eq(ga[0].delay_state.buffer_pos, a[0].delay_state.buffer_pos, "graph vs oracle: buffer_pos")


# ---------------------------------------------------------------------------------------------------- ArticulationView
@pytest.mark.parametrize("per_world", [1, 2])
@pytest.mark.parametrize("selection", ["slice", "indices"])
def test_actuator_parameters_on_the_gpu(oact, per_world, selection):
    from newton_b200.selection import ArticulationView

    if selection == "slice":
        model, pattern, kw = T.view_model(per_world), "arm", {}
    else:  # the chains' middle joints left out: an index-array dof selection
        model, pattern, kw = T.chain_view_model(per_world), "chain", {"exclude_joints": ["j1"]}
    gmodel = model.to(DEV)
    act, gact = model.actuators[0], gmodel.actuators[0]
    view, gview = ArticulationView(model, pattern, **kw), ArticulationView(gmodel, pattern, **kw)
    new = torch.arange(6.0 * per_world).reshape(3, 2 * per_world)
    mask = torch.tensor([True, False, True])
    with oact.host():
        view.set_actuator_parameter(act, act.controller, "kd", new, mask=mask)
        ref = view.get_actuator_parameter(act, act.controller, "kd")
    before = _lib.kernel_launch_count()
    gview.set_actuator_parameter(gact, gact.controller, "kd", new.to(DEV), mask=mask.to(DEV))
    got = gview.get_actuator_parameter(gact, gact.controller, "kd")
    assert _lib.kernel_launch_count() - before == 2
    _eq(got, ref, "kd")
    _eq(gact.controller.kd, act.controller.kd, "kd parameter")
    with pytest.raises(ValueError):
        gview.set_actuator_parameter(gact, gact.controller, "kd", new.to(DEV), mask=mask)  # mask on the host

"""newton_b200.controllers on the GPU (nb2_joint_impedance_step, both compiled variants of joint_impedance_kernel) against the CPU
oracle bit for bit (strict-fp library), plus the launch count, CUDA-graph capture with SolverFeatherstone, the capacity refusal,
a closed-loop tracking run and the NB2_FP=fast twin."""

import itertools
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import newton_b200
import oracle.controller as oc
from newton_b200 import ModelBuilder, _lib, scenes
from newton_b200.controllers import ControllerJointImpedance, ControllerJointImpedanceModelFree
from tests.helpers import word_diff

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = -12345.0


def _fill(inp, rng, scale=None):
    """Seeded values in every live input tensor of ``inp`` (mass matrices symmetric positive definite)."""
    for name, t in vars(inp).items():
        if t is None:
            continue
        if name == "mass_matrix":
            a = rng.normal(size=t.shape)
            t.copy_(torch.from_numpy(np.einsum("rij,rkj->rik", a, a) + 0.5 * np.eye(t.shape[-1])))
        elif name in ("stiffness", "damping"):
            t.copy_(torch.from_numpy(rng.uniform(0.0, 80.0, t.shape)))
        else:
            t.copy_(torch.from_numpy(rng.uniform(-1.5, 1.5, t.shape)))


def _pair(make):
    """The same controller on the CPU (oracle) and on the GPU, with identical seeded inputs; returns (cpu, gpu, inputs, outputs)."""
    cpu, gpu = make("cpu"), make(DEV)
    ci, co = cpu.input(), cpu.output()
    _fill(ci, np.random.default_rng(7))
    co.joint_f.fill_(SENTINEL)
    gi, go = gpu.input(), gpu.output()
    for name, t in vars(ci).items():
        if t is not None:
            getattr(gi, name).copy_(t)
    go.joint_f.fill_(SENTINEL)
    return cpu, gpu, (ci, co), (gi, go)


def _check(cpu, gpu, c_io, g_io):
    oc.step(cpu, inputs=c_io[0], outputs=c_io[1])
    gpu.step(inputs=g_io[0], outputs=g_io[1])
    torch.cuda.synchronize()
    got, ref = g_io[1].joint_f.cpu().numpy(), c_io[1].joint_f.numpy()
    assert word_diff(got, ref) == 0, f"{word_diff(got, ref)} words differ, max |diff| {np.max(np.abs(got - ref))}"
    return ref


# ---- model-free: every term combination, baked and live gains ------------------------------------------------------------
MF_DOFS = (9, 8, 1, 9, 3, 8, 1, 2)


def _model_free(device, flags, live):
    rng = np.random.default_rng(11)
    total, R, D = sum(MF_DOFS), len(MF_DOFS), max(MF_DOFS)
    sim = total + 13  # partial maps: the flat sim arrays are larger than the controlled dofs

    def perm():
        return torch.from_numpy(rng.permutation(sim)[:total].astype(np.int64)).to(torch.uint32)

    gains = torch.from_numpy(rng.uniform(0.0, 60.0, (2, R, D)).astype(np.float32))
    g, c, m, qdd = flags
    return ControllerJointImpedanceModelFree(
        robot_count=R, dofs_per_robot=torch.tensor(MF_DOFS, dtype=torch.int32), max_dofs=D, default_dof_indices=perm(),
        stiffness=None if live else gains[0], damping=None if live else gains[1], use_gravity_compensation=g,
        use_coriolis_compensation=c, use_inertia_decoupling=m, has_qdd_feedforward=qdd, joint_q_idx=perm(), joint_qd_idx=perm(),
        joint_q_des_idx=perm(), joint_qdd_idx=perm(), gravity_force_idx=perm(), coriolis_force_idx=perm(),
        joint_f_idx=perm().to(torch.int32), device=device)


@pytest.mark.parametrize("live", [False, True], ids=["baked", "live"])
@pytest.mark.parametrize("flags", list(itertools.product([False, True], repeat=4)),
                         ids=lambda f: "g%dc%dm%dqdd%d" % tuple(map(int, f)))
def test_model_free_bit_exact(cuda_lib, flags, live):
    cpu, gpu, c_io, g_io = _pair(lambda dev: _model_free(dev, flags, live))
    ref = _check(cpu, gpu, c_io, g_io)
    written = np.zeros(ref.size, bool)
    written[cpu._ports["joint_f"].host] = True
    assert (ref[~written] == SENTINEL).all() and (ref[written] != SENTINEL).all()


# ---- model-based ---------------------------------------------------------------------------------------------------------
def _model_based(builder, device, seed=5, **kw):
    R, n = builder.articulation_count, builder.joint_dof_count
    qd = [*builder.joint_qd_start, n]
    D = max(qd[e] - qd[s] for s, e in zip(builder.articulation_start, builder.articulation_end))
    rng = np.random.default_rng(seed)
    kp = torch.from_numpy(rng.uniform(10.0, 100.0, (R, D)).astype(np.float32))
    kd = torch.from_numpy(rng.uniform(1.0, 20.0, (R, D)).astype(np.float32))
    perm = torch.from_numpy(rng.permutation(n).astype(np.int64))
    return ControllerJointImpedance(builder, default_dof_indices=perm, stiffness=kp, damping=kd, joint_q_des_idx=perm.flip(0),
                                    device=device, **kw)


def _model_based_check(builder, **kw):
    cpu, gpu, c_io, g_io = _pair(lambda dev: _model_based(builder, dev, **kw))
    _check(cpu, gpu, c_io, g_io)
    for name in ("joint_q", "joint_qd", "body_q", "body_qd"):
        got, ref = getattr(gpu._state, name).cpu().numpy(), getattr(cpu._state, name).numpy()
        if name.startswith("body") and not (cpu._use_inertia or cpu._use_gravity or cpu._use_coriolis):
            continue
        assert word_diff(got, ref) == 0, f"internal state.{name}: {word_diff(got, ref)} words differ"


@pytest.mark.parametrize("flags", [(True, True, True, True), (True, False, False, False), (False, True, False, True),
                                   (False, False, True, False), (False, False, False, False)],
                         ids=lambda f: "g%dc%dm%dqdd%d" % tuple(map(int, f)))
def test_model_based_heterogeneous_fleet_bit_exact(cuda_lib, flags):
    g, c, m, qdd = flags
    _model_based_check(scenes.impedance_fleet_builder(96, ("panda", "ant", "pendulum")), use_gravity_compensation=g,
                       use_coriolis_compensation=c, use_inertia_decoupling=m, has_qdd_feedforward=qdd)


def test_model_based_4096_pandas_bit_exact(cuda_lib):
    _model_based_check(scenes.impedance_fleet_builder(4096, ("panda",)), seed=42)


def _chain(links):
    b = ModelBuilder()
    parent = -1
    for i in range(links):
        link = b.add_link(mass=1.0 + 0.01 * i, com=(0.1, 0.0, 0.0), inertia=np.eye(3) * 0.01)
        b.add_joint_revolute(parent, link, parent_xform=np.array([0.2 if parent >= 0 else 0.0, 0, 0, 0, 0, 0, 1.0]),
                             axis=(0.0, 1.0, 0.0) if i % 2 else (0.0, 0.0, 1.0))
        parent = link
    b.add_articulation(list(range(links)))
    return b


def test_long_chain_with_fewer_warps_per_cta_bit_exact(cuda_lib):
    # 40 links: 7 * 40^2 + 106 * 40 + 2 words = 61.9 KB per warp, so dyn_launch_config takes 2 warps per CTA instead of 4
    b = scenes.ModelBuilder()
    for _ in range(3):
        b.add_world(_chain(40))
    _model_based_check(b)


def test_chain_past_capacity_is_refused_without_a_launch(cuda_lib):
    b = _chain(90)  # > 227 KB of shared memory for one warp
    ctrl = _model_based(b, DEV)
    inp, out = ctrl.input(), ctrl.output()
    n0 = _lib.kernel_launch_count()
    with pytest.raises(_lib.Nb2Error, match="NB2_ERR_CAPACITY"):
        ctrl.step(inputs=inp, outputs=out)
    assert _lib.kernel_launch_count() == n0


# ---- launches, graphs, closed loop --------------------------------------------------------------------------------------
def test_one_launch_per_step(cuda_lib):
    for ctrl in (_model_based(scenes.impedance_fleet_builder(8, ("panda", "ant")), DEV), _model_free(DEV, (True, True, True, True), True)):
        inp, out = ctrl.input(), ctrl.output()
        ctrl.step(inputs=inp, outputs=out)
        n0 = _lib.kernel_launch_count()
        for _ in range(5):
            ctrl.step(inputs=inp, outputs=out)
        assert _lib.kernel_launch_count() - n0 == 5


def _closed_loop_setup(robots, gravity_compensation=True):
    b = scenes.impedance_fleet_builder(robots, ("panda",))
    for k in range(b.joint_dof_count):
        b.joint_target_ke[k] = 0.0
        b.joint_target_kd[k] = 0.0
    model = b.finalize(device=DEV)
    newton_b200.eval_fk(model, model.joint_q, model.joint_qd, model)
    n = model.joint_dof_count
    ctrl = ControllerJointImpedance(b, default_dof_indices=torch.arange(n, dtype=torch.int32), stiffness=torch.full((robots, 9), 100.0),
                                    damping=torch.full((robots, 9), 20.0), use_gravity_compensation=gravity_compensation, device=DEV)
    lo, hi = np.array(b.joint_limit_lower, np.float32), np.array(b.joint_limit_upper, np.float32)
    rng = np.random.default_rng(3)
    q_des = torch.from_numpy(lo + (hi - lo) * rng.uniform(0.3, 0.7, n).astype(np.float32)).to(DEV)
    return model, ctrl, q_des


def test_graph_capture_of_controller_and_featherstone_replays_bit_equal(cuda_lib):
    model, ctrl, q_des = _closed_loop_setup(16)
    solver = newton_b200.solvers.SolverFeatherstone(model)
    dt = 0.001

    def run(graph):
        s = [model.state(), model.state()]
        ctl = model.control()
        inp = ctrl.input()
        inp.joint_q_des.copy_(q_des)
        out = ctrl.output()
        out.joint_f = ctl.joint_f

        def frame():
            inp.joint_q, inp.joint_qd = s[0].joint_q, s[0].joint_qd
            ctrl.step(inputs=inp, outputs=out, dt=dt)
            for _ in range(4):
                solver.step(s[0], s[1], ctl, None, dt)
                s.reverse()

        if graph:
            stream = torch.cuda.Stream()
            stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(stream):
                frame()
            torch.cuda.synchronize()
            for st in s:
                st.assign(model.state())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                frame()
            for _ in range(10):
                g.replay()
        else:
            for _ in range(10):
                frame()
        torch.cuda.synchronize()
        return s[0]

    eager, graph = run(False), run(True)
    assert not torch.equal(eager.joint_q, model.joint_q)
    for name in ("joint_q", "joint_qd", "body_q"):
        assert torch.equal(getattr(eager, name), getattr(graph, name)), name


def _closed_loop_error(gravity_compensation):
    model, ctrl, q_des = _closed_loop_setup(32, gravity_compensation)
    solver = newton_b200.solvers.SolverFeatherstone(model)
    s0, s1, ctl = model.state(), model.state(), model.control()
    inp, out = ctrl.input(), ctrl.output()
    inp.joint_q_des.copy_(q_des)
    out.joint_f = ctl.joint_f
    dt = 0.001
    for _ in range(2000):  # 2 s
        inp.joint_q, inp.joint_qd = s0.joint_q, s0.joint_qd
        ctrl.step(inputs=inp, outputs=out, dt=dt)
        solver.step(s0, s1, ctl, None, dt)
        s0, s1 = s1, s0
    torch.cuda.synchronize()
    assert torch.isfinite(s0.joint_q).all()
    return float((s0.joint_q - q_des).abs().max())


def test_closed_loop_tracking_with_and_without_gravity_compensation(cuda_lib):
    err = _closed_loop_error(True)
    assert err < 1e-3, f"max |q - q_des| after 2 s with full compensation: {err:.3e}"
    err_no_g = _closed_loop_error(False)
    assert err_no_g > 1e-2, f"without gravity compensation the steady-state error should be visible, got {err_no_g:.3e}"


def test_fast_fp_twin_within_tolerance(cuda_lib):
    env = dict(os.environ, NB2_FP="fast")
    env.pop("NB2_LIB", None)
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "controller_fast_fp_worker.py")], env=env, capture_output=True,
                       text=True, timeout=600, cwd=ROOT)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    res = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("CONTROLLER_FAST_FP ")][-1].split(" ", 1)[1])
    assert res["lib"] == "libnewton_b200_fast.so"
    for name in ("model_free", "model_based"):
        assert res[name] < 1e-4, f"{name}: relative error {res[name]:.3e} of the fast twin"

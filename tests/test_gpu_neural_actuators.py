"""CUDA learned actuator networks (actuator_neural_step_kernel) against the CPU oracle (oracle/oracle_neural_actuator.h), bit for
bit: every float32 word of the output, the computed output and every array of the next state after each step, over
{MLP, LSTM} x {delay, none} x {0, 1, 3 clamps} x {unique, duplicate effort indices}, N = 1 and N off the tile, network
shapes from narrow to the largest that fits one CTA, the 4096-quadruped group, CUDA-graph replay inside a Featherstone
frame, the masked reset on the device, the capacity refusal and the NB2_FP=fast twin."""

import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from newton_b200 import _abi, _lib, scenes
from newton_b200.actuators import (
    Actuator,
    ClampingDCMotor,
    ClampingMaxEffort,
    ClampingPositionBased,
    ControllerNeuralLSTM,
    ControllerNeuralMLP,
    Delay,
)
from tests import neural_nets as NN
from tests import test_actuators as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def on():
    import oracle
    import oracle.actuator as on

    oracle.build()
    return on


def _eq(got, ref, what):
    g, r = got.detach().cpu().contiguous().numpy(), ref.detach().contiguous().numpy()
    assert g.shape == r.shape, what
    np.testing.assert_array_equal(g.view(np.int32), r.view(np.int32), err_msg=what)


def _state_arrays(s):
    out = [(n, getattr(s.controller_state, n)) for n in type(s.controller_state).__dataclass_fields__]
    if s.delay_state is not None:
        out += [(n, getattr(s.delay_state, n)) for n in ("buffer_pos", "buffer_vel", "buffer_act", "num_pushes", "write_idx")]
    return out


def run_pair(on, act, steps=20, seed=0, reset_at=None, scale=1.0):
    """Step ``act`` (CPU) on the oracle and its device copy with the same seeded inputs; compare after every step.  Returns the
    launches per GPU step."""
    gact = act._rebuilt(DEV)
    n_q = int(max(act.pos_indices.max(), act.target_pos_indices.max())) + 1
    n_qd = int(max(act.indices.max(), act.effort_indices.max())) + 1
    st, ctl = T.io(n_q, n_qd)
    ctl.computed = torch.zeros(n_qd)
    act.control_computed_output_attr = gact.control_computed_output_attr = "computed"
    gst = types.SimpleNamespace(**{k: v.to(DEV) for k, v in vars(st).items()})
    gctl = types.SimpleNamespace(**{k: v.to(DEV) for k, v in vars(ctl).items()})
    rng = np.random.default_rng(seed)
    cs, gs = [act.state(), act.state()], [gact.state(), gact.state()]
    launches = []
    for k in range(steps):
        for name in ("joint_q", "joint_qd", "joint_target_q", "joint_target_qd", "joint_act"):
            obj, gobj = (st, gst) if name in ("joint_q", "joint_qd") else (ctl, gctl)
            t = getattr(obj, name)
            t.copy_(torch.from_numpy((rng.normal(size=t.shape) * scale).astype(np.float32)))
            getattr(gobj, name).copy_(t)
        for o in ("joint_f", "computed"):
            getattr(ctl, o).zero_()
            getattr(gctl, o).zero_()
        on.step(act, st, ctl, cs[0], cs[1])
        before = _lib.kernel_launch_count()
        gact.step(gst, gctl, gs[0], gs[1])
        launches.append(_lib.kernel_launch_count() - before)
        torch.cuda.synchronize()
        for o in ("joint_f", "computed"):
            _eq(getattr(gctl, o), getattr(ctl, o), f"step {k}: {o}")
        for (name, g), (_, r) in zip(_state_arrays(gs[1]), _state_arrays(cs[1])):
            _eq(g, r, f"step {k}: {name}")
        cs.reverse()
        gs.reverse()
        if reset_at == k:
            mask = torch.from_numpy(rng.random(act.num_actuators) < 0.5)
            on.reset(cs[0], mask)
            gs[0].reset(mask.to(DEV))
            torch.cuda.synchronize()
            for (name, g), (_, r) in zip(_state_arrays(gs[0]), _state_arrays(cs[0])):
                _eq(g, r, f"after reset: {name}")
    return launches


_CKPT = {}


def _controller(tmp, kind, shape="small", seed=0):
    """A seeded checkpoint per (kind, shape), written once per module."""
    key = (kind, shape, seed)
    if key not in _CKPT:
        path = os.path.join(tmp, f"{kind}_{shape}_{seed}.pt2")
        if kind == "mlp":
            widths, meta = {"narrow": ([2, 1], {}), "small": ([6, 16, 8, 1], {"input_idx": [0, 2, 5], "input_order": "vel_pos"}),
                            "headline": ([6, 32, 32, 32, 1], {"input_idx": [0, 1, 2]}),
                            "largest": ([2, 200, 1], {})}[shape]
            meta.update(pos_scale=1.3, vel_scale=0.4, effort_scale=7.0)
            acts = ["elu", "softsign", "sigmoid", "relu", "tanh"][: len(widths) - 2]
            NN.save(NN.mlp(widths, acts or "relu", seed=seed, scale=2.0), path, metadata=meta)
        else:
            H, L = {"narrow": (1, 1), "small": (8, 2), "headline": (32, 2), "largest": (48, 2)}[shape]
            NN.save(NN.lstm(H, L, seed=seed), path, metadata={"num_layers": L, "hidden_size": H, "pos_scale": 2.0,
                                                              "effort_scale": 3.0}, kind="lstm")
        _CKPT[key] = path
    cls = ControllerNeuralMLP if kind == "mlp" else ControllerNeuralLSTM
    return cls(_CKPT[key])


@pytest.fixture(scope="module")
def ckpt_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("neural"))


def _clamps(n, count, rng):
    lut = ClampingPositionBased(lookup_positions=(-1.0, 0.0, 0.5, 1.0), lookup_efforts=(0.5, 2.0, 2.0, 4.0))
    chain = [ClampingMaxEffort(T.f32(rng.uniform(0.5, 3.0, n).tolist())),
             ClampingDCMotor(T.f32(rng.uniform(1.0, 5.0, n).tolist()), T.f32(rng.uniform(0.5, 3.0, n).tolist()),
                             T.f32(rng.uniform(0.5, 5.0, n).tolist())), lut]
    return chain[:count]


@pytest.mark.parametrize("kind", ["mlp", "lstm"])
@pytest.mark.parametrize("delay", [False, True])
@pytest.mark.parametrize("clamps", [0, 1, 3])
@pytest.mark.parametrize("dup", [False, True])
def test_matrix_bit_exact(on, ckpt_dir, kind, delay, clamps, dup):
    n = 150  # one full tile and a partial one
    rng = np.random.default_rng(n + clamps)
    eff = rng.integers(0, 40, n).tolist() if dup else list(range(n))
    act = Actuator(T.i32(list(range(n))), _controller(ckpt_dir, kind), clamping=_clamps(n, clamps, rng),
                   delay=Delay(T.i32(rng.integers(0, 4, n).tolist()), 3) if delay else None, effort_indices=T.i32(eff),
                   pos_indices=T.i32(rng.permutation(n).tolist()))
    launches = run_pair(on, act, steps=12, seed=clamps, reset_at=6)
    assert set(launches) == {2 if dup else 1}


@pytest.mark.parametrize("kind", ["mlp", "lstm"])
@pytest.mark.parametrize("shape", ["narrow", "small", "headline", "largest"])
@pytest.mark.parametrize("n", [1, 257])
def test_shapes_bit_exact(on, ckpt_dir, kind, shape, n):
    ctrl = _controller(ckpt_dir, kind, shape, seed=1)
    if shape == "largest":
        assert ctrl.smem_bytes() > 100 * 1024  # well past the 48 KB default: the opt-in path
    run_pair(on, Actuator(T.i32(list(range(n))), ctrl), steps=6, seed=n, scale=2.0)


@pytest.mark.parametrize("kind", ["mlp", "lstm"])
def test_4096_quadrupeds_bit_exact(on, ckpt_dir, kind):
    model = scenes.quadruped_actuated_model(4096, device="cpu")
    pd = model.actuators[0]
    n = pd.num_actuators
    rng = np.random.default_rng(3)
    act = Actuator(pd.indices, _controller(ckpt_dir, kind, "headline", seed=2), pos_indices=pd.pos_indices,
                   delay=Delay(T.i32(rng.integers(1, 4, n).tolist()), 3),
                   clamping=[ClampingDCMotor(T.f32([20.0] * n), T.f32([8.0] * n), T.f32([30.0] * n))])
    assert n == 4096 * 12
    run_pair(on, act, steps=20, seed=4, scale=0.5)


def test_graph_replay_in_featherstone_frame(on, tmp_path):
    """ModelBuilder.add_actuator(ControllerNeuralLSTM, index=..., model_path="net.pt2") stepped inside a captured CUDA graph
    with SolverFeatherstone: the replays equal the eager frames and the oracle's, bit for bit."""
    import newton_b200
    import oracle
    from newton_b200 import JointType

    path = NN.save(NN.lstm(16, 2, seed=5), tmp_path / "net.pt2", metadata={"num_layers": 2, "hidden_size": 16,
                                                                            "effort_scale": 20.0}, kind="lstm")
    quad = scenes.quadruped_builder()
    for k, j in enumerate(j for j in range(quad.joint_count) if quad.joint_type[j] == JointType.REVOLUTE):
        dof = quad.joint_qd_start[j]
        quad.add_actuator(ControllerNeuralLSTM, index=dof, pos_index=quad.joint_q_start[j], model_path=path, delay_steps=1 + k % 3)
        quad.joint_target_ke[dof] = quad.joint_target_kd[dof] = 0.0
    b = newton_b200.ModelBuilder()
    b.replicate(quad, 16)
    b.add_ground_plane(cfg=quad.default_shape_cfg)
    cpu_model = b.finalize()
    model = cpu_model.to(DEV)
    act = model.actuators[0]
    assert act.is_graphable() and isinstance(act.controller, ControllerNeuralLSTM)
    frames, substeps, dt = 3, 10, 0.001

    def run(graph):
        s, a, ctl = [model.state(), model.state()], [act.state(), act.state()], model.control()
        solver = newton_b200.solvers.SolverFeatherstone(model)

        def frame():
            for _ in range(substeps):
                ctl.joint_f.zero_()
                act.step(s[0], ctl, a[0], a[1], dt)
                solver.step(s[0], s[1], ctl, None, dt)
                s.reverse()
                a.reverse()

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
    for name in ("joint_q", "joint_qd"):
        _eq(getattr(graph[0], name), getattr(eager[0], name).cpu(), f"graph vs eager: {name}")
    for (name, g), (_, e) in zip(_state_arrays(ga[0]), _state_arrays(ea[0])):
        _eq(g, e.cpu(), f"graph vs eager: {name}")
    cact = cpu_model.actuators[0]
    s, a, ctl = [cpu_model.state(), cpu_model.state()], [cact.state(), cact.state()], cpu_model.control()
    solver = oracle.SolverFeatherstone(cpu_model)
    for _ in range(frames * substeps):
        ctl.joint_f.zero_()
        on.step(cact, s[0], ctl, a[0], a[1], dt)
        solver.step(s[0], s[1], ctl, None, dt)
        s.reverse()
        a.reverse()
    for name in ("joint_q", "joint_qd"):
        _eq(getattr(graph[0], name), getattr(s[0], name), f"graph vs oracle: {name}")
    for (name, g), (_, r) in zip(_state_arrays(ga[0]), _state_arrays(a[0])):
        _eq(g, r, f"graph vs oracle: {name}")


def test_capacity_refused_before_launch(ckpt_dir, tmp_path):
    big = ControllerNeuralMLP(NN.save(NN.mlp([2, 240, 1]), tmp_path / "big.pt2"))
    before = _lib.kernel_launch_count()
    with pytest.raises(_lib.Nb2Error, match="NB2_ERR_CAPACITY"):
        Actuator(T.i32([0, 1], DEV), big)
    assert _lib.kernel_launch_count() == before
    assert big.smem_bytes() > _abi.ACTUATOR_SMEM_MAX


def test_fast_fp_twin_within_tolerance():
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "neural_fast_fp_worker.py")
    env = dict(os.environ, NB2_FP="fast")
    out = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    line = next(ln for ln in out.stdout.splitlines() if ln.startswith("NEURAL_FAST_FP "))
    res = json.loads(line.split(" ", 1)[1])
    assert res["lib"] == "libnewton_b200_fast.so"
    # contraction and fp32 transcendentals move each activation by a few ulps; over 20 steps of the LSTM state the
    # effort stays within 1e-4 of its scale
    assert res["mlp"] < 1e-4 and res["lstm"] < 1e-4, res

"""Learned actuator networks (ControllerNeuralMLP / ControllerNeuralLSTM from Torch checkpoints) on the CPU oracle
(oracle/oracle_neural_actuator.h): the reference's Torch-path known answers, 50 seeded steps of every format x controller
against the reference's ``_compute_torch`` sequence in torch float32 and against the same module in float64, every supported
activation and layout, delay / clamps / duplicate effort indices, the builder, Model.to and shards, and every refusal.

Tolerances.  The oracle rounds each multiply and add to fp32 in one fixed order; torch float32 sums its GEMMs in another, so
the two differ by a few fp32 ulps of the largest partial sum of each dot product.  The bar |oracle - ref| <= 1e-5 (1 + |ref|)
is ~80 ulps at 1: it covers the re-associated sums of these widths (<= 64 terms) with room, and the LSTM's state error stays
at that level because its gates contract it.  Against float64 the same bar holds: fp32 rounding is then the whole error."""

import warnings

import numpy as np
import pytest
import torch

from newton_b200 import ModelBuilder, _abi, _lib
from newton_b200.actuators import (
    Actuator,
    ClampingDCMotor,
    ClampingMaxEffort,
    ControllerNeuralLSTM,
    ControllerNeuralMLP,
    Delay,
    load_metadata,
)
from tests import neural_nets as NN
from tests import test_actuators as T


@pytest.fixture(scope="module")
def on():
    import oracle
    import oracle.actuator as on

    oracle.build()
    return on


def _quiet(fn, *a):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        return fn(*a)


def _bar(got, ref, tol=1e-5):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    err = np.max(np.abs(got - ref))
    assert err <= tol * (1 + np.max(np.abs(ref))), f"error {err} vs scale {np.max(np.abs(ref))}"


def _drive(on, act, steps, seed=0, io=None, dt=None, after=None):
    """Step ``act`` on the oracle with seeded inputs; returns the per-step (inputs, joint_f, state) history."""
    n = act.num_actuators
    n_q = int(max(act.pos_indices.max(), act.target_pos_indices.max())) + 1
    n_qd = int(max(act.indices.max(), act.effort_indices.max())) + 1
    st, ctl = io if io is not None else T.io(n_q, n_qd)
    rng = np.random.default_rng(seed)
    s = [act.state(), act.state()]
    out = []
    for k in range(steps):
        for t in (st.joint_q, st.joint_qd, ctl.joint_target_q, ctl.joint_target_qd, ctl.joint_act):
            t.copy_(torch.from_numpy(rng.normal(size=t.shape).astype(np.float32)))
        ctl.joint_f.zero_()
        on.step(act, st, ctl, s[0], s[1], dt)
        out.append((st.joint_q.clone(), st.joint_qd.clone(), ctl.joint_target_q.clone(), ctl.joint_f.clone()))
        s.reverse()
        if after is not None:
            after(k, s[0])
    return out, s[0]


# ---------------------------------------------------------------------------------------------------- reference known answers
def _bias_mlp(bias):
    net = torch.nn.Sequential(torch.nn.Linear(2, 1))
    with torch.no_grad():
        net[0].weight.fill_(0.0)
        net[0].bias.fill_(bias)
    return net


def test_pt2_bias_only_known_answer(on, tmp_path):
    path = NN.save(_bias_mlp(7.0), tmp_path / "mlp.pt2", metadata={"effort_scale": 2.0})
    ctrl = ControllerNeuralMLP(model_path=path)
    assert ctrl.effort_scale == 2.0 and ctrl.is_stateful() and ctrl.is_graphable()
    act = Actuator(T.i32([0]), ctrl)
    st, ctl = T.io(1, 1, joint_target_q=T.f32([1.0]))
    on.step(act, st, ctl, act.state(), act.state())
    assert ctl.joint_f.item() == 14.0  # bias 7 * effort_scale 2


def test_dict_and_pt2_metadata(tmp_path):
    d = _quiet(ControllerNeuralMLP, NN.save(_bias_mlp(5.0), tmp_path / "m.pt", "dict", {"effort_scale": 4.0}))
    assert d.effort_scale == 4.0
    p = ControllerNeuralMLP(NN.save(_bias_mlp(1.0), tmp_path / "m.pt2", metadata={"torque_scale": 3.0, "pos_scale": 0.5}))
    assert (p.effort_scale, p.pos_scale, p.vel_scale) == (3.0, 0.5, 1.0)
    assert (p.input_order, p.input_idx, p.history_length) == ("pos_vel", [0], 1)


@pytest.mark.parametrize("kind", ["mlp", "lstm"])
def test_target_pos_indices(on, tmp_path, kind):
    # the error reads target_pos[target_pos_indices], not target_pos[pos_indices] (reference :715-769, :880-936)
    net = _bias_mlp(0.0) if kind == "mlp" else NN.lstm(4)
    if kind == "mlp":
        with torch.no_grad():
            net[0].weight.copy_(torch.tensor([[1.0, 0.0]]))
    cls = ControllerNeuralMLP if kind == "mlp" else ControllerNeuralLSTM
    ctrl = cls(NN.save(net, tmp_path / "n.pt2", metadata={"num_layers": 1, "hidden_size": 4}, kind=kind))
    act = Actuator(T.i32([0, 1]), ctrl, pos_indices=T.i32([3, 4]), target_pos_indices=T.i32([5, 6]))
    st, ctl = T.io(7, 2, joint_q=T.f32([0, 0, 0, 0.25, 0.5, 0, 0]), joint_target_q=T.f32([9, 9, 9, 9, 9, 1.0, 2.0]))
    on.step(act, st, ctl, act.state(), act.state())
    e = torch.tensor([0.75, 1.5])
    if kind == "mlp":
        np.testing.assert_array_equal(ctl.joint_f.numpy(), e.numpy())
    else:
        hc = [torch.zeros(1, 2, 4), torch.zeros(1, 2, 4)]
        _bar(ctl.joint_f, NN.torch_lstm_step(net, {}, e, torch.zeros(2), hc))


def test_lstm_config(tmp_path):
    # from the module (TorchScript keeps the lstm attribute), with metadata int coercion, the mismatch and the missing config
    ts = _quiet(ControllerNeuralLSTM, NN.save(NN.lstm(6, 2), tmp_path / "a.pt", "ts", {"num_layers": "2"}, kind="lstm"))
    assert (ts.num_layers, ts.hidden_size) == (2, 6)
    d = _quiet(ControllerNeuralLSTM, NN.save(NN.lstm(6, 2), tmp_path / "b.pt", "dict", {"hidden_size": 6.0}, kind="lstm"))
    assert (d.num_layers, d.hidden_size) == (2, 6)
    p = ControllerNeuralLSTM(NN.save(NN.lstm(5, 1), tmp_path / "c.pt2", metadata={"num_layers": 1.0, "hidden_size": "5"}, kind="lstm"))
    assert (p.num_layers, p.hidden_size) == (1, 5) and isinstance(p.hidden_size, int)
    with pytest.raises(ValueError, match="Metadata 'hidden_size' .* is 7, but the network's LSTM has hidden_size=6"):
        _quiet(ControllerNeuralLSTM, NN.save(NN.lstm(6, 1), tmp_path / "d.pt", "dict", {"hidden_size": 7}, kind="lstm"))
    with pytest.raises(ValueError, match="Cannot determine the LSTM configuration"):
        ControllerNeuralLSTM(NN.save(NN.lstm(5, 1), tmp_path / "e.pt2", kind="lstm"))
    with pytest.raises(ValueError, match="network.lstm must not be bidirectional"):
        _quiet(ControllerNeuralLSTM, NN.save(NN.LSTMNet(4, 1, bidirectional=True), tmp_path / "f.pt", "dict", kind="lstm"))
    bad = NN.lstm(4)
    bad.lstm.batch_first = False
    with pytest.raises(ValueError, match="network.lstm.batch_first must be True"):
        _quiet(ControllerNeuralLSTM, NN.save(bad, tmp_path / "g.pt", "dict", kind="lstm"))
    bad = NN.LSTMNet(4)
    bad.lstm = torch.nn.LSTM(3, 4, batch_first=True)
    with pytest.raises(ValueError, match="network.lstm.input_size must be 2"):
        _quiet(ControllerNeuralLSTM, NN.save(bad, tmp_path / "h.pt", "dict", kind="lstm"))


@pytest.mark.parametrize("fmt, text", [("ts", "TorchScript checkpoints"), ("dict", "dict checkpoints")])
def test_deprecation_warnings_point_at_caller(tmp_path, fmt, text):
    path = NN.save(_bias_mlp(1.0), tmp_path / "m.pt", fmt)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        ControllerNeuralMLP(model_path=path)
    hits = [w for w in caught if text in str(w.message)]
    assert len(hits) == 1 and hits[0].category is DeprecationWarning
    assert hits[0].filename == __file__
    with pytest.warns(DeprecationWarning, match=text):
        ControllerNeuralLSTM(NN.save(NN.lstm(3), tmp_path / "l.pt", fmt, kind="lstm"))


def test_load_metadata_without_warning(tmp_path):
    paths = [NN.save(_bias_mlp(1.0), tmp_path / "m.pt", "ts", {"effort_scale": 3.0}),
             NN.save(_bias_mlp(1.0), tmp_path / "m.pt2", metadata={"effort_scale": 3.0}),
             NN.save(_bias_mlp(1.0), tmp_path / "d.pt", "dict", {"effort_scale": 3.0})]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        assert [load_metadata(p) for p in paths] == [{"effort_scale": 3.0}] * 3
    assert not [w for w in caught if "checkpoints" in str(w.message)]


def test_masked_reset(on, tmp_path):
    for ctrl in (ControllerNeuralMLP(NN.save(NN.mlp([4, 8, 1]), tmp_path / "m.pt2", metadata={"input_idx": [0, 3]})),
                 ControllerNeuralLSTM(NN.save(NN.lstm(4, 2), tmp_path / "l.pt2", metadata={"num_layers": 2, "hidden_size": 4},
                                              kind="lstm"))):
        act = Actuator(T.i32([0, 1, 2, 3]), ctrl)
        _, s = _drive(on, act, 5)
        cs = s.controller_state
        arrays = [getattr(cs, n) for n in ctrl._STATE_NAMES]
        before = [a.clone() for a in arrays]
        assert all(a.abs().min() > 0 for a in before)
        mask = torch.tensor([True, False, True, False])
        on.reset(s, mask)
        for a, b in zip(arrays, before):
            assert (a[:, mask] == 0).all() and torch.equal(a[:, ~mask], b[:, ~mask])
        on.reset(s)
        assert all((a == 0).all() for a in arrays)
        with pytest.raises(ValueError, match="mask length"):
            cs.reset(torch.tensor([True]))


# ---------------------------------------------------------------------------------------------------- 50 steps against torch
def _torch_run(net, meta, kind, hist, steps):
    """The reference's torch sequence, fed the oracle's recorded inputs: efforts per step (float32 and float64)."""
    out = []
    for dtype in (torch.float32, torch.float64):
        state = [torch.zeros(hist, dtype=dtype), torch.zeros(hist, dtype=dtype)]
        efforts = []
        for q, qd, tq, _ in steps:
            e, v = (tq - q).to(dtype), qd.to(dtype)
            step = NN.torch_mlp_step if kind == "mlp" else NN.torch_lstm_step
            efforts.append(step(net, meta, e, v, state, dtype))
        out.append(efforts)
        net.to(torch.float32)
    return out


@pytest.mark.parametrize("fmt", ["pt2", "ts", "dict"])
@pytest.mark.parametrize("kind", ["mlp", "lstm"])
def test_formats_against_torch_50_steps(on, tmp_path, fmt, kind):
    if kind == "mlp":
        meta = {"input_idx": [0, 1, 2], "pos_scale": 0.8, "vel_scale": 0.3, "effort_scale": 5.0}
        net = NN.mlp([6, 32, 32, 32, 1], "softsign", seed=3)
        hist = (3, 64)
    else:
        meta = {"num_layers": 2, "hidden_size": 16, "pos_scale": 1.5, "vel_scale": 0.2, "effort_scale": 4.0}
        net = NN.lstm(16, 2, seed=3)
        hist = (2, 64, 16)
    path = NN.save(net, tmp_path / f"n.{'pt2' if fmt == 'pt2' else 'pt'}", fmt, meta, kind)
    cls = ControllerNeuralMLP if kind == "mlp" else ControllerNeuralLSTM
    act = Actuator(T.i32(list(range(64))), _quiet(cls, path))
    steps, _ = _drive(on, act, 50, seed=7)
    f32, f64 = _torch_run(net, meta, kind, hist, steps)
    for k, (*_, got) in enumerate(steps):
        _bar(got, f32[k])
        _bar(got, f64[k])


# ---------------------------------------------------------------------------------------------------- coverage
@pytest.mark.parametrize("act_name", sorted(NN.ACTS))
def test_every_activation_and_bias_free_layers(on, tmp_path, act_name):
    meta = {"input_idx": [0, 2, 5], "input_order": "vel_pos", "pos_scale": 2.0}
    net = NN.mlp([6, 12, 10, 1], act_name, seed=1, bias=[True, False, False], scale=2.0)
    ctrl = ControllerNeuralMLP(NN.save(net, tmp_path / "m.pt2", metadata=meta))
    assert [b is None for _, b, _, _ in ctrl._mlp.layers] == [False, True, True]
    act = Actuator(T.i32(list(range(9))), ctrl)
    steps, s = _drive(on, act, 12, seed=2)
    f32, f64 = _torch_run(net, meta, "mlp", (6, 9), steps)
    for k, (*_, got) in enumerate(steps):
        _bar(got, f32[k])
        _bar(got, f64[k])
    # history roll: entry t of the last state holds the error and velocity of t steps before the last step
    for t in range(6):
        q, qd, tq, _ = steps[-1 - t]
        np.testing.assert_array_equal(s.controller_state.pos_error_history[t].numpy(), (tq - q).numpy())
        np.testing.assert_array_equal(s.controller_state.vel_history[t].numpy(), qd.numpy())


def test_lstm_bias_free(on, tmp_path):
    net = NN.lstm(6, 2, seed=4, bias=False, head_bias=False)
    ctrl = ControllerNeuralLSTM(NN.save(net, tmp_path / "l.pt2", metadata={"num_layers": 2, "hidden_size": 6}, kind="lstm"))
    steps, _ = _drive(on, Actuator(T.i32(list(range(5))), ctrl), 20, seed=4)
    f32, f64 = _torch_run(net, {}, "lstm", (2, 5, 6), steps)
    for k, (*_, got) in enumerate(steps):
        _bar(got, f32[k])
        _bar(got, f64[k])


@pytest.mark.parametrize("kind", ["mlp", "lstm"])
def test_delay_clamps_and_duplicate_effort_indices(on, tmp_path, kind):
    """The network sees the delayed target; the clamp chain and the serial sum of repeated effort indices follow."""
    meta = {"num_layers": 1, "hidden_size": 4, "input_idx": [0, 1]}
    net = NN.mlp([4, 8, 1], "tanh", seed=5, scale=3.0) if kind == "mlp" else NN.lstm(4, 1, seed=5)
    cls = ControllerNeuralMLP if kind == "mlp" else ControllerNeuralLSTM
    ctrl = cls(NN.save(net, tmp_path / "n.pt2", metadata=meta, kind=kind))
    n, delays = 6, [0, 1, 2, 3, 1, 2]
    clamps = [ClampingMaxEffort(T.f32([0.3] * n)), ClampingDCMotor(T.f32([0.5] * n), T.f32([2.0] * n), T.f32([0.4] * n))]
    act = Actuator(T.i32(list(range(n))), ctrl, delay=Delay(T.i32(delays), 3), clamping=clamps, effort_indices=T.i32([0, 1, 1, 2, 0, 1]))
    act.control_computed_output_attr = "computed"
    st, ctl = T.io(n, n)
    ctl.computed = torch.zeros(n)
    seen = []

    def record(k, _):
        ctl.computed.zero_()

    steps, _ = _drive(on, act, 10, seed=6, io=(st, ctl), after=record)
    hist = (2, n) if kind == "mlp" else (1, n, 4)
    state = [torch.zeros(hist), torch.zeros(hist)]
    for k, (q, qd, tq, f) in enumerate(steps):
        seen.append(tq)
        tp = torch.stack([seen[max(0, k - d)][i] if d else tq[i] for i, d in enumerate(delays)])
        fn = NN.torch_mlp_step if kind == "mlp" else NN.torch_lstm_step
        computed = fn(net, meta, tp - q, qd, state)
        applied = torch.clamp(computed, -0.3, 0.3)
        v = torch.clamp(qd, -2.0 * (1 + 0.4 / 0.5), 2.0 * (1 + 0.4 / 0.5))
        applied = torch.minimum(torch.maximum(applied, torch.maximum(0.5 * (-1 - v / 2.0), torch.tensor(-0.4))),
                                torch.minimum(0.5 * (1 - v / 2.0), torch.tensor(0.4)))
        want = torch.zeros(n)
        for i, e in enumerate([0, 1, 1, 2, 0, 1]):
            want[e] += applied[i]
        _bar(f, want)
    assert act.has_duplicate_effort_indices


def test_builder_groups_by_model_path_and_model_to_shard(on, tmp_path):
    a = NN.save(NN.mlp([2, 8, 1], seed=1), tmp_path / "a.pt2")
    b = NN.save(NN.lstm(4, seed=2), tmp_path / "b.pt2", metadata={"num_layers": 1, "hidden_size": 4}, kind="lstm")
    c = NN.save(NN.mlp([2, 4, 1], seed=9), tmp_path / "c.pt2")
    t, (j1, j2) = T.two_joint_template()
    t.add_actuator(ControllerNeuralMLP, index=t.joint_qd_start[j1], model_path=a, delay_steps=1)
    t.add_actuator(ControllerNeuralMLP, index=t.joint_qd_start[j2], model_path=a, delay_steps=2)
    t.add_actuator(ControllerNeuralLSTM, index=t.joint_qd_start[j2], model_path=b)
    t.add_actuator(ControllerNeuralMLP, index=t.joint_qd_start[j1], model_path=c)
    builder = ModelBuilder()
    builder.replicate(t, 4)
    model = builder.finalize()
    groups = sorted((type(x.controller).__name__, x.controller.model_path, x.num_actuators) for x in model.actuators)
    assert groups == sorted([("ControllerNeuralMLP", a, 8), ("ControllerNeuralLSTM", b, 4), ("ControllerNeuralMLP", c, 4)])
    moved = model.to("cpu")
    for x, y in zip(model.actuators, moved.actuators):
        assert torch.equal(x.controller.weights, y.controller.weights)
        outs = []
        for m, act in ((model, x), (moved, y)):
            st, ctl = m.state(), m.control()
            st.joint_q.normal_(generator=torch.Generator().manual_seed(1))
            ctl.joint_target_q.fill_(0.3)
            on.step(act, st, ctl, act.state(), act.state())
            outs.append(ctl.joint_f)
        assert torch.equal(*outs) and outs[0].abs().max() > 0
    shard = model.shard(1, 2)  # worlds 2 and 3: their actuators rebased, each group's network kept whole
    assert sorted(x.num_actuators for x in shard.actuators) == [2, 2, 4]
    for act in shard.actuators:
        full = next(x for x in model.actuators if x.controller.model_path == act.controller.model_path)
        assert torch.equal(act.controller.weights, full.controller.weights)
        assert act.indices.min() >= 0 and act.indices.max() < shard.joint_dof_count


def test_view_parameters_refused(tmp_path):
    from newton_b200.selection import ArticulationView

    ctrl = ControllerNeuralMLP(NN.save(NN.mlp([2, 4, 1]), tmp_path / "m.pt2"))
    with pytest.raises(AttributeError, match="no per-actuator parameter 'kp'"):
        ArticulationView._actuator_param(ctrl, "kp")


# ---------------------------------------------------------------------------------------------------- refusals
class _Doubled(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(2, 4)
        self.b = torch.nn.Linear(4, 1)

    def forward(self, x):
        return 2.0 * self.b(torch.tanh(self.a(x)))


def test_refusals(tmp_path):
    with pytest.raises(NotImplementedError, match="export the network with torch.export.save"):
        ControllerNeuralMLP(str(tmp_path / "net.onnx"))
    bad = torch.nn.Sequential(torch.nn.Linear(2, 4), torch.nn.LayerNorm(4), torch.nn.Linear(4, 1))
    with pytest.raises(NotImplementedError, match="unsupported layer LayerNorm"):
        _quiet(ControllerNeuralMLP, NN.save(bad, tmp_path / "ln.pt", "dict"))
    with pytest.raises(NotImplementedError, match="unsupported operation aten.layer_norm"):
        ControllerNeuralMLP(NN.save(bad, tmp_path / "ln.pt2"))
    # a custom forward whose extracted chain (Linear, tanh-less Linear) misreads the network: caught by the probe check
    net = _Doubled()
    with pytest.raises(NotImplementedError, match="differs from the weights read out of it"):
        _quiet(ControllerNeuralMLP, NN.save(net, tmp_path / "c.pt", "dict"))
    with pytest.raises(NotImplementedError, match="input width is 4, expected 2 \\* len\\(input_idx\\) = 2"):
        ControllerNeuralMLP(NN.save(NN.mlp([4, 8, 1]), tmp_path / "w.pt2"))
    with pytest.raises(NotImplementedError, match="output width is 2, expected 1"):
        ControllerNeuralMLP(NN.save(NN.mlp([2, 8, 2]), tmp_path / "o.pt2"))
    with pytest.raises(ValueError, match="input_order must be 'pos_vel' or 'vel_pos'; got 'x'"):
        ControllerNeuralMLP(NN.save(NN.mlp([2, 4, 1]), tmp_path / "i.pt2", metadata={"input_order": "x"}))
    with pytest.raises(ValueError, match="input_idx must contain non-negative integers"):
        ControllerNeuralMLP(NN.save(NN.mlp([2, 4, 1]), tmp_path / "j.pt2", metadata={"input_idx": [-1]}))
    with pytest.raises(ValueError, match="requires 'model_path' argument"):
        ControllerNeuralMLP.resolve_arguments({})
    with pytest.raises(ValueError, match="requires a non-empty 'model_path'"):
        ControllerNeuralLSTM.resolve_arguments({"model_path": ""})
    ctrl = ControllerNeuralMLP(NN.save(NN.mlp([2, 4, 1]), tmp_path / "ok.pt2"))
    with pytest.raises(NotImplementedError, match="not differentiable"):
        Actuator(T.i32([0]), ctrl, requires_grad=True)


def test_capacity_refused_with_sizes(tmp_path):
    # 2 * 240 * 128 floats of scratch + weights > 227 KB
    ctrl = ControllerNeuralMLP(NN.save(NN.mlp([2, 240, 1]), tmp_path / "big.pt2"))
    with pytest.raises(_lib.Nb2Error, match=r"NB2_ERR_CAPACITY: .* needs \d+ bytes per CTA .* one CTA holds 232448"):
        Actuator(T.i32([0]), ctrl)
    ok = ControllerNeuralMLP(NN.save(NN.mlp([2, 200, 1]), tmp_path / "fits.pt2"))
    assert ok.smem_bytes() <= _abi.ACTUATOR_SMEM_MAX
    Actuator(T.i32([0]), ok)


def test_graphable_and_state_shapes(tmp_path):
    m = ControllerNeuralMLP(NN.save(NN.mlp([6, 4, 1]), tmp_path / "m.pt2", metadata={"input_idx": [0, 2, 5]}))
    st = m.state(7, "cpu")
    assert st.pos_error_history.shape == (6, 7) and st.vel_history.dtype == torch.float32
    lstm = ControllerNeuralLSTM(NN.save(NN.lstm(5, 3), tmp_path / "l.pt2", metadata={"num_layers": 3, "hidden_size": 5}, kind="lstm"))
    st = lstm.state(7, "cpu")
    assert st.hidden.shape == (3, 7, 5) and st.cell.shape == (3, 7, 5)
    act = Actuator(T.i32([0, 1]), lstm)
    assert act.is_graphable() and act.is_stateful()

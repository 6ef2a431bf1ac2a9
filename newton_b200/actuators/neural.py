"""Learned actuator networks (reference ``ControllerNeuralMLP`` / ``ControllerNeuralLSTM``, ``actuators/controllers/``) from
Torch checkpoints, stepped inside the fused actuator kernel (``csrc/nb2_actuator.cu``, ``actuator_neural_step_kernel``).

A checkpoint is loaded once on the host, its weights are read out of the module without running it, checked against one run
of the module on a seeded probe batch, and packed into one device buffer in the layout the kernel reads
(``include/newton_b200.h``, ``nb2_actuator_network``).  There is no torch path at step time: a network this module does not
recognise is refused at construction.

Checkpoint formats (the reference's Torch branch, ``actuators/utils.py``): ``.pt2`` from ``torch.export.save`` (preferred),
and the deprecated ``.pt`` from ``torch.jit.save`` and ``.pt`` / ``.pth`` from ``torch.save({"model": module, "metadata": {...}})``.
Metadata is a ``metadata.json`` extra file of the archive, or the dict's ``"metadata"``.
"""

from __future__ import annotations

import json
import os
import warnings
import zipfile
from dataclasses import dataclass
from typing import Any, ClassVar

import numpy as np
import torch

from .. import _abi
from .components import Controller

_METADATA_FILE = "metadata.json"
_TORCH_SUFFIXES = (".pt", ".pth", ".pt2")

# probe check: batch size, LSTM steps and the bound |module - extracted| <= _PROBE_TOL * (1 + |extracted|), float32 against
# float64 (fp32 rounding of a few dozen chained dot products stays below 1e-5 relative; a misread network is off by O(1))
_PROBE_BATCH, _PROBE_STEPS, _PROBE_TOL = 16, 3, 1e-4


def _archive_entries(path: str) -> set[str]:
    """Zip entry names with the archive-name prefix torch adds stripped (empty for a non-zip file)."""
    try:
        with zipfile.ZipFile(path) as zf:
            return {name.split("/", 1)[-1] for name in zf.namelist()}
    except (OSError, zipfile.BadZipFile):
        return set()


def _parse_metadata_json(text, path: str) -> dict[str, Any]:
    if not text:
        return {}
    try:
        metadata = json.loads(text)
    except json.JSONDecodeError as exc:
        raise ValueError(f"Invalid JSON in checkpoint metadata for '{path}'") from exc
    if not isinstance(metadata, dict):
        raise ValueError(f"Invalid checkpoint metadata for '{path}': expected a JSON object, got {type(metadata).__name__}")
    return metadata


def _check_path(path: str) -> None:
    ext = os.path.splitext(str(path))[1].lower()
    if ext == ".onnx":
        raise NotImplementedError(f"ONNX checkpoints are not supported ('{path}'); export the network with torch.export.save "
                                  f"to a .pt2 archive instead")
    if ext not in _TORCH_SUFFIXES:
        raise ValueError(f"Unsupported checkpoint '{path}': expected a .pt2, .pt or .pth Torch checkpoint")


def _load_torch_raw(path: str, warn: bool = True, stacklevel: int = 2) -> tuple[Any, dict[str, Any]]:
    """``(module, metadata)`` of a pt2 / TorchScript / dict checkpoint.  ``stacklevel`` of the deprecation warnings counts from
    this function's caller."""
    entries = _archive_entries(path)
    if "archive_format" in entries or "serialized_exported_program.json" in entries:
        extra = {_METADATA_FILE: ""}
        exported = torch.export.load(path, extra_files=extra)
        return exported.module(), _parse_metadata_json(extra[_METADATA_FILE], path)
    if "constants.pkl" in entries:  # torch.jit.save always writes constants.pkl; torch.save archives do not
        extra = {_METADATA_FILE: ""}
        net = torch.jit.load(path, map_location="cpu", _extra_files=extra)
        if warn:
            warnings.warn(f"Loading TorchScript checkpoints (torch.jit.save) is deprecated; re-export '{path}' as a pt2 archive "
                          f"via torch.export.save().", DeprecationWarning, stacklevel=stacklevel + 1)
        net.eval()
        return net, _parse_metadata_json(extra[_METADATA_FILE], path)
    checkpoint = torch.load(path, map_location="cpu", weights_only=False)
    if isinstance(checkpoint, dict):
        if "model" not in checkpoint:
            raise ValueError(f"Cannot load checkpoint at '{path}'; dict checkpoint has no 'model' key")
        if warn:
            warnings.warn(f"Loading dict checkpoints (torch.save) is deprecated; re-export '{path}' as a pt2 archive via "
                          f"torch.export.save().", DeprecationWarning, stacklevel=stacklevel + 1)
        net = checkpoint["model"]
        if hasattr(net, "eval"):
            net.eval()
        return net, checkpoint.get("metadata", {})
    raise ValueError(f"Cannot load checkpoint at '{path}'; expected a pt2 archive (torch.export.save), a TorchScript archive, "
                     f"or a dict with a 'model' key")


def load_metadata(path: str) -> dict[str, Any]:
    """The metadata of a Torch checkpoint, read from the archive's ``metadata.json`` entry without loading the network (a dict
    checkpoint keeps it inside the pickle and is loaded, without the deprecation warning)."""
    _check_path(path)
    try:
        with zipfile.ZipFile(path) as zf:
            entries = {name.split("/", 1)[-1]: name for name in zf.namelist()}
            entry = entries.get(f"extra/{_METADATA_FILE}") or entries.get(_METADATA_FILE)
            if entry is not None:
                return _parse_metadata_json(zf.read(entry), path)
            if "archive_format" in entries or "constants.pkl" in entries or "serialized_exported_program.json" in entries:
                return {}
    except (OSError, zipfile.BadZipFile):
        pass
    return _load_torch_raw(path, warn=False)[1]


# ---------------------------------------------------------------------------------------------------- reading the network
_ACT_MODULES = {"ReLU": _abi.NET_RELU, "ELU": _abi.NET_ELU, "Tanh": _abi.NET_TANH, "Sigmoid": _abi.NET_SIGMOID,
                "Softsign": _abi.NET_SOFTSIGN}
_ACT_NAMES = {v: k for k, v in _ACT_MODULES.items()}


def _f64(t) -> np.ndarray:
    return t.detach().to("cpu", torch.float64).numpy().copy()


def _kind(module) -> str:
    return getattr(module, "original_name", None) or type(module).__name__


def _mlp_chain_from_graph(gm) -> list:
    """``[("linear", W, b) | ("act", kind, alpha)]`` from a ``torch.export`` graph: a flat chain of aten.linear and the supported
    activations (Softsign appears as abs -> add(1) -> div)."""
    params = dict(gm.named_parameters())
    params.update(dict(gm.named_buffers()))

    def tensor(node):
        if node is None:
            return None
        if getattr(node, "op", None) != "get_attr" or node.target not in params:
            raise NotImplementedError(f"the network's Linear weights must be parameters, got {node}")
        return params[node.target]

    chain, pending_abs = [], {}
    for node in gm.graph.nodes:
        if node.op in ("placeholder", "get_attr", "output") or (node.op == "call_module" and str(node.target).startswith("_guards")):
            continue
        name = str(node.target)
        if name == "aten.linear.default":
            chain.append(("linear", tensor(node.args[1]), tensor(node.args[2] if len(node.args) > 2 else None)))
        elif name == "aten.relu.default":
            chain.append(("act", _abi.NET_RELU, 1.0))
        elif name == "aten.elu.default":
            alpha = float(node.args[1]) if len(node.args) > 1 else 1.0
            if any(float(a) != 1.0 for a in node.args[2:4]):
                raise NotImplementedError("the network's ELU has a scale or input_scale other than 1")
            chain.append(("act", _abi.NET_ELU, alpha))
        elif name == "aten.tanh.default":
            chain.append(("act", _abi.NET_TANH, 1.0))
        elif name == "aten.sigmoid.default":
            chain.append(("act", _abi.NET_SIGMOID, 1.0))
        elif name == "aten.abs.default":
            pending_abs[node] = node.args[0]
        elif name == "aten.add.Tensor" and node.args[0] in pending_abs and node.args[1] == 1:
            pending_abs[node] = pending_abs[node.args[0]]
        elif name == "aten.div.Tensor" and node.args[1] in pending_abs and pending_abs[node.args[1]] is node.args[0]:
            chain.append(("act", _abi.NET_SOFTSIGN, 1.0))
        else:
            raise NotImplementedError(f"unsupported operation {name} in the network's graph")
    return chain


def _mlp_chain_from_modules(module) -> list:
    """The chain from the leaf modules in registration order (``nn.Sequential``, TorchScript submodules)."""
    children = list(module.named_children())
    if not children:
        raise NotImplementedError(f"unsupported layer {_kind(module)}: the network holds no Linear / activation modules")
    chain = []
    for name, child in children:
        kind = _kind(child)
        if kind == "Linear":
            chain.append(("linear", child.weight, getattr(child, "bias", None)))
        elif kind in _ACT_MODULES:
            alpha = float(getattr(child, "alpha", 1.0)) if kind == "ELU" else 1.0
            chain.append(("act", _ACT_MODULES[kind], alpha))
        elif list(child.named_children()):
            chain += _mlp_chain_from_modules(child)
        else:
            raise NotImplementedError(f"unsupported layer {kind} ('{name}'); an MLP is Linear layers with ReLU, ELU, Tanh, "
                                      f"Sigmoid or Softsign between them")
    return chain


@dataclass
class _Mlp:
    layers: list  # (W float64 [out, in], b float64 [out] or None, activation kind, alpha)


def _read_mlp(net) -> _Mlp:
    chain = _mlp_chain_from_graph(net) if isinstance(net, torch.fx.GraphModule) else _mlp_chain_from_modules(net)
    layers = []
    for item in chain:
        if item[0] == "linear":
            layers.append([_f64(item[1]), None if item[2] is None else _f64(item[2]), _abi.NET_NONE, 1.0])
        else:
            if not layers or layers[-1][2] != _abi.NET_NONE:
                raise NotImplementedError(f"unsupported network: {_ACT_NAMES[item[1]]} must follow a Linear layer")
            layers[-1][2], layers[-1][3] = item[1], item[2]
    if not layers:
        raise NotImplementedError("unsupported network: no Linear layer found")
    if layers[-1][2] != _abi.NET_NONE:
        raise NotImplementedError("unsupported network: the last layer must be a Linear layer without activation")
    for (w, _, _, _), (w2, _, _, _) in zip(layers, layers[1:]):
        if w2.shape[1] != w.shape[0]:
            raise NotImplementedError(f"unsupported network: Linear widths {w.shape[0]} -> {w2.shape[1]} do not chain")
    if len(layers) > _abi.NET_MAX_LAYERS:
        raise NotImplementedError(f"unsupported network: {len(layers)} Linear layers, at most {_abi.NET_MAX_LAYERS}")
    return _Mlp([tuple(layer) for layer in layers])


def _act64(kind: int, a: np.ndarray, alpha: float) -> np.ndarray:
    if kind == _abi.NET_RELU:
        return np.where(a < 0, 0.0, a)
    if kind == _abi.NET_ELU:
        return np.where(a > 0, a, alpha * np.expm1(a))
    if kind == _abi.NET_TANH:
        return np.tanh(a)
    if kind == _abi.NET_SIGMOID:
        return 1.0 / (1.0 + np.exp(-a))
    if kind == _abi.NET_SOFTSIGN:
        return a / (1.0 + np.abs(a))
    return a


def _mlp_forward64(mlp: _Mlp, x: np.ndarray) -> np.ndarray:
    for w, b, kind, alpha in mlp.layers:
        x = x @ w.T + (b if b is not None else 0.0)
        x = _act64(kind, x, alpha)
    return x


@dataclass
class _Lstm:
    layers: list  # (W_ih [4H, in], W_hh [4H, H], b_ih [4H] or None, b_hh [4H] or None), float64
    head_w: np.ndarray  # [1, H]
    head_b: np.ndarray | None


def _read_lstm(net, num_layers: int, hidden_size: int) -> _Lstm:
    """The LSTM and its one ``Linear(hidden_size, 1)`` head from the module's parameters (every format names them alike)."""
    params = dict(net.named_parameters())
    lstm_keys = [k for k in params if k.rsplit(".", 1)[-1].startswith(("weight_ih_l", "weight_hh_l", "bias_ih_l", "bias_hh_l"))]
    prefixes = {k.rsplit(".", 1)[0] if "." in k else "" for k in lstm_keys}
    if len(prefixes) != 1:
        raise NotImplementedError(f"unsupported network: expected exactly one nn.LSTM, found {len(prefixes)}")
    prefix = next(iter(prefixes))
    p = (prefix + ".") if prefix else ""
    if any(k.endswith("_reverse") for k in lstm_keys) or any("weight_hr_l" in k for k in params):
        raise NotImplementedError("unsupported network: the LSTM is bidirectional or projected")
    found = sorted({int(k.rsplit("_l", 1)[1]) for k in lstm_keys})
    if found != list(range(num_layers)):
        raise ValueError(f"the network's LSTM has {len(found)} layers, the configuration says num_layers={num_layers}")
    has_bias = f"{p}bias_ih_l0" in params
    layers = []
    for k in range(num_layers):
        w_ih, w_hh = _f64(params[f"{p}weight_ih_l{k}"]), _f64(params[f"{p}weight_hh_l{k}"])
        if w_hh.shape != (4 * hidden_size, hidden_size) or w_ih.shape != (4 * hidden_size, 2 if k == 0 else hidden_size):
            raise ValueError(f"the network's LSTM layer {k} has weights {w_ih.shape} / {w_hh.shape}, which do not match "
                             f"hidden_size={hidden_size}")
        b = (_f64(params[f"{p}bias_ih_l{k}"]), _f64(params[f"{p}bias_hh_l{k}"])) if has_bias else (None, None)
        layers.append((w_ih, w_hh, *b))
    rest = {k: v for k, v in params.items() if k not in lstm_keys}
    weights = [k for k in rest if k.endswith("weight")]
    if len(weights) != 1 or set(rest) - {weights[0], weights[0][:-6] + "bias"}:
        raise NotImplementedError(f"unsupported network: expected exactly one Linear head after the LSTM, found parameters "
                                  f"{sorted(rest)}")
    head_w = _f64(rest[weights[0]])
    head_b = rest.get(weights[0][:-6] + "bias")
    if head_w.shape != (1, hidden_size):
        raise NotImplementedError(f"unsupported network: the head is Linear{tuple(head_w.shape[::-1])}, expected "
                                  f"Linear({hidden_size}, 1)")
    return _Lstm(layers, head_w, None if head_b is None else _f64(head_b))


def _sig(a):
    return 1.0 / (1.0 + np.exp(-a))


def _lstm_forward64(lstm: _Lstm, x: np.ndarray, h: np.ndarray, c: np.ndarray):
    """One step: x [B, 2], h / c [L, B, H] -> (effort [B, 1], h', c')."""
    h2, c2 = np.empty_like(h), np.empty_like(c)
    for k, (w_ih, w_hh, b_ih, b_hh) in enumerate(lstm.layers):
        a = x @ w_ih.T + h[k] @ w_hh.T
        if b_ih is not None:
            a = a + b_ih + b_hh
        i, f, g, o = np.split(a, 4, axis=1)
        c2[k] = _sig(f) * c[k] + _sig(i) * np.tanh(g)
        h2[k] = _sig(o) * np.tanh(c2[k])
        x = h2[k]
    y = x @ lstm.head_w.T + (lstm.head_b if lstm.head_b is not None else 0.0)
    return y, h2, c2


def _probe_fail(what: str, err: float, bound: float, path: str) -> NotImplementedError:
    return NotImplementedError(f"'{path}': the network's {what} differs from the weights read out of it ({err:.3g} > {bound:.3g}); "
                               f"its forward is not the supported chain (a custom forward or an unrecognised layer)")


def _close(got, want) -> tuple[float, float]:
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err = float(np.max(np.abs(got - want))) if got.size else 0.0
    return err, _PROBE_TOL * (1.0 + float(np.max(np.abs(want)) if want.size else 0.0))


def _run_module(net, *args):
    with torch.inference_mode():
        return net(*args)


# ---------------------------------------------------------------------------------------------------- the controllers
class _NeuralController(Controller):
    SHARED_PARAMS: ClassVar[set[str]] = {"model_path"}
    _KIND: ClassVar[int]

    @classmethod
    def resolve_arguments(cls, args: dict[str, Any]) -> dict[str, Any]:
        if "model_path" not in args:
            raise ValueError(f"{cls.__name__} requires 'model_path' argument")
        model_path = args["model_path"]
        if not model_path:
            raise ValueError(f"{cls.__name__} requires a non-empty 'model_path'")
        return {"model_path": model_path}

    def __init__(self, model_path: str):
        """Load ``model_path`` (``.pt2``, or the deprecated TorchScript ``.pt`` / dict ``.pt`` / ``.pth``), read and check its
        network and pack its weights.  Unsupported networks raise ``NotImplementedError``."""
        model_path = str(model_path)
        _check_path(model_path)
        self.model_path = model_path
        self.network, metadata = _load_torch_raw(model_path, stacklevel=2)  # the caller of the constructor
        self.metadata = metadata
        self.pos_scale = metadata.get("pos_scale", 1.0)
        self.vel_scale = metadata.get("vel_scale", 1.0)
        self.effort_scale = metadata.get("effort_scale", metadata.get("torque_scale", 1.0))
        self._configure(metadata)
        self.weights = torch.from_numpy(self._pack())  # float32, padded to whole float4s; moved to the device in finalize
        self._num_actuators = 0

    def finalize(self, device, num_actuators: int) -> None:
        self.weights = self.weights.to(device).contiguous()  # whole: the group shares one network (moved again by Model.to)
        self._num_actuators = num_actuators

    def is_stateful(self) -> bool:
        return True

    def is_graphable(self) -> bool:
        """True: the step is one fused kernel.  (The reference's Torch path runs the module through torch and is not.)"""
        return True

    def smem_bytes(self, lookup_entries: int = 0) -> int:
        """Shared memory of one CTA of the fused kernel (include/newton_b200.h, nb2_actuator_network)."""
        return 4 * (int(self.weights.numel()) + 2 * lookup_entries + self._scratch_floats())

    def _network_desc(self, current, nxt) -> _abi.ActuatorNetwork:
        w = _abi.ActuatorNetwork()
        w.weights = self.weights.data_ptr()
        w.weight_count = self._weight_count
        w.pos_scale, w.vel_scale, w.effort_scale = float(self.pos_scale), float(self.vel_scale), float(self.effort_scale)
        self._fill(w)
        n, dev, P = self._num_actuators, self.weights.device, _abi.ptr
        names = self._STATE_NAMES
        size = self._state_numel(n)
        w.state0_in, w.state1_in = (P(getattr(current, a), "f32", dev, size, f"current {a}") for a in names)
        w.state0_out, w.state1_out = (P(getattr(nxt, a), "f32", dev, size, f"next {a}") for a in names)
        if {w.state0_in, w.state1_in} & {w.state0_out, w.state1_out}:
            raise ValueError("current_act_state and next_act_state share network state storage")
        return w


def _reset_columns(mask, rows: int, width: int, a, b) -> None:
    """One ``nb2_actuator_network_reset`` launch (or its CPU oracle when the state lives on the host)."""
    from .actuator import _call

    n = int(a.shape[1])
    if mask is not None:
        if getattr(mask, "dtype", None) is not torch.bool or mask.dim() != 1:
            raise ValueError("reset mask must be a one-dimensional Boolean array")
        if len(mask) != n:
            raise ValueError(f"reset mask length ({len(mask)}) must match the actuator count ({n})")
        if str(mask.device) != str(a.device):
            raise ValueError(f"reset mask device ({mask.device}) must match the state device ({a.device})")
    P, dev = _abi.ptr, a.device
    _call("network_reset", dev, n, rows, width, P(mask, "bool", dev, n, "mask"), P(a, "f32", dev, a.numel(), "state"),
          P(b, "f32", dev, b.numel(), "state"))


class ControllerNeuralMLP(_NeuralController):
    """MLP actuator network (reference ``ControllerNeuralMLP``, Torch checkpoints): ``effort = net(x) * effort_scale`` with
    ``x`` the scaled position errors and joint velocities of the steps ``input_idx`` (0 = now, k = k steps ago), concatenated
    in ``input_order``.

    Supported networks: ``Linear -> act -> Linear -> ... -> Linear(., 1)`` with ``act`` one of ReLU, ELU(alpha), Tanh, Sigmoid,
    Softsign, biases optional, first width ``2 * len(input_idx)``.  Metadata: ``input_order`` ("pos_vel" / "vel_pos"),
    ``input_idx`` (default ``[0]``), ``pos_scale``, ``vel_scale``, ``effort_scale`` (or ``torque_scale``), all defaulting to 1."""

    _KIND = _abi.ACT_MLP
    _STATE_NAMES = ("pos_error_history", "vel_history")

    @dataclass
    class State(Controller.State):
        """History buffers of the MLP controller."""

        pos_error_history: Any = None
        """Position error history, shape ``[history_length, N]``."""
        vel_history: Any = None
        """Joint velocity history [m/s or rad/s], shape ``[history_length, N]``."""

        def reset(self, mask=None) -> None:
            """Zero every entry (``mask=None``) or the ``True`` actuators' columns, on the device."""
            _reset_columns(mask, int(self.pos_error_history.shape[0]), 1, self.pos_error_history, self.vel_history)

    def _configure(self, metadata) -> None:
        self.input_order = metadata.get("input_order", "pos_vel")
        if self.input_order not in ("pos_vel", "vel_pos"):
            raise ValueError(f"input_order must be 'pos_vel' or 'vel_pos'; got '{self.input_order}'")
        self.input_idx = list(metadata.get("input_idx", [0]))
        if any(i < 0 for i in self.input_idx):
            raise ValueError(f"input_idx must contain non-negative integers; got {self.input_idx}")
        if not 1 <= len(self.input_idx) <= _abi.NET_MAX_INPUTS:
            raise NotImplementedError(f"input_idx holds {len(self.input_idx)} entries; 1 to {_abi.NET_MAX_INPUTS} are supported")
        self.history_length = max(self.input_idx) + 1
        self._mlp = _read_mlp(self.network)
        widths = [self._mlp.layers[0][0].shape[1]] + [w.shape[0] for w, *_ in self._mlp.layers]
        if widths[0] != 2 * len(self.input_idx):
            raise NotImplementedError(f"the network's input width is {widths[0]}, expected 2 * len(input_idx) = "
                                      f"{2 * len(self.input_idx)}")
        if widths[-1] != 1:
            raise NotImplementedError(f"the network's output width is {widths[-1]}, expected 1 (one effort per actuator)")
        self.widths = widths
        self._probe()

    def _probe(self) -> None:
        x = np.random.default_rng(0).normal(size=(_PROBE_BATCH, self.widths[0]))
        try:
            got = _run_module(self.network, torch.from_numpy(x.astype(np.float32)))
        except Exception as exc:  # noqa: BLE001 - any failure of the module's own forward on the probe is a refusal
            raise NotImplementedError(f"'{self.model_path}': the network does not run on a [{_PROBE_BATCH}, {self.widths[0]}] "
                                      f"float32 batch: {exc}") from exc
        got = got[0] if isinstance(got, (tuple, list)) else got
        want = _mlp_forward64(self._mlp, x)
        if tuple(got.shape) != want.shape:
            raise NotImplementedError(f"'{self.model_path}': the network's output has shape {tuple(got.shape)}, expected "
                                      f"{want.shape}")
        err, bound = _close(got.double().numpy(), want)
        if not err <= bound:
            raise _probe_fail("output", err, bound, self.model_path)

    def _pack(self) -> np.ndarray:
        parts = []
        for w, b, _, _ in self._mlp.layers:
            parts.append(w.astype(np.float32).ravel())
            if b is not None:
                parts.append(b.astype(np.float32))
        flat = np.concatenate(parts)
        self._weight_count = int(flat.size)
        return np.concatenate([flat, np.zeros((-flat.size) % 4, np.float32)])

    def _scratch_floats(self) -> int:
        return 2 * max(self.widths) * _abi.NET_TILE

    def _fill(self, w) -> None:
        w.layer_count = len(self._mlp.layers)
        for k, width in enumerate(self.widths):
            w.widths[k] = width
        for k, (_, b, kind, alpha) in enumerate(self._mlp.layers):
            w.activation[k], w.alpha[k], w.has_bias[k] = kind, alpha, b is not None
        w.input_count = len(self.input_idx)
        for q, k in enumerate(self.input_idx):
            w.input_idx[q] = k
        w.vel_first = self.input_order == "vel_pos"
        w.history_length = self.history_length

    def _state_numel(self, n: int) -> int:
        return self.history_length * n

    def state(self, num_actuators: int, device) -> ControllerNeuralMLP.State:
        shape = (self.history_length, num_actuators)
        return ControllerNeuralMLP.State(pos_error_history=torch.zeros(shape, dtype=torch.float32, device=device),
                                         vel_history=torch.zeros(shape, dtype=torch.float32, device=device))


class ControllerNeuralLSTM(_NeuralController):
    """LSTM actuator network (reference ``ControllerNeuralLSTM``, Torch checkpoints): input ``[e * pos_scale, v * vel_scale]``
    for one time step, state ``(h, c)`` per layer, ``effort = head(h_top) * effort_scale``.

    Supported networks: one ``nn.LSTM`` (``batch_first=True``, ``input_size=2``, unidirectional, ``proj_size=0``, with or
    without bias) and exactly one ``Linear(hidden_size, 1)`` head on the last time step's output, called as
    ``net(x, (h, c)) -> (effort, (h, c))``.  ``num_layers`` / ``hidden_size`` come from the module's ``lstm`` attribute or
    from the metadata (which a ``.pt2`` archive must carry)."""

    _KIND = _abi.ACT_LSTM
    _STATE_NAMES = ("hidden", "cell")

    @dataclass
    class State(Controller.State):
        """Hidden and cell state of the LSTM controller."""

        hidden: Any = None
        """Hidden state, shape ``[num_layers, N, hidden_size]``."""
        cell: Any = None
        """Cell state, shape ``[num_layers, N, hidden_size]``."""

        def reset(self, mask=None) -> None:
            """Zero every entry (``mask=None``) or the ``True`` actuators' columns, on the device."""
            _reset_columns(mask, int(self.hidden.shape[0]), int(self.hidden.shape[2]), self.hidden, self.cell)

    def _configure(self, metadata) -> None:
        path = self.model_path
        lstm = getattr(self.network, "lstm", None)
        if lstm is not None and hasattr(lstm, "num_layers"):
            if not lstm.batch_first:
                raise ValueError("network.lstm.batch_first must be True")
            if lstm.input_size != 2:
                raise ValueError(f"network.lstm.input_size must be 2 (pos_error, vel); got {lstm.input_size}")
            if lstm.bidirectional:
                raise ValueError("network.lstm must not be bidirectional")
            if getattr(lstm, "proj_size", 0) != 0:
                raise ValueError(f"network.lstm.proj_size must be 0; got {lstm.proj_size}")
            self.num_layers, self.hidden_size = int(lstm.num_layers), int(lstm.hidden_size)
            for key, expected in (("num_layers", self.num_layers), ("hidden_size", self.hidden_size)):
                if key in metadata and int(metadata[key]) != expected:
                    raise ValueError(f"Metadata '{key}' in '{path}' is {metadata[key]}, but the network's LSTM has {key}={expected}")
        elif "num_layers" in metadata and "hidden_size" in metadata:
            self.num_layers, self.hidden_size = int(metadata["num_layers"]), int(metadata["hidden_size"])
        else:
            raise ValueError(f"Cannot determine the LSTM configuration for '{path}': the checkpoint does not expose an 'lstm' "
                             f"module (torch.nn.LSTM) and its metadata does not provide 'num_layers' and 'hidden_size'. Record "
                             f"both in the checkpoint metadata when exporting pt2 archives.")
        if not 1 <= self.num_layers <= _abi.NET_MAX_LAYERS or self.hidden_size < 1:
            raise NotImplementedError(f"num_layers={self.num_layers}, hidden_size={self.hidden_size}: 1 to "
                                      f"{_abi.NET_MAX_LAYERS} layers of at least one unit are supported")
        self._lstm = _read_lstm(self.network, self.num_layers, self.hidden_size)
        self._probe()

    def _probe(self) -> None:
        rng = np.random.default_rng(0)
        L, B, H = self.num_layers, _PROBE_BATCH, self.hidden_size
        h, c = rng.normal(size=(L, B, H)) * 0.5, rng.normal(size=(L, B, H)) * 0.5
        th, tc = torch.from_numpy(h.astype(np.float32)), torch.from_numpy(c.astype(np.float32))
        h, c = th.double().numpy(), tc.double().numpy()  # both sides start from the same float32 state
        for _ in range(_PROBE_STEPS):
            x = rng.normal(size=(B, 2)).astype(np.float32)
            try:
                out = _run_module(self.network, torch.from_numpy(x).unsqueeze(1), (th, tc))
                y, (th, tc) = out
            except Exception as exc:  # noqa: BLE001 - any failure of the module's own forward on the probe is a refusal
                raise NotImplementedError(f"'{self.model_path}': the network does not run as net(x [{B}, 1, 2], (h, c)) -> "
                                          f"(effort, (h, c)): {exc}") from exc
            want, h, c = _lstm_forward64(self._lstm, x.astype(np.float64), h, c)
            for what, g, r in (("effort", y, want), ("hidden state", th, h), ("cell state", tc, c)):
                if tuple(g.shape) != r.shape:
                    raise NotImplementedError(f"'{self.model_path}': the network's {what} has shape {tuple(g.shape)}, "
                                              f"expected {r.shape}")
                err, bound = _close(g.double().numpy(), r)
                if not err <= bound:
                    raise _probe_fail(what, err, bound, self.model_path)

    def _pack(self) -> np.ndarray:
        parts = []
        for w_ih, w_hh, b_ih, b_hh in self._lstm.layers:
            parts += [w_ih.ravel(), w_hh.ravel()] + ([b_ih, b_hh] if b_ih is not None else [])
        parts.append(self._lstm.head_w.ravel())
        if self._lstm.head_b is not None:
            parts.append(self._lstm.head_b)
        flat = np.concatenate(parts).astype(np.float32)
        self._weight_count = int(flat.size)
        return np.concatenate([flat, np.zeros((-flat.size) % 4, np.float32)])

    def _scratch_floats(self) -> int:
        return 4 * self.hidden_size * (_abi.NET_TILE + 1)

    def _fill(self, w) -> None:
        w.layer_count = self.num_layers
        w.widths[0], w.widths[1] = 2, self.hidden_size
        w.has_bias[0] = self._lstm.layers[0][2] is not None
        w.has_bias[1] = self._lstm.head_b is not None

    def _state_numel(self, n: int) -> int:
        return self.num_layers * n * self.hidden_size

    def state(self, num_actuators: int, device) -> ControllerNeuralLSTM.State:
        shape = (self.num_layers, num_actuators, self.hidden_size)
        return ControllerNeuralLSTM.State(hidden=torch.zeros(shape, dtype=torch.float32, device=device),
                                          cell=torch.zeros(shape, dtype=torch.float32, device=device))


NEURAL_CONTROLLERS = (ControllerNeuralMLP, ControllerNeuralLSTM)

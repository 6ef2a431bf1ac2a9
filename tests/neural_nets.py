"""Seeded learned actuator networks and their checkpoints for the neural-actuator tests, and the reference's Torch-path step
(``_compute_torch`` of ControllerNeuralMLP / ControllerNeuralLSTM) restated on plain tensors."""

from __future__ import annotations

import json
import os

import torch

ACTS = {"relu": torch.nn.ReLU, "elu": lambda: torch.nn.ELU(0.7), "tanh": torch.nn.Tanh, "sigmoid": torch.nn.Sigmoid,
        "softsign": torch.nn.Softsign}


def mlp(widths, act="softsign", seed=0, bias=True, scale=1.0):
    """``Linear -> act -> ... -> Linear`` with seeded weights; ``act`` is one name or one per hidden layer, ``bias`` one flag or
    one per layer."""
    g = torch.Generator().manual_seed(seed)
    acts = [act] * (len(widths) - 2) if isinstance(act, str) else list(act)
    biases = [bias] * (len(widths) - 1) if isinstance(bias, bool) else list(bias)
    layers = []
    for k, (a, b) in enumerate(zip(widths, widths[1:])):
        lin = torch.nn.Linear(a, b, bias=biases[k])
        with torch.no_grad():
            lin.weight.copy_(torch.randn(b, a, generator=g) * scale / a ** 0.5)
            if lin.bias is not None:
                lin.bias.copy_(torch.randn(b, generator=g) * 0.1)
        layers.append(lin)
        if k < len(widths) - 2:
            layers.append(ACTS[acts[k]]())
    return torch.nn.Sequential(*layers).eval()


class LSTMNet(torch.nn.Module):
    """The reference's test network shape: one LSTM and a Linear head on the last time step."""

    def __init__(self, hidden: int = 8, layers: int = 1, bias: bool = True, head_bias: bool = True, bidirectional: bool = False):
        super().__init__()
        self.lstm = torch.nn.LSTM(2, hidden, layers, batch_first=True, bias=bias, bidirectional=bidirectional)
        self.dec = torch.nn.Linear(hidden, 1, bias=head_bias)

    def forward(self, x: torch.Tensor, hc: tuple[torch.Tensor, torch.Tensor]) -> tuple[torch.Tensor, tuple[torch.Tensor, torch.Tensor]]:
        out, (h, c) = self.lstm(x, hc)
        return self.dec(out[:, -1, :]), (h, c)


def lstm(hidden=8, layers=1, seed=0, bias=True, head_bias=True):
    torch.manual_seed(seed)
    return LSTMNet(hidden, layers, bias, head_bias).eval()


def save(net, path, fmt="pt2", metadata=None, kind="mlp"):
    """Write ``net`` as ``fmt`` ("pt2", "ts" or "dict") with ``metadata``; returns the path."""
    path = str(path)
    meta = json.dumps(metadata or {})
    if fmt == "pt2":
        if kind == "mlp":
            args = (torch.randn(2, net[0].in_features),)
            dyn = ({0: torch.export.Dim("batch", min=1)},)
        else:
            L, H = net.lstm.num_layers, net.lstm.hidden_size
            b = torch.export.Dim("batch", min=2)
            args = (torch.randn(3, 1, 2), (torch.zeros(L, 3, H), torch.zeros(L, 3, H)))
            dyn = ({0: b}, ({1: b}, {1: b}))
        torch.export.save(torch.export.export(net, args, dynamic_shapes=dyn), path, extra_files={"metadata.json": meta})
    elif fmt == "ts":
        torch.jit.save(torch.jit.script(net), path, _extra_files={"metadata.json": meta})
    else:
        torch.save({"model": net, "metadata": metadata or {}}, path)
    assert os.path.exists(path)
    return path


def torch_mlp_step(net, meta, pos_error, vel, hist, dtype=torch.float32):
    """One ``_compute_torch`` step of ControllerNeuralMLP; ``hist`` = [pos_error_history, vel_history] is rolled in place."""
    idx = meta.get("input_idx", [0])
    ph, vh = hist
    pos_in = torch.stack([pos_error if i == 0 else ph[i - 1] for i in idx], dim=1)
    vel_in = torch.stack([vel if i == 0 else vh[i - 1] for i in idx], dim=1)
    ps, vs = meta.get("pos_scale", 1.0), meta.get("vel_scale", 1.0)
    if meta.get("input_order", "pos_vel") == "pos_vel":
        x = torch.cat([pos_in * ps, vel_in * vs], dim=1)
    else:
        x = torch.cat([vel_in * vs, pos_in * ps], dim=1)
    with torch.inference_mode():
        effort = net.to(dtype)(x.to(dtype))
    hist[0] = torch.cat([pos_error[None].to(ph.dtype), ph[:-1]])
    hist[1] = torch.cat([vel[None].to(vh.dtype), vh[:-1]])
    return effort.reshape(-1) * meta.get("effort_scale", meta.get("torque_scale", 1.0))


def torch_lstm_step(net, meta, pos_error, vel, hc, dtype=torch.float32):
    """One ``_compute_torch`` step of ControllerNeuralLSTM; ``hc`` = [h, c] is replaced in place."""
    x = torch.stack([pos_error * meta.get("pos_scale", 1.0), vel * meta.get("vel_scale", 1.0)], dim=1).unsqueeze(1)
    with torch.inference_mode():
        effort, (h, c) = net.to(dtype)(x.to(dtype), (hc[0].to(dtype), hc[1].to(dtype)))
    hc[0], hc[1] = h, c
    return effort.reshape(-1) * meta.get("effort_scale", meta.get("torque_scale", 1.0))

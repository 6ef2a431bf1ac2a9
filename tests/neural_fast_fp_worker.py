"""Worker of tests/test_gpu_neural_actuators.py::test_fast_fp_twin_within_tolerance: runs with NB2_FP=fast (the library is
chosen at import time) and prints, as one JSON line, the largest error of the MLP and LSTM efforts over 20 steps against the
CPU oracle, relative to the largest effort."""

import json
import os
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import oracle.actuator as on  # noqa: E402
from newton_b200 import _lib  # noqa: E402
from newton_b200.actuators import Actuator, ControllerNeuralLSTM, ControllerNeuralMLP  # noqa: E402
from tests import neural_nets as NN  # noqa: E402
from tests import test_actuators as T  # noqa: E402


def rel(ctrl, n=300, steps=20):
    act = Actuator(T.i32(list(range(n))), ctrl)
    gact = act._rebuilt("cuda:0")
    st, ctl = T.io(n, n)
    gst = types.SimpleNamespace(**{k: v.to("cuda:0") for k, v in vars(st).items()})
    gctl = types.SimpleNamespace(**{k: v.to("cuda:0") for k, v in vars(ctl).items()})
    cs, gs = [act.state(), act.state()], [gact.state(), gact.state()]
    rng = np.random.default_rng(0)
    worst = 0.0
    for _ in range(steps):
        for name in ("joint_q", "joint_qd", "joint_target_q"):
            obj, gobj = (st, gst) if name != "joint_target_q" else (ctl, gctl)
            getattr(obj, name).copy_(torch.from_numpy(rng.normal(size=n).astype(np.float32)))
            getattr(gobj, name).copy_(getattr(obj, name))
        ctl.joint_f.zero_()
        gctl.joint_f.zero_()
        on.step(act, st, ctl, cs[0], cs[1])
        gact.step(gst, gctl, gs[0], gs[1])
        got, ref = gctl.joint_f.cpu().numpy().astype(np.float64), ctl.joint_f.numpy().astype(np.float64)
        worst = max(worst, float(np.max(np.abs(got - ref)) / np.max(np.abs(ref))))
        cs.reverse()
        gs.reverse()
    return worst


def main():
    assert _lib.FP_MODE == "fast" and _lib.LIB_PATH.endswith("libnewton_b200_fast.so"), _lib.LIB_PATH
    with tempfile.TemporaryDirectory() as tmp:
        mlp = ControllerNeuralMLP(NN.save(NN.mlp([6, 32, 32, 32, 1], "softsign", seed=1), os.path.join(tmp, "m.pt2"),
                                          metadata={"input_idx": [0, 1, 2]}))
        lstm = ControllerNeuralLSTM(NN.save(NN.lstm(32, 2, seed=1), os.path.join(tmp, "l.pt2"),
                                            metadata={"num_layers": 2, "hidden_size": 32}, kind="lstm"))
        out = {"lib": os.path.basename(_lib.LIB_PATH), "mlp": rel(mlp), "lstm": rel(lstm)}
    print("NEURAL_FAST_FP " + json.dumps(out))


if __name__ == "__main__":
    main()

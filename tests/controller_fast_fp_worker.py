"""Worker of tests/test_gpu_controllers.py::test_fast_fp_twin_within_tolerance: runs with NB2_FP=fast (the library is chosen at
import time) and prints, as one JSON line, the largest error of both controllers against the CPU oracle, relative to the
largest torque."""

import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from newton_b200 import _lib, scenes  # noqa: E402
from tests import test_gpu_controllers as T  # noqa: E402


def rel(make):
    cpu, gpu, c_io, g_io = T._pair(make)
    T.oc.step(cpu, inputs=c_io[0], outputs=c_io[1])
    gpu.step(inputs=g_io[0], outputs=g_io[1])
    got, ref = g_io[1].joint_f.cpu().numpy().astype(np.float64), c_io[1].joint_f.numpy().astype(np.float64)
    return float(np.max(np.abs(got - ref)) / np.max(np.abs(ref)))


def main():
    assert _lib.FP_MODE == "fast" and _lib.LIB_PATH.endswith("libnewton_b200_fast.so"), _lib.LIB_PATH
    fleet = scenes.impedance_fleet_builder(96, ("panda", "ant", "pendulum"))
    out = {"lib": os.path.basename(_lib.LIB_PATH),
           "model_free": rel(lambda dev: T._model_free(dev, (True, True, True, True), True)),
           "model_based": rel(lambda dev: T._model_based(fleet, dev, has_qdd_feedforward=True))}
    print("CONTROLLER_FAST_FP " + json.dumps(out))


if __name__ == "__main__":
    main()

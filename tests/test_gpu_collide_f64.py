"""GPU: the CUDA collide stage against the CPU oracle (every float32 word) and the float64 collider of ``tests/f64_collide.py``.

Every case of ``tests/collide_cases.py`` (the generated pair worlds, the repository's scenes, the speculative scenes) runs in
``tests/collide_f64_worker.py`` under each collide switch that is read once per process: the 8-warp CTA forced (the models here are
small enough that the library would pick 1 warp, which is the default setting), one lane per pair in the write-out, and the fused
export; each at every lane width the model allows and with each of its broad phases.  The worker also steps XPBD once on contacts
collided with and without the export, fills a buffer smaller than the contact count, and in the default setting runs the bench
workload: 4096 quadrupeds, collide after each of 20 XPBD substeps, 16 sampled worlds compared per substep.
"""

import os
import subprocess
import sys

import numpy as np
import pytest

from tests import collide_cases as cases
from tests import f64_collide as F
from tests.collide_f64_worker import BENCH_SAMPLE, BENCH_SUBSTEPS, lane_runs
from tests.test_collide_f64 import FIELDS, collider, compare, oracle_contacts, overflow_prefix

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SETTINGS = {"default": {}, "warps8": {"NB2_COLLIDE_WARPS": "8"}, "pair_lanes": {"NB2_COLLIDE_LANE_PER_CONTACT": "0"},
            "fused_export": {"NB2_COLLIDE_FUSED_EXPORT": "1"}}


def _world_order(model, ref):
    """The oracle's rows (global sort-key order) stably re-ordered by world: the export's (world, key) order."""
    sw = model.numpy("shape_world")
    w = np.maximum(sw[ref["shape0"]], sw[ref["shape1"]])
    order = np.argsort(w, kind="stable")
    return {k: (v[order] if isinstance(v, np.ndarray) else v) for k, v in ref.items()}


def _sample(big, worlds, got, body_q):
    """The rows and bodies of the sampled ``worlds`` of the bench model, renumbered into a model of len(worlds) quadrupeds laid out
    the same way (per-world shapes and bodies, the ground plane last)."""
    from newton_b200 import scenes

    small = scenes.quadruped_model(len(worlds), seed=1)
    nw = int(big.world_count)
    ks, kb = (big.shape_count - 1) // nw, big.body_count // nw
    assert small.shape_count == len(worlds) * ks + 1 and small.body_count == len(worlds) * kb
    smap = np.full(big.shape_count, -1, np.int64)
    for j, w in enumerate(worlds):
        smap[w * ks:(w + 1) * ks] = np.arange(j * ks, (j + 1) * ks)
    smap[big.shape_count - 1] = small.shape_count - 1
    sw = big.numpy("shape_world")
    sel = np.isin(np.maximum(sw[got["shape0"]], sw[got["shape1"]]), worlds)
    sub = {k: got[k][sel] for k in FIELDS + ("shape0", "shape1")}
    sub["shape0"], sub["shape1"] = smap[sub["shape0"]].astype(np.int32), smap[sub["shape1"]].astype(np.int32)
    state = small.state()
    bq = body_q.reshape(-1, 7)
    state.body_q.copy_(__import__("torch").from_numpy(np.concatenate([bq[w * kb:(w + 1) * kb] for w in worlds])))
    return small, state, sub


@pytest.mark.parametrize("setting", list(SETTINGS))
def test_collide_matches_oracle_and_float64(oracle_lib, cuda_lib, tmp_path, setting):
    env = dict(os.environ, **SETTINGS[setting])
    args = ["bench"] if setting == "default" else []
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "collide_f64_worker.py"), str(tmp_path)] + args,
                       env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0 and "COLLIDE_F64_WORKER_DONE" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    all_cases = cases.all_cases()
    expected = {f"{label}__{L}__{bp}.npz" for label, m, phases, _ in all_cases for L in lane_runs(m) for bp in phases}
    expected |= {f"{label}__xpbd.npz" for label, _, _, _ in all_cases} | {"overflow.npz"}
    expected |= {f"bench__{s}.npz" for s in range(BENCH_SUBSTEPS)} if args else set()
    assert set(os.listdir(tmp_path)) == expected
    worst, near, runs = 0.0, 0, 0
    for label, model, phases, spec in all_cases:
        state = model.state()
        for bp in phases:
            ref = _world_order(model, oracle_contacts(oracle_lib, model, state, bp, speculative=spec))
            col = collider(model, state, bp, spec)
            for L in lane_runs(model):
                fn = f"{label}__{L}__{bp}.npz"
                got = dict(np.load(tmp_path / fn))
                assert int(got["count"]) == ref["count"], f"{fn}: {int(got['count'])} rows, oracle {ref['count']}"
                for k in ("shape0", "shape1") + FIELDS:
                    a, b = np.ascontiguousarray(got[k]), np.ascontiguousarray(ref[k])
                    assert a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32)), f"{fn}: {k} differs from the oracle"
                st = compare(model, state, got, col, label=fn + ": ", order="world")
                worst, near, runs = max(worst, st["ratio"]), near + st["near_rows"], runs + 1
        q = np.load(tmp_path / f"{label}__xpbd.npz")
        assert np.array_equal(q["exported"].view(np.int32), q["blocks_only"].view(np.int32)), f"{label}: export_contacts=False differs"
    ov = dict(np.load(tmp_path / "overflow.npz"))
    _, model, _, _ = cases.scene_models()[0]
    state = model.state()
    assert int(ov["count"]) == int(ov["cap"]) + 5
    overflow_prefix(collider(model, state), ov, int(ov["cap"]), "world")
    if args:
        from newton_b200 import scenes

        big = scenes.quadruped_model(4096, seed=1)
        sw = big.numpy("shape_world")
        for s in range(BENCH_SUBSTEPS):
            got = dict(np.load(tmp_path / f"bench__{s}.npz"))
            w_row = np.maximum(sw[got["shape0"]], sw[got["shape1"]])
            assert (np.diff(w_row) >= 0).all() and int(got["count"]) == len(w_row), f"substep {s}: export order or count"
            assert len(got["worlds"]) == BENCH_SAMPLE
            small, st_small, sub = _sample(big, got["worlds"], got, got["body_q"])
            st = compare(small, st_small, sub, F.Collider(small, st_small.body_q), label=f"bench substep {s}: ", order="world")
            worst, near, runs = max(worst, st["ratio"]), near + st["near_rows"], runs + 1
    print(f"\n{setting}: {runs} compared runs, largest ratio {worst:.2f}, knife-edge rows {near}")

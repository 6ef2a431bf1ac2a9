#!/usr/bin/env python
"""Device time per substep of the headline frame, split by graph node: clear_forces, collide (kernel and contact export
separately) and solver.step.

The scene and loop are bench.py's (4096 quadrupeds, SolverXPBD(iterations=8), 4 substeps per frame, settled 1.2 s first).  Two
independent measurements:

* CUDA events around eager calls, 4 x --substeps substeps per variant.  A spin kernel is queued first so that the host enqueues
  ahead of the device and the events see device time, not Python overhead.  The collide kernel alone is timed through a second
  pipeline with ``export_contacts=False``; the export is the difference.
* ``torch.profiler`` over --frames replays of the frame graph: kernel durations by name, and the idle gaps between the nodes of
  a frame.

  python scripts/frame_breakdown.py [--substeps 200] [--frames 50] [--trace DIR]

Prints the card, its power limit and SM clock, a table, and one JSON line.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402


def gpu_info(index: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # noqa: BLE001 - the card line is informative, the timings stand without it
        return {"unavailable": f"{type(e).__name__}: {e}"[:200]}


def category(name: str) -> str:
    if "collide_kernel" in name:
        return "collide_kernel"
    if "contact_export" in name:
        return "contact_export"
    if "contact_scan" in name:
        return "contact_scan"
    if "xpbd" in name:
        return "solver"
    if "fill" in name.lower() or "memset" in name.lower() or "elementwise" in name:
        return "clear_forces"
    return "other:" + name[:60]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--substeps", type=int, default=200, help="timed eager substeps per variant (events)")
    p.add_argument("--frames", type=int, default=50, help="profiled graph replays")
    p.add_argument("--envs", type=int, default=bench.ENVS_PER_GPU)
    p.add_argument("--trace", metavar="DIR", default=None, help="also write the profiler's chrome trace to DIR")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frame_breakdown.py measures device time: it needs a CUDA device")

    import newton_b200
    from newton_b200 import _lib

    bench.select_workload("quadruped_xpbd")
    S, DT = bench.SUBSTEPS, bench.DT
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    model = bench.build_scene(args.envs, seed=1).to(dev)
    pipeline = newton_b200.CollisionPipeline(model)
    pipeline_nx = newton_b200.CollisionPipeline(model, export_contacts=False)
    solver = bench.make_solver(newton_b200.solvers, model)
    states = [model.state(), model.state()]
    control = model.control()
    contacts = pipeline.contacts()

    def substep(pipe):
        states[0].clear_forces()
        pipe.collide(states[0], contacts)
        solver.step(states[0], states[1], control, contacts, DT)
        states.reverse()

    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
        for _ in range(int(round(1.2 * bench.FPS)) * S):  # bench.py's settle: 1.2 s of simulated time
            substep(pipeline)
    torch.cuda.synchronize()

    # ---- events around eager calls
    def eager(pipe, n):
        rows = []
        with torch.cuda.stream(stream):
            for _ in range(8):
                substep(pipe)
            chunk = 50
            for c0 in range(0, n, chunk):
                torch.cuda.synchronize()
                torch.cuda._sleep(50_000_000)  # ~25 ms spin: the host queues the chunk while the device is busy
                ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(min(chunk, n - c0))]
                for e in ev:
                    e[0].record(stream)
                    states[0].clear_forces()
                    e[1].record(stream)
                    pipe.collide(states[0], contacts)
                    e[2].record(stream)
                    solver.step(states[0], states[1], control, contacts, DT)
                    e[3].record(stream)
                    states.reverse()
                torch.cuda.synchronize()
                rows += [[e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), e[2].elapsed_time(e[3]), e[0].elapsed_time(e[3])] for e in ev]
        return np.asarray(rows) * 1e3  # us

    n = max(args.substeps, 200)
    with_export = eager(pipeline, n)
    without_export = eager(pipeline_nx, n)
    ev = {
        "clear_forces": float(np.median(with_export[:, 0])),
        "collide+export": float(np.median(with_export[:, 1])),
        "collide_kernel": float(np.median(without_export[:, 1])),
        "solver.step": float(np.median(with_export[:, 2])),
        "substep": float(np.median(with_export[:, 3])),
    }
    ev["contact_export"] = ev["collide+export"] - ev["collide_kernel"]

    # ---- profiler over replays of the frame graph (bench.py's capture)
    with torch.cuda.stream(stream):
        substep(pipeline)
    torch.cuda.synchronize()
    launches_before = _lib.kernel_launch_count()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        for _ in range(S):
            substep(pipeline)
    launches = _lib.kernel_launch_count() - launches_before
    for _ in range(10):
        graph.replay()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.frames):
            graph.replay()
            torch.cuda.synchronize()  # frames apart: the gaps below are the ones inside a frame
    trace_path = os.path.join(args.trace or "/tmp", "frame_breakdown.pt.trace.json")
    if args.trace:
        os.makedirs(args.trace, exist_ok=True)
    prof.export_chrome_trace(trace_path)
    with open(trace_path) as f:
        events = [e for e in json.load(f)["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    if not args.trace:
        os.remove(trace_path)
    events.sort(key=lambda e: e["ts"])
    # split into frames: a frame is S substeps, and a substep begins with the body_f zeroing of clear_forces
    frames, cur, seen = [], [], 0
    for e in events:
        if category(e["name"]) == "clear_forces":
            if seen and seen % S == 0:
                frames.append(cur)
                cur = []
            seen += 1
        cur.append(e)
    if cur:
        frames.append(cur)
    if len(frames) != args.frames:
        print(f"warning: the trace splits into {len(frames)} frames, {args.frames} were replayed", file=sys.stderr)
    per_cat: dict[str, list[float]] = {}
    gaps, spans = [], []
    for fr in frames:
        sums: dict[str, float] = {}
        for e in fr:
            sums[category(e["name"])] = sums.get(category(e["name"]), 0.0) + e["dur"]
        for k, v in sums.items():
            per_cat.setdefault(k, []).append(v / S)
        span = fr[-1]["ts"] + fr[-1]["dur"] - fr[0]["ts"]
        spans.append(span / S)
        gaps.append((span - sum(e["dur"] for e in fr)) / S)
    prof_us = {k: float(np.median(v)) for k, v in sorted(per_cat.items())}
    prof_us["gaps_between_nodes"] = float(np.median(gaps))
    prof_us["substep_span"] = float(np.median(spans))
    non_solver = prof_us["substep_span"] - prof_us.get("solver", 0.0)

    print(f"card: {card.get('name')}, power limit {card.get('power_limit')}, SM clock {card.get('sm_clock')} "
          f"(max {card.get('sm_clock_max')})")
    print(f"library: {_lib.LIB_PATH}")
    print(f"{args.envs} quadruped envs, XPBD {bench.ITERATIONS} it., {S} substeps/frame; live contacts "
          f"{int(contacts.rigid_contact_count.item())}; {launches} launches per frame graph")
    print(f"\nCUDA events around eager calls (median of {n} substeps, us per substep)")
    for k in ("clear_forces", "collide_kernel", "contact_export", "collide+export", "solver.step", "substep"):
        print(f"  {k:<28s} {ev[k]:9.2f}")
    print(f"\ntorch.profiler, frame graph replayed {len(frames)} times (median, us per substep)")
    for k, v in prof_us.items():
        print(f"  {k:<28s} {v:9.2f}")
    print(f"  {'non-solver (span - solver)':<28s} {non_solver:9.2f}")
    print(json.dumps({"card": card, "library": os.path.basename(_lib.LIB_PATH), "envs": args.envs, "launches_per_frame": launches,
                      "events_us": ev, "profiler_us": prof_us, "non_solver_us": non_solver}))


if __name__ == "__main__":
    main()

"""Times SensorTiledCamera.update on 4096 quadrupeds (seed 1) after 20 XPBD substeps, one 64 x 48 camera per base (vertical fov
58 deg, pitched down 30 deg, scenes.quadruped_camera_transforms), in two workloads:

  (a) quadruped_model: the robots and the ground plane;
  (b) quadruped_terrain_model: plus the visual-only global MESH terrain (256 x 256 seeded vertices, 130 050 triangles).

Per workload, device time per call from CUDA events over many calls, eager and replayed from a CUDA graph, for a depth-only
update and for all four channels; pixels (rays) per second; and the share of the HBM3 bandwidth of an H100 SXM (3.35 TB/s)
that the algorithmic bytes of the update take (the images written: 4 B per pixel for depth, 24 B for all four channels; the
ray table and transforms are a few hundred kB, read from L2).

The yardstick, timed the same way on the same pixels: world rays generated with torch (one rotation per pixel into
[N, 3] origin and direction tensors) plus newton_b200.intersect_ray, 28 B of rays in and 20 B out per pixel.  Its depth
must agree with the camera's within 1e-5 relative wherever it hits closer than max_distance (torch's rotation is not the
kernel's, bit for bit).  The card's name and power limit are read in the same run.  Prints one JSON line per workload;
writes nothing unless --out is given.

    python scripts/camera_bench.py [--envs 4096] [--iters 200] [--out results.json]
"""

from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import newton_b200  # noqa: E402
from newton_b200 import scenes  # noqa: E402
from newton_b200.sensors import SensorTiledCamera  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
YARDSTICK_BYTES_PER_RAY = 28 + 20


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def time_calls(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e3 / iters  # us per call


def time_graph(fn, iters, stream):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        fn()
    g.replay()
    torch.cuda.synchronize()
    return time_calls(g.replay, iters)


def quat_rotate(q, v):
    x, y, z, w = q.unbind(-1)
    vx, vy, vz = v.unbind(-1)
    c = 2.0 * w * w - 1.0
    d = 2.0 * (x * vx + y * vy + z * vz)
    return torch.stack([vx * c + x * d + (y * vz - z * vy) * w * 2.0, vy * c + y * d + (z * vx - x * vz) * w * 2.0,
                        vz * c + z * d + (x * vy - y * vx) * w * 2.0], dim=-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("camera_bench.py measures the CUDA kernels and needs a GPU")
    dev = "cuda:0"
    from tests.helpers import simulate

    results = []
    stream = torch.cuda.Stream()
    for name, build in (("robots_and_plane", scenes.quadruped_model), ("with_terrain", scenes.quadruped_terrain_model)):
        model = build(args.envs, seed=1).to(dev)
        state, _, _ = simulate(model, newton_b200.CollisionPipeline, newton_b200.solvers.SolverXPBD, substeps=20, dt=0.005,
                               solver_kwargs={"iterations": 8}, pipeline_kwargs={"reduce_contacts": False})
        torch.cuda.synchronize()
        model.bvh_refit_shapes(state)
        W = model.world_count
        width, height = scenes.CAMERA_SIZE
        sensor = SensorTiledCamera(model)
        rays = sensor.utils.compute_camera_rays_pinhole(width, height, camera_fovs=math.radians(scenes.CAMERA_FOV_DEG))
        Tf = scenes.quadruped_camera_transforms(model, state.body_q)
        imgs = {"depth_image": sensor.utils.create_depth_image_output(width, height),
                "forward_depth_image": sensor.utils.create_forward_depth_image_output(width, height),
                "shape_index_image": sensor.utils.create_shape_index_image_output(width, height),
                "normal_image": sensor.utils.create_normal_image_output(width, height)}
        n = W * width * height
        max_d = sensor.default_render_config.max_distance

        def depth_only():
            sensor.update(state, Tf, rays, depth_image=imgs["depth_image"])

        def all_channels():
            sensor.update(state, Tf, rays, **imgs)

        # yardstick: world rays in HBM from torch, then intersect_ray
        q = Tf[0, :, None, None, 3:7]
        origins, directions = torch.empty((n, 3), device=dev), torch.empty((n, 3), device=dev)
        worlds = torch.arange(W, dtype=torch.int32, device=dev).repeat_interleave(width * height)
        out = (torch.empty(n, device=dev), torch.empty(n, dtype=torch.int32, device=dev), torch.empty((n, 3), device=dev))

        def yardstick():
            origins.copy_((Tf[0, :, None, None, :3] + quat_rotate(q, rays[None, 0, :, :, 0])).reshape(n, 3))
            directions.copy_(quat_rotate(q, rays[None, 0, :, :, 1]).reshape(n, 3))
            newton_b200.intersect_ray(model, ray_origins=origins, ray_directions=directions, ray_worlds=worlds, out_dist=out[0],
                                      out_shape_id=out[1], out_normal=out[2])

        with torch.cuda.stream(stream):
            for _ in range(10):
                depth_only()
                all_channels()
                yardstick()
            torch.cuda.synchronize()
            t = {"depth_eager": time_calls(depth_only, args.iters), "all_eager": time_calls(all_channels, args.iters),
                 "yardstick_eager": time_calls(yardstick, args.iters), "depth_graph": time_graph(depth_only, args.iters, stream),
                 "all_graph": time_graph(all_channels, args.iters, stream), "yardstick_graph": time_graph(yardstick, args.iters, stream)}
            all_channels()
            yardstick()
        torch.cuda.synchronize()
        cam_d = imgs["depth_image"].reshape(-1).cpu().numpy().astype(np.float64)
        ys_d, ys_id = out[0].cpu().numpy().astype(np.float64), out[1].cpu().numpy()
        near = (ys_id >= 0) & (ys_d < max_d)
        rel = np.abs(cam_d[near] - ys_d[near]) / np.maximum(np.abs(ys_d[near]), 1e-30)
        cam_hit = imgs["shape_index_image"].reshape(-1).cpu().numpy() != 0xFFFFFFFF
        res = {"workload": name, "envs": W, "image": [width, height], "pixels": n, "card": card(),
               "update_us": {"depth_eager": round(t["depth_eager"], 2), "depth_graph": round(t["depth_graph"], 2),
                             "all_eager": round(t["all_eager"], 2), "all_graph": round(t["all_graph"], 2)},
               "yardstick_us": {"eager": round(t["yardstick_eager"], 2), "graph": round(t["yardstick_graph"], 2)},
               "speedup_depth_graph": round(t["yardstick_graph"] / t["depth_graph"], 2),
               "speedup_all_graph": round(t["yardstick_graph"] / t["all_graph"], 2),
               "pixels_per_s_depth_graph": round(n / (t["depth_graph"] * 1e-6)),
               "hbm_share_depth_graph": round(n * 4 / (t["depth_graph"] * 1e-6) / HBM_BYTES_PER_S, 4),
               "hbm_share_all_graph": round(n * 24 / (t["all_graph"] * 1e-6) / HBM_BYTES_PER_S, 4),
               "hbm_share_yardstick_graph": round(n * YARDSTICK_BYTES_PER_RAY / (t["yardstick_graph"] * 1e-6) / HBM_BYTES_PER_S, 4),
               "hit_fraction": round(float(cam_hit.mean()), 4),
               "yardstick_max_rel_depth_diff": float(rel.max()) if rel.size else 0.0,
               "hit_agreement": round(float((cam_hit == near).mean()), 6),
               "shapes_enabled": model.bvh_shape_count_enabled, "triangles": int(model._bvh_tri_face.numel())}
        print(json.dumps(res), flush=True)
        results.append(res)
        assert res["yardstick_max_rel_depth_diff"] <= 1e-5, res
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

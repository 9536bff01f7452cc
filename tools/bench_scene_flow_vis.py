"""The scene-flow figure, the reference's formulation vs emernerf_b200.flow_vis.visualize_scene_flow, on one GPU.

    python tools/bench_scene_flow_vis.py [--frames 200] [--points 100000] [--reps 3] [--out DIR]

Model and drive: the benchmark-size ``flow_feat`` field and ``SyntheticDrive`` of tools/bench_lidar_flow.py (200
scans of 10^5 points is an assumed size for a Waymo drive, not a measured one), with three cameras per frame added:
pinhole cameras 1920 x 1280 at the scan's ego position, looking ahead, left and right.  Two formulations, in the same
process, alternating call by call:
  reference  oracle.scene_flow_vis_ref: per drawn frame the boolean indexes, the camera mask with its inverse() per
             camera, query_flow, the in-place gate, two scene_flow_to_rgb calls and three .cpu() copies
  device     flow_vis.visualize_scene_flow: one select launch per frame, query_flow per frame, one colour launch per
             chunk, two host syncs
Reported per formulation: device time (CUDA events around the call) and wall time (ending in a synchronize) of each
call, host syncs per call (torch.cuda.set_sync_debug_mode("warn")) and CUDA kernels per call (torch.profiler, a
separate pass), and whether the two results are equal (coordinates and both colour lists bit for bit).  The GPU's name
and power limit come from the same run (nvidia-smi query, read only).  Writes DIR/bench_scene_flow_vis.json and prints
it.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import tempfile
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_lidar_flow import SyntheticDrive, Split, count_kernels, count_syncs, flow_field, gpu_info, timed  # noqa
from emernerf_b200 import flow_vis  # noqa: E402
from oracle import scene_flow_vis_ref  # noqa: E402

CAMS, WIDTH, HEIGHT, FOCAL = 3, 1920, 1280, 1000.0


class Cameras:
    """The attributes of a pixel source that the camera mask reads: per frame, three cameras at the ego position."""

    def __init__(self, frames: int, device="cuda"):
        self.num_cams, self.WIDTH, self.HEIGHT = CAMS, WIDTH, HEIGHT
        k = torch.tensor([[FOCAL, 0.0, WIDTH / 2], [0.0, FOCAL, HEIGHT / 2], [0.0, 0.0, 1.0]])
        self.intrinsics = k.repeat(frames * CAMS, 1, 1).to(device)
        mats = []
        for f in range(frames):
            for yaw in (0.0, math.pi / 3, -math.pi / 3):
                fwd = torch.tensor([math.cos(yaw), math.sin(yaw), 0.0], dtype=torch.float64)
                right = torch.linalg.cross(fwd, torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64))
                down = torch.linalg.cross(fwd, right)
                m = torch.eye(4, dtype=torch.float64)
                m[:3, 0], m[:3, 1], m[:3, 2] = right, down, fwd
                m[:3, 3] = torch.tensor([f * 0.5, 0.0, 2.0], dtype=torch.float64)
                mats.append(m.float())
        self.cam_to_worlds = torch.stack(mats).to(device)


def same(a, b) -> bool:
    keys = ("dynamic_coords", "dynamic_colors")
    for part in ("pred", "gt"):
        x, y = a[part], b[part]
        if x["vis_aabb"] != y["vis_aabb"] or [x["y_ratio"], x["z_ratio"]] != [y["y_ratio"], y["z_ratio"]]:
            return False
        for k in keys:
            if len(x[k]) != len(y[k]) or not all(np.array_equal(p.view(np.int32), q.view(np.int32))
                                                 for p, q in zip(x[k], y[k])):
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=tempfile.gettempdir())
    a = ap.parse_args()
    info = gpu_info()
    field = flow_field()
    ds = types.SimpleNamespace(full_lidar_set=Split(SyntheticDrive(a.frames, a.points), range(a.frames)),
                               pixel_source=Cameras(a.frames))
    cfg = types.SimpleNamespace()
    calls = {"reference": lambda: scene_flow_vis_ref.visualize_scene_flow(cfg, field, ds, device="cuda"),
             "device": lambda: flow_vis.visualize_scene_flow(cfg, field, ds, device="cuda")}
    results = {k: fn() for k, fn in calls.items()}             # warm-up; builds the device path's frame table
    device_ms = {k: [] for k in calls}
    wall_ms = {k: [] for k in calls}
    for _ in range(a.reps):
        for k, fn in calls.items():
            results[k], dev, wall = timed(fn)
            device_ms[k].append(round(dev, 2))
            wall_ms[k].append(round(wall, 2))
    r = results["device"]
    report = {
        "gpu": info,
        "frames": a.frames, "points_per_frame": a.points, "cameras": CAMS,
        "drawn_frames": len(r["pred"]["dynamic_coords"]),
        "drawn_points": int(sum(len(c) for c in r["pred"]["dynamic_coords"])),
        "device_ms": device_ms, "wall_ms": wall_ms,
        "host_syncs_per_call": {k: count_syncs(fn) for k, fn in calls.items()},
        "kernels_per_call": {k: count_kernels(fn) for k, fn in calls.items()},
        "equal": same(results["reference"], results["device"]),
    }
    text = json.dumps(report, indent=2)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_scene_flow_vis.json"), "w") as f:
        f.write(text)
    print(text)


if __name__ == "__main__":
    main()

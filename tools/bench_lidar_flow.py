"""Lidar scene-flow evaluation, the reference's formulation vs emernerf_b200.metrics.eval_lidar_flow, on one GPU.

    python tools/bench_lidar_flow.py [--frames 200] [--points 100000] [--reps 3] [--out DIR]

Model: the benchmark-size ``flow_feat`` field of bench.py (configs.make_cfg("flow_feat"), trained-like N(0, 0.5)
tables), in eval mode.  Drive: ``SyntheticDrive``, a Waymo-shaped lidar source generated on the device -- ``--frames``
scans of ``--points`` points each (200 scans of 10^5 points is an assumed size for a Waymo drive, not a measured one),
concatenated in scan order as the Waymo loader does, with flow labels, flow classes (-1 for one point in five) and
ground flags (one point in three).  Two formulations, in the same process, alternating call by call:
  reference  oracle.lidar_flow_ref: per frame the boolean indexes of get_render_rays, of the flow-class filter and of
             the ground removal, query_flow on the kept points, the in-place gate and the statistics on the host
  device     metrics.eval_lidar_flow: frames from the sampler's table, query_flow on every point, one kernel per chunk
Reported per formulation: device time (CUDA events around the call) and wall time (ending in a synchronize) of each
call, host syncs per call (torch.cuda.set_sync_debug_mode("warn")) and CUDA kernels per call (torch.profiler, a
separate pass), and the two results.  The GPU's name and power limit come from the same run (nvidia-smi query, read
only).  Writes DIR/bench_lidar_flow.json and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from emernerf_b200 import metrics  # noqa: E402
from emernerf_b200.configs import build_hot_path, make_cfg  # noqa: E402
from oracle import lidar_flow_ref  # noqa: E402


class SyntheticDrive:
    """The attributes of a Waymo lidar source that the flow evaluation reads, seeded, on the device, with the
    reference's boolean-index ``get_render_rays``."""
    timesteps = property(lambda self: self._timesteps)
    normalized_timestamps = property(lambda self: self._normalized_timestamps)

    def __init__(self, frames: int, points: int, seed: int = 0, device="cuda"):
        g = torch.Generator(device=device).manual_seed(seed)
        n = frames * points
        t = torch.arange(frames, device=device).repeat_interleave(points)
        ego = torch.stack([t.float() * 0.5, torch.zeros(n, device=device), torch.full((n,), 2.0, device=device)], -1)
        self.origins = ego + 0.05 * torch.randn(n, 3, generator=g, device=device)
        d = torch.randn(n, 3, generator=g, device=device) * torch.tensor([1.0, 1.0, 0.2], device=device)
        self.directions = torch.nn.functional.normalize(d, dim=-1)
        self.ranges = 2.0 + 73.0 * torch.rand(n, 1, generator=g, device=device)
        self._timesteps = t
        self._normalized_timestamps = t.float() / (frames - 1)
        moving = torch.rand(n, generator=g, device=device) < 0.3
        self.flows = torch.randn(n, 3, generator=g, device=device) * torch.where(moving, 0.5, 0.02)[:, None]
        self.flow_classes = torch.randint(0, 4, (n,), generator=g, device=device)
        self.flow_classes[torch.rand(n, generator=g, device=device) < 0.2] = -1
        self.grounds = torch.rand(n, generator=g, device=device) < 0.35
        self.device = torch.device(device)

    def get_render_rays(self, time_idx):
        return lidar_flow_ref.get_render_rays(self, time_idx)


class Split:
    """A SplitWrapper over every scan of the drive (the reference's ``full_lidar_set``)."""

    def __init__(self, datasource, split_indices):
        self.datasource, self.split_indices = datasource, list(split_indices)

    def __getitem__(self, idx):
        return self.datasource.get_render_rays(self.split_indices[idx])

    def __len__(self):
        return len(self.split_indices)


def flow_field():
    field, _, _, _ = build_hot_path(make_cfg("flow_feat"), device="cuda", table_std=0.5)
    return field.eval()


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except Exception as e:                      # noqa: BLE001 -- reported, not fatal
        return f"nvidia-smi unavailable: {e}"


def count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message) for w in caught)


def count_kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset")))


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    w0 = time.perf_counter()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1), (time.perf_counter() - w0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=tempfile.gettempdir())
    a = ap.parse_args()
    info = gpu_info()
    field = flow_field()
    drive = Split(SyntheticDrive(a.frames, a.points), range(a.frames))
    calls = {"reference": lambda: lidar_flow_ref.eval_lidar_flow(drive, field, True),
             "device": lambda: metrics.eval_lidar_flow(drive, field, True)}
    results = {k: fn() for k, fn in calls.items()}             # warm-up; builds the device path's frame table
    device_ms = {k: [] for k in calls}
    wall_ms = {k: [] for k in calls}
    for _ in range(a.reps):
        for k, fn in calls.items():
            results[k], dev, wall = timed(fn)
            device_ms[k].append(round(dev, 2))
            wall_ms[k].append(round(wall, 2))
    report = {
        "gpu": info,
        "frames": a.frames, "points_per_frame": a.points,
        "device_ms": device_ms, "wall_ms": wall_ms,
        "host_syncs_per_call": {k: count_syncs(fn) for k, fn in calls.items()},
        "kernels_per_call": {k: count_kernels(fn) for k, fn in calls.items()},
        "results": {k: {m: float(v) for m, v in r.items()} for k, r in results.items()},
    }
    text = json.dumps(report, indent=2)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_lidar_flow.json"), "w") as f:
        f.write(text)
    print(text)


if __name__ == "__main__":
    main()

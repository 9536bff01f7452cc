"""Camera-trajectory frames on one GPU: the ray generation of raygen.CameraTrajectory and whole frames through
render_rays.

    python tools/bench_trajectory.py [--frames 50] [--warmup 5] [--launches 500] [--out DIR]

Source: Waymo-shaped, 3 cameras x 20 timesteps of 640 x 960 (tools/bench_raybatch.py's tables, with each timestep's
cameras yawed so the rotations interpolate), rendered at downscale 0.5 (320 x 480 rays per frame), 4 frames per
keyframe and an offset, so most frames lie between keyframes.  Fields: the benchmarked static, dynamic and flow
configurations at full size (tests/golden/full_cases.py: 64 samples, proposal samples [128, 64]).
Reported:
  rays_ms      emer_trajectory_rays alone: CUDA events around each of --launches launches (the library's profile
               hook), mean and median per launch
  frame_ms     traj[k] + render_rays(..., return_decomposition=True) for --frames frames after --warmup, a host clock
               between two device synchronizes, per frame; per field variant
  rays_share   rays_ms (mean) / frame_ms
The GPU's name, power limit and maximum SM clock come from the same run (nvidia-smi query, read only).  Writes
DIR/bench_trajectory.json (DIR defaults to a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys
import tempfile
import time
import types

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests", "golden"))

from bench_raybatch import gpu_info, pixel_source  # noqa: E402
from emernerf_b200 import _lib, raygen  # noqa: E402
import errormap_cases as ec  # noqa: E402
import full_cases as fc  # noqa: E402

DEV = "cuda"
TIMESTEPS, CAMS = 20, 3


def source():
    s = ec.PixelSource()
    vars(s).update(vars(pixel_source(TIMESTEPS * CAMS, False)))
    # OpenCV cameras looking along the world's y axis, the rig yawing 9 degrees per timestep, each camera 50 apart
    c2w = s.cam_to_worlds
    for i in range(len(c2w)):
        yaw = math.radians(9 * (i // CAMS) + 50 * (i % CAMS - 1))
        c, si = math.cos(yaw), math.sin(yaw)
        Rz = torch.tensor([[c, -si, 0.0], [si, c, 0.0], [0.0, 0.0, 1.0]], device=DEV)
        fwd = torch.tensor([[1.0, 0.0, 0.0], [0.0, 0.0, 1.0], [0.0, -1.0, 0.0]], device=DEV)
        c2w[i, :3, :3] = Rz @ fwd
        c2w[i, :3, 3] = torch.tensor([2.0 * (i // CAMS), 0.0, 1.5], device=DEV)
    s._normalized_timestamps = (torch.arange(len(c2w), device=DEV) // CAMS).float() / (TIMESTEPS - 1)
    s._downscale_factor = 0.5
    return s


def models(variant):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder
    from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    field, props = fc.build_models(ns, variant)
    est = PropNetEstimator(None, None).to(DEV)
    field = field.to(DEV).eval()
    props = [p.to(DEV).eval() for p in props]
    return field, props, est.eval()


def rays_ms(traj, launches):
    rec = []
    _lib.set_profile(lambda name, args: name == "emer_trajectory_rays", rec)
    try:
        for j in range(launches):
            traj[j % len(traj)]
        torch.cuda.synchronize()
    finally:
        _lib.set_profile(None, None)
    t = [e0.elapsed_time(e1) for _, _, e0, e1 in rec]
    return {"mean": round(statistics.mean(t), 5), "median": round(statistics.median(t), 5), "launches": len(t)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_trajectory needs a CUDA device"
    from emernerf_b200.radiance_fields.render_utils import render_rays

    src = source()
    traj = raygen.CameraTrajectory(raygen.PixelRaySampler(src), frames_per_keyframe=4, offset=(0.5, 0.0, -1.0))
    h, w = traj[0]["origins"].shape[:2]
    result = {"info": gpu_info(), "size": [640, 960], "downscale": 0.5, "rays_per_frame": h * w,
              "items": len(traj), "frames_per_keyframe": 4}
    for _ in range(2):                                   # warm-up, then the measured pass
        result["rays_ms"] = rays_ms(traj, a.launches)
    print("rays", json.dumps(result["rays_ms"]), flush=True)
    cfg = fc.render_cfg()
    result["frame_ms"], result["rays_share"] = {}, {}
    step = max(1, len(traj) // (a.frames + a.warmup))
    for variant in ("static", "dynamic", "flow"):
        field, props, est = models(variant)
        with torch.no_grad():
            render = lambda k: render_rays(radiance_field=field, proposal_estimator=est, proposal_networks=props,
                                           data_dict=traj[k], cfg=cfg, return_decomposition=True)
            for j in range(a.warmup):
                render(j * step)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for j in range(a.frames):
                render(((a.warmup + j) * step) % len(traj))
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3 / a.frames
        result["frame_ms"][variant] = round(ms, 3)
        result["rays_share"][variant] = round(result["rays_ms"]["mean"] / ms, 6)
        print(variant, result["frame_ms"][variant], flush=True)
        del field, props, est
        torch.cuda.empty_cache()
    out_dir = a.out or tempfile.mkdtemp(prefix="bench_trajectory_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_trajectory.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()

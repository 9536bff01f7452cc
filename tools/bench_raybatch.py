"""Training-batch sampling, the reference's torch path vs emernerf_b200.raygen's samplers, on one GPU.

    python tools/bench_raybatch.py [--calls 200] [--warmup 20] [--out DIR]

Sources: 600 and 1000 images of 640 x 960 with sky and dynamic masks, error maps at buffer_downscale 16, and with or
without a [N, 46, 69, 64] feature map (the feature-lifting config); 8192 rays per call from 90 % of the images (a
candidate list, as the training split passes it), buffer_ratio 0 and 0.25; a lidar source of 4 M points over 200 scans.
Two formulations, in the same process, alternating call by call:
  reference  oracle.raybatch_ref: the reference's get_train_rays (torch.multinomial, list -> tensor copies, the
             feature gather through host indices)
  device     raygen.PixelRaySampler / raygen.LidarRaySampler (emer_topk_ratio + emer_pixel_batch)
Reported per configuration and formulation: device time per call from CUDA events, host wall time per call ending in
a synchronize (this shows the stalls), host syncs per call (torch.cuda.set_sync_debug_mode("warn")) and CUDA kernels
per call (torch.profiler, a separate pass).  The GPU's name and power limit come from the same run (nvidia-smi query,
read only).  Writes DIR/bench_raybatch.json (DIR defaults to a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from emernerf_b200 import raygen  # noqa: E402
from oracle import raybatch_ref  # noqa: E402
import raybatch_cases as rc  # noqa: E402

DEV = "cuda"
H, W, DS = 640, 960, 16


def pixel_source(n_images: int, features: bool):
    g = torch.Generator(device=DEV).manual_seed(n_images)
    s = rc.PixelSource()
    s.device = torch.device(DEV)
    s.data_cfg = types.SimpleNamespace(load_size=[H, W],
                                       sampler=types.SimpleNamespace(buffer_downscale=DS, buffer_ratio=0.25))
    s.images = torch.rand(n_images, H, W, 3, device=DEV, generator=g)
    s.sky_masks = (torch.rand(n_images, H, W, device=DEV, generator=g) > 0.7).float()
    s.dynamic_masks = (torch.rand(n_images, H, W, device=DEV, generator=g) > 0.9).float()
    s.features = torch.rand(n_images, 46, 69, 64, device=DEV, generator=g) if features else None
    s.featmap_downscale_factor = (46 / H, 69 / W) if features else None
    s._normalized_timestamps = torch.linspace(0, 1, n_images, device=DEV)
    s.cam_ids = torch.arange(n_images, device=DEV) % 3
    c2w = torch.eye(4, device=DEV).repeat(n_images, 1, 1)
    c2w[:, :3, 3] = torch.randn(n_images, 3, device=DEV, generator=g)
    s.cam_to_worlds = c2w
    K = torch.tensor([[1030.0, 0, 480.0], [0, 1030.0, 320.0], [0, 0, 1.0]], device=DEV)
    s.intrinsics = K.repeat(n_images, 1, 1)
    s.pixel_error_maps = torch.rand(n_images, H // DS, W // DS, device=DEV, generator=g)
    s.pixel_error_buffered = True
    return s


def lidar_source(n_points=4_000_000, scans=200):
    g = torch.Generator(device=DEV).manual_seed(1)
    s = rc.LidarSource()
    s.device = torch.device(DEV)
    s.origins = torch.randn(n_points, 3, device=DEV, generator=g)
    s.directions = torch.nn.functional.normalize(torch.randn(n_points, 3, device=DEV, generator=g), dim=-1)
    s.ranges = torch.rand(n_points, 1, device=DEV, generator=g) * 80
    s._timesteps = torch.sort(torch.randint(0, scans, (n_points,), device=DEV, generator=g)).values
    s._normalized_timestamps = s._timesteps.float() / (scans - 1)
    return s


def measure(fns, calls, warmup):
    """fns: name -> zero-argument call.  Alternates the formulations call by call."""
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    dev_ms = {k: 0.0 for k in fns}
    wall_ms = {k: 0.0 for k in fns}
    for _ in range(calls):
        for name, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            wall_ms[name] += (time.perf_counter() - t0) * 1e3
            dev_ms[name] += e0.elapsed_time(e1)
    res = {}
    for name, fn in fns.items():
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                fn()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        syncs = sum("synchroniz" in str(x.message) for x in w)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
        res[name] = {"device_ms": round(dev_ms[name] / calls, 4), "wall_ms": round(wall_ms[name] / calls, 4),
                     "host_syncs": syncs, "cuda_kernels": kernels}
    return res


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_raybatch needs a CUDA device"
    result = {"info": gpu_info(), "rays": a.rays, "calls": a.calls, "pixel": {}, "lidar": {}}
    for n_images in (600, 1000):
        for features in (False, True):
            src = pixel_source(n_images, features)
            cand = [i for i in range(n_images) if i % 10 != 3]
            for ratio in (0.0, 0.25):
                src.data_cfg.sampler.buffer_ratio = ratio
                sampler = raygen.PixelRaySampler(src)
                fns = {"reference": lambda: raybatch_ref.pixel_train_rays(src, a.rays, cand),
                       "device": lambda: sampler.get_train_rays(a.rays, cand)}
                key = f"{n_images}img_ratio{ratio}_{'feat' if features else 'nofeat'}"
                result["pixel"][key] = measure(fns, a.calls, a.warmup)
                print(key, json.dumps(result["pixel"][key]), flush=True)
            del src
            torch.cuda.empty_cache()
    lsrc = lidar_source()
    lcand = list(range(0, 200, 10)) + list(range(1, 200, 10))
    lsampler, cache = raygen.LidarRaySampler(lsrc), raybatch_ref.LidarCache()
    fns = {"reference": lambda: raybatch_ref.lidar_train_rays(lsrc, a.rays, lcand, cache),
           "device": lambda: lsampler.get_train_rays(a.rays, lcand)}
    result["lidar"]["4Mpts_200scans"] = measure(fns, a.calls, a.warmup)
    out_dir = a.out or tempfile.mkdtemp(prefix="bench_raybatch_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_raybatch.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()

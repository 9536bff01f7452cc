"""Per-image evaluation metrics, the reference's formulation vs emernerf_b200.metrics, on one GPU.

    python tools/bench_metrics.py [--iters 10] [--warmup 2] [--no-features] [--out DIR]

Workloads: seeded 640 x 960 and 160 x 240 images (the evaluation and low-res sizes), predictions noisy copies of the
targets in [0, 1], a ~5 % dynamic mask and (unless --no-features) 64-channel feature maps, three images per pass.
Two formulations, alternating in the same process:
  reference  what radiance_fields/video_utils.py:205-247 does per image: torch PSNRs (``.item()``), the boolean-indexed
             masked PSNRs with their ``sum() > 0`` checks, two device-to-host copies, and skimage's float32 SSIM twice
             (plain, and ``full=True`` for the masked mean) -- restated by oracle.metrics_ref on
             scipy.ndimage.uniform_filter, as skimage computes it; then the aggregation of :421-428
  device     metrics.image_metrics per image and one metrics.summarize
Reported per size and formulation: host wall time per image (ending in a synchronize), CUDA kernels and copies
(torch.profiler, a separate pass), emer_* library launches and host syncs (torch.cuda.set_sync_debug_mode("warn")).
For the kernel alone: CUDA-event time over many launches and its achieved bytes/s against the algorithmic bytes (both
images, the mask and both feature maps read once).  Also the largest difference of the device's SSIM and PSNR from
the reference's float32 values.  The GPU's name and power limit come from the same run (nvidia-smi query, read only).
Writes DIR/bench_metrics.json and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import warnings

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from emernerf_b200 import _lib, metrics  # noqa: E402
from oracle import metrics_ref  # noqa: E402

SIZES = ((640, 960), (160, 240))
IMAGES = 3
CF = 64


def make_images(h, w, features, dev):
    out = []
    for i in range(IMAGES):
        g = torch.Generator().manual_seed(100 * h + i)
        y = torch.rand(h, w, 3, generator=g)
        x = (y + 0.05 * torch.randn(h, w, 3, generator=g)).clamp(0, 1)
        m = (torch.rand(h, w, generator=g) < 0.05).float()
        d = {"rgb": x.to(dev), "pixels": y.to(dev), "dynamic_masks": m.to(dev)}
        if features:
            fy = torch.randn(h, w, CF, generator=g)
            d["dino_feat"], d["features"] = (fy + 0.1 * torch.randn(h, w, CF, generator=g)).to(dev), fy.to(dev)
        out.append(d)
    return out


def ref_psnr(prediction, target):           # datasets/metrics.py:31-47
    return (-10 * torch.log10(F.mse_loss(prediction, target))).item()


def reference(images):
    get_numpy = lambda x: x.squeeze().cpu().numpy()
    non_zero_mean = lambda x: sum(x) / len(x) if len(x) > 0 else -1
    psnrs, ssims, masked_psnrs, masked_ssims, feat_psnrs, masked_feat_psnrs = [], [], [], [], [], []
    for d in images:
        rgb = d["rgb"]
        psnrs.append(ref_psnr(rgb, d["pixels"]))
        ssims.append(metrics_ref.ssim(get_numpy(rgb), get_numpy(d["pixels"]), "fp32")[0])
        dynamic_mask = get_numpy(d["dynamic_masks"]).astype(bool)
        if dynamic_mask.sum() > 0:
            masked_psnrs.append(ref_psnr(rgb[dynamic_mask], d["pixels"][dynamic_mask]))
            masked_ssims.append(metrics_ref.ssim(get_numpy(rgb), get_numpy(d["pixels"]), "fp32", dynamic_mask)[1])
        if "dino_feat" in d:
            feat_psnrs.append(ref_psnr(d["dino_feat"], d["features"]))
            m = d["dynamic_masks"].squeeze().bool()
            if m.sum() > 0:
                masked_feat_psnrs.append(ref_psnr(d["dino_feat"][m], d["features"][m]))
    return {"psnr": non_zero_mean(psnrs), "ssim": non_zero_mean(ssims), "feat_psnr": non_zero_mean(feat_psnrs),
            "masked_psnr": non_zero_mean(masked_psnrs), "masked_ssim": non_zero_mean(masked_ssims),
            "masked_feat_psnr": non_zero_mean(masked_feat_psnrs)}


def device(images):
    per = [metrics.image_metrics(d["rgb"], d["pixels"], d["dynamic_masks"], d.get("dino_feat"), d.get("features"))
           for d in images]
    return metrics.summarize(per)


WAYS = {"reference": reference, "device": device}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except Exception as e:                      # noqa: BLE001 -- reported, not fatal
        return f"nvidia-smi unavailable: {e}"


def count_launches(fn, images):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    n0 = _lib.LAUNCHES
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(images)
        torch.cuda.synchronize()
    kernels = copies = 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if e.name.startswith(("Memcpy", "Memset")):
            copies += 1
        else:
            kernels += 1
    return kernels, copies, _lib.LAUNCHES - n0


def count_syncs(fn, images):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn(images)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return sum("synchroniz" in str(w.message) for w in caught)


def kernel_rate(d, reps):
    """Device time of one image_metrics launch, from CUDA events around the replay of a graph of ``reps`` launches (so
    the host's launch overhead is not in it), and its algorithmic bytes."""
    h, w, c = d["rgb"].shape
    nbytes = 2 * h * w * c * 4 + h * w * 4 + (2 * h * w * CF * 4 if "dino_feat" in d else 0)
    args = (d["rgb"], d["pixels"], d["dynamic_masks"], d.get("dino_feat"), d.get("features"))
    for _ in range(5):
        metrics.image_metrics(*args)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(reps):
            metrics.image_metrics(*args)
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(5):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / (5 * reps)
    return {"kernel_us": ms * 1e3, "algorithmic_bytes": nbytes, "achieved_GBps": nbytes / (ms * 1e-3) / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-features", action="store_true")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_metrics"),
                    help="directory for bench_metrics.json (default: under the system's temporary directory)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_metrics measures on a CUDA device"
    dev = torch.device("cuda")
    result = {"gpu": gpu_info(), "torch": torch.__version__, "images_per_pass": IMAGES, "iters": args.iters,
              "features": 0 if args.no_features else CF, "sizes": {}}
    for h, w in SIZES:
        images = make_images(h, w, not args.no_features, dev)
        for _ in range(args.warmup):
            for fn in WAYS.values():
                fn(images)
        wall = {k: [] for k in WAYS}
        values = {}
        for it in range(args.iters):
            for way in (("reference", "device") if it % 2 == 0 else ("device", "reference")):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                values[way] = WAYS[way](images)
                torch.cuda.synchronize()
                wall[way].append((time.perf_counter() - t0) * 1e3 / IMAGES)
        entry = {}
        for way, fn in WAYS.items():
            kernels, copies, lib = count_launches(fn, images)
            entry[way] = {"ms_per_image_median": statistics.median(wall[way]), "ms_per_image_min": min(wall[way]),
                          "cuda_kernels": kernels, "cuda_memcpy_memset": copies, "library_launches": lib,
                          "host_syncs": count_syncs(fn, images), "values": values[way]}
        entry["max_abs_diff"] = {k: abs(values["device"][k] - v) for k, v in values["reference"].items()}
        entry["kernel"] = kernel_rate(images[0], reps=50)
        if not args.no_features:
            entry["kernel_no_features"] = kernel_rate({k: images[0][k] for k in ("rgb", "pixels", "dynamic_masks")},
                                                      reps=50)
        result["sizes"][f"{h}x{w}"] = entry
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_metrics.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()

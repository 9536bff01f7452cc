"""The error-map refresh and the render rays, the reference's torch path vs emernerf_b200.raygen, on one GPU.

    python tools/bench_errormap.py [--calls 3] [--warmup 1] [--ray-calls 50] [--out DIR]

Source: 600 images of 640 x 960 with sky and dynamic masks and timestamps (tools/bench_raybatch.py's), error maps at
buffer_downscale 16 (40 x 60).  Fields: the benchmarked static and dynamic configurations at full size
(tests/golden/full_cases.py: 2^20 / 2^18-entry tables, 64 samples, proposal samples [128, 64]).
Two formulations, in the same process, alternating call by call:
  refresh      reference: oracle.errormap_ref.cache_step, the reference's train_emernerf.py:889-904 (render_pixels
                          image by image with its host copies, then update_pixel_error_maps on the host)
               device:    PixelRaySampler.refresh_pixel_error_maps
  render rays  get_render_rays of one image at downscale 1 and 1/4 (the evaluation videos): oracle.errormap_ref vs
               PixelRaySampler.get_render_rays
Both formulations render through the package's render_rays.  Reported per configuration and formulation: device time
per call from CUDA events, host wall time per call ending in a synchronize, host syncs per call
(torch.cuda.set_sync_debug_mode("warn")) and CUDA kernels per call (torch.profiler, a separate pass), with
tools/bench_raybatch.py's ``measure``; for the refresh also the launches through the library's C ABI per call, which
the profiler does not list.  The refreshed maps of the two formulations are compared: bit for bit, and the share of
pixels within 1e-4.  The GPU's
name, power limit and maximum SM clock come from the same run (nvidia-smi query, read only).  Writes
DIR/bench_errormap.json (DIR defaults to a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import types

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests", "golden"))

from bench_raybatch import gpu_info, measure, pixel_source  # noqa: E402
from emernerf_b200 import _lib, raygen  # noqa: E402
from oracle import errormap_ref  # noqa: E402
import errormap_cases as ec  # noqa: E402
import full_cases as fc  # noqa: E402

DEV = "cuda"


def source():
    s = ec.PixelSource()
    vars(s).update(vars(pixel_source(600, False)))
    s._downscale_factor = 1.0
    return s


def models(variant):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder
    from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    field, props = fc.build_models(ns, variant)
    return field.to(DEV), [p.to(DEV) for p in props], PropNetEstimator(None, None).to(DEV)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ray-calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_errormap needs a CUDA device"
    from emernerf_b200.radiance_fields.render_utils import render_rays

    result = {"info": gpu_info(), "images": 600, "size": [640, 960], "buffer_downscale": 16, "refresh": {},
              "render_rays": {}}
    ref_src, dev_src = source(), source()
    sampler = raygen.PixelRaySampler(dev_src)
    cfg = fc.render_cfg()
    for variant in ("static", "dynamic"):
        field, props, est = models(variant)
        fns = {"reference": lambda: errormap_ref.cache_step(ref_src, field, est, props, cfg, render_rays),
               "device": lambda: sampler.refresh_pixel_error_maps(field, est, props, cfg)}
        result["refresh"][variant] = measure(fns, a.calls, a.warmup)
        # the reference's rays differ from the kernel's in the last bits of the view directions (within 1e-6)
        diff = (ref_src.pixel_error_maps - dev_src.pixel_error_maps).abs()
        result["refresh"][variant]["maps_bit_identical"] = bool(torch.equal(ref_src.pixel_error_maps,
                                                                            dev_src.pixel_error_maps))
        result["refresh"][variant]["maps_within_1e-4"] = round(float((diff <= 1e-4).float().mean()), 6)
        for name, fn in fns.items():
            before = _lib.LAUNCHES
            fn()
            result["refresh"][variant][name]["library_launches"] = _lib.LAUNCHES - before
        print(variant, json.dumps(result["refresh"][variant]), flush=True)
        del field, props, est, fns
        torch.cuda.empty_cache()
    for name, d in (("1", 1.0), ("1_4", 0.25)):
        ref_src._downscale_factor = dev_src._downscale_factor = d
        fns = {"reference": lambda: errormap_ref.get_render_rays(ref_src, 17),
               "device": lambda: sampler.get_render_rays(17)}
        result["render_rays"][name] = measure(fns, a.ray_calls, 5)
        print(name, json.dumps(result["render_rays"][name]), flush=True)
    out_dir = a.out or tempfile.mkdtemp(prefix="bench_errormap_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_errormap.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()

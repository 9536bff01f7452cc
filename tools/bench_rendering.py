"""The body of ``rendering``, op-by-op torch vs the fused emer_render_* kernels, on one GPU.

    python tools/bench_rendering.py [--iters 200] [--warmup 20] [--out DIR]

Workloads (seeded random field results at the shapes the field hands to ``rendering``):
  dynamic     R = 8192, S = 64: static + dynamic densities and colours, sky colour        -- forward + backward
  flow        dynamic + shadow, flows as 3-wide column slices of [R, S, 6] rows            -- forward + backward
  flow_feat   flow + 64-channel static / dynamic features, feature sky and PE              -- forward + backward
  eval_decomp flow_feat at R = 16384, S = 64 with return_decomposition=True, no grad      -- forward only
Each runs two ways, alternating in the same process: ``torch`` (EMER_RENDERING=torch, the default: emer_composite_*,
one emer_accumulate_* per accumulated quantity, the blend in torch ops) and ``fused`` (one emer_render_fwd, one
emer_render_bwd).  The backward feeds fixed upstream gradients to rgb, opacity, depth, shadow_ratio and dino_feat.
Reported per workload and way: device time (CUDA events; median and min), CUDA kernel launches and memory copies / sets
(torch.profiler, a separate pass), and the largest relative difference of the two ways' outputs.  The GPU's name, power
limit and SM clock limit are read in the same run (nvidia-smi query, read only).  Writes DIR/bench_rendering.json and
prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from emernerf_b200.radiance_fields import render_utils  # noqa: E402

C = 64
WORKLOADS = {
    "dynamic": (8192, 64, ("rgb_sky",), True),
    "flow": (8192, 64, ("shadow_ratio", "flows"), True),
    "flow_feat": (8192, 64, ("shadow_ratio", "flows", "rgb_sky", "dino"), True),
    "eval_decomp": (16384, 64, ("shadow_ratio", "flows", "rgb_sky", "dino"), False),
}
GRAD_OUTPUTS = ("rgb", "opacity", "depth", "shadow_ratio", "dino_feat")


def make_results(r, s, extra, grad, dev):
    g = torch.Generator().manual_seed(0)
    rnd = lambda *shape: torch.rand(*shape, generator=g).to(dev)       # noqa: E731
    delta = rnd(r, s) * 0.05 + 0.01
    t0 = 2.0 + torch.cumsum(delta, -1) - delta
    t1 = t0 + delta
    res = {"static_density": rnd(r, s) * 2.0, "dynamic_density": rnd(r, s) * 2.0,
           "static_rgb": rnd(r, s, 3), "dynamic_rgb": rnd(r, s, 3)}
    if "rgb_sky" in extra:
        res["rgb_sky"] = rnd(r, 3)
    if "shadow_ratio" in extra:
        res["shadow_ratio"] = rnd(r, s, 1)
    if "dino" in extra:
        res.update(static_dino_feat=rnd(r, s, C), dynamic_dino_feat=rnd(r, s, C), dino_sky_feat=rnd(r, C),
                   dino_pe=rnd(r, C))
    leaves = {k: v.requires_grad_(grad) for k, v in res.items()}
    if "flows" in extra:
        flow = rnd(r, s, 6)
        res["forward_flow"], res["backward_flow"] = flow[..., :3], flow[..., 3:]
    return t0, t1, res, leaves


def step(way, work, data, ups):
    t0, t1, res, leaves = data
    r, s, extra, train = WORKLOADS[work]
    render_utils.RENDERING = way
    for v in leaves.values():
        v.grad = None

    def query_fn(a, b):
        out = dict(res)
        out["density"] = out["static_density"] + out["dynamic_density"]
        return out

    with torch.set_grad_enabled(train):
        out = render_utils.rendering(t0, t1, query_fn, return_decomposition=not train)
        if train:
            keys = [k for k in GRAD_OUTPUTS if k in out]
            torch.autograd.backward([out[k] for k in keys], [ups[k] for k in keys])
    return out


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except Exception as e:                      # noqa: BLE001 -- reported, not fatal
        return f"nvidia-smi unavailable: {e}"


def count_launches(way, work, data, ups):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(way, work, data, ups)
        torch.cuda.synchronize()
    kernels = copies = 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if e.name.startswith(("Memcpy", "Memset")):
            copies += 1
        else:
            kernels += 1
    return kernels, copies


def max_rel_diff(a, b):
    worst = 0.0
    for k, v in b.items():
        if k == "extras" or k not in a:
            continue
        d = (a[k].detach().double() - v.detach().double()).abs().max().item()
        worst = max(worst, d / max(v.detach().double().abs().max().item(), 1e-30))
    return worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_rendering"),
                    help="directory for bench_rendering.json (default: under the system's temporary directory)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rendering measures on a CUDA device"
    dev = torch.device("cuda")
    result = {"gpu": gpu_info(), "torch": torch.__version__, "iters": args.iters, "workloads": {}}
    for work, (r, s, extra, train) in WORKLOADS.items():
        data = make_results(r, s, extra, train, dev)
        g = torch.Generator().manual_seed(1)
        ups = {"rgb": torch.randn(r, 3, generator=g).to(dev), "opacity": torch.randn(r, 1, generator=g).to(dev),
               "depth": torch.randn(r, 1, generator=g).to(dev), "shadow_ratio": torch.randn(r, 1, generator=g).to(dev),
               "dino_feat": torch.randn(r, C, generator=g).to(dev)}
        outs = {}
        for _ in range(args.warmup):
            for way in ("torch", "fused"):
                outs[way] = step(way, work, data, ups)
        dev_ms = {"torch": [], "fused": []}
        torch.cuda.synchronize()
        for it in range(args.iters):
            for way in (("torch", "fused") if it % 2 == 0 else ("fused", "torch")):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(way, work, data, ups)
                e1.record()
                torch.cuda.synchronize()
                dev_ms[way].append(e0.elapsed_time(e1))
        entry = {"rays": r, "samples": s, "backward": train}
        for way in ("torch", "fused"):
            kernels, copies = count_launches(way, work, data, ups)
            entry[way] = {"device_ms_median": statistics.median(dev_ms[way]), "device_ms_min": min(dev_ms[way]),
                          "cuda_kernels": kernels, "cuda_memcpy_memset": copies}
        entry["speedup_median"] = entry["torch"]["device_ms_median"] / entry["fused"]["device_ms_median"]
        entry["outputs_max_rel_diff"] = max_rel_diff(outs["fused"], outs["torch"])
        if train:
            grads = {}
            for way in ("torch", "fused"):
                step(way, work, data, ups)
                grads[way] = {k: v.grad.clone() for k, v in data[3].items()}
            entry["grads_max_rel_diff"] = max_rel_diff(grads["fused"], grads["torch"])
        result["workloads"][work] = entry
        del data
        torch.cuda.empty_cache()
    render_utils.RENDERING = "torch"
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_rendering.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()

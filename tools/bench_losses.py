"""Forward + backward of the training losses, eager torch vs emernerf_b200.loss, on one GPU.

    python tools/bench_losses.py [--iters 200] [--warmup 20] [--out DIR]

Workloads (R = 8192 rays, S = 64 samples, seeded; targets from emernerf_b200.synthetic, predictions random):
  lidar      range (l2), line of sight (epsilon 2.5, coef 0.1), lidar dynamic sparsity   -- the lidar pass
  static     rgb l2 + opacity-based sky                                                 -- the pixel pass, by config
  dynamic    static + dynamic sparsity + shadow
  flow_feat  dynamic + feature l2 (64 channels)
  cycle      the flow variants' cycle loss (coef 0.01) and its four flow statistics (train_emernerf.py:700-740), the
             flows 3-wide column slices of [R, S, 6] rows as the flow MLP writes them
Each set runs two ways, alternating in the same process: ``torch`` -- the reference's arithmetic restated op by op
(boolean indexing in the range loss, as the reference) -- and ``fused`` -- the emernerf_b200.loss classes.
Reported per set and way: device time (CUDA events), host wall time (ending in a synchronize), CUDA kernel launches
and memory copies / sets (torch.profiler, a separate pass), and host synchronisations (counted under
torch.cuda.set_sync_debug_mode("warn")).  The GPU's name and power limit are read in the same run (nvidia-smi query,
read only).  Writes DIR/bench_losses.json and prints it.  Losses only: this is not a training-step time.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile
import time
import warnings

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from emernerf_b200 import loss as fused_loss  # noqa: E402
from emernerf_b200 import synthetic  # noqa: E402

R, S, EPS = 8192, 64, 2.5
SETS = {
    "lidar": ("range", "line_of_sight", "lidar_dynamic"),
    "static": ("rgb", "sky"),
    "dynamic": ("rgb", "sky", "dynamic", "shadow"),
    "flow_feat": ("rgb", "sky", "dynamic", "shadow", "feature"),
    "cycle": ("cycle",),
}
LEAVES = ("rgb", "opacity", "depth", "weights", "dynamic_density", "shadow_ratio", "dino_feat", "flow_fwd_query",
          "flow_bwd_query")


def make_inputs(dev):
    pix = synthetic.pixel_batch(R, seed=0, features=True, device=dev)
    lid = synthetic.lidar_batch(R, seed=0, device=dev)
    g = torch.Generator().manual_seed(1)
    rnd = lambda *s: torch.rand(*s, generator=g).to(dev)
    x = {
        "pixels": pix["pixels"], "sky_masks": pix["sky_masks"], "features": pix["features"],
        "lidar_ranges": lid["lidar_ranges"],
        "rgb": rnd(R, 3), "opacity": rnd(R, 1).clamp(1e-6, 1.0), "depth": rnd(R, 1) * 90.0,
        "weights": rnd(R, S) * 0.05, "t_vals": torch.sort(rnd(R, S) * 100.0, -1).values,
        "dynamic_density": rnd(R, S) * 2.0, "shadow_ratio": rnd(R, 1), "dino_feat": rnd(R, 64),
    }
    # the flow MLP's [R, S, 6] outputs at the samples and at the two warped queries
    x["flow"] = rnd(R, S, 6) * 2.0 - 1.0
    x["flow_fwd_query"] = rnd(R, S, 6) * 2.0 - 1.0
    x["flow_bwd_query"] = rnd(R, S, 6) * 2.0 - 1.0
    for k in LEAVES:
        x[k].requires_grad_()
    return x


# ------------------------------------------------------------------ the reference's arithmetic, eager torch, fp32
def flow_extras(x):
    return {"forward_flow": x["flow"][..., :3], "backward_flow": x["flow"][..., 3:],
            "forward_pred_backward_flow": x["flow_fwd_query"][..., 3:],
            "backward_pred_forward_flow": x["flow_bwd_query"][..., :3]}


def torch_term(name, x):
    if name == "cycle":
        ex = flow_extras(x)
        cycle = 0.5 * ((ex["forward_flow"].detach() + ex["forward_pred_backward_flow"]) ** 2
                       + (ex["backward_flow"].detach() + ex["backward_pred_forward_flow"]) ** 2).mean()
        x["stats"] = {"max_forward_flow_norm": ex["forward_flow"].detach().norm(dim=-1).max(),
                      "max_backward_flow_norm": ex["backward_flow"].detach().norm(dim=-1).max(),
                      "max_forward_pred_backward_flow_norm": ex["forward_pred_backward_flow"].norm(dim=-1).max(),
                      "max_backward_pred_forward_flow_norm": ex["backward_pred_forward_flow"].norm(dim=-1).max()}
        return cycle * 0.01
    if name == "rgb":
        return F.mse_loss(x["rgb"].squeeze(), x["pixels"].squeeze(), reduction="none").mul(1.0).mean() * 1.0
    if name == "sky":
        return F.binary_cross_entropy(x["opacity"].squeeze(), 1 - x["sky_masks"].float(), reduction="none").mean() * 1e-3
    if name == "feature":
        return F.mse_loss(x["dino_feat"].squeeze(), x["features"].squeeze(), reduction="none").mul(1.0).mean() * 0.5
    if name in ("dynamic", "lidar_dynamic"):
        return x["dynamic_density"].mean() * 0.01
    if name == "shadow":
        return x["shadow_ratio"].mean() * 0.01
    if name == "range":
        pred, gt = x["depth"].squeeze(), x["lidar_ranges"].squeeze()
        valid = (gt > 0.01) & (gt < 80)
        nd = lambda d: torch.clamp(d / 80, 0.0, 1.0)
        return F.mse_loss(nd(pred[valid]), nd(gt[valid]), reduction="none").mean() * 1.0
    # line of sight: accumulate_along_rays(values, mask) is (values[..., None] * mask).sum(-2)
    gt, t, w = x["lidar_ranges"].squeeze(), x["t_vals"].detach().squeeze(), x["weights"]
    depth_mask = gt > 0
    gt = gt.unsqueeze(-1)
    empty = (t < gt - EPS).unsqueeze(-1)
    near = ((t > gt - EPS) & (t < gt + EPS)).unsqueeze(-1)
    sig = EPS / 3
    dirac = (1 / math.sqrt(2 * torch.pi * sig**2)) * torch.exp(-((t - gt) ** 2) / (2 * sig**2))
    e = (w.square()[..., None] * empty).sum(-2).mean()
    n = ((w - dirac).square()[..., None] * near).sum(-2).mean()
    return ((e + n) * depth_mask * 1.0).mean() * 0.1


FUSED = {
    "rgb": lambda: fused_loss.RealValueLoss(loss_type="l2", coef=1.0, name="rgb"),
    "sky": lambda: fused_loss.SkyLoss(loss_type="opacity_based", coef=1e-3),
    "feature": lambda: fused_loss.RealValueLoss(loss_type="l2", coef=0.5, name="feature"),
    "dynamic": lambda: fused_loss.DynamicRegularizationLoss(loss_type="sparsity", coef=0.01),
    "lidar_dynamic": lambda: fused_loss.DynamicRegularizationLoss(loss_type="sparsity", coef=0.01),
    "shadow": lambda: fused_loss.DynamicRegularizationLoss(name="shadow", loss_type="sparsity", coef=0.01),
    "range": lambda: fused_loss.DepthLoss(loss_type="l2", coef=1.0),
    "line_of_sight": lambda: fused_loss.LineOfSightLoss(coef=0.1),
    "cycle": lambda: None,
}


def fused_term(fn, name, x):
    if name == "cycle":
        cycle, x["stats"] = fused_loss.flow_cycle_loss(flow_extras(x))
        return cycle
    if name == "rgb":
        return fn(x["rgb"], x["pixels"])
    if name == "sky":
        return fn(x["opacity"], x["sky_masks"])
    if name == "feature":
        return fn(x["dino_feat"], x["features"])
    if name == "dynamic":
        return fn(x["dynamic_density"])
    if name == "lidar_dynamic":
        return fn(x["dynamic_density"], name="lidar_dynamic")
    if name == "shadow":
        return fn(x["shadow_ratio"])
    if name == "range":
        return fn(x["depth"], x["lidar_ranges"], name="lidar_range_loss")
    return fn(x["depth"], x["lidar_ranges"], x["weights"], x["t_vals"], epsilon=EPS, name="lidar_line_of_sight",
              coef_decay=1.0)


def step(way, names, x, fns):
    for k in LEAVES:
        x[k].grad = None
    x.pop("stats", None)
    if way == "torch":
        total = sum(torch_term(n, x) for n in names)
    else:
        total = sum(v for n in names for v in fused_term(fns[n], n, x).values())
    total.backward()
    return total


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except Exception as e:                      # noqa: BLE001 -- reported, not fatal
        return f"nvidia-smi unavailable: {e}"


def count_launches(way, names, x, fns):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(way, names, x, fns)
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


def count_syncs(way, names, x, fns):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            step(way, names, x, fns)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return sum("synchroniz" in str(w.message) for w in caught)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_losses"),
                    help="directory for bench_losses.json (default: under the system's temporary directory)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_losses measures on a CUDA device"
    dev = torch.device("cuda")
    x = make_inputs(dev)
    fns = {k: f() for k, f in FUSED.items()}
    result = {"gpu": gpu_info(), "torch": torch.__version__, "rays": R, "samples": S, "iters": args.iters,
              "sets": {}}
    for set_name, names in SETS.items():
        for _ in range(args.warmup):
            for way in ("torch", "fused"):
                step(way, names, x, fns)
        dev_ms = {"torch": [], "fused": []}
        host_ms = {"torch": [], "fused": []}
        values, stats = {}, {}
        torch.cuda.synchronize()
        for it in range(args.iters):
            for way in (("torch", "fused") if it % 2 == 0 else ("fused", "torch")):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record()
                total = step(way, names, x, fns)
                e1.record()
                torch.cuda.synchronize()
                host_ms[way].append((time.perf_counter() - t0) * 1e3)
                dev_ms[way].append(e0.elapsed_time(e1))
                values[way] = total.item()
                if "stats" in x:
                    stats[way] = {k: v.item() for k, v in x["stats"].items()}
        entry = {}
        for way in ("torch", "fused"):
            kernels, copies = count_launches(way, names, x, fns)
            entry[way] = {
                "device_ms_median": statistics.median(dev_ms[way]), "device_ms_min": min(dev_ms[way]),
                "host_wall_ms_median": statistics.median(host_ms[way]), "host_wall_ms_min": min(host_ms[way]),
                "cuda_kernels": kernels, "cuda_memcpy_memset": copies,
                "host_syncs": count_syncs(way, names, x, fns), "loss": values[way],
            }
        entry["loss_rel_diff"] = abs(values["fused"] - values["torch"]) / max(abs(values["torch"]), 1e-30)
        if stats:
            entry["stats_max_rel_diff"] = max(abs(stats["fused"][k] - v) / max(abs(v), 1e-30)
                                              for k, v in stats["torch"].items())
        result["sets"][set_name] = entry
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_losses.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()

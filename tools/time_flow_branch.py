"""Time the flow configs' field pass with EMER_FLOW_BRANCH=layers and =fused, alternating, with CUDA events.

    python tools/time_flow_branch.py [--variant flow|flow_feat] [--rays 8192] [--samples 64] [--reps 20] [--dump DIR]

The benchmark's field (configs.build_hot_path, N(0, 0.3) tables) is evaluated on one synthetic pixel batch of
rays x samples points (524 288 by default) laid along the rays, in training mode with a fixed warp noise: forward,
then backward of a sum of squares of every differentiable output.  Each switch is timed over --reps passes after
warm-up, in alternating blocks; the medians of forward and forward + backward are printed, with the GPU's name and
power limit.  --dump DIR writes each switch's outputs as DIR/<switch>_<key>.npy for comparison between builds.
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from emernerf_b200 import _ops, configs, synthetic


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", default="flow", choices=["flow", "flow_feat"])
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dump", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_flow_branch: no CUDA device")
    dev = torch.device("cuda")
    cfg = configs.make_cfg(args.variant, num_samples=args.samples)
    field = configs.build_hot_path(cfg, dev, table_std=0.3, capturable=False, optimizer="torch")[0]
    field.train()
    b = {k: v.to(dev) for k, v in synthetic.pixel_batch(args.rays, cfg.data.num_timesteps, 3, seed=0,
                                                          features=args.variant == "flow_feat").items()}
    S = args.samples
    tv = torch.linspace(1.0, 80.0, S, device=dev).expand(args.rays, S)
    d = b["viewdirs"][:, None, :].expand(-1, S, -1)
    pos = b["origins"][:, None, :] + d * tv[..., None]
    sub = {k: v.reshape(args.rays, -1)[:, :1].expand(args.rays, S) for k, v in b.items()
           if k in ("normed_timestamps", "img_idx", "cam_idx")}
    sub["pixel_coords"] = b["pixel_coords"]
    field._noise_override = torch.rand(args.rays, S, 1, generator=torch.Generator().manual_seed(1)).to(dev)
    params = [p for p in field.parameters() if p.requires_grad]

    def fwd():
        return field(pos, d, sub)

    def step():
        out = fwd()
        loss = sum((v.float() ** 2).mean() for v in out.values() if torch.is_tensor(v) and v.requires_grad)
        torch.autograd.grad(loss, params, allow_unused=True)
        return out

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    res = {sw: {"fwd": [], "step": []} for sw in ("layers", "fused")}
    for _ in range(args.rounds):
        for sw in ("layers", "fused"):
            _ops.FLOW_BRANCH = sw
            for _ in range(args.warmup):
                step()
            res[sw]["fwd"] += [timed(fwd) for _ in range(args.reps)]
            res[sw]["step"] += [timed(step) for _ in range(args.reps)]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"{args.variant}: {args.rays} rays x {S} samples = {args.rays * S} points; {gpu}")
    for sw in ("layers", "fused"):
        f, s = statistics.median(res[sw]["fwd"]), statistics.median(res[sw]["step"])
        print(f"  EMER_FLOW_BRANCH={sw:6s}  forward {f:7.3f} ms   forward + backward {s:7.3f} ms")
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        for sw in ("layers", "fused"):
            _ops.FLOW_BRANCH = sw
            with torch.no_grad():
                out = fwd()
            for k, v in out.items():
                if torch.is_tensor(v):
                    np.save(os.path.join(args.dump, f"{sw}_{k}.npy"), v.float().cpu().numpy())


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""The reference's training iteration (train_emernerf.py:612-855: a pixel pass and a lidar pass, two or three Adam
steps) run eagerly, as users run the loop, against ``train.CapturedIteration``, alternating in one process.

    python tools/bench_iteration.py [--rays 8192] [--iters 200] [--blocks 4] [--variants static dynamic flow flow_feat]

Per variant: the benchmark's field (``make_cfg(small=False)``: 2^20-entry tables, 64 samples, proposal samples
[128, 64]) with FusedAdam, the reference's schedulers and the package's losses, ``--rays`` pixel and ``--rays`` lidar
rays per iteration drawn by the device samplers from the test fixture sources (12 images of 64 x 96, uniform rays;
500 lidar points).  The eager loop is the restatement the tests use as their oracle
(tests/captured_iteration_cases.reference_iteration), with the ``.item()`` reads the loop makes; the captured run
drains its logged values once per block.  Iterations start at step 3000 of a 25 000-step schedule (steady state of
the proposal schedule, line of sight on).  Reported per iteration: milliseconds (CUDA events over each block, blocks
alternating), Python-side library launches, host syncs (torch's sync debug mode over 20 separate iterations) and
the reserved memory each arm adds: its setup plus its peak over the warm-up, above what the emptied cache held
before the arm was built (so the eager arm's state is not counted in the captured arm's figure).  One JSON line per variant, after the card's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]

import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable: {e}"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q}


def count_syncs(fn, n):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        for _ in range(n):
            fn()
    torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message).lower() for w in caught) / n


def run_variant(variant, args):
    import captured_iteration_cases as cic
    from emernerf_b200 import _lib

    kw = dict(pixel_rays=args.rays, lidar_rays=args.rays, num_iters=25000, start_iter=2000, decay_steps=2000,
              small=False)
    step = {"eager": 3000, "captured": 3000}

    def footprint(build, run):
        """Reserved memory an arm adds: its setup, then its peak over the warm-up, above what the cache held
        (emptied) before the setup was built."""
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_reserved()
        torch.cuda.reset_peak_memory_stats()
        made = build()
        for _ in range(args.warmup):
            run()
        torch.cuda.synchronize()
        return made, torch.cuda.max_memory_reserved() - base

    def one_eager():
        cic.reference_iteration(holder["eager"], step["eager"])
        step["eager"] += 1

    def one_captured():
        holder["it"](step["captured"])
        step["captured"] += 1

    def make_eager():
        s = cic.make_setup(variant, **kw)
        s.dataset.pixel_source.pixel_error_buffered = False
        return s

    def make_captured():
        s = cic.make_setup(variant, **kw)
        s.dataset.pixel_source.pixel_error_buffered = False
        return cic.captured(s)

    holder = {}
    eager, mem_eager = footprint(lambda: holder.setdefault("eager", make_eager()), one_eager)
    it, mem_captured = footprint(lambda: holder.setdefault("it", make_captured()), one_captured)
    it.drain()
    graphs = sum(g.graph is not None for g in it._graphs.values())

    per = args.iters // args.blocks
    ms = {"eager": 0.0, "captured": 0.0}
    launches = {"eager": 0, "captured": 0}
    for _ in range(args.blocks):
        for name, fn in (("eager", one_eager), ("captured", one_captured)):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n0 = _lib.LAUNCHES
            e0.record()
            for _ in range(per):
                fn()
            if name == "captured":
                it.drain()
            e1.record()
            torch.cuda.synchronize()
            launches[name] += _lib.LAUNCHES - n0
            ms[name] += e0.elapsed_time(e1)
    n = per * args.blocks
    syncs = {"eager": count_syncs(one_eager, 20), "captured": count_syncs(one_captured, 20)}
    it.drain()
    return {"variant": variant, "rays_per_pass": args.rays, "iterations_timed": n,
            "ms_per_iteration": {k: v / n for k, v in ms.items()},
            "speedup": ms["eager"] / ms["captured"],
            "python_library_launches_per_iteration": {k: v / n for k, v in launches.items()},
            "host_syncs_per_iteration": syncs,
            "reserved_by_arm_mib": {"eager": mem_eager / 2**20, "captured": mem_captured / 2**20},
            "captured_graphs": graphs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--blocks", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--variants", nargs="+", default=["static", "dynamic", "flow", "flow_feat"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_iteration.py needs a CUDA device")
    print(json.dumps(card()), flush=True)
    for v in args.variants:
        print(json.dumps(run_variant(v, args)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

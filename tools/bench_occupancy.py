"""Few-shot occupancy evaluation, the reference's formulation vs emernerf_b200.metrics, on one GPU.

    python tools/bench_occupancy.py [--frames 3] [--centroid-frames 20] [--occupied 0.1] [--out DIR]

Model: the benchmark-size ``flow_feat`` field of bench.py (configs.make_cfg("flow_feat"), trained-like N(0, 0.5)
tables), in eval mode.  Frames: seeded voxel centres on Occ3D's 0.4 m (100 x 200 x 16) and 0.1 m (800 x 1600 x 64)
grids, the front half of the grid as the reference's get_occ keeps it, ``--occupied`` of those voxels occupied, and
random labels of 15 classes.  Two formulations, in the same process:
  reference  oracle.occupancy_ref: per frame a density pass, boolean indexing, a second pass with the feature head,
             the cosine kNN and per-class ``.item()`` reads; centroids from the concatenated kept features
  device     metrics.collect_centroids / metrics.eval_few_shot_occ: one field pass per chunk, one kernel per chunk
Reported per grid and formulation: eval_few_shot_occ's wall time per frame (ending in a synchronize), host syncs per
frame (torch.cuda.set_sync_debug_mode("warn")), CUDA kernels per frame (torch.profiler, a separate pass) and the
peak memory of collect_centroids over ``--centroid-frames`` train frames.  For the kernels alone: CUDA-event time of
each over repeated launches on one 2^20-voxel chunk, and its achieved bytes/s for n (4 C + 12) bytes.  The GPU's name
and power limit come from the same run (nvidia-smi query, read only).  Writes DIR/bench_occupancy.json and prints it.
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

from emernerf_b200 import _lib, _ops, metrics  # noqa: E402
from emernerf_b200.configs import build_hot_path, make_cfg  # noqa: E402
from oracle import occupancy_ref  # noqa: E402

GRIDS = {"0.4m": (100, 200, 16), "0.1m": (800, 1600, 64)}
AABB = {"0.4m": ((0.0, -40.0, -1.0), 0.4), "0.1m": ((0.0, -80.0, -5.0), 0.1)}      # datasets/waymo.py:577-586
N_CLASSES = 15


class SeededOcc:
    """get_occ(i): the occupied voxels of frame i, generated on the device (nothing held between frames)."""

    def __init__(self, grid, occupied, timesteps=200):
        self.grid, self.occupied, self.timesteps = grid, occupied, timesteps
        self.label_mapping = {j: f"class{j}" for j in range(N_CLASSES)}
        x, y, z = GRIDS[grid]
        self.front = (x // 2, y, z)
        self.n = int(self.front[0] * y * z * occupied)

    def get_occ(self, index):
        g = torch.Generator(device="cuda").manual_seed(index)
        x, y, z = self.front
        flat = torch.randperm(x * y * z, generator=g, device="cuda")[:self.n]
        ijk = torch.stack([flat // (y * z) + x, flat // z % y, flat % z], -1).float()
        (ox, oy, oz), v = AABB[self.grid]
        coords = torch.stack([ijk[:, 0] * v + ox + v / 2, ijk[:, 1] * v + oy + v / 2, ijk[:, 2] * v + oz + v / 2], -1)
        labels = torch.randint(0, N_CLASSES, (self.n,), generator=g, device="cuda")
        return coords, labels, torch.full((self.n,), index / (self.timesteps - 1), device="cuda")


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
    torch.cuda.synchronize()
    return sum("synchroniz" in str(w.message) for w in caught)


def count_kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset")))


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return peak


def kernel_rates(field, ds, reps=50):
    """CUDA-event time of each occupancy kernel on one chunk of the field's real outputs."""
    coords, labels, t = ds.get_occ(0)
    n = min(metrics.OCC_CHUNK_POINTS, labels.numel())
    with torch.no_grad():
        out = field.forward(positions=coords[:n], data_dict={"normed_timestamps": t[:n]}, combine_static_dynamic=True,
                            query_feature_head=True, query_pe_head=False)
    feat, dens, lab = out["dino_feat"].contiguous(), out["density"].reshape(-1).contiguous(), labels[:n].contiguous()
    c, k = feat.shape[1], N_CLASSES
    sums = torch.zeros(k, c, dtype=torch.float64, device="cuda")
    counts = torch.zeros(2 * k + 2, dtype=torch.int64, device="cuda")
    cen = torch.randn(k, c, device="cuda")
    bank = torch.arange(k, device="cuda")
    ws = _ops._ptr(metrics._occ_workspace(feat.device))
    common = (_ops._ptr(feat), c, c, _ops._ptr(dens), 1, _ops._ptr(lab), n)
    launches = {
        "emer_occ_accumulate": lambda: _lib.call("emer_occ_accumulate", *common, k, 0.2, _ops._ptr(sums),
                                                 _ops._ptr(counts), ws, _ops._stream()),
        "emer_occ_classify": lambda: _lib.call("emer_occ_classify", *common, _ops._ptr(cen), k, _ops._ptr(bank), 0.2,
                                               _ops._ptr(counts), ws, _ops._stream()),
    }
    res = {}
    nbytes = n * (4 * c + 12)
    for name, fn in launches.items():
        for _ in range(5):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / reps
        res[name] = {"n": n, "channels": c, "classes": k, "us": round(us, 2), "bytes": nbytes,
                     "GB_per_s": round(nbytes / us / 1e3, 1),
                     "kept_fraction": round(float((dens > 0.2).float().mean()), 3)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--centroid-frames", type=int, default=20)
    ap.add_argument("--occupied", type=float, default=0.1)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_occupancy"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_occupancy measures on a GPU"
    field, _, _, _ = build_hot_path(make_cfg("flow_feat"), device="cuda", table_std=0.5)
    field.eval()
    result = {"gpu": gpu_info(), "torch": torch.__version__, "grids": {}}
    forms = {"reference": occupancy_ref, "device": metrics}
    for grid in GRIDS:
        ds = SeededOcc(grid, args.occupied)
        test = list(range(100, 100 + args.frames))
        row = {"voxels_per_frame": ds.n}
        for name, mod in forms.items():
            cen, bank = mod.collect_centroids([0], ds, field, "cuda")
            mod.eval_few_shot_occ([99], ds, field, "cuda", cen, bank)          # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = mod.eval_few_shot_occ(test, ds, field, "cuda", cen, bank)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3 / len(test)
            syncs = count_syncs(lambda: mod.eval_few_shot_occ(test[:1], ds, field, "cuda", cen, bank))
            kernels = count_kernels(lambda: mod.eval_few_shot_occ(test[:1], ds, field, "cuda", cen, bank))
            peak = peak_bytes(lambda: mod.collect_centroids(list(range(args.centroid_frames)), ds, field, "cuda"))
            row[name] = {"ms_per_frame": round(ms, 2), "host_syncs_per_frame": syncs, "cuda_kernels_per_frame": kernels,
                         "collect_centroids_peak_MB": round(peak / 2**20, 1),
                         "micro_accuracy": got["micro_accuracy"], "num_measured_points": got["num_measured_points"]}
        row["kernels"] = kernel_rates(field, ds)
        result["grids"][grid] = row
        print(json.dumps({grid: row}), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_occupancy.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()

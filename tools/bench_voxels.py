"""The voxel lifting on one GPU: ``emernerf_b200.voxels.visualize_voxels`` beside the reference's loop
(``oracle.voxels_ref``, on the same drop-in renderer and field) in the same process.

    python tools/bench_voxels.py [--timesteps 12] [--calls 3] [--voxel-size 0.3] [--out DIR]

Field: the benchmark-size ``flow_feat`` configuration (``configs.make_cfg("flow_feat")``, tables N(0, 0.5^2), every
density exponent raised by DENSITY_SHIFT so that the static gate keeps voxels).  Source:
tools/bench_trajectory.py's Waymo-shaped rig of 3 cameras, --timesteps timesteps, rendered at downscale 0.25
(160 x 240 rays per image), bound to ``raygen.PixelRaySampler``.  Reported per call, after one warm-up call of each:
  wall_ms            host clock between device synchronizes, both versions, alternating
  split_ms           the new version's phases: rendering and marking (mark_images), PCA, compaction and query
  syncs              host syncs (torch's sync debug mode, counted) of one call of each version
  library_launches   launches through the library's C ABI per call (the reference loop's torch kernels not counted)
  kernel_ms          CUDA-event time of each new kernel per call (the library's profile hook), summed
The per-image render dominates both versions.  The GPU's name and power limit come from the same run.  Writes
DIR/bench_voxels.json (DIR defaults to a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time
import types
import warnings

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests", "golden"))

import bench_trajectory as bt  # noqa: E402
from bench_raybatch import gpu_info  # noqa: E402
from emernerf_b200 import _lib, configs, raygen, voxels  # noqa: E402
from oracle import voxels_ref  # noqa: E402

DEV = "cuda"
DENSITY_SHIFT = 1.0
KERNELS = ("emer_voxel_mark", "emer_voxel_compact", "emer_voxel_select")


class PixelSet:
    def __init__(self, sampler, n):
        self.sampler, self.n = sampler, n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return dict(self.sampler.get_render_rays(i))


def dataset(timesteps):
    bt.TIMESTEPS = timesteps
    src = bt.source()
    src._downscale_factor = 0.25
    sampler = raygen.PixelRaySampler(src)
    src.get_render_rays = sampler.get_render_rays
    ps = types.SimpleNamespace(unique_normalized_timestamps=torch.unique(src._normalized_timestamps))
    return types.SimpleNamespace(full_pixel_set=PixelSet(sampler, len(src.cam_to_worlds)), num_cams=bt.CAMS,
                                 pixel_source=ps)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def count_syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(x.message) for x in w)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timesteps", type=int, default=12)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--voxel-size", type=float, default=0.3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_voxels needs a CUDA device"
    from emernerf_b200.radiance_fields.render_utils import render_rays

    cfg = configs.make_cfg("flow_feat")
    field, props, est, _ = configs.build_hot_path(cfg, DEV, table_std=0.5)
    with torch.no_grad():                  # +1 on every density exponent: the random-init densities sit below 0.5
        for m in [field] + list(props):
            for k, v in m.named_parameters():
                if k.endswith("base_mlp.2.bias"):
                    v[0] += DENSITY_SHIFT
    cfg.render.vis_voxel_size = a.voxel_size
    ds = dataset(a.timesteps)
    new = lambda: voxels.visualize_voxels(cfg, field, est, props, ds, is_dynamic=True)  # noqa: E731
    ref = lambda: voxels_ref.visualize_voxels(cfg, field, est, props, ds, DEV, True, render_rays,  # noqa: E731
                                              voxels.robust_pca)
    result = {"info": gpu_info(), "images": len(ds.full_pixel_set), "rays_per_image": 160 * 240,
              "voxel_size": a.voxel_size}
    torch.manual_seed(0)
    got_new, _ = timed(new)
    torch.manual_seed(0)
    got_ref, _ = timed(ref)
    result["static_voxels"] = {"new": len(got_new["coords"]), "reference": len(got_ref["coords"])}
    result["dynamic_groups"] = {"new": [len(x) for x in got_new["dynamic_coords"]],
                                "reference": [len(x) for x in got_ref["dynamic_coords"]]}
    walls = {"new": [], "reference": []}
    for _ in range(a.calls):
        for name, fn in (("new", new), ("reference", ref)):
            walls[name].append(round(timed(fn)[1], 2))
    result["wall_ms"] = walls
    geo = voxels.VoxelGeometry(field.aabb, a.voxel_size)
    (static, groups, patches), t_mark = timed(lambda: voxels.mark_images(cfg, field, est, props, ds, geo, True))
    pca, t_pca = timed(lambda: voxels.robust_pca(torch.cat(patches), m=2.5))
    _, t_compact = timed(lambda: voxels.compact([static] + [groups[j] for j in sorted(groups)]))
    result["split_ms"] = {"render_and_mark": round(t_mark, 2), "pca": round(t_pca, 2),
                          "compact": round(t_compact, 2),
                          "query_and_copy": round(min(walls["new"]) - t_mark - t_pca - t_compact, 2)}
    result["syncs"] = {"new": count_syncs(new), "reference": count_syncs(ref)}
    launches = {}
    for name, fn in (("new", new), ("reference", ref)):
        before = _lib.LAUNCHES
        fn()
        launches[name] = _lib.LAUNCHES - before
    result["library_launches"] = launches
    rec = []
    _lib.set_profile(lambda name, args: name in KERNELS, rec)
    try:
        new()
        torch.cuda.synchronize()
    finally:
        _lib.set_profile(None, None)
    kernel = {k: {"ms": 0.0, "launches": 0} for k in KERNELS}
    for name, _, e0, e1 in rec:
        kernel[name]["ms"] += e0.elapsed_time(e1)
        kernel[name]["launches"] += 1
    result["kernel_ms"] = {k: {"ms": round(v["ms"], 4), "launches": v["launches"]} for k, v in kernel.items()}
    out_dir = a.out or tempfile.mkdtemp(prefix="bench_voxels_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_voxels.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()

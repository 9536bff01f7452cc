"""The evaluation videos on one GPU: ``emernerf_b200.video.render_videos`` beside the reference's ``render`` +
``save_videos`` loop (``oracle.video_ref``, on the same drop-in renderer and field), alternating, with the same
writer that discards its frames.

    python tools/bench_videos.py [--timesteps 6] [--downscale 1] [--calls 2] [--variants static,dynamic,flow_feat]
                                 [--out DIR]

Scene: tools/bench_trajectory.py's Waymo-shaped rig, 3 cameras of 640 x 960, --timesteps timesteps, rendered at
--downscale through ``raygen.PixelRaySampler``; the flow_feat source carries feature maps.  Fields: the benchmark
configurations (``configs.make_cfg``, tables N(0, 0.5^2)), the feature PCA a seeded random basis.  The turbo map is
videos_cases' seeded table (matplotlib is not needed).  Reported per variant:
  s_per_timestep   host clock between device synchronizes, per timestep, both versions, alternating, every call
  syncs            host syncs of one call (torch's sync debug mode, counted), per timestep
  peak_rss_mb      peak host RSS of a process that builds the scene and makes one call, each version on its own
  frames_equal     whether both versions wrote the same frames (depth bin-edge pixels aside, as the tests allow)
With imageio importable, a second pass times one call of each with imageio's writer into a temporary directory.
The GPU's name and power limit come from the same run.  Writes DIR/bench_videos.json (DIR defaults to a temporary
directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import resource
import subprocess
import sys
import tempfile
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(ROOT)
sys.path.insert(0, ROOT)
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests", "golden"))

DEV = "cuda"
CAMS = 3
KEYS = {
    "static": ["gt_rgbs", "rgbs", "depths", "median_depths", "gt_sky_masks", "sky_masks"],
    "dynamic": ["gt_rgbs", "rgbs", "static_rgbs", "dynamic_rgbs", "shadow_reduced_static_rgbs",
                "shadow_only_static_rgbs", "depths", "static_depths", "dynamic_depths", "median_depths",
                "gt_sky_masks", "sky_masks"],
    "flow_feat": ["gt_rgbs", "rgbs", "dynamic_rgbs", "depths", "dynamic_depths", "forward_flows", "backward_flows",
                  "dino_feats", "gt_dino_feats", "dino_feats_pe_free", "dino_pe", "static_dino_feats",
                  "dynamic_dino_feats", "dynamic_rgb_on_static_dinos", "dynamic_dino_on_static_rgbs", "sky_masks"],
}


class PixelSet:
    split = "full"

    def __init__(self, sampler, n):
        self.sampler, self.n = sampler, n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return dict(self.sampler.get_render_rays(i))


def scene(variant: str, timesteps: int, downscale: float):
    """(cfg, field, proposal networks, estimator, dataset, cameras) of one variant on the device."""
    import bench_raybatch as br
    import errormap_cases as ec
    from emernerf_b200 import configs, raygen

    cfg = configs.make_cfg(variant)
    field, props, est, _ = configs.build_hot_path(cfg, DEV, table_std=0.5)
    field.eval(), est.eval(), [p.eval() for p in props]
    feature = variant == "flow_feat"
    if feature:
        g = torch.Generator(device=DEV).manual_seed(5)
        field.feats_reduction_mat.copy_(torch.randn(field.feats_reduction_mat.shape, device=DEV, generator=g))
        field.feat_color_min.fill_(-2.0)
        field.feat_color_max.fill_(2.0)
    s = ec.PixelSource()
    vars(s).update(vars(br.pixel_source(timesteps * CAMS, feature)))
    c2w = s.cam_to_worlds
    for i in range(len(c2w)):                     # tools/bench_trajectory.py's rig
        yaw = math.radians(9 * (i // CAMS) + 50 * (i % CAMS - 1))
        c, si = math.cos(yaw), math.sin(yaw)
        rz = torch.tensor([[c, -si, 0.0], [si, c, 0.0], [0.0, 0.0, 1.0]], device=DEV)
        fwd = torch.tensor([[1.0, 0.0, 0.0], [0.0, 0.0, 1.0], [0.0, -1.0, 0.0]], device=DEV)
        c2w[i, :3, :3] = rz @ fwd
        c2w[i, :3, 3] = torch.tensor([2.0 * (i // CAMS), 0.0, 1.5], device=DEV)
    s._normalized_timestamps = (torch.arange(len(c2w), device=DEV) // CAMS).float() / max(timesteps - 1, 1)
    s._downscale_factor = downscale
    sampler = raygen.PixelRaySampler(s)
    return cfg, field, props, est, PixelSet(sampler, len(c2w)), CAMS


class Discard:
    def append_data(self, frame):
        pass

    def close(self):
        pass


class Keep(Discard):
    def __init__(self, sink):
        self.sink = sink

    def append_data(self, frame):
        self.sink.append(np.array(frame, copy=True))


def new_call(parts, ts, keys, get_writer):
    from emernerf_b200 import video

    cfg, field, props, est, ds, cams = parts
    video._get_writer = get_writer
    return video.render_videos(cfg, field, est, props, ds, os.path.join(tempfile.gettempdir(), "bench_videos.mp4"),
                               ts, keys, cams, verbose=False, compute_metrics=False)


def ref_call(parts, ts, keys, get_writer):
    import videos_cases as vc
    from emernerf_b200 import flow_vis, voxels
    from emernerf_b200.radiance_fields.render_utils import render_rays
    from oracle import video_ref

    cfg, field, props, est, ds, cams = parts
    return video_ref.render_videos(cfg, field, est, props, ds, os.path.join(tempfile.gettempdir(),
                                   "bench_videos_ref.mp4"), ts, keys, cams, verbose=False, render_rays=render_rays,
                                   robust_pca=voxels.robust_pca, scene_flow_to_rgb=flow_vis.scene_flow_to_rgb,
                                   cmap=video_ref.Colormap(vc.turbo_table()), get_writer=get_writer)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


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


def setup():
    import videos_cases as vc
    from emernerf_b200 import video

    video.load_turbo_lut = vc.turbo_lut           # matplotlib's table is not needed to time the frames


def one_call(which, variant, ts, downscale):
    """Subprocess body: build the scene, make one call, report the peak RSS."""
    setup()
    parts = scene(variant, ts, downscale)
    fn = new_call if which == "new" else ref_call
    fn(parts, ts, KEYS[variant], lambda path, **kw: Discard())
    torch.cuda.synchronize()
    print(json.dumps({"peak_rss_mb": resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024}))


def peak_rss(which, variant, ts, downscale):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--rss-child", which, "--variants", variant,
                        "--timesteps", str(ts), "--downscale", str(downscale)], capture_output=True, text=True,
                       timeout=1800)
    if r.returncode != 0:
        return {"error": r.stderr[-800:]}
    return json.loads(r.stdout.strip().splitlines()[-1])["peak_rss_mb"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timesteps", type=int, default=6)
    ap.add_argument("--downscale", type=float, default=1.0)
    ap.add_argument("--calls", type=int, default=2)
    ap.add_argument("--variants", default="static,dynamic,flow_feat")
    ap.add_argument("--rss-child", default=None)
    ap.add_argument("--no-rss", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_videos needs a CUDA device"
    if a.rss_child:
        one_call(a.rss_child, a.variants, a.timesteps, a.downscale)
        return
    import videos_cases as vc
    from bench_raybatch import gpu_info

    setup()
    ts = a.timesteps
    result = {"info": gpu_info(), "timesteps": ts, "cams": CAMS, "downscale": a.downscale, "variants": {}}
    for variant in a.variants.split(","):
        parts = scene(variant, ts, a.downscale)
        keys = KEYS[variant]
        h, w = parts[4][0]["origins"].shape[:2]
        got = {"new": [], "reference": []}
        torch.manual_seed(0)
        new_call(parts, ts, keys, lambda path, **kw: Keep(got["new"]))
        torch.manual_seed(0)
        ref_call(parts, ts, keys, lambda path, **kw: Keep(got["reference"]))
        a_, b_ = np.stack(got["new"]), np.stack(got["reference"])
        diff = (a_ != b_).any(-1) if a_.shape == b_.shape else None
        row = {"rays_per_image": int(h * w), "rows": int(a_.shape[1] // h),
               "frames_equal": diff is not None and not diff.any(),
               "differing_pixels": None if diff is None else int(diff.sum()), "frame_pixels": int(a_[..., 0].size)}
        times = {"new": [], "reference": []}
        for _ in range(a.calls):
            for name, fn in (("new", new_call), ("reference", ref_call)):
                times[name].append(round(timed(lambda: fn(parts, ts, keys, lambda path, **kw: Discard())) / ts, 4))
        row["s_per_timestep"] = times
        row["syncs_per_timestep"] = {
            name: round(count_syncs(lambda: fn(parts, ts, keys, lambda path, **kw: Discard())) / ts, 2)
            for name, fn in (("new", new_call), ("reference", ref_call))}
        try:
            import imageio  # noqa: F401

            d = tempfile.mkdtemp(prefix="bench_videos_")
            writer = lambda path, **kw: imageio.get_writer(os.path.join(d, os.path.basename(path)), **kw)  # noqa
            row["s_per_timestep_imageio"] = {name: round(timed(lambda: fn(parts, ts, keys, writer)) / ts, 4)
                                             for name, fn in (("new", new_call), ("reference", ref_call))}
        except ImportError:
            row["s_per_timestep_imageio"] = "imageio not importable: not measured"
        parts = None
        torch.cuda.empty_cache()
        if not a.no_rss:
            row["peak_rss_mb"] = {name: peak_rss(name, variant, ts, a.downscale) for name in ("new", "reference")}
        result["variants"][variant] = row
        print(json.dumps({variant: row}), flush=True)
    out_dir = a.out or tempfile.mkdtemp(prefix="bench_videos_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_videos.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()

"""Per-level timing of the hash-grid forward / backward kernels on ray-coherent points.

    python tools/microbench_grid.py [--rays 8192] [--samples 64]

Points are the real sample positions of one render pass of the bench model (proposal-resampled, so
consecutive lanes of a warp are consecutive samples of a ray).  Each level is timed alone through a
one-level descriptor, then the full grid; CUDA events, 20 repetitions after 3 warm-ups."""
import argparse
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from emernerf_b200 import _lib, _ops, configs, synthetic
from emernerf_b200.grid_desc import GridDesc


def timeit(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def one_level(desc: GridDesc, l: int) -> GridDesc:
    d = GridDesc.__new__(GridDesc)
    d.n_dims, d.n_levels, d.n_feat = desc.n_dims, 1, desc.n_feat
    d.scales, d.resolutions = [desc.scales[l]], [desc.resolutions[l]]
    d.offsets, d.hashed = [desc.offsets[l], desc.offsets[l + 1]], [desc.hashed[l]]
    c = type(desc.c)()
    c.n_dims, c.n_levels, c.n_feat = desc.n_dims, 1, desc.n_feat
    c.scale[0], c.resolution[0], c.hashed[0] = desc.scales[l], desc.resolutions[l], int(desc.hashed[l])
    c.offset[0], c.offset[1] = desc.offsets[l], desc.offsets[l + 1]
    d.c = c
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--samples", type=int, default=64)
    a = ap.parse_args()
    dev = "cuda"
    cfg = configs.make_cfg("static", num_samples=a.samples)
    field, props, est, _ = configs.build_hot_path(cfg, dev, table_std=0.3)
    field.train()
    batch = synthetic.pixel_batch(a.rays, device=dev)
    from emernerf_b200.radiance_fields.render_utils import render_rays

    with torch.no_grad():
        out = render_rays(field, est, props, batch, cfg)
    t = out["extras"]["t_vals"]
    pos = batch["origins"][:, None, :] + batch["viewdirs"][:, None, :] * t[..., None]
    x = _ops.contract(pos.reshape(-1, 3), field.aabb, None, True).contiguous()
    n = x.shape[0]
    desc = field.xyz_encoder.desc
    table = field.xyz_encoder.tcnn_encoding.params.detach()
    inside = ((x > 0) & (x < 1)).all(-1).float().mean().item()
    print(f"points {n}, inside-cube fraction {inside:.3f}")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t_: ctypes.c_void_p(t_.data_ptr())
    for l in list(range(desc.n_levels)) + [-1]:
        d = desc if l < 0 else one_level(desc, l)
        y = torch.empty(n, d.n_output_dims, device=dev)
        dy = torch.randn(n, d.n_output_dims, device=dev)
        dt = torch.zeros_like(table)
        f = timeit(lambda: _lib.call("emer_grid_fwd", ctypes.byref(d.c), P(x), P(table), P(y), n, st))
        b = timeit(lambda: _lib.call("emer_grid_bwd", ctypes.byref(d.c), P(x), P(table), P(dy), P(dt), None, n, st))
        xr = torch.rand_like(x)
        br = timeit(lambda: _lib.call("emer_grid_bwd", ctypes.byref(d.c), P(xr), P(table), P(dy), P(dt), None, n, st))
        name = "all" if l < 0 else f"L{l} res={desc.resolutions[l]:5d} {'hash' if desc.hashed[l] else 'dense'}"
        print(f"{name:22s} fwd {f * 1e3:8.1f} us   bwd(table) {b * 1e3:8.1f} us   bwd on uniform-random points {br * 1e3:8.1f} us")


if __name__ == "__main__":
    main()

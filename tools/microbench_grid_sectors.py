"""The hash grid's gather and table scatter against the whole-sector ceiling of their output layout.

    python tools/microbench_grid_sectors.py [--rays 8192] [--samples 64] [--reps 50] [--build-dir DIR]
                                            [--lib NAME=PATH ...]

`y` (and the scatter's `dy`) is row-major [N, L*F], 160 B per point for the 10 x 4 grids, and a level group
writes only its levels' part of each row.  This times, at the real sample positions of one render pass of the
bench model (524 288 ray-coherent points), builds of csrc/grid.cu compiled into --build-dir (a temporary directory by
default):

    shipped        the library's kernels
    level_major    EMER_GRID_DIAG_LEVEL_MAJOR: the same schedule writing / reading a private level-major [L, N, F]
                   buffer, i.e. whole sectors in contiguous runs -- the ceiling for any schedule of [N, L*F]

--lib NAME=PATH adds another build of the library (e.g. a previous commit's, built from its grid.cu and error.cu) to
the comparison; --lib builds come first and the first build is the reference.  Every build runs twice, alternating,
with CUDA events around each launch (median of --reps after warm-up), and its forward is checked bit for bit
against the reference's (level-major outputs transposed back).  Then the same for the 4-D dynamic grid (10 x 4, 2^18)
at the same points with a per-ray time coordinate."""
import argparse
import ctypes
import hashlib
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from emernerf_b200 import _lib, _ops, build, configs, synthetic
from emernerf_b200.grid_desc import GridDesc
from oracle import hotpath

VARIANTS = {
    "shipped": [],
    "level_major": ["-DEMER_GRID_DIAG_LEVEL_MAJOR=1"],
}


def build_variant(out_dir, name, defines):
    srcs = [os.path.join(build.CSRC, f) for f in ("grid.cu", "error.cu")]
    h = hashlib.sha256(" ".join(defines).encode())
    for p in srcs + [os.path.join(build.CSRC, "common.cuh")]:
        h.update(open(p, "rb").read())
    so = os.path.join(out_dir, f"grid_{name}_{h.hexdigest()[:12]}.so")
    if not os.path.exists(so):
        cmd = [build._nvcc()] + build.NVCC_FLAGS + defines + ["-shared", "-o", so] + srcs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {name}:\n{r.stderr}")
    return so


def open_lib(path):
    lib = ctypes.CDLL(path)
    for fn in ("emer_grid_fwd", "emer_grid_bwd"):
        getattr(lib, fn).argtypes = _lib._SIGNATURES[fn]
        getattr(lib, fn).restype = ctypes.c_int
    lib.emer_last_error.restype = ctypes.c_char_p
    return lib


def median_ms(fn, reps, warm=5):
    for _ in range(warm):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    return statistics.median(e0.elapsed_time(e1) for e0, e1 in ev)


def checked(lib, name, *args):
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise RuntimeError(f"{name}: {lib.emer_last_error().decode()}")


def run_grid(label, desc, x, libs, reps):
    n, L, F = x.shape[0], desc.n_levels, desc.n_feat
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t_: ctypes.c_void_p(t_.data_ptr())
    g = torch.Generator(device="cuda").manual_seed(0)
    table = torch.randn(desc.n_params, device="cuda", generator=g) * 0.3
    dy = torch.randn(n, L * F, device="cuda", generator=g)
    dt = torch.zeros_like(table)
    y = torch.empty(n, L * F, device="cuda")
    base = None
    print(f"\n{label}: {n} points, {L} levels x {F}, table {desc.n_params * 4 / 2**20:.1f} MiB")
    for name, lib in libs + libs:          # twice, to show the spread
        fwd = lambda: checked(lib, "emer_grid_fwd", ctypes.byref(desc.c), P(x), P(table), P(y), n, st)
        bwd = lambda: checked(lib, "emer_grid_bwd", ctypes.byref(desc.c), P(x), P(table), P(dy), P(dt), None, n, st)
        tf, tb = median_ms(fwd, reps), median_ms(bwd, reps)
        fwd()
        torch.cuda.synchronize()
        out = y.view(L, n, F).permute(1, 0, 2).reshape(n, L * F) if name == "level_major" else y
        if base is None:
            base, same = out.clone(), "reference"
        else:
            same = "bit-identical" if torch.equal(out, base) else f"DIFFERS (max {(out - base).abs().max().item():.3g})"
        print(f"  {name:16s} fwd {tf * 1e3:7.1f} us   bwd(table) {tb * 1e3:7.1f} us   fwd {same}")

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--build-dir", default=None)
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH")
    ap.add_argument("--variants", default=",".join(VARIANTS))
    ap.add_argument("--build-only", action="store_true")
    a = ap.parse_args()
    out_dir = a.build_dir or tempfile.mkdtemp(prefix="grid_sectors_")
    os.makedirs(out_dir, exist_ok=True)
    paths = [tuple(s.split("=", 1)) for s in a.lib]
    paths += [(v, build_variant(out_dir, v, VARIANTS[v])) for v in a.variants.split(",")]
    if a.build_only:
        print("\n".join(p for _, p in paths))
        return
    libs = [(name, open_lib(p)) for name, p in paths]

    dev = "cuda"
    print(torch.cuda.get_device_name(), os.popen("nvidia-smi --query-gpu=power.limit,clocks.max.sm,clocks.sm "
                                                 "--format=csv,noheader").read().strip())
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
    run_grid("static grid", field.xyz_encoder.desc, x, libs, a.reps)
    tr = torch.rand(a.rays, 1, 1, device=dev).expand(a.rays, t.shape[1], 1).reshape(-1, 1)
    x4 = torch.cat([x, tr], -1).contiguous()
    run_grid("4-D dynamic grid", GridDesc(4, hotpath.hash_encoder_config(10, 32, 8192, 18, 4)), x4, libs, a.reps)
    print(torch.cuda.get_device_name(), os.popen("nvidia-smi --query-gpu=power.limit,clocks.max.sm,clocks.sm "
                                                 "--format=csv,noheader").read().strip())


if __name__ == "__main__":
    main()

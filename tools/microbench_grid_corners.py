"""The hash-grid gathers and scatters against the ceiling of fetching each x-neighbour corner pair in one load.

    python tools/microbench_grid_corners.py [--rays 8192] [--samples 64] [--reps 50] [--build-dir DIR]
                                            [--csrc DIR] [--lib NAME=PATH ...] [--variants shipped,xhigh_reuse]
                                            [--build-only]

Corners c and c ^ 1 of a cell differ only in x.  This times, at the sample positions of one render pass of the bench
model (8192 rays: 524 288 ray-coherent points for the field grids, and the two proposal levels as the bench runs them,
n = 128 from a flat CDF and n = 64 from its output), builds of csrc/grid.cu + csrc/prop_level.cu compiled into
--build-dir (a temporary directory by default):

    shipped        the library's kernels
    xhigh_reuse    EMER_GRID_DIAG_XHIGH_REUSE: the x-high corner of each pair is not loaded and takes the x-low
                   corner's value.  Its outputs are wrong; its time bounds what any way of fetching a pair in one
                   instruction can save.

--lib NAME=PATH adds another build of the same three files (e.g. a previous commit's, made with --csrc DIR
--build-only) to the comparison; --lib builds come first and the first build is the reference.  Every build runs
twice, alternating, with CUDA events around each launch (median of --reps after warm-up).  Outputs are checked bit for
bit against the reference build's: the grid forwards, and the proposal levels' s, t and CDF rows (and the backward's
d_enc).  Kernels timed: grid_fwd_kernel<3,4,1> / grid_bwd_table_kernel<3,4,1> (static grid), grid_fwd_kernel<4,4,1> /
grid_bwd_table_kernel<4,4,1> (4-D dynamic grid, 10 x 4, 2^18), prop_level_kernel<8> at both levels,
prop_level_bwd_kernel<8> at both levels, and grid_fwd_kernel<3,1,8> / grid_bwd_table_kernel<3,1,8> at the n = 64
level's points."""
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

from emernerf_b200 import build  # noqa: E402  (no torch needed to build)

VARIANTS = {
    "shipped": [],
    "xhigh_reuse": ["-DEMER_GRID_DIAG_XHIGH_REUSE=1"],
}
FILES = ("grid.cu", "prop_level.cu", "error.cu")


def build_variant(out_dir, name, defines, csrc):
    srcs = [os.path.join(csrc, f) for f in FILES]
    h = hashlib.sha256(" ".join(defines).encode())
    for p in srcs + sorted(os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")):
        h.update(open(p, "rb").read())
    so = os.path.join(out_dir, f"corners_{name}_{h.hexdigest()[:12]}.so")
    if not os.path.exists(so):
        inc = os.path.join(os.path.dirname(os.path.dirname(csrc)), "include")
        flags = [f for f in build.NVCC_FLAGS if f not in ("-I",) and not os.path.isabs(f)]
        cmd = [build._nvcc()] + flags + ["-I", inc, "-I", csrc] + defines + ["-shared", "-o", so] + srcs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {name}:\n{r.stderr}")
    return so


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--build-dir", default=None)
    ap.add_argument("--csrc", default=build.CSRC, help="source tree of the builds made here")
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH")
    ap.add_argument("--variants", default=",".join(VARIANTS))
    ap.add_argument("--build-only", action="store_true")
    a = ap.parse_args()
    out_dir = a.build_dir or tempfile.mkdtemp(prefix="grid_corners_")
    os.makedirs(out_dir, exist_ok=True)
    paths = [tuple(s.split("=", 1)) for s in a.lib]
    paths += [(v, build_variant(out_dir, v, VARIANTS[v], os.path.abspath(a.csrc)))
              for v in a.variants.split(",") if v]
    if a.build_only:
        print("\n".join(p for _, p in paths))
        return
    run(a, paths)


def run(a, paths):
    import torch

    from emernerf_b200 import _lib, _ops, configs, synthetic
    from emernerf_b200.grid_desc import GridDesc
    from oracle import hotpath

    def open_lib(path):
        lib = ctypes.CDLL(path)
        for fn in ("emer_grid_fwd", "emer_grid_bwd", "emer_prop_level", "emer_prop_level_bwd"):
            getattr(lib, fn).argtypes = _lib._SIGNATURES[fn]
            getattr(lib, fn).restype = ctypes.c_int
        lib.emer_last_error.restype = ctypes.c_char_p
        return lib

    libs = [(name, open_lib(p)) for name, p in paths]
    main_lib = _lib.load()

    def median_ms(fn, reps=a.reps, warm=5):
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

    def same(out, base):
        if base is None:
            return "reference"
        return "bit-identical" if all(torch.equal(o, b) for o, b in zip(out, base)) else "DIFFERS"

    P = lambda t_: ctypes.c_void_p(t_.data_ptr() if t_ is not None else 0)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def card():
        q = os.popen("nvidia-smi --query-gpu=power.limit,clocks.max.sm,clocks.sm --format=csv,noheader").read().strip()
        return f"{torch.cuda.get_device_name()}, {q}"

    print(card())
    dev = "cuda"
    cfg = configs.make_cfg("static", num_samples=a.samples)
    field, props, est, _ = configs.build_hot_path(cfg, dev, table_std=0.3)
    field.train()
    batch = synthetic.pixel_batch(a.rays, device=dev)
    from emernerf_b200.radiance_fields.render_utils import render_rays

    levels = []                                  # the proposal levels' calls, as the render made them
    orig = _ops.prop_level

    def capture(*args, **kw):
        out = orig(*args, **kw)
        levels.append((args, kw))
        return out

    _ops.prop_level = capture
    try:
        with torch.no_grad():
            out = render_rays(field, est, props, batch, cfg)
    finally:
        _ops.prop_level = orig
    t = out["extras"]["t_vals"]
    pos = batch["origins"][:, None, :] + batch["viewdirs"][:, None, :] * t[..., None]
    x = _ops.contract(pos.reshape(-1, 3), field.aabb, None, True).contiguous()
    tr = torch.rand(a.rays, 1, 1, device=dev).expand(a.rays, t.shape[1], 1).reshape(-1, 1)
    x4 = torch.cat([x, tr], -1).contiguous()
    grids = [("static grid", field.xyz_encoder.desc, x),
             ("4-D dynamic grid", GridDesc(4, hotpath.hash_encoder_config(10, 32, 8192, 18, 4)), x4)]

    # ---- field grids: gather and table scatter
    for label, desc, xg in grids:
        n, L, F = xg.shape[0], desc.n_levels, desc.n_feat
        g = torch.Generator(device="cuda").manual_seed(0)
        table = torch.randn(desc.n_params, device="cuda", generator=g) * 0.3
        dy = torch.randn(n, L * F, device="cuda", generator=g)
        dt = torch.zeros_like(table)
        y = torch.empty(n, L * F, device="cuda")
        base = None
        print(f"\n{label}: {n} points, {L} levels x {F}, table {desc.n_params * 4 / 2**20:.1f} MiB")
        for name, lib in libs + libs:
            fwd = lambda: checked(lib, "emer_grid_fwd", ctypes.byref(desc.c), P(xg), P(table), P(y), n, st)
            bwd = lambda: checked(lib, "emer_grid_bwd", ctypes.byref(desc.c), P(xg), P(table), P(dy), P(dt), None, n,
                                  st)
            tf, tb = median_ms(fwd), median_ms(bwd)
            fwd()
            torch.cuda.synchronize()
            s = same([y], base)
            if base is None:
                base = [y.clone()]
            print(f"  {name:16s} fwd {tf * 1e3:7.1f} us   bwd(table) {tb * 1e3:7.1f} us   fwd {s}")

    # ---- proposal levels (prop_level_kernel<8>, prop_level_bwd_kernel<8>) and the proposal grid at their points
    print(f"\nproposal levels: {a.rays} rays, n = {[lv[0][2] for lv in levels]}")
    g = torch.Generator(device="cuda").manual_seed(1)
    bwd_in = []
    for args, kw in levels:
        r, n = args[0].shape[0], args[2]
        s_, t_, c_, sig = orig(*args, **dict(kw, want_sigma=True))
        bwd_in.append((t_, sig, torch.rand(r, n + 1, device=dev, generator=g) * 1e-3))
    pdesc = levels[-1][0][11]
    r_last, n_last = levels[-1][0][0].shape[0], levels[-1][0][2]
    xc = torch.empty(r_last * n_last, 3, device=dev)
    d_enc = torch.empty(r_last * n_last, pdesc.n_output_dims, device=dev)
    base = None
    for name, lib in libs + libs:
        _lib._LIB = lib
        try:
            res, outs = [], []
            for li, (args, kw) in enumerate(levels):
                res.append(median_ms(lambda: orig(*args, **kw)))
                outs += list(orig(*args, **kw))
            for li, (args, kw) in enumerate(levels):
                (o, d_, aabb, unb, desc, tab, w0, b0, w1) = (args[7], args[8], args[9], args[10], args[11],
                                                             args[12], args[13], args[14], args[15])
                t_, sig, dcdf = bwd_in[li]
                r, n = t_.shape[0], t_.shape[1] - 1
                xcl = torch.empty(r * n, 3, device=dev)
                del_ = torch.empty(r * n, desc.n_output_dims, device=dev)
                acc = [torch.zeros_like(w0), torch.zeros_like(b0), torch.zeros(w1.numel(), device=dev),
                       torch.zeros(1, device=dev)]
                box, o, d_ = aabb.reshape(-1).contiguous(), o.contiguous(), d_.contiguous()
                w1c = w1.reshape(-1).contiguous()
                call = lambda: checked(lib, "emer_prop_level_bwd", ctypes.byref(desc.c), P(t_), P(sig), P(dcdf), n,
                                       P(o), P(d_), P(box), int(unb), P(tab), P(w0), P(b0), P(w1c), P(xcl), P(del_),
                                       P(acc[0]), P(acc[1]), P(acc[2]), P(acc[3]), r, st)
                res.append(median_ms(call))
                call()
                outs.append(del_.clone())
                if li == len(levels) - 1:
                    xc.copy_(xcl)
                    d_enc.copy_(del_)
        finally:
            _lib._LIB = main_lib
        torch.cuda.synchronize()
        # the proposal grid (8 x 1) alone at the last level's sample positions
        npt = xc.shape[0]
        ptab = levels[-1][0][12]
        yp = torch.empty(npt, pdesc.n_output_dims, device=dev)
        dtp = torch.zeros_like(ptab)
        pf = lambda: checked(lib, "emer_grid_fwd", ctypes.byref(pdesc.c), P(xc), P(ptab), P(yp), npt, st)
        pb = lambda: checked(lib, "emer_grid_bwd", ctypes.byref(pdesc.c), P(xc), P(ptab), P(d_enc), P(dtp), None,
                             npt, st)
        tpf, tpb = median_ms(pf), median_ms(pb)
        pf()
        torch.cuda.synchronize()
        outs.append(yp.clone())
        s = same(outs, base)
        if base is None:
            base = outs
        nl = len(levels)
        fw = "  ".join(f"n={lv[0][2]} {res[i] * 1e3:6.1f}" for i, lv in enumerate(levels))
        bw = "  ".join(f"n={lv[0][2]} {res[nl + i] * 1e3:6.1f}" for i, lv in enumerate(levels))
        print(f"  {name:16s} prop_level us: {fw}   bwd us: {bw}   grid<3,1,8> fwd {tpf * 1e3:6.1f} "
              f"bwd(table) {tpb * 1e3:6.1f} us ({npt} points)   s/t/cdf/d_enc/fwd {s}")
    print(card())


if __name__ == "__main__":
    main()

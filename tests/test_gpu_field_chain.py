"""emer_field_bwd (csrc/field_fused.cu): the fused field chain's data gradients through the C ABI, every output buffer
on its own against an fp64 restatement of include/emer_b200.h (emer_field_bwd), in all six instantiations
<k_enc in {32, 40, 64}, n_feat in {64, 128}>.

Inputs: ReLU-sparse saved activations (about half of every mask is an exact zero), colours within 1e-4 of 0 and 1,
densities above e^15 (where the backward clamps) and below 1e-30, the head's weight blocks as column views of
[64, c + 64] / [64, 128 + c] matrices (c = 49: row strides 113 / 177; c = 33), every subset of the optional upstream
gradients the product passes, ragged last tiles and last rays, and sizes at which each warpgroup of the persistent grid
walks at least three tiles.

Bars (relative to each buffer's max-abs): 2e-5 for every buffer, the bar of test_gpu_field_wgrad.py.  3xTF32 gives
about 1e-6; one dropped product of a stage gives tf32's ~5e-4.  Measured maxima over the matrix on an H100 80GB HBM3
at 400 W: dz2 9.6e-8, dz1 9.3e-7, dZ0 1.8e-6, dF 2.2e-6, dzb 3.0e-6, d_enc 3.6e-6, d_ray_bias[:, :64] 1.4e-6,
d_ray_bias[:, 64:] 8.9e-7.

The unmarked companion runs the same reference against tests/cabi_emulator.py at small sizes, so the formula is
checked on a machine without a GPU and the emulator the CPU suite trusts is pinned to it."""
import ctypes
import math

import pytest
import torch

import cabi_emulator
from helpers import rel_err

DEV = "cuda"
E15 = math.exp(15.0)
TOL = 2e-5
INSTANCES = [(k, f) for k in (32, 40, 64) for f in (64, 128)]
N_RAGGED = 64 * 1400 + 37          # 1401 tiles: >= 3 per warpgroup of a 132-SM x 3-warpgroup grid, last tile 37 rows
N_EVEN = 128 * 700                 # a multiple of every S below
UPSTREAM = {                       # which of d_rgb, d_sigma, d_geo, d_sem are given
    "all": ("d_rgb", "d_sigma", "d_geo", "d_sem"),
    "rgb": ("d_rgb",),
    "sigma_geo": ("d_sigma", "d_geo"),
    "sem": ("d_sem",),
    "no_sem": ("d_rgb", "d_sigma", "d_geo"),
}


def _cases(sizes):
    """(k_enc, n_feat, n, S, upstream, c, ld_denc_pad): every instantiation at every size, then the upstream subsets
    and the S % 32 != 0 launch (no per-ray sums) at the largest size."""
    out = []
    for i, (k, f) in enumerate(INSTANCES):
        for j, (n, S) in enumerate(sizes):
            out.append((k, f, n, S, "all", (49, 33)[(i + j) % 2], 8 * ((i + j) % 2)))
    n = sizes[-2][0]
    out += [(40, 64, n, 32, "rgb", 49, 0), (40, 128, n, 64, "sigma_geo", 49, 8), (32, 128, n, 32, "sem", 33, 0),
            (64, 128, n, 128, "no_sem", 49, 8), (40, 128, n, 64, "no_sem", 33, 0), (40, 64, n, 48, "all", 49, 8),
            (32, 128, n, 96, "all", 33, 0)]
    return out


GPU_CASES = _cases([(1, 32), (63, 32), (N_RAGGED, 64), (N_EVEN, 128)])
CPU_CASES = _cases([(1, 32), (63, 32), (64 * 5 + 37, 64), (128 * 3, 128)])


def _inputs(k_enc, n_feat, n, S, upstream, c, ld_denc, seed, dev):
    """The kernel's inputs and (sentinel-filled) outputs.  d_sigma is scaled by 1 / clamp(sigma, 1, e^15), so every
    row's d_sigma * min(sigma, e^15) is O(1): rows above e^15 neither hide the others nor are hidden by them."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    u = lambda *s: torch.rand(*s, generator=g)
    x = dict(hb=r(n, 64).relu(), hg=r(n, 128).relu(), h1=r(n, 64).relu())
    rgb = u(n, 3) * 0.98 + 0.01
    rgb[0::5, 0] = u(len(range(0, n, 5))) * 1e-4 + 1e-7
    rgb[2::5, 1] = 1.0 - (u(len(range(2, n, 5))) * 1e-4 + 1e-7)
    sigma = torch.exp(r(n))
    sigma[1::7] = E15 * (1.0 + 30.0 * u(len(range(1, n, 7))))
    sigma[4::7] = 1e-31 * (0.5 + u(len(range(4, n, 7))))
    x.update(rgb=rgb, sigma=sigma)
    x["d_rgb"], x["d_sigma"] = r(n, 3), r(n) / sigma.clamp(1.0, E15)
    x["d_geo"], x["d_sem"] = r(n, 64) * 0.3, r(n, 64) * 0.3
    for k in ("d_rgb", "d_sigma", "d_geo", "d_sem"):
        if k not in UPSTREAM[upstream] or (k == "d_sem" and n_feat == 64):
            x[k] = None
    x.update(wb0=r(64, k_enc) / k_enc ** 0.5, wb1=r(n_feat, 64) / 8, w0=r(64, c + 64) / (c + 64) ** 0.5,
             w1=r(64, 128 + c) / (128 + c) ** 0.5, w2=r(3, 64) / 8)
    nan = float("nan")
    R = (n + S - 1) // S
    o = dict(dz2=torch.full((n, 3), nan), dz1=torch.full((n, 64), nan), d1=torch.full((n, 128), nan),
             dzb=torch.full((n, 64), nan), d_enc=torch.full((n, k_enc + ld_denc), -7.0),
             d_rb=r(R, 128) * 0.1 if S % 32 == 0 else None)
    o["d_enc"][:, :k_enc] = nan
    mv = lambda d: {k: None if v is None else v.to(dev) for k, v in d.items()}
    return mv(x), mv(o)


def _launch(call, stream, x, o, k_enc, n_feat, c, S, n, dz2=True):
    P = lambda t: ctypes.c_void_p(0 if t is None else t.data_ptr())
    w0, w1 = x["w0"], x["w1"]
    call("emer_field_bwd", P(x["d_rgb"]), P(x["rgb"]), P(x["d_sigma"]), P(x["sigma"]), P(x["d_geo"]), P(x["d_sem"]),
         P(x["hb"]), P(x["hg"]), P(x["h1"]), P(x["wb0"]), k_enc, P(x["wb1"]), n_feat, P(w0[:, c:]), w0.stride(0),
         P(w1[:, :64]), P(w1[:, 64 + c:]), w1.stride(0), P(x["w2"]), P(o["dz2"] if dz2 else None), P(o["dz1"]),
         P(o["d1"]), P(o["dzb"]), P(o["d_enc"]), o["d_enc"].stride(0), P(o["d_rb"]), S, n, stream)


def _reference(x, k_enc, n_feat, c, S, n):
    """include/emer_b200.h's formula for emer_field_bwd in fp64; the ray sums are the increments of d_ray_bias."""
    d = {k: None if v is None else v.double() for k, v in x.items()}
    w0, w1 = d["w0"], d["w1"]
    z2 = torch.zeros((n, 3), dtype=torch.float64, device=d["rgb"].device)
    if d["d_rgb"] is not None:
        z2 = d["d_rgb"] * d["rgb"] * (1.0 - d["rgb"])
    z1 = (z2 @ d["w2"]) * (d["h1"] > 0)
    z0 = (z1 @ w1[:, :64]) * (d["hg"][:, :64] > 0)
    dF = z1 @ w1[:, 64 + c:] + z0 @ w0[:, c:]
    if d["d_geo"] is not None:
        dF = dF + d["d_geo"]
    if d["d_sigma"] is not None:
        dF[:, 0] += d["d_sigma"] * d["sigma"].clamp(max=E15)
    dhb = dF @ d["wb1"][:64]
    if n_feat == 128 and d["d_sem"] is not None:
        dhb = dhb + d["d_sem"] @ d["wb1"][64:]
    zb = dhb * (d["hb"] > 0)
    ray = torch.arange(n, device=z0.device) // S
    sums = torch.zeros(((n + S - 1) // S, 128), dtype=torch.float64, device=z0.device)
    sums.index_add_(0, ray, torch.cat([z0, z1], 1))
    return dict(dz2=z2, dz1=z1, dZ0=z0, dF=dF, dzb=zb, d_enc=zb @ d["wb0"], rb0=sums[:, :64], rb1=sums[:, 64:])


def _check(x, o, rb_before, k_enc, n_feat, c, S, n):
    """{buffer: relative error}; asserts the buffers the kernel must leave alone."""
    want = _reference(x, k_enc, n_feat, c, S, n)
    got = dict(dz1=o["dz1"], dZ0=o["d1"][:, :64], dF=o["d1"][:, 64:], dzb=o["dzb"], d_enc=o["d_enc"][:, :k_enc])
    if x["d_rgb"] is not None:
        got["dz2"] = o["dz2"]
    else:          # no colour gradient: dz2 is not written
        assert bool(o["dz2"].isnan().all())
    # the padding columns of d_enc's rows are not written
    assert bool((o["d_enc"][:, k_enc:] == -7.0).all())
    errs = {k: rel_err(v, want[k]) for k, v in got.items()}
    if o["d_rb"] is not None:
        rb = rb_before.double()
        errs["rb0"] = rel_err(o["d_rb"][:, :64], rb[:, :64] + want["rb0"])
        errs["rb1"] = rel_err(o["d_rb"][:, 64:], rb[:, 64:] + want["rb1"])
    return errs


def _ids(cases):
    return [f"k{k}-f{f}-n{n}-S{S}-{u}-c{c}-pad{p}" for k, f, n, S, u, c, p in cases]


@pytest.mark.gpu
@pytest.mark.parametrize("k_enc,n_feat,n,S,upstream,c,pad", GPU_CASES, ids=_ids(GPU_CASES))
def test_field_bwd_buffers_vs_fp64(k_enc, n_feat, n, S, upstream, c, pad):
    """Each output buffer of one emer_field_bwd launch within its bar of fp64; d_ray_bias accumulates into a non-zero
    buffer; d_enc's padding columns and, without d_rgb, dz2 stay as they were."""
    from emernerf_b200 import _lib, _ops

    x, o = _inputs(k_enc, n_feat, n, S, upstream, c, pad, seed=n + 7 * k_enc + n_feat + S + c, dev=DEV)
    rb_before = None if o["d_rb"] is None else o["d_rb"].clone()
    _ops._need_cuda(x["rgb"])
    _launch(_lib.call, _ops._stream(), x, o, k_enc, n_feat, c, S, n)
    torch.cuda.synchronize()
    errs = _check(x, o, rb_before, k_enc, n_feat, c, S, n)
    print(" ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    for k, e in errs.items():
        assert e < TOL, (k, e, errs)


@pytest.mark.gpu
@pytest.mark.parametrize("k_enc,n_feat", INSTANCES)
def test_field_bwd_repeatable_and_dz2_optional(k_enc, n_feat):
    """Two launches on the same inputs give bit-identical dz2 / dz1 / d1 / dzb / d_enc (no atomics there; only the
    per-ray sums of d_ray_bias may differ, within rounding); a launch without dz2 writes the same other buffers."""
    from emernerf_b200 import _lib, _ops

    n, S, c = N_RAGGED, 64, 49
    runs = []
    for dz2 in (True, True, False):
        x, o = _inputs(k_enc, n_feat, n, S, "all", c, 8, seed=11 + k_enc + n_feat, dev=DEV)
        _ops._need_cuda(x["rgb"])
        _launch(_lib.call, _ops._stream(), x, o, k_enc, n_feat, c, S, n, dz2=dz2)
        runs.append(o)
    torch.cuda.synchronize()
    a, b, no_dz2 = runs
    for k in ("dz2", "dz1", "d1", "dzb", "d_enc"):
        assert torch.equal(a[k].nan_to_num(-1.0), b[k].nan_to_num(-1.0)), k
        assert not bool(a[k].isnan().any()), k
        if k != "dz2":
            assert torch.equal(a[k], no_dz2[k]), k
    assert bool(no_dz2["dz2"].isnan().all())
    assert rel_err(a["d_rb"], b["d_rb"]) < 1e-6 and rel_err(a["d_rb"], no_dz2["d_rb"]) < 1e-6


@pytest.mark.gpu
def test_field_gradient_sinks_and_side_stream_match_autograd(monkeypatch):
    """The product's RadianceField (static config, small tables: k_enc = 40 through the fused chain), 256 rays x 64
    samples, a loss on rgb and density, from the same weights and inputs three ways: (a) plain autograd, (b) FusedAdam's
    gradient sinks on the main stream, (c) sinks with the weight gradients on the side stream, joined before they are
    read.  Every parameter's gradient, read before any step, agrees across the three within the rounding of reordered
    atomic sums (2e-6; measured on an H100 80GB HBM3 at 400 W: at most 4.1e-7); so do the per-ray column blocks of
    the head's w0 / w1, where (c) adds its part after the join."""
    from emernerf_b200 import _lib, _ops, configs, synthetic
    from emernerf_b200.optim import FusedAdam

    R, S = 256, 64
    cfg = configs.make_cfg("static", small=True, num_samples=S)
    field, _, _, _ = configs.build_hot_path(cfg, DEV, table_std=0.3, seed=4)
    field.train()
    batch = synthetic.pixel_batch(R, seed=4, device=DEV)
    g = torch.Generator().manual_seed(4)
    t = torch.sort(torch.rand(R, S, generator=g) * 40.0 + 1.0, dim=-1).values.to(DEV)
    dirs = batch["viewdirs"][:, None, :].expand(R, S, 3)
    pos = batch["origins"][:, None, :] + dirs * t[..., None]
    data = {k: batch[k][:, None].expand(R, S) for k in ("img_idx", "normed_timestamps")}
    g_rgb, g_den = torch.randn(R, S, 3, generator=g).to(DEV), torch.randn(R, S, generator=g).to(DEV)
    params = dict(field.named_parameters())

    def run(mode):
        _ops.clear_grad_sinks()
        monkeypatch.setattr(_ops, "WGRAD_STREAM", mode == "side")
        for p in params.values():
            p.grad = None
        if mode != "autograd":
            FusedAdam(params.values(), lr=1e-3)
        out = field(pos, dirs, data)
        loss = (out["rgb"] * g_rgb).sum() + (out["density"] * g_den).sum()
        rec = []
        _lib.set_profile(lambda name, args: True, rec)
        try:
            loss.backward()
        finally:
            _lib.set_profile(None, None)
        names = {r[0] for r in rec}
        assert {"emer_field_bwd", "emer_field_wgrad"} <= names, names
        if mode == "side":
            assert len(_ops._AFTER_JOIN) == 2          # the head's w0 / w1 blocks, added after the join
        _ops.join_side_streams()
        torch.cuda.synchronize()
        grads = {k: torch.zeros_like(p) if p.grad is None else p.grad.detach().clone() for k, p in params.items()}
        _ops.clear_grad_sinks()
        for p in params.values():
            p.grad = None
        return grads

    runs = {m: run(m) for m in ("autograd", "main", "side")}
    w0, w1 = "rgb_head.layers.0.weight", "rgb_head.layers.1.weight"
    c = params[w0].shape[1] - 64
    blocks = {k: (lambda v: v) for k in params}
    blocks.update({w0 + "[:, :c]": lambda v: v[:, :c], w1 + "[:, 64:64+c]": lambda v: v[:, 64:64 + c]})
    a = runs["autograd"]
    worst = {}
    for name, f in blocks.items():
        key = name.split("[")[0]
        want = f(a[key])
        if float(want.abs().max()) == 0.0:
            for m in ("main", "side"):
                assert float(f(runs[m][key]).abs().max()) == 0.0, (name, m)
            continue
        worst[name] = max(rel_err(f(runs[m][key]), want) for m in ("main", "side"))
    print(" ".join(f"{k} {v:.1e}" for k, v in worst.items()))
    assert w0 + "[:, :c]" in worst and w1 + "[:, 64:64+c]" in worst and "xyz_encoder.tcnn_encoding.params" in worst
    for name, e in worst.items():
        assert e < 2e-6, (name, e)


@pytest.mark.parametrize("k_enc,n_feat,n,S,upstream,c,pad", CPU_CASES, ids=_ids(CPU_CASES))
def test_field_bwd_emulator_vs_fp64(k_enc, n_feat, n, S, upstream, c, pad):
    """The same reference and bars against tests/cabi_emulator.py's emer_field_bwd on host memory."""
    x, o = _inputs(k_enc, n_feat, n, S, upstream, c, pad, seed=n + 7 * k_enc + n_feat + S + c, dev="cpu")
    rb_before = None if o["d_rb"] is None else o["d_rb"].clone()
    _launch(lambda name, *a: getattr(cabi_emulator, name)(*a), None, x, o, k_enc, n_feat, c, S, n)
    errs = _check(x, o, rb_before, k_enc, n_feat, c, S, n)
    for k, e in errs.items():
        assert e < TOL, (k, e, errs)

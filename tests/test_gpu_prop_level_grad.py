"""Gradients of the proposal networks against fp64.

On the steps that update the proposal networks, their whole gradient comes from ``emer_interlevel_loss`` (loss ->
d_cdf) and ``emer_prop_level_bwd`` + the grid scatter (d_cdf -> table, W0, b0, w1, b1).  The level backward runs
persistent CTAs: ``min(ceil(R / 8), 3 * SMs)`` CTAs of 8 warps, each warp walking rays ``wid, wid + grid * 8, ...``
with the weight gradients held in registers until one flush per CTA.  These tests hold it to an fp64 restatement of
the level (``_level_fp64``):

* case by case through ``_ops.prop_level_train``: both instantiations (4 and 8 levels x 1 feature), n at the edges of
  the 32-wide scans and of the 257-edge limit, ray counts at which warps walk one ray and several (the benchmark's
  8192 among them), first and second levels, bounded and unbounded fields, saturated and vanishing densities, and
  d_cdf rows with exact zeros;
* the production step: both proposal levels evaluating ONE network (DESIGN.md Q21) through ``PropNetEstimator``, the
  anti-aliased interlevel loss, and ``FusedAdam``'s gradient sinks.

Bars are relative to the max-abs of the fp64 result: CDF 1e-5; gradients 2e-5 up to 2e5 contributing samples and
5e-5 beyond (the bars of test_gpu_layer_instantiations.py); s and t bit-exact.  The sinks of the production step:
5e-5 against the fp64 levels driven by the interlevel kernel's own d_cdf and against the fp64 gradient of the loss.
"""
import math

import pytest
import torch

from helpers import rel_err
from oracle import adapters, hotpath, nerfacc_ref as nf, tcnn_ref

DEV = "cuda"
KIND = "uniform_lindisp"
NEAR, FAR = 0.1, 1000.0
E15 = math.exp(15.0)
AABB = [-20.0, -20.0, -5.0, 20.0, 20.0, 10.0]
NAMES = ("table", "w0", "b0", "w1", "b1")


class _TruncExp(torch.autograd.Function):
    """trunc_exp in the precision of its input (nerf_utils.py:59-75 of the reference): forward exp(x), backward
    g * exp(min(x, 15)).  ``hotpath.density_activation`` always computes in fp32."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(torch.clamp(x, max=15.0))


def _fma_chain32(enc: torch.Tensor, w0: torch.Tensor, b0: torch.Tensor) -> torch.Tensor:
    """h = b0 + W0 enc in fp32 with the kernels' fmaf order (one fmaf per input, in input order).  ``enc`` is the fp64
    interpolation rounded to fp32, not pl_encode's own fp32 features, so for a unit within rounding of zero this is
    an approximation of the kernel's sign, not a reproduction of it."""
    h = b0.float().expand(enc.shape[0], -1)
    e, w = enc.float(), w0.float()
    for i in range(e.shape[1]):
        h = (e[:, i:i + 1].double() * w[:, i].double() + h.double()).float()
    return h


def _level_fp64(t_edges, origins, dirs, aabb, unbounded, desc, geom, table, w0, b0, w1, b1, dtype=torch.float64,
                stats=None):
    """One proposal level's (sigma [R, n], cdf [R, n+1]) from its t edges, differentiable w.r.t. table, w0, b0, w1, b1.

    The discrete choices are the kernel's: the interval midpoints ``o + d (t0 + t1) / 2``, the contraction and its
    in-box selector are computed in fp32 (``hotpath.contract_points``, bit-exact with the device), the corner
    indices are the device's own (``_ops.grid_indices``; on the CPU, ``tcnn_ref``'s, which they equal bit for bit)
    and the corner weights are ``tcnn_ref``'s fp32 weights.  Everything after that is computed in ``dtype``: the
    interpolation, Linear(LF, 64), ReLU, Linear(64, 1), trunc_exp(raw - 1) with its backward clamp at exp(15),
    sigma * delta, the exclusive sum and 1 - exp(-E), and a last CDF column of 1.

    ReLU: where a hidden pre-activation lies within 1e-6 of its own scale (|b0| + |W0| |enc|) of zero, the fp32 kernel
    and this evaluation may disagree on its sign.  For those units only the mask is taken from an fp32 evaluation
    (``_fma_chain32``: the kernel's fmaf order on fp32-rounded features, an approximation of the kernel's choice);
    their count is written to ``stats["relu_near_zero"]``."""
    R, m = t_edges.shape
    n = m - 1
    dev = t_edges.device
    with torch.no_grad():
        t0, t1 = t_edges[:, :-1], t_edges[:, 1:]
        pos = origins[:, None, :] + dirs[:, None, :] * (t0 + t1)[..., None] / 2.0
        xc = hotpath.contract_points(pos.reshape(-1, 3), aabb.reshape(-1), unbounded)
        dev_idx = None
        if xc.is_cuda:
            from emernerf_b200 import _ops

            dev_idx = _ops.grid_indices(xc, desc).long()
        corners = []
        for lvl in range(geom.n_levels):
            idx, w, _, _ = tcnn_ref.corner_indices_and_weights(xc, geom, lvl)
            if dev_idx is not None:
                assert torch.equal(idx, dev_idx[:, lvl]), f"corner indices of level {lvl}"
            corners.append((idx, w.to(dtype)))
        del dev_idx
    F = geom.n_feat
    tab = table.to(dtype).view(-1, F)
    enc = torch.cat([(w[:, :, None] * tab[idx]).sum(1) for idx, w in corners], 1)
    w0d, b0d = w0.to(dtype), b0.to(dtype)
    h = enc @ w0d.T + b0d
    with torch.no_grad():
        scale = enc.abs() @ w0d.abs().T + b0d.abs()
        near = h.abs() < 1e-6 * scale
        on = h > 0
        n_near = int(near.sum())
        if n_near:
            on = torch.where(near, _fma_chain32(enc, w0, b0) > 0, on)
    if stats is not None:
        stats["relu_near_zero"] = n_near
    raw = (h * on) @ w1.to(dtype).reshape(-1, 1) + b1.to(dtype).reshape(1, 1)
    sigma = _TruncExp.apply(raw.view(R, n) - 1.0)
    sd = sigma * (t1 - t0).to(dtype)
    e_excl = torch.cumsum(torch.cat([torch.zeros(R, 1, dtype=dtype, device=dev), sd[:, :-1]], 1), 1)
    cdf = torch.cat([1.0 - torch.exp(-e_excl), torch.ones(R, 1, dtype=dtype, device=dev)], 1)
    return sigma, cdf


def _density_field(levels, unbounded, seed, device, b1=None, max_resolution=None, log2_hashmap_size=None, std=0.5):
    """A proposal DensityField (``levels`` x 1 feature) with an N(0, std) table; ``b1`` overrides the output bias."""
    from emernerf_b200.radiance_fields import build_density_field

    torch.manual_seed(seed)
    big = levels == 8
    net = build_density_field(n_input_dims=3, n_levels=levels,
                              max_resolution=max_resolution or (512 if big else 96),
                              log2_hashmap_size=log2_hashmap_size or (15 if big else 12), n_features_per_level=1,
                              unbounded=unbounded)
    net.set_aabb(AABB)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        tp = net.xyz_encoder.tcnn_encoding.params
        tp.copy_(torch.randn(tp.shape, generator=g) * std)
        if b1 is not None:
            net.base_mlp[2].bias.fill_(b1)
    return net.to(device)


def _params(net):
    lin = [m for m in net.base_mlp if isinstance(m, torch.nn.Linear)]
    return [net.xyz_encoder.tcnn_encoding.params, lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias]


def _rays(R, seed, device):
    g = torch.Generator().manual_seed(seed)
    origins = torch.randn(R, 3, generator=g) * 2.0
    dirs = torch.randn(R, 3, generator=g)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    return origins.to(device), dirs.to(device)


# ------------------------------------------------------------------------------------------------- CPU: the restatement
@pytest.mark.parametrize("levels,unbounded", [(8, True), (4, False)])
def test_restatement_in_fp32_matches_the_oracle(levels, unbounded):
    """``_level_fp64`` evaluated in fp32 on the CPU (tcnn_ref's corner indices) reproduces the oracle's DensityField +
    transmittance (radiance_field.py:825-841 -> render_utils.py:314-324 of the reference) within fp32 rounding, and
    so do its autograd gradients.  What differs is only the summation order of the interpolation (a sum of eight
    products here, an fmaf chain in the oracle) and of the two layers."""
    R, n = 48, 40
    net = _density_field(levels, unbounded, seed=11, device="cpu")
    spec = adapters.spec_from_module(net)
    origins, dirs = _rays(R, 12, "cpu")
    if not unbounded:
        origins = origins * 4.0                                     # some rays start outside the box as well
    g = torch.Generator().manual_seed(13)
    prev_s = torch.tensor([[0.0, 1.0]]).repeat(R, 1)
    iv, _ = nf.importance_sampling(nf.RayIntervals(prev_s), prev_s.clone(), n, True, jitter=torch.rand(R, 1, generator=g))
    t = hotpath._s_to_t(KIND, iv.vals, NEAR, FAR)
    up = torch.randn(R, n + 1, generator=g)

    sd = adapters.cpu_state_dict(net, requires_grad=True)
    pos = origins[:, None, :] + dirs[:, None, :] * (t[:, :-1] + t[:, 1:])[..., None] / 2.0
    sig_want = hotpath.density_field_forward(sd, spec, pos)["density"].squeeze(-1)
    trans, _ = nf.render_transmittance_from_density(t[:, :-1], t[:, 1:], sig_want)
    cdf_want = 1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], -1)
    keys = ["xyz_encoder.tcnn_encoding.params", "base_mlp.0.weight", "base_mlp.0.bias", "base_mlp.2.weight",
            "base_mlp.2.bias"]
    want = torch.autograd.grad((cdf_want * up).sum(), [sd[k] for k in keys])

    ps = [sd[k].detach().clone().requires_grad_(True) for k in keys]
    stats = {}
    sig, cdf = _level_fp64(t, origins, dirs, net.aabb, unbounded, None, spec.geom("xyz"), *ps, dtype=torch.float32,
                           stats=stats)
    got = torch.autograd.grad((cdf * up).sum(), ps)
    assert sig.dtype == torch.float32 and cdf.shape == (R, n + 1)
    assert torch.equal(cdf[:, -1], torch.ones(R))
    assert rel_err(sig, sig_want) < 2e-6, rel_err(sig, sig_want)
    assert rel_err(cdf, cdf_want) < 2e-6, rel_err(cdf, cdf_want)
    for name, a, b in zip(NAMES, got, want):
        assert rel_err(a, b) < 1e-5, (name, rel_err(a, b))
    assert stats["relu_near_zero"] == 0


# ------------------------------------------------------------------------------------------------- GPU
class _Touched:
    """Stands in for FusedAdam's bookkeeping: the ``mark`` / ``touched`` pair a sink is registered with."""

    def __init__(self):
        self._touched = set()

    def mark(self, p):
        self._touched.add(id(p))

    def touched(self, p):
        return id(p) in self._touched


@pytest.fixture
def restore_sinks():
    """The gradient-sink registry is global: whatever a test registers or clears is put back afterwards."""
    from emernerf_b200 import _ops

    saved = dict(_ops._GRAD_SINKS)
    yield
    _ops._GRAD_SINKS.clear()
    _ops._GRAD_SINKS.update(saved)


def _grad_bar(samples: int) -> float:
    return 2e-5 if samples <= 200000 else 5e-5


def _multi_rays() -> int:
    """Two full rounds of the persistent level backward plus five rays: every warp walks at least two rays."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 2 * (3 * sms * 8) + 5


def _d_cdf(R, n, seed):
    """Random upstream gradient with whole rows of zeros, zero tails (samples behind the last non-zero entry get
    d_raw == 0 exactly, the warp-uniform skip of the unit layout) and a large last column, which must have no effect
    (cdf[:, n] is the constant 1)."""
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(R, n + 1, generator=g)
    r = torch.arange(R)
    d[r % 5 == 3] = 0.0
    start = torch.randint(0, n + 1, (R,), generator=g)
    d[(r % 7 == 2)[:, None] & (torch.arange(n + 1)[None, :] >= start[:, None])] = 0.0
    d[:, n] = 1e3 * torch.randn(R, generator=g)
    return d.to(DEV)


# (levels, n, R, previous level, unbounded, b1): "multi" = _multi_rays(); previous level "first" = the uniform
# [0, 1], "second" = this network's own 128-interval output (m1 = 129), "spike" = all of the previous level's mass
# in s in [0, 2e-8] (t within ~4e-6 of the near plane: deltas of ~2.5e-7, so sigma > e^15 still leaves sigma * delta
# ~ 1 and the clamped backward branch carries gradient), "spike_far" = the same with a last, empty bin up to s = 1,
# into which the last edge of rays with jitter > 0.5 falls: that interval reaches t = 1000, and its sigma * delta
# (~3e9) outweighs the ray's prefix (~20) by more than 2^24 -- an exclusive scan formed as inclusive sum minus the own
# term returns 0 there (cdf = 0 after cdf = 1).  Stratified jitter everywhere.
CASES = {
    "lf4_n1_r1": (4, 1, 1, "first", True, None),
    "lf8_n1_r37_second": (8, 1, 37, "second", True, None),
    "lf4_n31_r37_bounded": (4, 31, 37, "first", False, None),
    "lf8_n32_r37_clamp": (8, 32, 37, "spike", True, 16.0),
    "lf8_n32_r37_clamp_far": (8, 32, 37, "spike_far", True, 16.0),
    "lf8_n33_r37_second": (8, 33, 37, "second", True, None),
    "lf8_n33_r37_flat": (8, 33, 37, "first", True, -25.0),
    "lf8_n255_r37": (8, 255, 37, "first", True, None),
    "lf4_n256_r37_second_bounded": (4, 256, 37, "second", False, None),
    "lf8_n128_multi": (8, 128, "multi", "first", True, None),
    "lf8_n64_multi_second": (8, 64, "multi", "second", True, None),
    "lf4_n128_multi_bounded": (4, 128, "multi", "first", False, None),
    "lf8_n128_r8192": (8, 128, 8192, "first", True, None),
    "lf8_n64_r8192_second": (8, 64, 8192, "second", True, None),
}


def _previous_level(kind, net, R, origins, dirs, s_min, s_max, seed):
    from emernerf_b200 import _ops

    first = torch.arange(2, device=DEV, dtype=torch.float32).repeat(R, 1)
    if kind == "first":
        return first, first.clone()
    if kind == "spike":
        s = torch.tensor([0.0, 2e-8], device=DEV).repeat(R, 1)
        return s, s.clone() / 2e-8
    if kind == "spike_far":
        s = torch.tensor([0.0, 2e-8, 1.0], device=DEV).repeat(R, 1)
        return s, torch.tensor([0.0, 1.0, 1.0], device=DEV).repeat(R, 1)
    g = torch.Generator().manual_seed(seed)
    bias = torch.rand(R, generator=g).to(DEV)
    s, _, cdf = _ops.prop_level(first, first.clone(), 128, bias, s_min, s_max, KIND, origins, dirs, net.aabb,
                                net.unbounded, net.xyz_encoder.desc, *_params(net))
    return s, cdf


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_level_backward_vs_fp64(case, restore_sinks):
    """``emer_prop_level_bwd`` + the grid scatter through ``_ops.prop_level_train``: the CDF and all five gradients
    against ``_level_fp64`` + autograd of sum(cdf * d_cdf).  Every gradient buffer is a registered sink that starts
    non-zero and marked touched, so the kernels must ADD to it (and ``.grad`` stays None); s and t must equal the
    no-grad launch bit for bit, and every CDF row must be non-decreasing."""
    from emernerf_b200 import _ops

    levels, n, R, prev, unbounded, b1 = CASES[case]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if R == "multi":
        R = _multi_rays()
        assert R > 3 * sms * 8
    seed = sum(map(ord, case))
    net = _density_field(levels, unbounded, seed, DEV, b1=b1)
    desc, geom = net.xyz_encoder.desc, adapters.spec_from_module(net).geom("xyz")
    origins, dirs = _rays(R, seed + 2, DEV)
    s_min, s_max = hotpath.s_bounds(KIND, NEAR, FAR)
    prev_s, prev_cdf = _previous_level(prev, net, R, origins, dirs, s_min, s_max, seed + 3)
    bias = torch.rand(R, generator=torch.Generator().manual_seed(seed + 4)).to(DEV)
    # persistent grid of the backward: rays per warp = ceil(R / (CTAs * 8))
    ctas = min(-(-R // 8), 3 * sms)
    rays_per_warp = -(-R // (ctas * 8))
    if R >= 3 * sms * 8:
        assert rays_per_warp >= 2, rays_per_warp

    params = [p.detach().clone().requires_grad_(True) for p in _params(net)]
    touch = _Touched()
    sinks = [torch.zeros_like(p) for p in params]
    for p, s in zip(params, sinks):
        _ops.register_grad_sink(p, s, touch.mark, touch.touched)
        touch.mark(p)                                   # "another term wrote it first": no zeroing, accumulate
    args = (prev_s, prev_cdf, n, bias, s_min, s_max, KIND, origins, dirs, net.aabb, unbounded, desc)
    s0, t0, cdf0 = _ops.prop_level(*args, *params)
    s1, t1, cdf1 = _ops.prop_level_train(*args, *params)
    assert torch.equal(s0, s1) and torch.equal(t0, t1) and torch.equal(cdf0, cdf1)
    assert cdf1.requires_grad and not s1.requires_grad and not t1.requires_grad
    assert (cdf1[:, 1:] - cdf1[:, :-1]).min().item() >= -1e-6, "CDF decreases along a ray"

    stats = {}
    p64 = [p.detach().double().requires_grad_(True) for p in params]
    sigma, cdf = _level_fp64(t1, origins, dirs, net.aabb, unbounded, desc, geom, *p64, stats=stats)
    if b1 is not None and b1 > 0:
        # both branches of trunc_exp's backward, and gradient reaching the clamped samples
        assert (sigma > E15).any() and (sigma < E15).any()
    if b1 is not None and b1 < 0:
        assert sigma.max().item() < 1e-6 and cdf[:, :-1].max().item() < 1e-3
    e_cdf = rel_err(cdf1, cdf)
    d_cdf = _d_cdf(R, n, seed + 5)
    want = torch.autograd.grad((cdf * d_cdf.double()).sum(), p64)
    del cdf, sigma

    g = torch.Generator(device=DEV).manual_seed(seed + 6)
    # pre-fill at a quarter of the gradient's scale (so fp32 rounding of pre-fill + gradient stays below the bar), or
    # of 1 where the fp64 gradient is exactly zero (n = 1: cdf = [0, 1] is constant): the kernels must add, never
    # overwrite, in every row
    pre = [torch.randn(s.shape, device=DEV, generator=g) * 0.25 * (w.abs().max().item() or 1.0)
           for s, w in zip(sinks, want)]
    for s, p in zip(sinks, pre):
        s.copy_(p)
    (cdf1 * d_cdf).sum().backward()
    torch.cuda.synchronize()

    errs = {k: rel_err(s.double() - p.double(), w) for k, s, p, w in zip(NAMES, sinks, pre, want)}
    bar = _grad_bar(R * n)
    print(f"{case}: R={R} rays/warp={rays_per_warp} cdf {e_cdf:.2e} "
          + " ".join(f"{k} {e:.2e}" for k, e in errs.items())
          + f" (bar {bar:.0e}, relu near zero {stats['relu_near_zero']})")
    assert all(p.grad is None for p in params)
    assert all(id(p) in touch._touched for p in params)
    assert e_cdf < 1e-5, e_cdf
    for k, e in errs.items():
        assert e < bar, (k, e)


# ------------------------------------------------------------------------------------------------- the production step
def _interlevel(s, cdf, prop_s, prop_cdf, r, dtype=torch.float64, chunk=1024, reduce=True):
    """One level's anti-aliased interlevel term in ``dtype`` (the restatement of test_gpu_kernels.py::
    test_interlevel_loss_value_and_gradient_vs_oracle, nerfacc_prop_net.py:22-60,182-240 of the reference): blur the
    final histogram, integrate it, interpolate at the level's edges, hinge against the level's weights.  Only
    ``prop_cdf`` carries gradient; the dense bracketing masks are built ``chunk`` rays at a time.  ``reduce=False``:
    the [R, n] terms instead of their mean."""
    with torch.no_grad():
        s_, ps_, cdf_ = s.to(dtype), prop_s.to(dtype), cdf.to(dtype)
        w_n = (cdf_[:, 1:] - cdf_[:, :-1]) / (s_[:, 1:] - s_[:, :-1])
        c, w = hotpath.blur_stepfun(s_, w_n, r)
        area = 0.5 * (w[:, 1:] + w[:, :-1]) * (c[:, 1:] - c[:, :-1])
        cd = torch.cat([torch.zeros_like(area[:, :1]), torch.cumsum(area, -1)], -1)
        w_s = torch.cat([torch.diff(hotpath.sorted_interp_quad(ps_[i:i + chunk], c[i:i + chunk], w[i:i + chunk],
                                                               cd[i:i + chunk]), dim=-1)
                         for i in range(0, s.shape[0], chunk)])
    wp = prop_cdf[:, 1:] - prop_cdf[:, :-1]
    terms = (w_s - wp).clamp_min(0) ** 2 / (wp + 1e-5)
    return terms.mean() if reduce else terms


# Sinks against the fp64 gradient of the whole loss.  Measured on an NVIDIA H100 80GB HBM3 at 700 W: table 2.9e-5,
# MLP 2e-6 to 9e-6 (emer_interlevel_loss computes its row in fp64: its d_cdf is 5e-8 off fp64, where the same formula
# evaluated in fp32 is 3.7e-3 off at pulse width 0.003).
LOSS_BAR = 5e-5


@pytest.mark.gpu
def test_both_levels_into_the_optimizer_sinks(restore_sinks):
    """The proposal update of the benchmark's step: ``PropNetEstimator.sampling(requires_grad=True)`` with proposal
    samples [128, 64] at 8192 rays, both level closures bound to ONE 8 x 1 proposal network (DESIGN.md Q21), the
    anti-aliased interlevel loss against a synthetic final level (65 edges, opacity < 1) and ``backward`` into
    ``FusedAdam``'s gradient sinks.  Each sink must hold the fp64 gradient of the same loss (the interlevel
    restatement composed with ``_level_fp64`` of both levels at the kernel's own edges):

    * table sink untouched and holding garbage: the first level's backward zeroes it, the second adds -- it ends up
      holding exactly the gradient;
    * every sink pre-filled and marked touched (another term wrote it first): pre-fill + gradient;
    * ``.grad`` stays the optimizer's sink view (autograd adds nothing of its own);
    * without sinks, ``.grad`` accumulates over two backward passes."""
    from emernerf_b200 import _ops, configs
    from emernerf_b200.optim import FusedAdam
    from emernerf_b200.third_party.nerfacc_prop_net import FusedProposalLevel, PropNetEstimator

    R, samples, final = 8192, [128, 64], 64
    cfg = configs.make_cfg("static")
    pe = cfg.nerf.propnet.xyz_encoder
    net = _density_field(pe.n_levels_per_prop[-1], True, 29, "cpu", max_resolution=pe.max_resolution_per_prop[-1],
                         log2_hashmap_size=pe.lgo2_hashmap_size_per_prop[-1], std=0.3)
    net.set_aabb(configs.AABB)
    net = net.to(DEV)
    params = _params(net)
    opt = FusedAdam([{"params": params[:1]}, {"params": params[1:]}], lr=0.01, eps=1e-15, weight_decay=1e-5,
                    betas=(0.9, 0.99), flatten_params=True)
    sinks = [p.grad for p in params]
    est = PropNetEstimator(opt, None, enable_anti_aliasing_loss=True,
                           anti_aliasing_pulse_width=cfg.nerf.propnet.anti_aliasing_pulse_width).to(DEV)
    g = torch.Generator().manual_seed(30)
    lo, hi = torch.tensor(configs.AABB[:3]), torch.tensor(configs.AABB[3:])
    origins = (lo + (hi - lo) * (0.25 + 0.5 * torch.rand(R, 3, generator=g))).to(DEV)
    dirs = torch.randn(R, 3, generator=g)
    dirs = (dirs / dirs.norm(dim=-1, keepdim=True)).to(DEV)
    jit = [torch.rand(R, generator=g).to(DEV) for _ in range(len(samples) + 1)]
    est._jitter_override = jit
    w = torch.rand(R, final, generator=g) ** 4 + 1e-6
    excl = torch.cumsum(torch.cat([torch.zeros(R, 1), w[:, :-1]], -1), -1) / w.sum(-1, keepdim=True)
    trans = (1.0 - torch.rand(R, 1, generator=g) * 0.98 * excl).to(DEV)      # opacity < 1

    fused = FusedProposalLevel(origins, dirs, net)

    def closure(t0, t1):
        raise AssertionError("the level must run fused")
    closure.emer_fused = fused
    fns = [closure, closure]                      # Q21: every level evaluates the last proposal network

    def step():
        est.prop_cache.clear()
        est.sampling(fns, samples, final, R, NEAR, FAR, KIND, stratified=True, requires_grad=True)
        cache = [(iv.vals, cdf) for iv, cdf, _ in est.prop_cache]
        for _, cdf in cache[:-1]:
            cdf.retain_grad()                     # d_cdf as emer_interlevel_loss hands it to the level backward
        est.compute_loss(trans).backward()
        torch.cuda.synchronize()
        return cache

    # fp64 reference at the kernel's own edges: the levels again through the no-grad launch (bit-identical s)
    opt.zero_grad()
    cache = step()
    s_min, s_max = hotpath.s_bounds(KIND, NEAR, FAR)
    prev_s = torch.arange(2, device=DEV, dtype=torch.float32).repeat(R, 1)
    prev_cdf = prev_s
    p64 = [p.detach().double().requires_grad_(True) for p in params]
    geom = adapters.spec_from_module(net).geom("xyz")
    final_s, _ = cache[-1]
    final_cdf = 1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], -1)
    loss64, chain64 = 0.0, 0.0
    for lvl, n in enumerate(samples):
        s, t, cdf = _ops.prop_level(prev_s, prev_cdf, n, jit[lvl], s_min, s_max, KIND, origins, dirs, net.aabb, True,
                                    net.xyz_encoder.desc, *params)
        assert torch.equal(s, cache[lvl][0]) and torch.equal(cdf, cache[lvl][1].detach())
        _, cdf64 = _level_fp64(t, origins, dirs, net.aabb, True, net.xyz_encoder.desc, geom, *p64)
        r = est.pulse_width[lvl]
        loss64 = loss64 + _interlevel(final_s, final_cdf, s, cdf64, r)
        # the interlevel kernel's d_cdf against fp64 and against the same restatement in fp32, at the kernel's CDF
        d_kernel = cache[lvl][1].grad
        at = cdf.double().requires_grad_(True)
        (d64,) = torch.autograd.grad(_interlevel(final_s, final_cdf, s, at, r), at)
        at32 = cdf.clone().requires_grad_(True)
        (d32,) = torch.autograd.grad(_interlevel(final_s, final_cdf, s, at32, r, torch.float32), at32)
        print(f"level {lvl}: d_cdf of emer_interlevel_loss {rel_err(d_kernel, d64):.2e}, "
              f"of the fp32 restatement {rel_err(d32, d64):.2e} (vs fp64)")
        chain64 = chain64 + (cdf64 * d_kernel.double()).sum()
        prev_s, prev_cdf = s, cdf
    want = torch.autograd.grad(loss64, p64, retain_graph=True)
    want_chain = torch.autograd.grad(chain64, p64)
    scale = [x.abs().max().item() for x in want]
    assert all(v > 0 for v in scale)

    def check(tag, got):
        """``got`` against the fp64 chain driven by the kernel's d_cdf (the level backward and the sinks alone: 5e-5)
        and against the fp64 gradient of the whole loss (LOSS_BAR)."""
        for ref, bar, what in ((want_chain, 5e-5, "level"), (want, LOSS_BAR, "loss")):
            errs = {k: rel_err(a, b) for k, a, b in zip(NAMES, got, ref)}
            print(f"sinks, {tag}, vs fp64 {what}: " + " ".join(f"{k} {e:.2e}" for k, e in errs.items()))
            for k, e in errs.items():
                assert e < bar, (tag, what, k, e)

    # 1. untouched table sink holding garbage (the other sinks zero, as step() leaves them): exactly the gradient
    opt.zero_grad()
    sinks[0].fill_(7.0)
    step()
    assert all(p.grad.data_ptr() == s.data_ptr() for p, s in zip(params, sinks))
    assert all(id(p) in opt._touched for p in params)
    check("untouched", [s.double() for s in sinks])

    # 2. pre-filled and touched: pre-fill + gradient
    opt.zero_grad()
    gp = torch.Generator(device=DEV).manual_seed(31)
    pre = [torch.randn(s.shape, device=DEV, generator=gp) * 0.25 * v for s, v in zip(sinks, scale)]
    for p, s, f in zip(params, sinks, pre):
        s.copy_(f)
        opt._mark(p)
    step()
    assert all(p.grad.data_ptr() == s.data_ptr() for p, s in zip(params, sinks))
    check("touched", [s.double() - f.double() for s, f in zip(sinks, pre)])

    # 3. no sinks: the ordinary autograd path, accumulating in .grad
    _ops.clear_grad_sinks()
    for p in params:
        p.grad = None
    step()
    step()
    assert all(p.grad is not None and p.grad.data_ptr() != s.data_ptr() for p, s in zip(params, sinks))
    check("no sinks, two passes", [p.grad.double() / 2.0 for p in params])

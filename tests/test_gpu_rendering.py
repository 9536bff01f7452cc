"""emer_render_fwd / emer_render_bwd (csrc/render.cu) on the GPU.

* Against ``oracle.hotpath.rendering`` (the reference's ``rendering``) run in float64 on CPU, on random inputs over
  every presence combination of the field's results: outputs within 1e-5 relative to their max-abs, the gradients of
  every input (``torch.autograd.grad`` on the fp64 graph) within 1e-5 of theirs.  The oracle builds its median split as
  an fp32 CPU tensor, so the median depth is compared with an fp32 run of it.
* Same device: weights, trans, opacity, depth and median depth bit-identical to emer_composite_fwd's; two launches
  bit-identical (no float atomics in either direction).
* ``render_rays`` / ``rendering`` with ``EMER_RENDERING=fused`` on the golden cases and the full-size fixtures at pinned
  samples, at the bars of tests/test_gpu_golden.py and tests/test_gpu_fullsize.py, and within 1e-5 of the switch-off
  outputs."""
import pytest
import torch

import cases
import test_gpu_fullsize as fullsize
import test_gpu_golden as golden
from helpers import assert_close_dict, rel_err
from oracle import hotpath

pytestmark = pytest.mark.gpu
DEV = "cuda"
C = 64
KEYS = {"sigma": "density", "sigma_s": "static_density", "sigma_d": "dynamic_density", "rgb": "rgb",
        "rgb_s": "static_rgb", "rgb_d": "dynamic_rgb", "shadow": "shadow_ratio", "rgb_sky": "rgb_sky",
        "dino": "dino_feat", "dino_s": "static_dino_feat", "dino_d": "dynamic_dino_feat", "dino_sky": "dino_sky_feat",
        "dino_pe": "dino_pe"}
# what a static / dynamic / dynamic-with-shadow / flow / feature field hands to rendering
COMBOS = {
    "static": ("rgb",),
    "static_feat_sky_pe": ("rgb", "rgb_sky", "dino", "dino_sky", "dino_pe"),
    "dynamic": ("sigma_s", "sigma_d", "rgb_s", "rgb_d", "rgb_sky"),
    "dynamic_shadow": ("sigma_s", "sigma_d", "rgb_s", "rgb_d", "shadow", "rgb_sky"),
    "flow": ("sigma_s", "sigma_d", "rgb_s", "rgb_d", "shadow", "flows"),
    "flow_feat": ("sigma_s", "sigma_d", "rgb_s", "rgb_d", "shadow", "rgb_sky", "dino_s", "dino_d", "dino_sky",
                  "dino_pe", "flows"),
}


def make_inputs(combo, r, s, seed=0):
    """fp32 CPU inputs, well conditioned in fp32: every sample's sigma*delta is >= 0.01 (the fp32 alpha = 1 - exp(-x)
    of the reference carries a relative error of ~3e-8 / x, and the static / dynamic ratio gradients peak where sigma is
    smallest), and every ray's optical depth is <= 6, so no ray's fp32 opacity reaches the clamp at 1."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *shape: torch.rand(*shape, generator=g)        # noqa: E731
    delta = rnd(r, s) * 0.02 + 0.02
    t0 = 0.5 + torch.cumsum(delta, -1) - delta
    t1 = t0 + delta
    have = COMBOS[combo]
    ins = {}
    if "sigma_s" in have:
        ins["sigma_s"], ins["sigma_d"] = rnd(r, s) * 0.5 + 0.25, rnd(r, s) * 0.5 + 0.25
        ins["sigma"] = ins["sigma_s"] + ins["sigma_d"]
    else:
        ins["sigma"] = rnd(r, s) + 0.5
    for k in have:
        if k in ("rgb", "rgb_s", "rgb_d"):
            ins[k] = rnd(r, s, 3)
        elif k == "shadow":
            ins[k] = rnd(r, s, 1)
        elif k == "rgb_sky":
            ins[k] = rnd(r, 3)
        elif k in ("dino", "dino_s", "dino_d"):
            ins[k] = torch.randn(r, s, C, generator=g)
        elif k in ("dino_sky", "dino_pe"):
            ins[k] = torch.randn(r, C, generator=g)
    flows = None
    if "flows" in have:
        buf = torch.randn(r, s, 6, generator=g)
        flows = (buf[..., :3], buf[..., 3:])
    return t0, t1, ins, flows


def oracle(t0, t1, ins, flows, decomposition, dtype=torch.float64, grad=False):
    leaves = {k: v.to(dtype).requires_grad_(grad) for k, v in ins.items()}
    res = {KEYS[k]: v for k, v in leaves.items()}
    if flows is not None:
        res["forward_flow"], res["backward_flow"] = (f.to(dtype) for f in flows)
    with torch.set_grad_enabled(grad):
        out = hotpath.rendering(t0.to(dtype), t1.to(dtype), res, return_decomposition=decomposition)
    return out, leaves


def run(t0, t1, ins, flows, decomposition, grad=False):
    from emernerf_b200 import _ops

    dev = {k: v.to(DEV).requires_grad_(grad) for k, v in ins.items()}
    fl = None if flows is None else tuple(f.to(DEV) for f in flows)
    if fl is not None:                  # column slices of one [R, S, 6] buffer, as the flow head writes them
        buf = torch.cat([flows[0], flows[1]], -1).to(DEV)
        fl = (buf[..., :3], buf[..., 3:])
    with torch.set_grad_enabled(grad):
        out = _ops.render(t0.to(DEV), t1.to(DEV), dev, flows=fl, decomposition=decomposition)
    return out, dev


NAMES = {"dino": "dino_feat"}


def _check_outputs(got, want, want32, flow_scale=None):
    """1e-5 of the max-abs; the flow sums (signed terms that cancel) against the max-abs of the sums of |w f|; the
    median depth equal to the fp32 oracle's except on rays whose fp64 cumulative weight passes within 1e-5 of 0.5, where
    the order of the sum decides the index (emer_composite_fwd's median, which it equals bit for bit, does the same)."""
    for k, v in got.items():
        ref = want["extras"][k] if k in ("weights", "trans") else want[NAMES.get(k, k)]
        if k == "median_depth":
            ref = want32[k]
        assert tuple(v.shape) == tuple(ref.shape), (k, v.shape, ref.shape)
        if not v.numel():
            continue
        if k == "median_depth":
            off = (v.cpu() != ref).squeeze(-1)
            cw = torch.cumsum(want["extras"]["weights"][off], -1)
            assert ((cw - 0.5).abs().min(-1).values < 1e-5).all(), int(off.sum())
        elif k in ("forward_flow", "backward_flow"):
            err = (v.double().cpu() - ref).abs().max().item()
            assert err <= 1e-5 * flow_scale[k], (k, err, flow_scale[k])
        else:
            assert rel_err(v, ref) <= 1e-5, (k, rel_err(v, ref))


SHAPES = [(1, 1), (1, 48), (1, 64), (1, 100), (0, 64), (8193, 48), (8193, 100)]


@pytest.mark.parametrize("decomposition", [False, True])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{r}x{s}" for r, s in SHAPES])
@pytest.mark.parametrize("combo", list(COMBOS))
def test_forward_matches_fp64_oracle(combo, shape, decomposition):
    if shape[0] == 8193 and decomposition and combo not in ("flow", "flow_feat", "static"):
        pytest.skip("the large batch covers the decomposition on the flow variants")
    t0, t1, ins, flows = make_inputs(combo, *shape)
    got, _ = run(t0, t1, ins, flows, decomposition)
    want, _ = oracle(t0, t1, ins, flows, decomposition)
    want32, _ = oracle(t0, t1, ins, flows, False, dtype=torch.float32)
    expect = {"weights", "trans", "opacity", "depth", "median_depth", "rgb"}
    if "dino" in ins or "dino_s" in ins:
        expect |= {"dino"} | ({"dino_pe_free"} if "dino_pe" in ins else set())
    if "shadow" in ins:
        expect.add("shadow_ratio")
    if decomposition and "sigma_s" in ins:
        expect |= {"static_opacity", "dynamic_opacity", "static_depth", "dynamic_depth", "static_rgb", "dynamic_rgb"}
        if "shadow" in ins:
            expect |= {"shadow_reduced_static_rgb", "shadow_only_static_rgb", "shadow"}
        if flows is not None:
            expect |= {"forward_flow", "backward_flow"}
        if "dino_s" in ins:
            expect |= {"static_dino", "dynamic_dino"}
    assert set(got) == expect
    scale = None
    if decomposition and flows is not None and "sigma_s" in ins and shape[0]:
        absolute, _ = oracle(t0, t1, ins, tuple(f.abs() for f in flows), True)
        scale = {k: absolute[k].abs().max().item() for k in ("forward_flow", "backward_flow")}
    _check_outputs(got, want, want32, scale)


GRAD_SHAPES = [(1, 1), (1, 48), (1, 64), (1, 100), (0, 64), (8193, 64), (8193, 100)]


@pytest.mark.parametrize("shape", GRAD_SHAPES, ids=[f"{r}x{s}" for r, s in GRAD_SHAPES])
@pytest.mark.parametrize("combo", list(COMBOS))
def test_backward_matches_fp64_oracle(combo, shape):
    if shape[0] == 8193 and shape[1] == 100 and combo not in ("flow_feat", "static_feat_sky_pe"):
        pytest.skip("the largest batch covers the feature variants")
    t0, t1, ins, flows = make_inputs(combo, *shape, seed=1)
    got, dev = run(t0, t1, ins, flows, False, grad=True)
    want, leaves = oracle(t0, t1, ins, flows, False, grad=True)
    g = torch.Generator().manual_seed(7)
    outs, gouts, wouts = [], [], []
    for k, v in got.items():
        if k == "median_depth":
            continue
        up = torch.randn(v.shape, generator=g, dtype=torch.float64)
        outs.append(v)
        gouts.append(up.float().to(DEV))
        ref = want["extras"][k] if k in ("weights", "trans") else want[NAMES.get(k, k)]
        wouts.append((ref, up))
    names = list(dev)
    d = torch.autograd.grad(outs, [dev[k] for k in names], gouts, allow_unused=True)
    wd = torch.autograd.grad([w for w, _ in wouts], [leaves[k] for k in names], [u for _, u in wouts],
                             allow_unused=True)
    for k, a, b in zip(names, d, wd):
        assert (a is None) == (b is None), k
        if a is None or a.numel() == 0:
            continue
        assert a.shape == b.shape, k
        err = (a.double().cpu() - b).abs().max().item()
        scale = b.abs().max().item()
        assert err <= 1e-5 * max(scale, 1e-30), (k, err, scale)


@pytest.mark.parametrize("combo", list(COMBOS))
def test_scan_bit_identical_to_composite_and_deterministic(combo):
    from emernerf_b200 import _ops

    t0, t1, ins, flows = make_inputs(combo, 8193, 100, seed=2)
    a, dev = run(t0, t1, ins, flows, False, grad=True)
    w, tr, op, dep, med, _ = _ops.composite(t0.to(DEV), t1.to(DEV), dev["sigma"].detach())
    for k, v in (("weights", w), ("trans", tr), ("opacity", op), ("depth", dep), ("median_depth", med)):
        assert torch.equal(a[k], v), k
    b, dev2 = run(t0, t1, ins, flows, False, grad=True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    def loss(o):
        return sum((v * (i + 1)).sum() for i, (k, v) in enumerate(o.items()) if k != "median_depth")

    ga = torch.autograd.grad(loss(a), list(dev.values()))
    gb = torch.autograd.grad(loss(b), list(dev2.values()))
    for k, x, y in zip(dev, ga, gb):
        assert torch.equal(x, y), k
    c, _ = run(t0, t1, ins, flows, True)
    d, _ = run(t0, t1, ins, flows, True)
    for k in c:
        assert torch.equal(c[k], d[k]), k


# ------------------------------------------------------------------------------------ end to end with the switch on
@pytest.fixture
def fused(monkeypatch):
    from emernerf_b200.radiance_fields import render_utils

    monkeypatch.setattr(render_utils, "RENDERING", "fused")


@pytest.mark.parametrize("case", list(cases.CASES))
@pytest.mark.parametrize("mode", ["eval", "lidar", "train"])
def test_fused_render_rays_matches_reference_outputs(fused, case, mode):
    golden.test_render_rays_matches_reference_outputs(case, mode)


@pytest.mark.parametrize("case", list(cases.CASES))
def test_fused_training_gradients_match_reference(fused, case):
    golden.test_training_gradients_and_proposal_loss_match_reference(case)


@pytest.mark.parametrize("case", list(cases.CASES))
def test_fused_compositing_at_reference_samples(fused, case):
    golden.test_field_and_compositing_at_reference_samples(case)


@pytest.mark.parametrize("variant", fullsize.fc.VARIANTS)
def test_fused_full_size_at_reference_samples(fused, variant):
    fullsize.test_full_size_field_and_compositing_at_reference_samples(variant)


@pytest.mark.parametrize("case", list(cases.CASES))
@pytest.mark.parametrize("mode", ["eval", "train"])
def test_switch_on_and_off_agree(monkeypatch, case, mode):
    from emernerf_b200.radiance_fields import render_utils
    from oracle import adapters

    outs, grads = {}, {}
    for how in ("torch", "fused"):
        monkeypatch.setattr(render_utils, "RENDERING", how)
        g, field, props, est = golden._build(case)
        out, names = fullsize._launch_names(lambda: golden._render(g, field, props, est, mode))
        assert ("emer_render_fwd" in names) == (how == "fused"), names
        outs[how] = out
        if mode == "train":
            adapters.parity_loss(out).backward()
            grads[how] = {k: v.grad.clone() for k, v in field.named_parameters() if v.grad is not None}
    assert_close_dict(outs["fused"], outs["torch"], 1e-5)
    if mode == "train":
        assert set(grads["fused"]) == set(grads["torch"])
        for k in grads["torch"]:
            # the hash-grid scatter adds with float atomics, so two backward passes differ in the last bits
            assert rel_err(grads["fused"][k], grads["torch"][k]) < 1e-3, k

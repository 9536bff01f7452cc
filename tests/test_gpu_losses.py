"""emernerf_b200.loss on the GPU: every class against the reference's goldens and, at full size (8192 x 64 and a
ragged 8191), against an fp64 restatement of the reference's arithmetic; bit-identical repeats; accumulation into a
non-zero .grad under a 1024 upstream factor; no host sync; CUDA-graph capture of the lidar-pass set; and the field's
and proposal networks' parameter gradients of a whole pixel + lidar pass against the torch formulation."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import loss_cases as lc
from test_losses_cpu import check_case

pytestmark = pytest.mark.gpu
DEV = "cuda"
COEF = {"RealValueLoss": 1.0, "SkyLoss": 0.01, "DepthLoss": 1.0, "LineOfSightLoss": 1.0,
        "DynamicRegularizationLoss": 1.0}


def _real(kind, d):
    if kind == "l1":
        return d.abs()
    if kind == "l2":
        return d * d
    return torch.where(d.abs() < 1.0, 0.5 * d * d, d.abs() - 0.5)


def restated(case, inp, f32):
    """The reference's arithmetic in the dtype of ``inp``; mask decisions on the fp32 inputs ``f32``, as the fp32
    reference takes them."""
    _, cls, ctor, args, kw = case
    a = [inp[k] for k in args]
    coef = ctor.get("coef", COEF[cls])
    if cls == "RealValueLoss":
        return (_real(ctor.get("loss_type", "l2"), a[0] - a[1]) * kw.get("coef", 1.0)).mean() * coef
    if cls == "SkyLoss":
        if ctor["loss_type"] == "opacity_based":
            return F.binary_cross_entropy(a[0].squeeze(), 1 - a[1], reduction="none").mean() * coef
        return ((a[0] ** 2).sum(-1) * a[1]).mean() * coef
    if cls == "DepthLoss":
        mx = float(ctor.get("upper_bound", 80))
        gt32 = f32[args[1]].squeeze()
        valid = (gt32 > 0.01) & (gt32 < mx)
        nd = lambda d: torch.clamp(d.squeeze()[valid] / mx, 0.0, 1.0)
        return _real(ctor.get("loss_type", "l2"), nd(a[0]) - nd(a[1])).mean() * coef
    if cls == "LineOfSightLoss":
        eps = kw["epsilon"]
        gt32, t32 = f32[args[1]].squeeze()[:, None], f32["t_vals"]
        lo, hi = gt32 - np.float32(eps), gt32 + np.float32(eps)
        empty, near = t32 < lo, (t32 > lo) & (t32 < hi)
        w, t, g = a[2], inp["t_vals"], a[1].squeeze()[:, None]
        sig = eps / 3
        dirac = 1 / math.sqrt(2 * math.pi * sig ** 2) * torch.exp(-((t - g) ** 2) / (2 * sig ** 2))
        sight = (w * w * empty).sum(-1).mean() + ((w - dirac) ** 2 * near).sum(-1).mean()
        return (sight * (gt32[:, 0] > 0) * kw.get("coef_decay", 1.0)).mean() * coef
    if ctor.get("loss_type", "sparsity") == "sparsity":
        return a[0].mean() * coef
    k = ctor.get("entropy_skewness", 2.0)
    r = a[0] / (a[0] + a[1] + 1e-7)
    c = (r ** k).clamp(1e-6, 1 - 1e-6)
    return (-(c * c.log()) + -(1 - c) * (1 - c).log()).mean() * coef


@pytest.mark.parametrize("case", lc.CASES, ids=[c[0] for c in lc.CASES])
def test_loss_on_cuda_matches_reference_golden(case):
    from emernerf_b200 import loss

    check_case(loss, case, DEV)


@pytest.mark.parametrize("r", [8192, 8191])
@pytest.mark.parametrize("case", lc.CASES, ids=[c[0] for c in lc.CASES])
def test_full_size_against_fp64(case, r):
    from emernerf_b200 import loss

    x = lc.make_inputs(seed=3, r=r, s=64, edges=False)
    key, value, grads = lc.run_case(loss, x, case, DEV)
    inp = {k: v.double().requires_grad_(k in lc.GRAD_INPUTS) for k, v in x.items()}
    want = restated(case, inp, x)
    if not torch.isfinite(want):
        assert torch.isnan(value)
        return
    assert abs(value.item() - want.item()) <= 1e-5 * abs(want.item()), (value.item(), want.item())
    wanted = [k for k in grads]
    refs = torch.autograd.grad(want, [inp[k] for k in wanted], allow_unused=True)
    for k, gr in zip(wanted, refs):
        gr = torch.zeros_like(inp[k]) if gr is None else gr
        scale = gr.abs().max().item()
        err = (grads[k].double().cpu() - gr).abs().max().item()
        assert err <= 1e-6 * max(scale, 1e-30), (k, err, scale)


def _lidar_set(loss, x, eps=2.5, decay=0.5):
    depth = loss.DepthLoss(loss_type="l2")(x["depth"], x["lidar_ranges"], name="lidar_range_loss")
    los = loss.LineOfSightLoss(coef=0.1)(x["depth"], x["lidar_ranges"], x["weights"], x["t_vals"], epsilon=eps,
                                          name="lidar_line_of_sight", coef_decay=decay)
    dyn = loss.DynamicRegularizationLoss(coef=0.01)(x["dynamic_density"], x["static_density"], name="lidar_dynamic")
    return {**depth, **los, **dyn}


def _inputs(seed=5, r=8192):
    return {k: v.to(DEV).requires_grad_(k in lc.GRAD_INPUTS) for k, v in lc.make_inputs(seed, r, 64).items()}


def test_bit_identical_repeats():
    from emernerf_b200 import loss

    outs = []
    for _ in range(2):
        x = _inputs()
        vals = _lidar_set(loss, x)
        vals.update(loss.RealValueLoss(name="feature", coef=0.5)(x["dino_feat"], x["features"]))
        vals.update(loss.DynamicRegularizationLoss(loss_type="entropy", entropy_skewness=1.1)(
            x["dynamic_density"], x["static_density"]))
        sum(vals.values()).backward()
        outs.append(({k: v.detach().clone() for k, v in vals.items()},
                     {k: x[k].grad.clone() for k in ("depth", "weights", "dino_feat", "dynamic_density",
                                                      "static_density")}))
    for a, b in zip(outs[0], outs[1]):
        for k in a:
            assert torch.equal(a[k], b[k]) or (torch.isnan(a[k]).all() and torch.isnan(b[k]).all()), k


def test_gradients_accumulate_with_scaled_upstream():
    from emernerf_b200 import loss

    x = _inputs()
    sum(_lidar_set(loss, x).values()).backward()
    base = {k: x[k].grad.clone() for k in ("depth", "weights", "dynamic_density")}
    y = _inputs()
    for k in base:
        y[k].grad = torch.ones_like(y[k])
    scaler = torch.amp.GradScaler("cuda", init_scale=1024.0)
    scaler.scale(sum(_lidar_set(loss, y).values())).backward()
    for k, g in base.items():
        assert torch.allclose(y[k].grad, 1.0 + 1024.0 * g, rtol=1e-6, atol=1e-6), k


def test_no_host_sync():
    from emernerf_b200 import loss

    x = _inputs()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        total = 0
        for _, cls, ctor, args, kwargs in lc.CASES:
            total = total + next(iter(getattr(loss, cls)(**ctor)(*[x[a] for a in args], **kwargs).values()))
        total.backward()
        loss.compute_line_of_sight_loss(x["lidar_ranges"], x["weights"], x["t_vals"]).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_lidar_set_in_a_cuda_graph():
    from emernerf_b200 import loss

    static = _inputs(seed=7)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for k in static:
                static[k].grad = None
            sum(_lidar_set(loss, static).values()).backward()
    torch.cuda.current_stream().wait_stream(side)
    for k in static:
        static[k].grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        vals = _lidar_set(loss, static)
        sum(vals.values()).backward()
    for seed in (11, 12):
        fresh = _inputs(seed=seed)
        with torch.no_grad():
            for k in static:
                static[k].copy_(fresh[k])
        graph.replay()
        want = _lidar_set(loss, fresh)
        sum(want.values()).backward()
        torch.cuda.synchronize()
        for k in want:
            assert torch.equal(vals[k], want[k]), k
        for k in ("depth", "weights", "dynamic_density"):
            assert torch.equal(static[k].grad, fresh[k].grad), k


def _torch_pixel(out, batch):
    rgb = F.mse_loss(out["rgb"], batch["pixels"], reduction="none").mean()
    sky = F.binary_cross_entropy(out["opacity"].squeeze(), 1 - batch["sky_masks"], reduction="none").mean() * 0.001
    return rgb + sky


def _torch_lidar(out, batch, eps=2.5):
    gt = batch["lidar_ranges"].squeeze()
    valid = (gt > 0.01) & (gt < 80)
    nd = lambda d: torch.clamp(d / 80, 0.0, 1.0)
    depth = F.mse_loss(nd(out["depth"].squeeze()[valid]), nd(gt[valid]), reduction="none").mean()
    w, t = out["extras"]["weights"], out["extras"]["t_vals"].detach()
    g = gt[:, None]
    empty, near = t < g - eps, (t > g - eps) & (t < g + eps)
    sig = eps / 3
    dirac = (1 / math.sqrt(2 * torch.pi * sig ** 2)) * torch.exp(-((t - g) ** 2) / (2 * sig ** 2))
    sight = (w.square() * empty).sum(-1).mean() + ((w - dirac).square() * near).sum(-1).mean()
    return depth + (sight * (gt > 0) * 0.5).mean() * 0.1


def test_pixel_and_lidar_pass_parameter_gradients():
    from emernerf_b200 import loss
    from test_gpu_golden import _build, _render

    g, field, props, est = _build("static")
    params = [p for p in field.parameters()] + [p for m in props for p in m.parameters()]
    rgb_fn, sky_fn = loss.RealValueLoss(), loss.SkyLoss(loss_type="opacity_based", coef=0.001)
    depth_fn, los_fn = loss.DepthLoss(), loss.LineOfSightLoss(coef=0.1)
    for mode in ("train", "lidar"):
        batch = g.tensors("in/lidar" if mode == "lidar" else "in/pixel", DEV)
        out = _render(g, field, props, est, mode)
        if mode == "train":
            new = {**rgb_fn(out["rgb"], batch["pixels"]), **sky_fn(out["opacity"], batch["sky_masks"])}
        else:
            new = {**depth_fn(out["depth"], batch["lidar_ranges"], name="lidar_range_loss"),
                   **los_fn(out["depth"], batch["lidar_ranges"], out["extras"]["weights"], out["extras"]["t_vals"],
                            epsilon=2.5, name="lidar_line_of_sight", coef_decay=0.5)}
        total = sum(new.values())
        g_new = torch.autograd.grad(total, params, allow_unused=True)
        out = _render(g, field, props, est, mode)                  # the same seeded pass, for the torch formulation
        ref = _torch_pixel(out, batch) if mode == "train" else _torch_lidar(out, batch)
        assert abs(total.item() - ref.item()) <= 1e-5 * abs(ref.item())
        g_ref = torch.autograd.grad(ref, params, allow_unused=True)
        n = 0
        for p, a, b in zip(params, g_new, g_ref):
            assert (a is None) == (b is None)
            if a is None:
                continue
            n += 1
            scale = b.abs().max().item()
            assert (a - b).abs().max().item() <= 1e-4 * max(scale, 1e-30), (mode, tuple(p.shape))
        assert n > 0

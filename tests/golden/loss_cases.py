"""Inputs and cases of the training-loss fixture (tests/golden/losses.npz, written by make_golden_losses.py).

Every loss class of the reference's loss/base.py with the options the shipped configurations reach, at R = 136 rays x
S = 48 samples (neither a multiple of the kernels' warp or CTA widths), on seeded inputs with hand-built edge rows:
opacity at 1e-6 and 1, ranges at 0, 0.01, 80 and beyond, predicted depths beyond the 80 m bound, t_vals exactly at
gt -+ epsilon, densities whose entropy ratio is clamped.
"""
from __future__ import annotations

import torch

R, S = 136, 48

# name, class, constructor kwargs, positional input keys, call kwargs
CASES = [
    ("rgb_l1", "RealValueLoss", dict(loss_type="l1"), ("rgb", "pixels"), {}),
    ("rgb_l2", "RealValueLoss", dict(loss_type="l2", coef=1.0, name="rgb"), ("rgb", "pixels"), {}),
    ("rgb_smooth_l1", "RealValueLoss", dict(loss_type="smooth_l1", coef=2.0), ("rgb", "pixels"), dict(coef=0.5)),
    ("feature_l2", "RealValueLoss", dict(loss_type="l2", coef=0.5, name="feature"), ("dino_feat", "features"), {}),
    ("feature_smooth_l1", "RealValueLoss", dict(loss_type="smooth_l1", coef=0.5, name="feature"),
     ("dino_feat", "features"), {}),
    ("sky_opacity", "SkyLoss", dict(loss_type="opacity_based", coef=0.001), ("opacity", "sky_masks"), {}),
    ("sky_weights", "SkyLoss", dict(loss_type="weights_based"), ("weights", "sky_masks"), {}),
    ("depth_l2", "DepthLoss", dict(loss_type="l2", coef=1.0), ("depth", "lidar_ranges"), dict(name="lidar_range_loss")),
    ("depth_l1", "DepthLoss", dict(loss_type="l1"), ("depth", "lidar_ranges"), {}),
    ("depth_smooth_l1", "DepthLoss", dict(loss_type="smooth_l1", coef=0.5, upper_bound=60),
     ("depth", "lidar_ranges"), {}),
    ("depth_empty", "DepthLoss", dict(loss_type="l2"), ("depth", "no_ranges"), dict(name="lidar_range_loss")),
    ("los_eps6", "LineOfSightLoss", dict(loss_type="my", name="line_of_sight", coef=0.1),
     ("depth", "lidar_ranges", "weights", "t_vals"), dict(epsilon=6.0, name="lidar_line_of_sight", coef_decay=0.5)),
    ("los_eps2_5", "LineOfSightLoss", dict(coef=0.1), ("depth", "lidar_ranges", "weights", "t_vals"),
     dict(epsilon=2.5)),
    ("los_empty", "LineOfSightLoss", dict(coef=0.1), ("depth", "no_ranges", "weights", "t_vals"), dict(epsilon=2.5)),
    ("dynamic_sparsity", "DynamicRegularizationLoss", dict(loss_type="sparsity", coef=0.01),
     ("dynamic_density", "static_density"), {}),
    ("dynamic_lidar", "DynamicRegularizationLoss", dict(loss_type="sparsity", coef=0.01),
     ("dynamic_density", "static_density"), dict(name="lidar_dynamic")),
    ("dynamic_entropy_1_1", "DynamicRegularizationLoss", dict(loss_type="entropy", coef=0.01, entropy_skewness=1.1),
     ("dynamic_density", "static_density"), {}),
    ("dynamic_entropy_2", "DynamicRegularizationLoss", dict(loss_type="entropy"), ("dynamic_density", "static_density"),
     {}),
    ("shadow", "DynamicRegularizationLoss", dict(name="shadow", loss_type="sparsity", coef=0.01), ("shadow_ratio",), {}),
]

# inputs that receive gradients (leaves with requires_grad in both the reference run and the tests)
GRAD_INPUTS = ("rgb", "dino_feat", "opacity", "depth", "weights", "dynamic_density", "static_density", "shadow_ratio")

CLASSES = ("Loss", "RealValueLoss", "SkyLoss", "DepthLoss", "LineOfSightLoss", "DynamicRegularizationLoss")
FUNCTIONS = ("normalize_depth", "dirac_delta_approx", "compute_line_of_sight_loss")


def make_inputs(seed: int = 0, r: int = R, s: int = S, edges: bool = True):
    """The fixture's inputs are these (seed 0, default sizes); losses.npz keeps only their digest (``digest``)."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *shape: torch.rand(*shape, generator=g)
    x = {
        "rgb": rnd(r, 3),
        "pixels": rnd(r, 3),
        "dino_feat": torch.randn(r, 64, generator=g),
        "features": rnd(r, 64),
        "opacity": (rnd(r, 1) * (1 - 1e-6) + 1e-6).clamp(1e-6, 1.0),
        "sky_masks": (rnd(r) < 0.3).float(),
        "depth": rnd(r, 1) * 90.0,
        "lidar_ranges": rnd(r, 1) * 79.5 + 0.5,
        "weights": rnd(r, s) * 0.05,
        "t_vals": rnd(r, s) * 100.0,
        "dynamic_density": torch.exp(torch.randn(r, s, generator=g)),
        "static_density": torch.exp(torch.randn(r, s, generator=g)),
        "shadow_ratio": rnd(r, 1),
    }
    x["no_ranges"] = torch.zeros(r, 1)
    if edges:
        x["opacity"][0:4] = 1e-6
        x["opacity"][4:8] = 1.0
        x["sky_masks"][0:8:2] = 1.0
        x["sky_masks"][1:8:2] = 0.0
        gt = x["lidar_ranges"]
        gt[0:8, 0] = torch.tensor([0.0, 0.01, 80.0, 85.0, 1e-3, 0.0100001, 79.99999, 120.0])
        x["depth"][8:16, 0] = torch.tensor([80.0, 81.0, 95.0, 0.0, 79.9, 200.0, 80.0001, 60.0])
        # samples exactly at gt -+ epsilon (the strict inequalities of the masks), in the fp32 of the masks
        for rows, eps in ((slice(16, 32), 6.0), (slice(32, 48), 2.5)):
            g_r = gt[rows]
            x["t_vals"][rows, 0:1] = g_r - eps
            x["t_vals"][rows, 1:2] = g_r + eps
            x["t_vals"][rows, 2:3] = g_r
            x["t_vals"][rows, 3:4] = torch.nextafter(g_r - eps, torch.full_like(g_r, 1e9))
        # entropy: ratios 0 (clamped at 1e-6), ~1 (clamped at 1 - 1e-6), and both densities zero
        x["dynamic_density"][0, :] = 0.0
        x["static_density"][1, :] = 0.0
        x["dynamic_density"][2, :] = 0.0
        x["static_density"][2, :] = 0.0
        x["weights"][3, :] = 0.0
    return x


def digest(x: dict) -> dict:
    """Per input: float64 sum and sum of squares, to tell that regenerated inputs are the fixture's."""
    return {k: torch.stack([v.double().sum(), v.double().square().sum()]) for k, v in x.items()}


def run_case(module, x: dict, case: tuple, device="cpu"):
    """Runs one case through ``module``'s loss classes (the reference's or emernerf_b200.loss) on ``device``:
    (returned key, value, {input: gradient of the value}) -- gradients only for a finite value."""
    name, cls, ctor, args, kwargs = case
    inp = {k: v.to(device).clone().requires_grad_(k in GRAD_INPUTS) for k, v in x.items()}
    (key, value), = getattr(module, cls)(**ctor)(*[inp[a] for a in args], **kwargs).items()
    grads = {}
    wanted = [a for a in dict.fromkeys(args) if a in GRAD_INPUTS]
    if value.requires_grad and torch.isfinite(value):
        got = torch.autograd.grad(value, [inp[a] for a in wanted], allow_unused=True)
        grads = {a: torch.zeros_like(inp[a]) if gr is None else gr for a, gr in zip(wanted, got)}
    return key, value, grads

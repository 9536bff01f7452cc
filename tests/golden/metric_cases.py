"""Inputs and cases of the evaluation-metric fixture (tests/golden/metrics.npz, written by make_golden_metrics.py).

Seeded CPU inputs for the reference's compute_psnr, compute_valid_depth_rmse and compute_scene_flow_metrics: PSNR of a
training ray batch, of a noisy image and of identical images (+inf); depth RMSE over rays with zero, negative and
positive ranges, a [R, 1] column against [R], and a batch without a valid ray (NaN); scene flow on a noisy lidar-like
frame, with zero predictions and zero labels mixed in, and a frame whose labels are all below the 0.1 angle threshold
(angle error NaN).  Sizes are not multiples of the kernels' warp or CTA widths.
"""
from __future__ import annotations

from typing import Dict

import torch

# name, reference function, input keys (positional)
CASES = [
    ("psnr_rays", "compute_psnr", ("rgb", "pixels")),
    ("psnr_image", "compute_psnr", ("image_pred", "image")),
    ("psnr_identical", "compute_psnr", ("image", "image")),
    ("depth_rays", "compute_valid_depth_rmse", ("depth", "ranges")),
    ("depth_column", "compute_valid_depth_rmse", ("depth_col", "ranges")),
    ("depth_no_valid", "compute_valid_depth_rmse", ("depth", "no_ranges")),
    ("flow_frame", "compute_scene_flow_metrics", ("flow_pred", "flow_labels")),
    ("flow_zeros", "compute_scene_flow_metrics", ("flow_pred_zeros", "flow_labels_zeros")),
    ("flow_small", "compute_scene_flow_metrics", ("flow_pred", "flow_labels_small")),
]
FLOW_KEYS = ("EPE3D", "acc3d_strict", "acc3d_relax", "outlier", "angle_error")


def make_inputs(seed: int = 0) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g)
    rgb = rnd(1001, 3)
    image = rnd(37, 53, 3)
    ranges = rnd(1001) * 80.0
    ranges[::7] = 0.0
    ranges[3::11] = -1.0
    labels = torch.randn(1, 4099, 3, generator=g) * 0.5
    pred = labels + torch.randn(1, 4099, 3, generator=g) * 0.08
    pred_z, labels_z = pred.clone(), labels.clone()
    pred_z[0, ::5] = 0.0
    labels_z[0, 2::9] = 0.0
    labels_z[0, 4::13] = pred_z[0, 4::13]          # exact matches: the dot product reaches the clamp
    return {
        "rgb": rgb,
        "pixels": (rgb + 0.05 * torch.randn(1001, 3, generator=g)).clamp(0, 1),
        "image": image,
        "image_pred": (image + 0.1 * torch.randn(37, 53, 3, generator=g)).clamp(0, 1),
        "depth": ranges + torch.randn(1001, generator=g),
        "depth_col": (ranges + torch.randn(1001, generator=g))[:, None],
        "ranges": ranges,
        "no_ranges": -rnd(1001),
        "flow_pred": pred,
        "flow_labels": labels,
        "flow_pred_zeros": pred_z,
        "flow_labels_zeros": labels_z,
        "flow_labels_small": labels * 0.1 / 3.0,
    }

"""Seeded sources and render results for the error-map refresh, shared by make_golden_errormap.py (which runs the
reference's own ``get_render_rays`` and ``update_pixel_error_maps`` on them) and the tests.

The sources are raybatch_cases' (12 images of 64 x 96, error maps of 4 x 6) with the reference's
``_downscale_factor`` set: "full" carries masks, features and timestamps, "bare" none of them.  ``render_results``
builds the lists ``render_pixels`` hands to ``update_pixel_error_maps``, from a seeded generator."""
from __future__ import annotations

import numpy as np
import torch

import raybatch_cases as rc

SOURCES = ("full", "bare")
# 1/3 does not divide the image: 21 x 32
DOWNSCALES = {"1": 1.0, "1_4": 1 / 4, "1_16": 1 / 16, "1_3": 1 / 3}
IMAGES = {"1": (5,), "1_4": (0, 5, 11), "1_16": (0, 5, 11), "1_3": (0, 5, 11)}     # per downscale
# name -> (with dynamic opacities: None = no key, "empty" = an empty list, True = one per image; constant map; NaN)
UPDATES = {
    "plain": (None, False, False),
    "dynamic": (True, False, False),
    "empty_dynamic": ("empty", False, False),
    "constant": (None, True, False),
    "nan": (None, False, True),
}


class PixelSource(rc.PixelSource):
    """raybatch_cases' stand-in with the property get_render_rays reads."""
    downscale_factor = property(lambda self: self._downscale_factor)


def fill(src, case: str, d: float = 1.0):
    rc.fill_pixel(src, case)
    src._downscale_factor = d
    return src


def render_results(case: str):
    """The dict of numpy lists render_pixels returns, as far as update_pixel_error_maps reads it."""
    dyn, constant, nan = UPDATES[case]
    g = torch.Generator().manual_seed(300 + list(UPDATES).index(case))
    n, h, w = rc.N_IMAGES, rc.HEIGHT // rc.DOWNSCALE, rc.WIDTH // rc.DOWNSCALE
    gt = torch.rand(n, h, w, 3, generator=g)
    rgb = torch.rand(n, h, w, 3, generator=g)
    if constant:
        gt, rgb = torch.full_like(gt, 0.5), torch.full_like(rgb, 0.25)
    if nan:
        rgb[3, 1, 2, 0] = float("nan")
    out = {"gt_rgbs": [a.numpy() for a in gt], "rgbs": [a.numpy() for a in rgb]}
    if dyn == "empty":
        out["dynamic_opacities"] = []
    elif dyn:
        op = torch.rand(n, h, w, generator=g)
        op[0, 0, :3] = torch.tensor([0.1, np.nextafter(np.float32(0.1), np.float32(1)), 0.0999999])  # around 0.1f
        out["dynamic_opacities"] = [a.numpy() for a in op]
    return out

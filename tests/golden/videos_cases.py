"""Seeded per-image render products for the evaluation videos, shared by make_golden_videos.py (which runs the
reference's own ``render`` + ``save_videos`` on them) and the tests.

Each case names a field variant (which products ``render_rays`` returns), a tile size, cameras, timestamps, keys and
the writer mode.  ``results(case, i)`` and ``data(case, i)`` are image i's render results and dataset item, from a
CPU generator seeded per case and image; ``Model`` carries the PCA the feature products use.  ``turbo_table()`` is a
seeded 256-entry RGBA table standing in for matplotlib's turbo (no colour data of matplotlib's is kept here): some of
its entries are exact multiples of 1/255, whose float64 ``255 * x`` truncates below the integer.  The "edges" cases
put values just outside [0, 1], exactly 0 and 1, depths at lo and hi, depth 0, negative depths, NaN and infinities,
and float32 values next to every k / 255 (``near_steps``)."""
from __future__ import annotations

import types

import numpy as np
import torch

MARGIN = 1e-4                # a depth pixel is not firm where v * 256 lies within MARGIN of an integer
FEAT, PE = 8, 6              # feature and positional-embedding channels
DEPTH_LO, DEPTH_HI = 4.0, 120

VARIANTS = {
    # name: products of render_rays beyond rgb / depth / opacity
    "static": ("median_depth",),
    "dynamic": ("static_rgb", "dynamic_rgb", "static_depth", "static_opacity", "dynamic_depth", "dynamic_opacity",
                "median_depth", "shadow_reduced_static_rgb", "shadow_only_static_rgb"),
    "flow": ("static_rgb", "dynamic_rgb", "static_depth", "static_opacity", "dynamic_depth", "dynamic_opacity",
             "forward_flow", "backward_flow"),
    "feature": ("static_rgb", "dynamic_rgb", "static_depth", "static_opacity", "dynamic_depth", "dynamic_opacity",
                "dino_feat", "static_dino", "dynamic_dino"),
    "feature_pe": ("static_rgb", "dynamic_rgb", "static_depth", "static_opacity", "dynamic_depth", "dynamic_opacity",
                   "dino_feat", "static_dino", "dynamic_dino", "dino_pe_free", "dino_pe"),
}

DEFAULT_KEYS = ["gt_rgbs", "rgbs", "depths"]
DYNAMIC_KEYS = ["gt_rgbs", "rgbs", "static_rgbs", "dynamic_rgbs", "shadow_reduced_static_rgbs",
                "shadow_only_static_rgbs", "depths", "static_depths", "dynamic_depths", "median_depths",
                "gt_sky_masks", "sky_masks"]
FLOW_KEYS = ["gt_rgbs", "rgbs", "depths", "dynamic_rgbs", "forward_flows", "backward_flows", "opacities_missing"]
FEATURE_KEYS = ["gt_rgbs", "rgbs", "dino_feats", "gt_dino_feats", "dino_feats_pe_free", "dino_pe",
                "static_dino_feats", "dynamic_dino_feats", "dynamic_rgb_on_static_dinos", "dynamic_dino_on_static_rgbs",
                "depths", "static_depths"]

# name: variant, (H, W), cameras, timestamps, keys, separate, save_images, edges
CASES = {
    "static": dict(variant="static", hw=(8, 12), cams=3, ts=2, keys=DEFAULT_KEYS + ["median_depths", "sky_masks"]),
    "dynamic": dict(variant="dynamic", hw=(8, 12), cams=2, ts=2, keys=DYNAMIC_KEYS),
    "flow": dict(variant="flow", hw=(8, 12), cams=2, ts=2, keys=FLOW_KEYS),
    "feature": dict(variant="feature", hw=(8, 12), cams=2, ts=2, keys=FEATURE_KEYS),
    "feature_pe": dict(variant="feature_pe", hw=(8, 12), cams=2, ts=2, keys=FEATURE_KEYS),
    "single": dict(variant="dynamic", hw=(8, 12), cams=3, ts=1, keys=DEFAULT_KEYS + ["dynamic_depths"], png=True),
    "separate": dict(variant="dynamic", hw=(8, 12), cams=2, ts=3,
                     keys=["gt_rgbs", "rgbs", "depths", "dynamic_depths", "gt_sky_masks", "sky_masks",
                           "forward_flows"], separate=True, save_images=True),
    "one_cam": dict(variant="flow", hw=(8, 12), cams=1, ts=3, keys=["rgbs", "forward_flows", "depths"]),
    "odd": dict(variant="dynamic", hw=(17, 29), cams=2, ts=2, keys=["rgbs", "dynamic_depths", "sky_masks"]),
    "edges": dict(variant="dynamic", hw=(8, 12), cams=2, ts=2, keys=DYNAMIC_KEYS, edges=True),
    "edges_no_depth": dict(variant="dynamic", hw=(8, 12), cams=2, ts=2,
                           keys=["gt_rgbs", "rgbs", "static_rgbs", "gt_sky_masks", "sky_masks"], edges=True),
}


def spec(case: str) -> dict:
    s = dict(separate=False, save_images=False, png=False, edges=False)
    s.update(CASES[case])
    return s


def save_path(case: str) -> str:
    return f"videos/{case}.png" if spec(case)["png"] else f"videos/{case}.mp4"


def n_images(case: str) -> int:
    s = spec(case)
    return s["cams"] * s["ts"]


def turbo_table() -> np.ndarray:
    """[256, 4] float64 RGBA in [0, 1], alpha 1."""
    g = np.random.default_rng(2024)
    rgb = g.random((256, 3))
    rgb[::7] = g.integers(0, 256, (len(rgb[::7]), 3)) / 255.0     # k / 255: 255 * x lands just below k for some k
    rgb[0], rgb[255] = [0.1882, 0.0706, 0.2314], [0.4784, 0.0157, 0.0078]
    return np.concatenate([rgb, np.ones((256, 1))], axis=1)


def turbo_lut() -> np.ndarray:
    """The table as the package takes it: trunc(255 * colour) in float64, [256, 3] uint8."""
    return (255 * np.clip(turbo_table()[:, :3], 0, 1)).astype(np.uint8)


def near_steps() -> np.ndarray:
    """float32 values within 3 ulps of every k / 255 in [0, 1]: where a float32 and a float64 ``255 * x`` would
    truncate apart if any value could (no float32 in [0, 1] does: checked over all of them)."""
    out = []
    for k in range(1, 256):
        x = np.float32(k / 255.0)
        lo, hi = x, x
        out.append(x)
        for _ in range(3):
            lo, hi = np.nextafter(lo, np.float32(0)), np.nextafter(hi, np.float32(2))
            out += [lo, hi]
    v = np.array(out, np.float32)
    return v[(v >= 0) & (v <= 1)]


def depth_v(d, op):
    """The reference's v of visualize_depth (numpy 2: float32 curve, float64 from there)."""
    with np.errstate(all="ignore"):
        curve = -np.log(np.asarray(d, np.float32) + 1e-6)
        lo, hi = -np.log(DEPTH_LO + 1e-6), -np.log(DEPTH_HI + 1e-6)
        v = np.nan_to_num(np.clip((curve - np.minimum(lo, hi)) / np.abs(hi - lo), 0, 1))
        return v * np.asarray(op, np.float32)


def firm_tile(d, op):
    """False where v * 256 lies within MARGIN of a bin edge.  Near 0 and 256 both neighbours give the same entry
    (under is the first colour, over the last), so only the interior edges 1..255 count."""
    with np.errstate(all="ignore"):
        s = depth_v(d, op) * 256
        k = np.round(s)
        return ~((np.abs(s - k) <= MARGIN) & (k >= 1) & (k <= 255))


class Model:
    """The attributes ``render`` reads of the model: the registered PCA, and ``eval``."""

    def __init__(self, device="cpu"):
        g = torch.Generator().manual_seed(77)
        self.feats_reduction_mat = (torch.randint(-4, 5, (FEAT, 3), generator=g).float() / 8).to(device)
        self.feat_color_min = torch.tensor([-1.0, -0.75, -1.25], device=device)
        self.feat_color_max = torch.tensor([1.0, 1.25, 0.5], device=device)

    def eval(self):
        return self


def _gen(case: str, i: int, salt: int) -> torch.Generator:
    return torch.Generator().manual_seed(1000 * (list(CASES).index(case) + 1) + 10 * i + salt)


def _unit(g, h, w, c):
    """Mostly [0, 1], with a few values just outside."""
    x = torch.rand(h, w, c, generator=g) * 1.02 - 0.01
    return x


def _depth(g, h, w):
    return torch.exp(torch.rand(h, w, 1, generator=g) * (np.log(300.0) - np.log(0.5)) + np.log(0.5))


def _edges(x: torch.Tensor, k: int) -> torch.Tensor:
    """Overwrite the first pixels of x [h, w, c] with edge values (k varies them per product)."""
    vals = torch.tensor([0.0, 1.0, -0.0, 1.0000001, -1e-7, 2.0, -3.0, float("nan"), float("inf"), -float("inf"),
                         0.5, 0.999999])
    vals = torch.cat([vals, torch.from_numpy(near_steps()[::41])])
    flat = x.reshape(-1)
    n = min(len(vals), flat.numel())
    flat[:n] = torch.roll(vals, k)[:n]
    return x


def _depth_edges(d: torch.Tensor, op: torch.Tensor) -> None:
    vals = torch.tensor([DEPTH_LO, float(DEPTH_HI), 0.0, -1e-6, -1.0, float("nan"), float("inf"), 1e-7, 3.999999,
                         120.00001, 1e6, 50.0])
    n = len(vals)
    d.reshape(-1)[:n] = vals
    ops = torch.tensor([1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.0, float("nan"), 1.0000001, -0.5, float("inf")])
    op.reshape(-1)[n:2 * n] = ops
    d.reshape(-1)[n:2 * n] = 10.0


def results(case: str, i: int):
    s = spec(case)
    h, w = s["hw"]
    g = _gen(case, i, 1)
    prods = VARIANTS[s["variant"]]
    r = {"rgb": _unit(g, h, w, 3), "depth": _depth(g, h, w), "opacity": torch.rand(h, w, 1, generator=g)}
    for k in prods:
        if k.endswith("_rgb"):
            r[k] = _unit(g, h, w, 3)
        elif k.endswith("depth"):
            r[k] = _depth(g, h, w)
        elif k.endswith("opacity"):
            r[k] = torch.rand(h, w, 1, generator=g)
        elif k.endswith("_flow"):
            r[k] = torch.randn(h, w, 3, generator=g) * 0.8
        elif k in ("dino_feat", "static_dino", "dynamic_dino"):
            r[k] = torch.randint(-8, 9, (h, w, FEAT), generator=g).float() / 16
        elif k == "dino_pe_free":
            r[k] = torch.randn(h, w, FEAT, generator=g)
        elif k == "dino_pe":
            r[k] = torch.randn(h, w, PE, generator=g)
    if s["edges"]:
        for j, k in enumerate(sorted(r)):
            if r[k].shape[-1] == 3 and k != "forward_flow" and k != "backward_flow":
                _edges(r[k], j)
        _depth_edges(r["depth"], r["opacity"])
        if "dynamic_depth" in r:
            _depth_edges(r["dynamic_depth"], r["dynamic_opacity"])
    return r


def data(case: str, i: int):
    s = spec(case)
    h, w = s["hw"]
    g = _gen(case, i, 2)
    d = {"pixels": torch.rand(h, w, 3, generator=g), "sky_masks": (torch.rand(h, w, generator=g) < 0.3).float(),
         "img_idx": torch.full((h, w), i, dtype=torch.long)}
    if s["variant"].startswith("feature"):
        d["features"] = torch.randint(-8, 9, (h, w, FEAT), generator=g).float() / 16
    return d


class Dataset:
    split = "full"

    def __init__(self, case: str, device="cpu"):
        self.case, self.device = case, device

    def __len__(self):
        return n_images(self.case)

    def __getitem__(self, i):
        return {k: v.to(self.device) for k, v in data(self.case, i).items()}


def fake_render_rays(device="cpu"):
    """A ``render_rays`` returning image i's seeded results (i from the item's ``img_idx``)."""
    def render_rays(radiance_field=None, proposal_estimator=None, proposal_networks=None, data_dict=None, cfg=None,
                    return_decomposition=True, **kw):
        i = int(data_dict["img_idx"].reshape(-1)[0])
        return {k: v.to(device) for k, v in results(radiance_field.case, i).items()}
    return render_rays


def model(case: str, device="cpu"):
    m = Model(device)
    m.case = case
    return m


cfg = types.SimpleNamespace()

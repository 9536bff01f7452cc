"""Torch restatement of the reference's error-map refresh: ``ScenePixelSource.get_render_rays``
(datasets/base/pixel_source.py:733-846), ``update_pixel_error_maps`` (:491-517) and the cache step of the training
loop (train_emernerf.py:889-904), which renders every image through ``render_pixels`` / ``render``
(radiance_fields/video_utils.py:50-103, 104-468).

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.  The GPU tests hold ``PixelRaySampler.get_render_rays``,
``update_pixel_error_maps`` and ``refresh_pixel_error_maps`` to it (tests/test_gpu_errormap.py), and
tools/bench_errormap.py times ``cache_step`` as the reference's path; tests/test_errormap_cpu.py pins
``get_render_rays`` and ``update_pixel_error_maps`` against the reference's own methods
(tests/golden/errormap.npz).  ``source`` is any object with the reference source's attributes; the downscale factor
is an argument instead of the source's ``update_downscale_factor`` / ``reset_downscale_factor`` pair.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch
from torch import Tensor


def _get_rays(x: Tensor, y: Tensor, c2w: Tensor, K: Tensor):
    """get_rays, pixel_source.py:39-76, for one camera ([1, 4, 4], [1, 3, 3])."""
    cam = torch.nn.functional.pad(torch.stack([(x - K[:, 0, 2] + 0.5) / K[:, 0, 0],
                                               (y - K[:, 1, 2] + 0.5) / K[:, 1, 1]], dim=-1), (0, 1), value=1.0)
    d = (cam[:, None, :] * c2w[:, :3, :3]).sum(dim=-1)
    nrm = torch.linalg.norm(d, dim=-1, keepdims=True)
    return torch.broadcast_to(c2w[:, :3, -1], d.shape), d / (nrm + 1e-8), nrm


def get_render_rays(source, img_idx: int, d: Optional[float] = None) -> Dict[str, Tensor]:
    """pixel_source.py:733-846 at downscale d (default: ``source.downscale_factor``)."""
    d = source.downscale_factor if d is None else d
    rgb = source.images[img_idx]
    if d != 1.0:
        rgb = torch.nn.functional.interpolate(rgb.unsqueeze(0).permute(0, 3, 1, 2), scale_factor=d, mode="bicubic",
                                              antialias=True).squeeze(0).permute(1, 2, 0)
        h, w = rgb.shape[:2]
    else:
        h, w = source.HEIGHT, source.WIDTH
    x, y = torch.meshgrid(torch.arange(w), torch.arange(h), indexing="xy")
    x, y = x.flatten().to(source.device), y.flatten().to(source.device)
    out = {}
    K = source.intrinsics[img_idx] * d
    K[2, 2] = 1.0
    o, v, nrm = _get_rays(x, y, source.cam_to_worlds[img_idx][None], K[None])
    out.update(origins=o.reshape(h, w, 3), viewdirs=v.reshape(h, w, 3), direction_norm=nrm.reshape(h, w, 1),
               pixel_coords=torch.stack([y / h, x / w], dim=-1).float().reshape(h, w, 2))
    ts = source.normalized_timestamps
    if ts is not None:
        out["normed_timestamps"] = torch.full((h, w), ts[img_idx], dtype=torch.float32)
    out["img_idx"] = torch.full((h, w), img_idx, dtype=torch.long)
    out["cam_idx"] = torch.full((h, w), source.cam_ids[img_idx], dtype=torch.long)
    out["pixels"] = rgb

    def nearest(m):
        if d == 1.0:
            return m
        return torch.nn.functional.interpolate(m[None, None], scale_factor=d, mode="nearest")[0, 0]

    if source.sky_masks is not None:
        out["sky_masks"] = nearest(source.sky_masks[img_idx])
    if source.dynamic_masks is not None:
        out["dynamic_masks"] = nearest(source.dynamic_masks[img_idx].float())
    if source.features is not None:
        # get_features (:439-468) with downscale = featmap_downscale_factor / d
        sy, sx = (s / d for s in source.featmap_downscale_factor)
        fy, fx = (y * sy).long(), (x * sx).long()
        out["features"] = source.features[img_idx, fy.cpu(), fx.cpu()].reshape(h, w, -1)
    return out


def update_pixel_error_maps(source, render_results) -> None:
    """pixel_source.py:491-517: the error on the host, then the min-max normalisation on the source's device."""
    if source.pixel_error_maps is None:
        return
    gt = torch.from_numpy(np.stack(render_results["gt_rgbs"], axis=0))
    pred = torch.from_numpy(np.stack(render_results["rgbs"], axis=0))
    maps = torch.abs(gt - pred).mean(dim=-1)
    assert maps.shape == source.pixel_error_maps.shape
    if "dynamic_opacities" in render_results and len(render_results["dynamic_opacities"]) > 0:
        dyn = torch.from_numpy(np.stack(render_results["dynamic_opacities"], axis=0))
        maps[dyn > 0.1] *= 5
    maps = maps.to(source.device)
    source.pixel_error_maps = (maps - maps.min()) / (maps.max() - maps.min())
    source.pixel_error_buffered = True


def _numpy(t: Tensor) -> np.ndarray:
    return t.squeeze().cpu().numpy()                    # get_numpy, video_utils.py:44


@torch.no_grad()
def cache_step(source, model, proposal_estimator, proposal_networks, cfg, render_rays, render_rays_of=None) -> None:
    """train_emernerf.py:889-904 with the package's ``render_rays``: ``render_pixels`` over every image at
    ``1 / buffer_downscale`` with ``return_decomposition=True`` and ``compute_metrics=False``, keeping the host copies
    ``render`` makes for the static and dynamic fields (video_utils.py:150-213; no flow, feature or shadow head), then
    ``update_pixel_error_maps``.  ``render_rays_of(i, d)`` replaces ``get_render_rays`` when given."""
    model.eval()                                         # render_pixels, video_utils.py:70-75
    for p in proposal_networks:
        p.eval()
    proposal_estimator.eval()
    d = 1 / source.buffer_downscale
    keys = ("rgbs", "gt_rgbs", "static_rgbs", "dynamic_rgbs", "depths", "opacities", "static_depths",
            "static_opacities", "dynamic_depths", "dynamic_opacities", "median_depths", "sky_masks")
    res = {k: [] for k in keys}
    for i in range(len(source.images)):
        data = get_render_rays(source, i, d) if render_rays_of is None else render_rays_of(i, d)
        for k, v in data.items():                        # :152-154
            data[k] = v.cuda(non_blocking=True)
        out = render_rays(radiance_field=model, proposal_estimator=proposal_estimator,
                          proposal_networks=proposal_networks, data_dict=data, cfg=cfg, return_decomposition=True)
        res["rgbs"].append(_numpy(out["rgb"]))                                         # :158
        res["gt_rgbs"].append(_numpy(data["pixels"]))                                  # :160
        if "static_rgb" in out:
            res["static_rgbs"].append(_numpy(out["static_rgb"]))                        # :162
        if "dynamic_rgb" in out:                                                       # :163-170
            green = (torch.tensor([0.0, 177, 64]) / 255.0).to(out["dynamic_rgb"].device)
            dy = out["dynamic_rgb"] * out["dynamic_opacity"] + green * (1 - out["dynamic_opacity"])
            res["dynamic_rgbs"].append(_numpy(dy))
        res["depths"].append(_numpy(out["depth"]))                                     # :185-186
        res["opacities"].append(_numpy(out["opacity"]))                                # :188
        if "static_depth" in out:                                                      # :189-191
            res["static_depths"].append(_numpy(out["static_depth"]))
            res["static_opacities"].append(_numpy(out["static_opacity"]))
        if "dynamic_depth" in out:                                                     # :192-194
            res["dynamic_depths"].append(_numpy(out["dynamic_depth"]))
            res["dynamic_opacities"].append(_numpy(out["dynamic_opacity"]))
        elif "median_depth" in out:                                                    # :195-196
            res["median_depths"].append(_numpy(out["median_depth"]))
        if "sky_masks" in data:                                                        # :198-199
            res["sky_masks"].append(_numpy(data["sky_masks"]))
    update_pixel_error_maps(source, res)

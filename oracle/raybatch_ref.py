"""Torch restatement of the reference's training-batch samplers: ``ScenePixelSource.get_train_rays`` with its
uniform and error-map samplers (datasets/base/pixel_source.py:564-731) and ``SceneLidarSource.get_train_rays``
(datasets/base/lidar_source.py:223-308).

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.  The GPU tests run it on the device as the reference's torch path
(tests/test_gpu_raybatch.py), and tools/bench_raybatch.py times it.  It makes the reference's generator calls in the
reference's order, including ``torch.multinomial`` itself, and the reference's tensor ops, so on one device it gives
the reference's batch and leaves the generator where the reference leaves it; tests/test_raybatch_cpu.py pins it
against the reference's own methods (tests/golden/raybatch.npz).  ``source`` is any object with the reference
source's attributes.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
from torch import Tensor


def _as_index_tensor(candidate_indices, n_images: int, device) -> Tensor:
    if candidate_indices is None:
        return torch.arange(n_images).to(device)
    if isinstance(candidate_indices, Tensor):
        return candidate_indices
    return torch.tensor(candidate_indices).to(device)


def _uniform(source, n: int, candidate_indices):
    cand = _as_index_tensor(candidate_indices, len(source.images), source.device)
    pick = torch.randint(0, len(cand), size=(n,), device=source.device)
    x = torch.randint(0, source.WIDTH, size=(n,), device=source.device)
    y = torch.randint(0, source.HEIGHT, size=(n,), device=source.device)
    return cand[pick], y.long(), x.long()


def _importance(source, n: int, candidate_indices):
    cand = _as_index_tensor(candidate_indices, len(source.images), source.device)
    h = source.HEIGHT // source.buffer_downscale
    w = source.WIDTH // source.buffer_downscale
    j = torch.multinomial(source.pixel_error_maps[cand].reshape(-1), n, replacement=False)
    plane = h * w
    img = cand[j // plane]
    row, col = (j % plane) // w, j % w
    y = (row * source.buffer_downscale).long()
    x = (col * source.buffer_downscale).long()
    dev = source.images.device
    y = y + torch.randint(0, source.buffer_downscale, (n,), device=dev)
    x = x + torch.randint(0, source.buffer_downscale, (n,), device=dev)
    return img, y.clamp(0, source.HEIGHT - 1), x.clamp(0, source.WIDTH - 1)


def _rays(x: Tensor, y: Tensor, c2w: Tensor, K: Tensor):
    cam = torch.stack([(x - K[:, 0, 2] + 0.5) / K[:, 0, 0], (y - K[:, 1, 2] + 0.5) / K[:, 1, 1],
                       torch.ones_like(K[:, 0, 0])], dim=-1)
    d = (cam[:, None, :] * c2w[:, :3, :3]).sum(dim=-1)
    nrm = torch.linalg.norm(d, dim=-1, keepdims=True)
    return torch.broadcast_to(c2w[:, :3, 3], d.shape), d / (nrm + 1e-8), nrm


@torch.no_grad()
def pixel_train_rays(source, num_rays: int, candidate_indices=None) -> Dict[str, Tensor]:
    if source.buffer_ratio > 0 and source.pixel_error_buffered:
        n_i = int(num_rays * source.buffer_ratio)
        parts = [_uniform(source, num_rays - n_i, candidate_indices), _importance(source, n_i, candidate_indices)]
        img, y, x = (torch.cat([a[i] for a in parts]) for i in range(3))
    else:
        img, y, x = _uniform(source, num_rays, candidate_indices)
    out: Dict[str, Optional[Tensor]] = {}
    o, d, nrm = _rays(x, y, source.cam_to_worlds[img], source.intrinsics[img])
    out.update(origins=o, viewdirs=d, direction_norms=nrm,
               pixel_coords=torch.stack([y / source.HEIGHT, x / source.WIDTH], dim=-1))
    ts = source.normalized_timestamps
    out["normed_timestamps"] = None if ts is None else ts[img]
    out["img_idx"] = torch.ones_like(x) * img
    out["cam_idx"] = source.cam_ids[img]
    out["pixels"] = None if source.images is None else source.images[img, y, x]
    out["sky_masks"] = None if source.sky_masks is None else source.sky_masks[img, y, x]
    out["dynamic_masks"] = None if source.dynamic_masks is None else source.dynamic_masks[img, y, x].float()
    if source.features is not None:
        s = source.featmap_downscale_factor
        sy, sx = (s, s) if isinstance(s, float) else s
        fy, fx = (y * sy).long(), (x * sx).long()
        out["features"] = source.features[img, fy.cpu(), fx.cpu()]
    return {k: v for k, v in out.items() if v is not None}


class LidarCache:
    """The reference keeps the points of the last candidate set on the source; this keeps them here."""

    def __init__(self):
        self.indices, self.arrays = None, None


@torch.no_grad()
def lidar_train_rays(source, num_rays: int, candidate_indices, cache: LidarCache) -> Dict[str, Tensor]:
    if candidate_indices is None:
        idx = torch.randint(0, len(source.origins), size=(num_rays,), device=source.device)
        arrays = cache.arrays
    else:
        cand = candidate_indices if isinstance(candidate_indices, Tensor) else \
            torch.tensor(candidate_indices, device=source.device)
        if cache.indices is None or not torch.equal(cand, cache.indices):
            keep = torch.zeros_like(source.timesteps, dtype=torch.bool)
            for c in cand:
                keep |= source.timesteps == c
            cache.indices = cand
            cache.arrays = tuple(a[keep] for a in (source.origins, source.directions, source.ranges,
                                                   source.normalized_timestamps))
        arrays = cache.arrays
        idx = torch.randint(0, len(arrays[0]), size=(num_rays,), device=source.device)
    o, d, r, t = (a[idx] for a in arrays)
    return {"lidar_origins": o, "lidar_viewdirs": d, "lidar_ranges": r, "lidar_normed_timestamps": t}

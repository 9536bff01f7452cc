"""Seeded pixel and lidar sources for the training-batch samplers, shared by make_golden_raybatch.py (which runs the
reference's own ``get_train_rays`` on them) and the tests (which run the samplers and the oracle on them).

A source is any object carrying the reference source's attributes; ``fill_pixel`` / ``fill_lidar`` set them on an
instance of the reference's class as on the stand-ins below, from a seeded generator that leaves the default one
alone.  Every array is small: 12 images of 64 x 96, error maps of 4 x 6 (buffer_downscale 16)."""
from __future__ import annotations

import types

import torch

N_IMAGES, HEIGHT, WIDTH, DOWNSCALE = 12, 64, 96, 16
FEAT_H, FEAT_W, FEAT_C = 7, 10, 8
N_POINTS, N_SCANS = 500, 10

# name -> (ratio, buffered, with optional sources, candidates, rays per call, calls, seed)
PIXEL_CASES = {
    "full": (0.25, True, True, [0, 2, 3, 5, 7, 8, 11], 96, 2, 1),
    "bare": (0.25, True, False, None, 101, 2, 2),
    "uniform": (0.0, True, True, "tensor", 96, 2, 3),
    "all_importance": (1.0, True, True, [1, 4, 6, 9, 10], 60, 2, 4),
    "unbuffered": (0.25, False, True, [0, 1, 2], 50, 1, 5),
}
# name -> (candidate sets of successive calls, rays per call, seed)
LIDAR_CASES = {
    "lists": ([[1, 3, 4, 8], [1, 3, 4, 8], [0, 2, 9]], 64, 6),
    "tensor": ([[0, 1], "tensor", "tensor"], 33, 7),
}
LIDAR_TENSOR_CANDIDATES = [2, 5, 6, 7]


class PixelSource:
    """The attributes and properties of ScenePixelSource that get_train_rays reads."""
    HEIGHT = property(lambda self: self.data_cfg.load_size[0])
    WIDTH = property(lambda self: self.data_cfg.load_size[1])
    buffer_downscale = property(lambda self: self.data_cfg.sampler.buffer_downscale)
    buffer_ratio = property(lambda self: self.data_cfg.sampler.buffer_ratio)
    normalized_timestamps = property(lambda self: self._normalized_timestamps)


class LidarSource:
    """The attributes and properties of SceneLidarSource that get_train_rays reads."""
    timesteps = property(lambda self: self._timesteps)
    normalized_timestamps = property(lambda self: self._normalized_timestamps)


def fill_pixel(src, case: str):
    ratio, buffered, optional, _, _, _, seed = PIXEL_CASES[case]
    g = torch.Generator().manual_seed(100 + seed)
    n, h, w = N_IMAGES, HEIGHT, WIDTH
    src.device = torch.device("cpu")
    src.data_cfg = types.SimpleNamespace(load_size=[h, w],
                                         sampler=types.SimpleNamespace(buffer_downscale=DOWNSCALE, buffer_ratio=ratio))
    src.images = torch.rand(n, h, w, 3, generator=g)
    src.cam_ids = torch.arange(n) % 3
    c2w = torch.eye(4).repeat(n, 1, 1)
    c2w[:, :3, :3] = torch.linalg.qr(torch.randn(n, 3, 3, generator=g))[0]
    c2w[:, :3, 3] = torch.randn(n, 3, generator=g) * 10
    src.cam_to_worlds = c2w
    K = torch.zeros(n, 3, 3)
    K[:, 0, 0] = 80 + 10 * torch.rand(n, generator=g)
    K[:, 1, 1] = 80 + 10 * torch.rand(n, generator=g)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = w / 2 + torch.rand(n, generator=g), h / 2 + torch.rand(n, generator=g), 1.0
    src.intrinsics = K
    maps = torch.rand(n, h // DOWNSCALE, w // DOWNSCALE, generator=g)
    maps[maps < 0.1] = 0.0                                  # some weights exactly zero
    src.pixel_error_maps = maps
    src.pixel_error_buffered = buffered
    if optional:
        src.sky_masks = (torch.rand(n, h, w, generator=g) > 0.7).float()
        src.dynamic_masks = (torch.rand(n, h, w, generator=g) > 0.8).float()
        src.features = torch.rand(n, FEAT_H, FEAT_W, FEAT_C, generator=g)
        src.featmap_downscale_factor = (FEAT_H / h, FEAT_W / w)
        src._normalized_timestamps = torch.linspace(0, 1, n)
    else:
        src.sky_masks = src.dynamic_masks = src.features = src._normalized_timestamps = None
        src.featmap_downscale_factor = None
    return src


def pixel_candidates(case: str, device="cpu"):
    cand = PIXEL_CASES[case][3]
    if cand == "tensor":
        return torch.tensor([0, 4, 5, 6, 11], device=device)
    return cand


def fill_lidar(src, case: str):
    seed = LIDAR_CASES[case][2]
    g = torch.Generator().manual_seed(200 + seed)
    src.device = torch.device("cpu")
    src.origins = torch.randn(N_POINTS, 3, generator=g)
    src.directions = torch.nn.functional.normalize(torch.randn(N_POINTS, 3, generator=g), dim=-1)
    src.ranges = torch.rand(N_POINTS, 1, generator=g) * 50
    src._timesteps = torch.sort(torch.randint(0, N_SCANS, (N_POINTS,), generator=g)).values
    src._normalized_timestamps = src._timesteps.float() / (N_SCANS - 1)
    return src


def lidar_candidates(case: str, call: int, device="cpu"):
    c = LIDAR_CASES[case][0][call]
    return torch.tensor(LIDAR_TENSOR_CANDIDATES, device=device) if c == "tensor" else c


def to_device(src, device):
    """Move every tensor attribute (the reference's ``to()``)."""
    for k, v in list(vars(src).items()):
        if isinstance(v, torch.Tensor):
            setattr(src, k, v.to(device))
    src.device = torch.device(device)
    return src

"""Seeded sources and cases for the camera trajectories, shared by make_golden_trajectory.py (which runs the
reference's own ``get_rays`` on the interpolated poses) and the tests.

"main" is 3 cameras x 5 timesteps of 24 x 40 pixels in the reference's timestep-major order (image t * 3 + c), with
sky masks and timestamps.  Its poses hold the segments the interpolation treats apart:
  - camera 0, timesteps 1 -> 2: the same pose twice (quaternion dot 1: the normalised lerp);
  - camera 1, timesteps 2 -> 3: rotations of 119 and 121 degrees about -x, whose quaternions come out of Shepperd's
    branches nearly opposite (dot ~ -0.999: the sign flip);
  - camera 2, timesteps 0 -> 1: a 170 degree yaw about the world's z axis (the shorter arc is 170, not 190 degrees).
"single" is one timestep of the same cameras, without sky masks or timestamps."""
from __future__ import annotations

import types

import numpy as np
import torch

import errormap_cases as ec

N_CAMS, N_TIMESTEPS, HEIGHT, WIDTH = 3, 5, 24, 40
OFFSET = (0.4, -0.3, 1.2)
ZERO = (0.0, 0.0, 0.0)
# name -> (source, downscale, frames per keyframe, offset)
CASES = {
    "m1": ("main", 1.0, 1, ZERO),
    "m3_half": ("main", 0.5, 3, ZERO),
    "m3_half_offset": ("main", 0.5, 3, OFFSET),
    "m4": ("main", 1.0, 4, ZERO),
    "m4_offset": ("main", 1.0, 4, OFFSET),
    "single": ("single", 1.0, 3, OFFSET),
}
# the special segments of "main": (camera, first timestep)
NLERP_SEGMENT, FLIP_SEGMENT, YAW_SEGMENT = (0, 1), (1, 2), (2, 0)


def rot(axis, deg: float) -> np.ndarray:
    """Rotation [3, 3] (fp64) by deg degrees about axis (Rodrigues)."""
    k = np.asarray(axis, dtype=np.float64)
    k = k / np.linalg.norm(k)
    t = np.deg2rad(deg)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(t) * Kx + (1 - np.cos(t)) * Kx @ Kx


X, Z = (1, 0, 0), (0, 0, 1)
FORWARD = rot(X, -90)                                  # an OpenCV camera looking along the world's y axis


def rotations():
    """[camera][timestep] -> rotation [3, 3]."""
    base = rot((0.2, 1.0, 0.1), 30)
    cam0 = [base, rot(Z, 10) @ base, rot(Z, 10) @ base, rot(Z, 25) @ rot(X, 5) @ base, rot(Z, 40) @ base]
    cam1 = [rot(X, -80), rot(X, -100), rot(X, -119), rot(X, -121), rot((1.0, 0.2, 0.1), -140)]
    cam2 = [rot(Z, yaw) @ FORWARD for yaw in (0, 170, 200, 230, 235)]
    return [cam0, cam1, cam2]


def fill(src, name: str, d: float = 1.0):
    """Fill a source object (the reference's class or errormap_cases' stand-in) with the "main" or "single" tables."""
    n_t = N_TIMESTEPS if name == "main" else 1
    n = n_t * N_CAMS
    g = torch.Generator().manual_seed(400 + n_t)
    src.device = torch.device("cpu")
    src.data_cfg = types.SimpleNamespace(load_size=[HEIGHT, WIDTH], sampler=types.SimpleNamespace(
        buffer_downscale=4, buffer_ratio=0.0))
    src.images = torch.rand(n, HEIGHT, WIDTH, 3, generator=g)
    src.cam_ids = torch.arange(n) % N_CAMS
    rots = rotations()
    c2w = torch.eye(4).repeat(n, 1, 1)
    K = torch.zeros(n, 3, 3)
    for t in range(n_t):
        for c in range(N_CAMS):
            i = t * N_CAMS + c
            c2w[i, :3, :3] = torch.from_numpy(rots[c][t])
            c2w[i, :3, 3] = torch.tensor([2.0 * t + 0.5 * c, 0.3 * t - 0.2 * c, 1.5 + 0.1 * t])
            K[i, 0, 0], K[i, 1, 1] = 30.0 + c + 0.5 * t, 31.0 + 0.25 * c
            K[i, 0, 2], K[i, 1, 2], K[i, 2, 2] = WIDTH / 2 + 0.25 * c, HEIGHT / 2 - 0.25 * t, 1.0
    src.cam_to_worlds, src.intrinsics = c2w, K
    src.pixel_error_maps, src.pixel_error_buffered = None, False
    src.dynamic_masks = src.features = src.featmap_downscale_factor = None
    if name == "main":
        src.sky_masks = (torch.rand(n, HEIGHT, WIDTH, generator=g) > 0.7).float()
        src._normalized_timestamps = (torch.arange(n) // N_CAMS).float() / (N_TIMESTEPS - 1)
    else:
        src.sky_masks = src._normalized_timestamps = None
    src._downscale_factor = d
    return src


def source(name: str, d: float = 1.0):
    return fill(ec.PixelSource(), name, d)


def segment(name: str, m: int, k: int):
    """(image a, image b, i, camera) of item k of a trajectory over every camera of source ``name``: the layout
    ``CameraTrajectory`` promises, restated."""
    n_t = N_TIMESTEPS if name == "main" else 1
    frame, c = divmod(k, N_CAMS)
    seg, i = divmod(frame, m)
    if seg == n_t - 1:
        return seg * N_CAMS + c, seg * N_CAMS + c, 0, c
    return seg * N_CAMS + c, (seg + 1) * N_CAMS + c, i, c


def num_items(name: str, m: int) -> int:
    n_t = N_TIMESTEPS if name == "main" else 1
    return ((n_t - 1) * m + 1) * N_CAMS


def golden_items(case: str):
    """The items trajectory.npz keeps: with m > 1 the frames inside each camera's special segment, with m = 1 the
    middle timestep, and every item of "single"."""
    name, _, m, _ = CASES[case]
    items = range(num_items(name, m))
    if name == "single":
        return list(items)
    if m == 1:
        return [k for k in items if k // N_CAMS == N_TIMESTEPS // 2]
    special = dict((NLERP_SEGMENT, FLIP_SEGMENT, YAW_SEGMENT))
    return [k for k in items if divmod(k // N_CAMS, m)[0] == special[k % N_CAMS] and (k // N_CAMS) % m]

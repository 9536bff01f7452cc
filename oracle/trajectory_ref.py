"""Numpy / torch restatement of ``emer_trajectory_rays`` (csrc/errormap.cu): the render rays of a camera between two
keyframe images, for ``raygen.CameraTrajectory``.

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.  The pose is interpolated in fp64 numpy (slerp of the rotations as
unit quaternions with the shorter-arc sign flip, a normalised lerp above a dot product of 0.9995, lerp of the origins,
then the offset along the frame's axes), rounded to fp32, and the rays are the reference's ``get_rays``
(datasets/base/pixel_source.py:39-76, as restated in errormap_ref) on that pose with keyframe a's intrinsics scaled as
``get_render_rays`` scales them.  tests/golden/make_golden_trajectory.py runs the reference's own ``get_rays`` on the
same poses; tests/test_trajectory_cpu.py holds this module to that file and tests/test_gpu_trajectory.py holds the
kernel to this module.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import numpy as np
import torch
from torch import Tensor

from .errormap_ref import _get_rays

NLERP_DOT = 0.9995


def rotation_to_quat(R: np.ndarray) -> np.ndarray:
    """Unit quaternion (w, x, y, z) of a rotation [3, 3] by Shepperd's branches: w when the trace is positive,
    otherwise the largest diagonal entry's component, which comes out positive."""
    R = np.asarray(R, dtype=np.float64)
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    if tr > 0:
        s = 2.0 * np.sqrt(1.0 + tr)
        q = [0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = 2.0 * np.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2])
        q = [(R[2, 1] - R[1, 2]) / s, 0.25 * s, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s]
    elif R[1, 1] > R[2, 2]:
        s = 2.0 * np.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2])
        q = [(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, 0.25 * s, (R[1, 2] + R[2, 1]) / s]
    else:
        s = 2.0 * np.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1])
        q = [(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, 0.25 * s]
    q = np.array(q)
    return q / np.linalg.norm(q)


def quat_to_rotation(q: np.ndarray) -> np.ndarray:
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def quat_dot(A: np.ndarray, B: np.ndarray) -> float:
    """q_a . q_b of two c2w matrices' rotations, before the sign flip."""
    return float(rotation_to_quat(A[:3, :3]) @ rotation_to_quat(B[:3, :3]))


def slerp(qa: np.ndarray, qb: np.ndarray, f: float) -> np.ndarray:
    dot = float(qa @ qb)
    if dot < 0:
        qb, dot = -qb, -dot
    if dot > NLERP_DOT:
        q = qa + f * (qb - qa)
        return q / np.linalg.norm(q)
    th0 = np.arccos(dot)
    th = th0 * f
    return (np.sin(th0 - th) * qa + np.sin(th) * qb) / np.sin(th0)


def frame_pose(A, B, i: int, m: int, offset: Sequence[float] = (0.0, 0.0, 0.0)) -> np.ndarray:
    """The frame's c2w [4, 4] in fp32 between c2w matrices A and B (fp32) at fraction i / m: A's rotation and origin
    when i == 0, otherwise the fp64 slerp and lerp; then origin + R offset in fp64, rounded."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    if i == 0:
        R, o = A[:3, :3], A[:3, 3]
    else:
        f = i / m
        R = quat_to_rotation(slerp(rotation_to_quat(A[:3, :3]), rotation_to_quat(B[:3, :3]), f))
        o = A[:3, 3] + f * (B[:3, 3] - A[:3, 3])
    out = np.eye(4, dtype=np.float32)
    out[:3, :3] = R
    out[:3, 3] = o + R @ np.asarray(offset, dtype=np.float64)
    return out


def frame_time(ta: float, tb: float, i: int, m: int) -> np.float32:
    """t_a + (i / m)(t_b - t_a), every operation in fp32."""
    f32 = np.float32
    return f32(ta) + (f32(i) / f32(m)) * (f32(tb) - f32(ta))


def frame_rays(source, a: int, b: int, i: int, m: int, cam: int, offset=(0.0, 0.0, 0.0), d: Optional[float] = None,
               get_rays=None) -> Dict[str, Tensor]:
    """The frame's rays on the source's device with ``get_render_rays``' keys, order, shapes and dtypes (without the
    ground-truth ones); ``get_rays`` defaults to the restatement of the reference's."""
    get_rays = _get_rays if get_rays is None else get_rays
    d = source.downscale_factor if d is None else d
    dev = source.cam_to_worlds.device
    h, w = source.HEIGHT, source.WIDTH
    if d != 1.0:                                         # the size of get_render_rays' resized image
        img = source.images[a][None].permute(0, 3, 1, 2)
        h, w = torch.nn.functional.interpolate(img, scale_factor=d, mode="bicubic", antialias=True).shape[2:]
    c2w = source.cam_to_worlds.cpu().numpy()
    pose = torch.from_numpy(frame_pose(c2w[a], c2w[b], i, m, offset)).to(dev)
    K = source.intrinsics[a] * d
    K[2, 2] = 1.0
    x, y = torch.meshgrid(torch.arange(w), torch.arange(h), indexing="xy")
    x, y = x.flatten().to(dev), y.flatten().to(dev)
    o, v, nrm = get_rays(x, y, pose[None], K[None])
    out = dict(origins=o.reshape(h, w, 3), viewdirs=v.reshape(h, w, 3), direction_norm=nrm.reshape(h, w, 1),
               pixel_coords=torch.stack([y / h, x / w], dim=-1).float().reshape(h, w, 2))
    ts = source.normalized_timestamps
    if ts is not None:
        t = ts.cpu().numpy()
        out["normed_timestamps"] = torch.full((h, w), float(frame_time(t[a], t[b], i, m)), dtype=torch.float32,
                                              device=dev)
    out["img_idx"] = torch.full((h, w), a if 2 * i <= m else b, dtype=torch.long, device=dev)
    out["cam_idx"] = torch.full((h, w), cam, dtype=torch.long, device=dev)
    if source.sky_masks is not None:
        out["sky_masks"] = torch.zeros((h, w), dtype=torch.float32, device=dev)
    return out

"""CPU emulator of emer_trajectory_rays (csrc/errormap.cu) -- TEST INFRASTRUCTURE ONLY.

A host restatement through the same raw pointers and sizes ``raygen.CameraTrajectory`` hands to the library: the pose
is oracle/trajectory_ref.py's (fp64, rounded to fp32), the ray ``cabi_emulator.emer_gen_rays``' with keyframe a's
intrinsics scaled by d, as errormap_emulator computes ``get_render_rays``.  ``install(monkeypatch)`` installs
``errormap_emulator`` (and through it the rest of the ABI) and routes this entry point here.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

import cabi_emulator
import errormap_emulator
from cabi_emulator import _require, _vec, _view, emer_gen_rays
from oracle import trajectory_ref

_I64 = dict(ctype=ctypes.c_int64, dtype=np.int64)


def emer_trajectory_rays(in_ref, out_ref, stream):
    a, o = in_ref._obj, out_ref._obj
    h, w, N = a.h, a.w, a.n_images
    i, m = a.frac_num, a.frac_den
    _require(h > 0 and w > 0, "emer_trajectory_rays: empty image")
    _require(0 <= a.image_a < N and 0 <= a.image_b < N, "emer_trajectory_rays: keyframes out of range")
    _require(0 <= i < m, "emer_trajectory_rays: fraction not in [0, 1)")
    _require(all(np.isfinite(list(a.offset))), "emer_trajectory_rays: non-finite offset")
    _require(a.c2w and a.intrinsics and o.origins and o.viewdirs and o.norms and o.pixel_coords and o.img_idx and
             o.cam_idx, "emer_trajectory_rays: NULL pointer")
    _require(not o.timestamps or a.timestamps, "emer_trajectory_rays: timestamps without a source")
    c2w = _view(a.c2w, N, 16).view(N, 4, 4).numpy()
    pose = torch.from_numpy(trajectory_ref.frame_pose(c2w[a.image_a], c2w[a.image_b], i, m, list(a.offset)))
    K = (_view(a.intrinsics, N, 9)[a.image_a] * a.downscale).contiguous()
    n = h * w
    y = torch.arange(h).repeat_interleave(w).float()
    x = torch.arange(w).repeat(h).float()
    emer_gen_rays(None, x.data_ptr(), y.data_ptr(), pose.data_ptr(), K.data_ptr(), 0, None, h, w, o.origins,
                  o.viewdirs, o.norms, o.pixel_coords, None, n, stream)
    if o.timestamps:
        ts = _vec(a.timestamps, N).numpy()
        _vec(o.timestamps, n).fill_(float(trajectory_ref.frame_time(ts[a.image_a], ts[a.image_b], i, m)))
    _vec(o.img_idx, n, **_I64).fill_(a.image_a if 2 * i <= m else a.image_b)
    _vec(o.cam_idx, n, **_I64).fill_(a.cam_id)
    if o.sky_masks:
        _vec(o.sky_masks, n).zero_()


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: this kernel here, everything else in errormap_emulator."""
    if name != "emer_trajectory_rays":
        return errormap_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    emer_trajectory_rays(*args)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib

    errormap_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)

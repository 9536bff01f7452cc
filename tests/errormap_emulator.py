"""CPU emulator of the render-ray and error-map entry points of the C ABI (emer_image_rays, emer_error_map,
emer_error_map_normalize; csrc/errormap.cu) -- TEST INFRASTRUCTURE ONLY.

Host restatements through the same raw pointers and sizes the product hands to the library.  ``install(monkeypatch)``
installs ``raybatch_emulator`` (and through it the rest of the ABI) and routes these three entry points here, so
``PixelRaySampler.get_render_rays`` and ``update_pixel_error_maps`` run on CPU tensors in the ``-m "not gpu"`` suite.
As in raybatch_emulator, the ray is ``cabi_emulator.emer_gen_rays``' and the pixel coordinates are ``y / h`` as torch
divides on the host; the kernel computes ``y * (1 / h)``, as torch does on CUDA.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

import cabi_emulator
import raybatch_emulator
from cabi_emulator import _addr, _require, _vec, _view, emer_gen_rays

_I64 = dict(ctype=ctypes.c_int64, dtype=np.int64)


def _words(workspace):
    return np.ctypeslib.as_array((ctypes.c_uint32 * 4).from_address(_addr(workspace)))


def emer_image_rays(in_ref, out_ref, stream):
    a, o = in_ref._obj, out_ref._obj
    n_img, h, w, H, W = a.n_images, a.h, a.w, a.height, a.width
    n = n_img * h * w
    if n == 0:
        return
    _require(a.c2w and a.intrinsics and o.origins and o.viewdirs and o.norms and o.pixel_coords and o.img_idx,
             "emer_image_rays: NULL pointer")
    _require(not o.features or 1 <= a.feat_c <= 256, "emer_image_rays: features need 1 <= C <= 256")
    first, last = a.first_image, a.first_image + n_img
    k = torch.arange(n_img).repeat_interleave(h * w)
    y = torch.arange(h).repeat_interleave(w).repeat(n_img)
    x = torch.arange(w).repeat(h * n_img)
    img = first + k
    C = _view(a.c2w, last, 16)[first:last].contiguous()
    K = (_view(a.intrinsics, last, 9)[first:last] * a.downscale).contiguous()
    xf, yf = x.float(), y.float()
    emer_gen_rays(k.data_ptr(), xf.data_ptr(), yf.data_ptr(), C.data_ptr(), K.data_ptr(), 0, None, h, w, o.origins,
                  o.viewdirs, o.norms, o.pixel_coords, None, n, stream)
    _vec(o.img_idx, n, **_I64).copy_(img)
    if o.cam_idx:
        _vec(o.cam_idx, n, **_I64).copy_(_vec(a.cam_ids, last, **_I64)[img])
    if o.timestamps:
        _vec(o.timestamps, n).copy_(_vec(a.timestamps, last)[img])
    sy = torch.floor(yf * a.mask_scale_y).long().clamp(max=H - 1)
    sx = torch.floor(xf * a.mask_scale_x).long().clamp(max=W - 1)
    for src, dst in ((a.sky_masks, o.sky_masks), (a.dynamic_masks, o.dynamic_masks)):
        if dst:
            _vec(dst, n).copy_(_vec(src, last * H * W).view(last, H, W)[img, sy, sx])
    if o.features:
        fh, fw, fc = a.feat_h, a.feat_w, a.feat_c
        fy = (yf * a.feat_scale_y).long().clamp(max=fh - 1)
        fx = (xf * a.feat_scale_x).long().clamp(max=fw - 1)
        _view(o.features, n, fc).copy_(_view(a.features, last * fh * fw, fc).view(last, fh, fw, fc)[img, fy, fx])


def emer_error_map(gt, rgb, opacity, n, out, workspace, stream):
    _require(n >= 0, "emer_error_map: negative pixel count")
    if n == 0:
        return
    _require(_addr(gt) and _addr(rgb) and _addr(out) and _addr(workspace), "emer_error_map: NULL pointer")
    e = (_view(gt, n, 3) - _view(rgb, n, 3)).abs()
    e = ((e[:, 0] + e[:, 1]) + e[:, 2]) / 3
    if _addr(opacity):
        e = torch.where(_vec(opacity, n) > 0.1, e * 5, e)
    _vec(out, n).copy_(e)
    bits = e.numpy().view(np.uint32)
    ws = _words(workspace)
    ws[1] = max(ws[1], bits.max())
    ws[0] = max(ws[0], (~bits).max())


def emer_error_map_normalize(out, n, workspace, stream):
    _require(_addr(out) and _addr(workspace), "emer_error_map_normalize: NULL pointer")
    ws = _words(workspace)
    lo = torch.from_numpy(np.array([~ws[0]], dtype=np.uint32).view(np.float32))[0]
    hi = torch.from_numpy(np.array([ws[1]], dtype=np.uint32).view(np.float32))[0]
    m = _vec(out, n)
    m.copy_((m - lo) / (hi - lo))
    ws[:] = 0


ENTRY_POINTS = ("emer_image_rays", "emer_error_map", "emer_error_map_normalize")


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: these kernels here, everything else in raybatch_emulator."""
    if name not in ENTRY_POINTS:
        return raybatch_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib, raygen

    raybatch_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(raygen, "_MAP_WS", {})

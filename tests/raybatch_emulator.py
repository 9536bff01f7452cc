"""CPU emulator of the training-batch entry points of the C ABI (emer_topk_ratio, emer_pixel_batch;
csrc/raybatch.cu) -- TEST INFRASTRUCTURE ONLY.

Host restatements through the same raw pointers and sizes the product hands to the library.  ``install(monkeypatch)``
installs ``cabi_emulator`` (the rest of the ABI) and routes these two entry points here, so
``emernerf_b200.raygen.PixelRaySampler`` runs on CPU tensors, with the CPU generator, in the ``-m "not gpu"`` suite.
The ray of each pixel is ``cabi_emulator.emer_gen_rays``'s, and the pixel coordinates are ``y / H`` as torch divides
on the host; the kernel computes ``y * (1 / H)``, as torch does on CUDA.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

import cabi_emulator
from cabi_emulator import _addr, _require, _vec, _view, emer_gen_rays

TOPK_MAX_K = 16384                  # EMER_TOPK_MAX_K
_I64 = dict(ctype=ctypes.c_int64, dtype=np.int64)


def emer_topk_ratio(p, plane, cand, n_cand, q, k, out_idx, workspace, stream):
    _require(_addr(p) and _addr(cand) and _addr(q) and _addr(out_idx) and _addr(workspace),
             "emer_topk_ratio: NULL pointer")
    _require(plane > 0 and n_cand > 0, "emer_topk_ratio: empty map")
    m = plane * n_cand
    _require(m < 2 ** 31, "emer_topk_ratio: too many keys")
    _require(1 <= k <= min(TOPK_MAX_K, m), "emer_topk_ratio: k outside [1, min(EMER_TOPK_MAX_K, M)]")
    c = _vec(cand, n_cand, **_I64)
    keys = _view(p, int(c.max()) + 1, plane)[c].reshape(-1) / _vec(q, m)
    # by descending key, then ascending index (a stable sort keeps equal keys in index order)
    _vec(out_idx, k, **_I64).copy_(torch.sort(keys, descending=True, stable=True).indices[:k])


def emer_pixel_batch(in_ref, out_ref, stream):
    a, o = in_ref._obj, out_ref._obj
    n_u, n_i = a.n_uniform, a.n_importance
    n = n_u + n_i
    if n == 0:
        return
    H, W = a.height, a.width
    _require(a.cand and a.c2w and a.intrinsics and o.img_idx and o.origins and o.viewdirs and o.norms
             and o.pixel_coords, "emer_pixel_batch: NULL pointer")
    _require(not o.features or 1 <= a.feat_c <= 256, "emer_pixel_batch: features need 1 <= C <= 256")
    imgs, ys, xs = [], [], []
    if n_u:
        n_cand = int(_vec(a.u_pick, n_u, **_I64).max()) + 1
        imgs.append(_vec(a.cand, n_cand, **_I64)[_vec(a.u_pick, n_u, **_I64)])
        ys.append(_vec(a.u_y, n_u, **_I64).clone())
        xs.append(_vec(a.u_x, n_u, **_I64).clone())
    if n_i:
        sel = _vec(a.i_sel, n_i, **_I64)
        plane = a.map_h * a.map_w
        c, row, col = sel // plane, (sel % plane) // a.map_w, sel % a.map_w
        imgs.append(_vec(a.cand, int(c.max()) + 1, **_I64)[c])
        ys.append((row * a.map_downscale + _vec(a.i_dy, n_i, **_I64)).clamp(0, H - 1))
        xs.append((col * a.map_downscale + _vec(a.i_dx, n_i, **_I64)).clamp(0, W - 1))
    img, y, x = torch.cat(imgs), torch.cat(ys), torch.cat(xs)
    n_img = int(img.max()) + 1
    _vec(o.img_idx, n, **_I64).copy_(img)
    if o.cam_idx:
        _vec(o.cam_idx, n, **_I64).copy_(_vec(a.cam_ids, n_img, **_I64)[img])
    if o.pixels:
        _view(o.pixels, n, 3).copy_(_view(a.images, n_img * H * W, 3).view(n_img, H, W, 3)[img, y, x])
    for src, dst in ((a.sky_masks, o.sky_masks), (a.dynamic_masks, o.dynamic_masks)):
        if dst:
            _vec(dst, n).copy_(_vec(src, n_img * H * W).view(n_img, H, W)[img, y, x])
    if o.timestamps:
        _vec(o.timestamps, n).copy_(_vec(a.timestamps, n_img)[img])
    if o.features:
        fh, fw, fc = a.feat_h, a.feat_w, a.feat_c
        fy = (y.float() * a.feat_scale_y).long().clamp(max=fh - 1)
        fx = (x.float() * a.feat_scale_x).long().clamp(max=fw - 1)
        _view(o.features, n, fc).copy_(_view(a.features, n_img * fh * fw, fc).view(n_img, fh, fw, fc)[img, fy, fx])
    # the ray and the pixel coordinates as torch computes them on the host; the kernel's y * (1 / H) is what torch
    # computes on CUDA
    xf, yf = x.float(), y.float()
    emer_gen_rays(o.img_idx, xf.data_ptr(), yf.data_ptr(), a.c2w, a.intrinsics, 0, None, H, W, o.origins, o.viewdirs,
                  o.norms, o.pixel_coords, None, n, stream)


ENTRY_POINTS = ("emer_topk_ratio", "emer_pixel_batch")


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: the training-batch kernels here, everything else in cabi_emulator."""
    if name not in ENTRY_POINTS:
        return cabi_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib, raygen

    cabi_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(raygen, "_WS", {})

"""CPU emulator of the evaluation-metric entry points of the C ABI (emer_image_metrics, emer_depth_rmse,
emer_scene_flow_metrics; csrc/metrics.cu) -- TEST INFRASTRUCTURE ONLY.

Host restatements through the same raw pointers, row strides and sizes the product hands to the library, with the fp64
arithmetic of ``oracle.metrics_ref``.  ``install(monkeypatch)`` installs ``cabi_emulator`` (the rest of the ABI) and
routes these three entry points here, so ``emernerf_b200.metrics`` runs on CPU tensors in the ``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import numpy as np

import cabi_emulator
from cabi_emulator import _addr, _require, _view
from oracle import metrics_ref

IMAGE_OUT = ("psnr", "ssim", "masked_psnr", "masked_ssim", "feat_psnr", "masked_feat_psnr", "mask_count")


def _out(ptr, n):
    return _view(ptr, 1, n, ctype=ctypes.c_double, dtype=np.float64)[0]


def emer_image_metrics(pred, target, h, w, c, mask, fx, ld_fx, fy, ld_fy, cf, out, workspace, stream):
    _require(all(_addr(p) for p in (pred, target, out, workspace)), "emer_image_metrics: NULL pointer")
    _require(1 <= c <= 4, f"emer_image_metrics: {c} channels (1..4)")
    _require(h >= 7 and w >= 7, f"emer_image_metrics: {h}x{w} image is smaller than the 7x7 SSIM window")
    _require(bool(_addr(fx)) == bool(_addr(fy)), "emer_image_metrics: one feature map without the other")
    feats = None
    if _addr(fx):
        _require(1 <= cf <= 256, f"emer_image_metrics: {cf} feature channels (1..256)")
        _require(ld_fx >= cf and ld_fy >= cf, "emer_image_metrics: feature row stride below the channel count")
        feats = [_view(p, h * w, cf, ld).numpy().reshape(h, w, cf) for p, ld in ((fx, ld_fx), (fy, ld_fy))]
    x = _view(pred, h * w, c).numpy().reshape(h, w, c)
    y = _view(target, h * w, c).numpy().reshape(h, w, c)
    m = None if not _addr(mask) else _view(mask, h, w).numpy() != 0
    with np.errstate(all="ignore"):
        got = metrics_ref.image_metrics(x, y, m, *(feats or (None, None)))
    o = _out(out, 11)
    for i, k in enumerate(IMAGE_OUT):
        o[i] = got[k]
    for i, v in enumerate((x.min(), x.max(), y.min(), y.max())):     # numpy's extrema propagate NaN, as the kernel's
        o[7 + i] = float(v)


def emer_depth_rmse(pred, target, n, out, workspace, stream):
    _require(all(_addr(p) for p in (pred, target, out, workspace)), "emer_depth_rmse: NULL pointer")
    _require(n >= 0, "emer_depth_rmse: negative size")
    p = _view(pred, 1, n).numpy()[0]
    t = _view(target, 1, n).numpy()[0]
    o = _out(out, 3)
    o[0], o[1] = metrics_ref.valid_depth_rmse(p, t)
    with np.errstate(all="ignore"):
        o[2] = metrics_ref.psnr(p, t) if n else float("nan")


def emer_scene_flow_metrics(pred, labels, n, out, workspace, stream):
    _require(all(_addr(p) for p in (pred, labels, out, workspace)), "emer_scene_flow_metrics: NULL pointer")
    _require(n >= 0, "emer_scene_flow_metrics: negative size")
    stats, counts = metrics_ref.scene_flow_metrics(_view(pred, n, 3).numpy(), _view(labels, n, 3).numpy())
    o = _out(out, 7)
    for i, k in enumerate(("EPE3D", "acc3d_strict", "acc3d_relax", "outlier", "angle_error")):
        o[i] = stats[k]
    o[5], o[6] = counts["angle"], n


ENTRY_POINTS = ("emer_image_metrics", "emer_depth_rmse", "emer_scene_flow_metrics")


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: the metrics here, everything else in ``cabi_emulator``."""
    if name not in ENTRY_POINTS:
        return cabi_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    import torch

    from emernerf_b200 import _lib, metrics

    cabi_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(metrics, "_WS", {})
    monkeypatch.setattr(metrics, "_numpy_device", lambda: torch.device("cpu"))

"""Restatement of the reference's evaluation metrics -- TEST INFRASTRUCTURE (see ``oracle/__init__.py``).

``datasets/metrics.py``'s compute_psnr, compute_valid_depth_rmse and compute_scene_flow_metrics, and
``skimage.metrics.structural_similarity`` as the reference calls it (data_range=1.0, channel_axis=-1, full=True for
the masked SSIM of ``radiance_fields/video_utils.py:223-231``), in two modes:

  * ``"fp64"``: every step in float64 on float64 copies of the inputs (the yardstick of csrc/metrics.cu);
  * ``"fp32"``: the reference's own float32 path.  skimage keeps float32 images in float32: each
    ``scipy.ndimage.uniform_filter`` output is float32, so are the products and the map; the crop mean is taken in
    float64 and stored into a float32 per-channel array whose mean is float32; the masked mean of the full map is a
    float32 numpy mean.  PSNR is torch's float32 ``F.mse_loss`` and ``log10``.

skimage is not a dependency here; ``ssim`` restates its defaults (7x7 uniform window, 'reflect' border, sample
covariance 49/48, K1 = 0.01, K2 = 0.03).  The fp64 box filter (``box7``) is our own and is checked against
``scipy.ndimage.uniform_filter`` by the tests.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch

WIN = 7
PAD = (WIN - 1) // 2
COV_NORM = WIN * WIN / (WIN * WIN - 1.0)
C1 = (0.01 * 1.0) ** 2
C2 = (0.03 * 1.0) ** 2
FLOW_DOT_MAX = float(np.float32(1 - 1e-7))      # torch rounds the clamp bounds to the fp32 tensor's dtype


def box7(a: np.ndarray) -> np.ndarray:
    """7x7 mean of a 2-D float64 array with scipy's 'reflect' border (d c b a | a b c d)."""
    p = np.pad(np.asarray(a, np.float64), PAD, mode="symmetric")
    return np.lib.stride_tricks.sliding_window_view(p, (WIN, WIN)).sum(axis=(-2, -1)) / (WIN * WIN)


def _ssim_channel(x: np.ndarray, y: np.ndarray, mode: str) -> Tuple[float, np.ndarray]:
    """(crop mean, full map) of one channel, as skimage's 2-D structural_similarity(full=True)."""
    if mode == "fp64":
        filt = box7
        x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    else:
        from scipy.ndimage import uniform_filter

        filt = lambda a: uniform_filter(a, size=WIN)
        x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    ux, uy = filt(x), filt(y)
    uxx, uyy, uxy = filt(x * x), filt(y * y), filt(x * y)
    vx = COV_NORM * (uxx - ux * ux)
    vy = COV_NORM * (uyy - uy * uy)
    vxy = COV_NORM * (uxy - ux * uy)
    a1, a2, b1, b2 = 2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2
    s = (a1 * a2) / (b1 * b2)
    return float(s[PAD:-PAD, PAD:-PAD].mean(dtype=np.float64)), s


def ssim(x: np.ndarray, y: np.ndarray, mode: str = "fp64", mask: Optional[np.ndarray] = None) -> Tuple[float, float]:
    """(ssim, masked_ssim) of [H, W, C] images; masked_ssim is NaN without a mask or with an empty one."""
    x, y = np.asarray(x), np.asarray(y)
    if x.shape[0] < WIN or x.shape[1] < WIN:
        raise ValueError("win_size exceeds image extent")
    dt = np.float64 if mode == "fp64" else np.float32
    per, maps = zip(*(_ssim_channel(x[..., c], y[..., c], mode) for c in range(x.shape[-1])))
    mssim = float(np.asarray(per, dtype=dt).mean())
    full = np.stack(maps, axis=-1)
    m = None if mask is None else np.asarray(mask).astype(bool)
    masked = float(full[m].mean()) if m is not None and m.sum() > 0 else float("nan")
    return mssim, masked


def psnr(pred, target, mode: str = "fp64") -> float:
    """-10 log10(mean squared error) over all elements."""
    if mode == "fp64":
        d = np.asarray(pred, np.float64) - np.asarray(target, np.float64)
        with np.errstate(divide="ignore"):
            return float(-10.0 * np.log10(np.mean(d * d)))
    p = torch.as_tensor(np.asarray(pred, np.float32))
    t = torch.as_tensor(np.asarray(target, np.float32))
    return float(-10 * torch.log10(torch.nn.functional.mse_loss(p, t)))


def image_metrics(pred, target, mask=None, feat_pred=None, feat_target=None, mode: str = "fp64") -> Dict[str, float]:
    """The metric block of video_utils.render for one image (every key; undefined metrics are NaN)."""
    pred, target = np.asarray(pred), np.asarray(target)
    nan = float("nan")
    m = None if mask is None else np.asarray(mask).reshape(pred.shape[:2]).astype(bool)
    s, ms = ssim(pred, target, mode, m)
    out = {"psnr": psnr(pred, target, mode), "ssim": s, "masked_ssim": ms, "masked_psnr": nan, "feat_psnr": nan,
           "masked_feat_psnr": nan, "mask_count": nan if m is None else float(m.sum())}
    have = m is not None and m.sum() > 0
    if have:
        out["masked_psnr"] = psnr(pred[m], target[m], mode)
    if feat_pred is not None:
        fp, ft = np.asarray(feat_pred), np.asarray(feat_target)
        out["feat_psnr"] = psnr(fp, ft, mode)
        if have:
            out["masked_feat_psnr"] = psnr(fp[m], ft[m], mode)
    return out


def valid_depth_rmse(pred, target) -> Tuple[float, int]:
    """(sqrt(mean((p - t)^2) over t > 0), count) in float64; NaN over no valid ray."""
    p = np.asarray(pred, np.float64).reshape(-1)
    t = np.asarray(target, np.float64).reshape(-1)
    v = t > 0
    if not v.any():
        return float("nan"), 0
    d = p[v] - t[v]
    return float(np.sqrt(np.mean(d * d))), int(v.sum())


def scene_flow_metrics(pred, labels) -> Tuple[Dict[str, float], Dict[str, int]]:
    """(the five NSFP statistics in float64, the counts behind the fractions and the angle mean)."""
    p = np.asarray(pred, np.float64).reshape(-1, 3)
    lab = np.asarray(labels, np.float64).reshape(-1, 3)
    n = p.shape[0]
    l2 = np.sqrt(np.sum((p - lab) ** 2, -1))
    ln = np.sqrt(np.sum(lab * lab, -1))
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = l2 / (ln + 1e-20)
        counts = {"acc3d_strict": int(((l2 < 0.05) | (rel < 0.05)).sum()),
                  "acc3d_relax": int(((l2 < 0.1) | (rel < 0.1)).sum()),
                  "outlier": int(((l2 > 0.3) | (rel > 0.1)).sum())}
        keep = ln > 0.1
        ul = lab / (ln[:, None] + 1e-7)
        up = p / (np.sqrt(np.sum(p * p, -1))[:, None] + 1e-7)
        dot = np.sum(ul[keep] * up[keep], -1)
        nan = dot != dot
        dot = np.clip(dot, -FLOW_DOT_MAX, FLOW_DOT_MAX)
        dot[nan] = 0.0
        angle = float(np.mean(np.arccos(dot))) if dot.size else float("nan")
        out = {"EPE3D": float(np.mean(l2)) if n else float("nan"), "angle_error": angle}
        for k, c in counts.items():
            out[k] = c / n if n else float("nan")
    counts["angle"] = int(keep.sum())
    return out, counts

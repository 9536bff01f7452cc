"""CPU emulator of the scene-flow figure's entry points of the C ABI (emer_flow_vis_select, emer_flow_vis_color;
csrc/flow_vis.cu) -- TEST INFRASTRUCTURE ONLY.

Host restatements in numpy through the same raw pointers, row strides and sizes the product hands to the library:
fp32 with one rounding per operation where the kernels round so (the projection's fma chain through fp64, where the
product of two floats is exact), numpy's ``hypot`` and ``arctan2`` for thrust's ``abs`` and ``arg``, and the wheel of
``oracle.scene_flow_vis_ref``.  ``install(monkeypatch)`` installs ``lidar_flow_emulator`` (and through it the rest of
the ABI) and routes these two entry points here, so ``emernerf_b200.flow_vis`` runs end to end on CPU tensors in the
``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import numpy as np

import cabi_emulator
import lidar_flow_emulator
from cabi_emulator import _addr, _require, _view
from oracle.scene_flow_vis_ref import WHEEL

MAX_ROWS, MAX_CAMS = 1 << 24, 16
SCALE_NONE, SCALE_HOST, SCALE_DEVICE = 0, 1, 2
_F32 = np.float32
_WHEEL = WHEEL.numpy().astype(_F32)


def flow_rgb(x, y, scale_mode, scale, bright):
    """The colours [n, 3] of flows (x, y) [n] as csrc/flow_color.cuh computes them."""
    x, y = np.asarray(x, _F32), np.asarray(y, _F32)
    with np.errstate(all="ignore"):
        re = x + (y * _F32(0) - _F32(0) * _F32(1))
        im = _F32(0) + (y * _F32(1) + _F32(0) * _F32(0))
        radius = np.hypot(re, im).astype(_F32)
        angle = np.arctan2(im, re).astype(_F32)
        if scale_mode == SCALE_HOST:
            radius = radius * _F32(scale)
        elif scale_mode == SCALE_DEVICE and _F32(scale) > 0:
            radius = radius / _F32(scale)
        angle = np.where(angle < 0, angle + _F32(2 * np.pi), angle).astype(_F32)
        angle = (angle * _F32(54 / (2 * np.pi))).astype(_F32)
        bad = np.isnan(radius) | np.isnan(angle)
        a = np.where(bad, _F32(0), angle)
        frac = np.fmod(a, _F32(1)).astype(_F32)
        i0 = np.clip(np.trunc(a), 0, 55).astype(np.int64)
        i1 = np.clip(np.ceil(a), 0, 55).astype(np.int64)
        hue = _WHEEL[i0] * (_F32(1) - frac)[:, None] + _WHEEL[i1] * frac[:, None]
        r = radius[:, None]
        over = r > 1
        inv = np.where(over, _F32(1) / np.where(over, r, _F32(1)), _F32(0)).astype(_F32)
        if bright:
            c = np.where(over, hue * inv, _F32(255) - r * (_F32(255) - hue))
        else:
            c = np.where(over, _F32(255) - inv * (_F32(255) - hue), hue * r)
        c = (c.astype(_F32) * _F32(_F32(1) / _F32(255))).astype(_F32)
    c[bad] = np.nan
    return c


def flow_radius(x, y):
    with np.errstate(all="ignore"):
        re = np.asarray(x, _F32) + (np.asarray(y, _F32) * _F32(0) - _F32(0))
        im = _F32(0) + (np.asarray(y, _F32) * _F32(1) + _F32(0))
        return np.hypot(re, im).astype(_F32)


def in_view(q, mats, w, h):
    """get_valid_lidar_mask of the points q [n, 3] for the dense matrices [cams, 4, 4]."""
    seen = np.zeros(len(q), bool)
    q64 = q.astype(np.float64)
    for m in mats:
        pr = []
        for r in range(3):
            acc = _F32(0) * np.zeros(len(q), _F32)
            for k in range(3):
                acc = (np.float64(m[r, k]) * q64[:, k] + acc.astype(np.float64)).astype(_F32)
            pr.append(acc + m[r, 3])
        with np.errstate(all="ignore"):
            den = pr[2] + _F32(1e-6)
            u, v = pr[0] / den, pr[1] / den
            seen |= (u >= 0) & (u < _F32(w)) & (v >= 0) & (v < _F32(h)) & (pr[2] > 0)
    return seen


def emer_flow_vis_select(origins, ld_o, viewdirs, ld_d, ranges, ld_r, times, ld_t, flows, ld_f, classes, ld_c, n,
                         lidar2img, cams, width, height, points, out_times, rows9, count, frame_counts, workspace,
                         stream):
    _require(0 <= n <= MAX_ROWS, f"emer_flow_vis_select: {n} points")
    _require(1 <= cams <= MAX_CAMS, f"emer_flow_vis_select: {cams} cameras")
    _require(_addr(count) and _addr(frame_counts) and _addr(workspace), "emer_flow_vis_select: NULL pointer")
    if n == 0:
        return
    o = _view(origins, n, 3, ld_o).numpy()
    d = _view(viewdirs, n, 3, ld_d).numpy()
    r = _view(ranges, n, 1, ld_r).numpy()
    t = _view(times, n, 1, ld_t).numpy()[:, 0]
    f = _view(flows, n, 3, ld_f).numpy()
    cls = _view(classes, n, 1, ld_c, ctype=ctypes.c_int64, dtype=np.int64).numpy()[:, 0]
    mats = _view(lidar2img, cams * 4, 4).numpy().reshape(cams, 4, 4)
    labelled = cls != -1
    q = (o + r * d).astype(_F32)
    keep = labelled.copy()
    keep[labelled] = in_view(q[labelled], mats, width, height)
    cnt = _view(count, 1, 1, ctype=ctypes.c_int64, dtype=np.int64)[0].numpy()
    fc = _view(frame_counts, 1, 2, ctype=ctypes.c_int64, dtype=np.int64)[0].numpy()
    base, k = int(cnt[0]), int(keep.sum())
    fc[0] += int(labelled.sum())
    fc[1] += k
    if k:
        _view(points, base + k, 3).numpy()[base:] = q[keep]
        _view(out_times, 1, base + k).numpy()[0, base:] = t[keep]
        out = _view(rows9, base + k, 9).numpy()[base:]
        out[:, 0:3] = q[keep]
        out[:, 6:9] = flow_rgb(f[keep, 0], f[keep, 1], SCALE_HOST, _F32(1) / _F32(2), True)
    cnt[0] = base + k


def emer_flow_vis_color(flow, ld_flow, density, threshold, n, scale_mode, radius_scale, device_radius, bright, colors,
                        ld_colors, radius, stream):
    _require(n >= 0, "emer_flow_vis_color: negative size")
    _require(scale_mode in (SCALE_NONE, SCALE_HOST, SCALE_DEVICE), f"emer_flow_vis_color: scale mode {scale_mode}")
    if n == 0:
        return
    _require(_addr(flow) and ld_flow >= 2, "emer_flow_vis_color: flow rows")
    _require(_addr(colors) or _addr(radius), "emer_flow_vis_color: neither colours nor radii to write")
    fl = _view(flow, n, 2, ld_flow).numpy().copy()
    if _addr(density):
        gate = _view(density, 1, n).numpy()[0] < _F32(threshold)
        fl[gate] *= _F32(0)
    if not _addr(colors):
        _view(radius, 1, n).numpy()[0] = flow_radius(fl[:, 0], fl[:, 1])
        return
    scale = _F32(radius_scale)
    if scale_mode == SCALE_HOST:
        with np.errstate(divide="ignore"):
            scale = _F32(1) / scale
    elif scale_mode == SCALE_DEVICE:
        scale = _view(device_radius, 1, 1).numpy()[0, 0]
    _view(colors, n, 3, ld_colors).numpy()[:] = flow_rgb(fl[:, 0], fl[:, 1], scale_mode, scale, bool(bright))


ENTRY_POINTS = ("emer_flow_vis_select", "emer_flow_vis_color")


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: the scene-flow figure's kernels here, the rest in the other
    emulators."""
    if name not in ENTRY_POINTS:
        return lidar_flow_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib, flow_vis

    lidar_flow_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(flow_vis, "_WS", {})

"""CPU emulator of the evaluation video frames' entry point of the C ABI (emer_video_compose; csrc/video.cu) -- TEST
INFRASTRUCTURE ONLY.

A numpy restatement through the same raw pointers, descriptors and sizes the product hands to the library: float32
with one rounding per operation where the kernel rounds so, the depth curve's float64 log rounded once to float32, the
rest of the depth path in float64, and matplotlib's index rule.  ``install(monkeypatch)`` installs
``scene_flow_vis_emulator`` (and through it the rest of the ABI), routes this entry point here and replaces the pinned
host frames, the copy event and its wait by host stand-ins, so ``emernerf_b200.video`` runs end to end on CPU tensors
in the ``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

import cabi_emulator
import scene_flow_vis_emulator
from cabi_emulator import _addr, _require, _view

RGB, DEPTH, BLEND, GRAY = 0, 1, 2, 3
MAX_TILES, MAX_PIXELS = 32, 1 << 26
_F32 = np.float32
CURVE_LO = -np.log(4.0 + 1e-6)
CURVE_HI = -np.log(120 + 1e-6)
WAITS = []          # one entry per frame the writer waited for


def to8b(x, f64: bool) -> np.ndarray:
    """(255 * np.clip(x, 0, 1)).astype(np.uint8) of float32 values, the product in float64 or float32; NaN gives 0."""
    x = np.asarray(x, _F32)
    with np.errstate(invalid="ignore"):
        c = np.clip(x.astype(np.float64) if f64 else x, 0, 1)
        v = (255 * c) if f64 else (_F32(255) * c).astype(_F32)
    v = np.where(np.isnan(v), 0, v)
    return v.astype(np.uint8)


def blend(a, alpha, b) -> np.ndarray:
    """np.clip(a * alpha + b * (1 - alpha), 0, 1) on float32 arrays ([n, 3], [n, 1], [n, 3])."""
    a, alpha, b = (np.asarray(t, _F32) for t in (a, alpha, b))
    with np.errstate(invalid="ignore", over="ignore"):
        return np.clip(a * alpha + b * (_F32(1) - alpha), _F32(0), _F32(1))


def depth_index(depth, opacity) -> np.ndarray:
    """The turbo entry of each depth pixel, -1 for the "bad" colour (csrc/video.cuh: video_depth_index)."""
    d, w = np.asarray(depth, _F32), np.asarray(opacity, _F32)
    with np.errstate(all="ignore"):
        x = d + _F32(1e-6)
        curve = -(np.log(x.astype(np.float64)).astype(_F32))
        v = (curve.astype(np.float64) - np.minimum(CURVE_LO, CURVE_HI)) / np.abs(CURVE_HI - CURVE_LO)
        v = np.nan_to_num(np.clip(v, 0, 1))
        v = v * w.astype(np.float64)
        s = v * 256.0
        idx = np.where(s < 0, 0, np.where(s >= 256, 255, np.trunc(np.where(np.isfinite(s), s, 0)))).astype(np.int64)
    return np.where(np.isnan(v), -1, idx)


def tile_rgb(kind: int, ins, invert: bool, f64: bool, lut: np.ndarray) -> np.ndarray:
    """The [n, 3] uint8 pixels of one tile from its float32 inputs (rows of C)."""
    if kind == RGB:
        return to8b(ins[0], f64)
    if kind == DEPTH:
        i = depth_index(ins[0][:, 0], ins[1][:, 0])
        out = lut[np.maximum(i, 0)].copy()
        out[i < 0] = 0
        return out
    if kind == BLEND:
        return to8b(blend(ins[0], ins[1], ins[2]), f64)
    v = np.asarray(ins[0][:, 0], _F32)
    if invert:
        v = _F32(1) - v
    return np.repeat(to8b(v, f64)[:, None], 3, axis=1)


def emer_video_compose(frame, frame_w, tiles, n_tiles, height, width, col, lut, stream):
    _require(_addr(frame) and tiles is not None, "emer_video_compose: NULL pointer")
    _require(1 <= n_tiles <= MAX_TILES, f"emer_video_compose: {n_tiles} tiles")
    _require(height >= 1 and width >= 1 and height * width <= MAX_PIXELS, "emer_video_compose: tile size")
    _require(col >= 0 and (col + 1) * width <= frame_w, "emer_video_compose: column")
    n = height * width
    table = None
    rows_needed = 0
    specs = []
    for i in range(n_tiles):
        t = tiles[i]
        _require(t.kind in (RGB, DEPTH, BLEND, GRAY), f"emer_video_compose: tile {i} of kind {t.kind}")
        _require(t.row >= 0, f"emer_video_compose: tile {i} at row {t.row}")
        chans = {RGB: (3,), DEPTH: (1, 1), BLEND: (3, 1, 3), GRAY: (1,)}[t.kind]
        _require(all(t.inputs[k] for k in range(len(chans))), f"emer_video_compose: tile {i} lacks an input")
        if t.kind == DEPTH:
            _require(_addr(lut), "emer_video_compose: a depth tile without the colour table")
            table = _view(lut, 256, 3, ctype=ctypes.c_uint8, dtype=np.uint8).numpy()
        ins = [_view(t.inputs[k], n, c).numpy() for k, c in enumerate(chans)]
        specs.append((t.kind, ins, t.row, bool(t.invert), bool(t.f64)))
        rows_needed = max(rows_needed, t.row + 1)
    out = _view(frame, rows_needed * height, frame_w * 3, ctype=ctypes.c_uint8, dtype=np.uint8).numpy()
    out = out.reshape(rows_needed * height, frame_w, 3)
    for kind, ins, row, invert, f64 in specs:
        px = tile_rgb(kind, ins, invert, f64, table).reshape(height, width, 3)
        out[row * height:(row + 1) * height, col * width:(col + 1) * width] = px


ENTRY_POINTS = ("emer_video_compose",)


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: the video kernel here, the rest in the other emulators."""
    if name not in ENTRY_POINTS:
        return scene_flow_vis_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib, video

    scene_flow_vis_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(video, "_LUT", {})
    monkeypatch.setattr(video, "_host_frame", lambda shape: torch.empty(shape, dtype=torch.uint8))
    monkeypatch.setattr(video, "_record", lambda dev: None)
    monkeypatch.setattr(video, "_wait", lambda ev: WAITS.append(ev))

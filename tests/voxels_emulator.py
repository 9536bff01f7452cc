"""CPU emulator of the voxel-lifting entry points of the C ABI (emer_voxel_mark, emer_voxel_compact,
emer_voxel_select; csrc/voxels.cu) -- TEST INFRASTRUCTURE ONLY.

Host restatements in numpy through the same raw pointers, row strides, sizes and host structs the product hands to the
library: fp32 with one rounding per operation where the kernels round so, the colour's dot product in fp64.
``install(monkeypatch)`` installs ``errormap_emulator`` (and through it the rest of the ABI, with the render rays of
``raygen.PixelRaySampler``) and routes these three entry points here, so ``emernerf_b200.voxels.visualize_voxels`` runs
end to end on CPU tensors in the ``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import numpy as np

import cabi_emulator
import errormap_emulator
from cabi_emulator import _addr, _require, _view

MAX_GRIDS, MAX_ROWS, MAX_CHANNELS = 32, 1 << 24, 256
_F32 = np.float32


def _grid(g):
    _require(g is not None and _addr(g.bits), "emer_voxel_grid: NULL grid")
    res = [int(v) for v in g.res]
    _require(min(res) >= 1 and res[0] * res[1] * res[2] <= 1 << 32, "emer_voxel_grid: resolution")
    return np.array(list(g.min), _F32), np.array(list(g.voxel_size), _F32), res


def _words(g, res):
    n = (res[0] * res[1] * res[2] + 31) // 32
    return np.ctypeslib.as_array((ctypes.c_uint32 * n).from_address(_addr(g.bits)))


def voxel_index(p, lo, vs, res):
    """Linear voxel index of each end point [n, 3] (fp32), -1 where it marks nothing."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        q = (p - lo) / vs
        ok = np.all((q > _F32(-1)) & (q.astype(np.float64) < np.array(res, np.float64)), axis=1)
        idx = np.where(ok[:, None], q, 0).astype(np.int64)
    lin = (idx[:, 0] * res[1] + idx[:, 1]) * res[2] + idx[:, 2]
    return np.where(ok, lin, -1)


def _mark(g, o, d, t):
    lo, vs, res = _grid(g)
    with np.errstate(invalid="ignore", over="ignore"):
        p = o + d * t[:, None]
    lin = voxel_index(p, lo, vs, res)
    lin = lin[lin >= 0]
    words = _words(g, res)
    np.bitwise_or.at(words, lin >> 5, (np.uint32(1) << (lin & 31).astype(np.uint32)))


def emer_voxel_mark(origins, ld_o, viewdirs, ld_d, depth, ld_t, dyn_depth, ld_dd, n, max_depth, static, dynamic,
                    stream):
    _require(n >= 0, "emer_voxel_mark: negative size")
    s = static._obj
    dyn = dynamic._obj if dynamic is not None and _addr(dynamic._obj.bits) else None
    _grid(s)
    if n == 0:
        return
    _require(_addr(origins) and _addr(viewdirs) and _addr(depth), "emer_voxel_mark: NULL pointer")
    _require(dyn is None or _addr(dyn_depth), "emer_voxel_mark: a dynamic grid without dynamic depths")
    o = _view(origins, n, 3, ld_o).numpy()
    d = _view(viewdirs, n, 3, ld_d).numpy()
    t = _view(depth, n, 1, ld_t).numpy()[:, 0]
    with np.errstate(invalid="ignore"):
        near = t < _F32(max_depth)
    _mark(s, o[near], d[near], t[near])
    if dyn is not None:
        _mark(dyn, o, d, _view(dyn_depth, n, 1, ld_dd).numpy()[:, 0])


def set_voxels(g):
    """(linear indices of the set voxels in order, world coordinates [m, 3] fp32) of one grid struct."""
    lo, vs, res = _grid(g)
    bits = np.unpackbits(_words(g, res).view(np.uint8), bitorder="little")
    lin = np.nonzero(bits)[0].astype(np.int64)
    ijk = np.stack([lin // (res[1] * res[2]), (lin // res[2]) % res[1], lin % res[2]], 1)
    return lin, lo + ijk.astype(_F32) * vs


def emer_voxel_compact(grids, n_grids, counts, coords, workspace, stream):
    _require(1 <= n_grids <= MAX_GRIDS, f"emer_voxel_compact: {n_grids} grids (1..{MAX_GRIDS})")
    _require(_addr(counts) and _addr(workspace), "emer_voxel_compact: NULL pointer")
    cnt = _view(counts, 1, n_grids, ctype=ctypes.c_int64, dtype=np.int64)[0].numpy()
    for g in range(n_grids):
        lin, xyz = set_voxels(grids[g])
        if not _addr(coords):
            cnt[g] = len(lin)
        elif len(lin):
            _view(coords, grids[g].first_row + len(lin), 3).numpy()[grids[g].first_row:] = xyz


def select_rows(dens, threshold, n):
    """torch's CUDA mean of the stacked columns > threshold: the sum from 0 in order, times n / (n k) in fp32."""
    s = _F32(0)
    for d in dens:
        s = s + d
    with np.errstate(invalid="ignore"):
        return s * (_F32(n) / _F32(n * len(dens))) > _F32(threshold)


def colours(f, m, lo, hi):
    c = (f.astype(np.float64) @ m.astype(np.float64)).astype(_F32)
    with np.errstate(invalid="ignore", divide="ignore"):
        v = (c - lo) / (hi - lo)
        return np.where(np.isnan(v), v, np.clip(v, _F32(0), _F32(1)))


def emer_voxel_select(d0, d1, d2, k, threshold, points, feat, ld_feat, c, reduction, cmin, cmax, n, out_points,
                      out_colors, count, workspace, stream):
    _require(1 <= k <= 3, f"emer_voxel_select: {k} density columns (1..3)")
    _require(0 <= n <= MAX_ROWS, f"emer_voxel_select: {n} rows")
    _require(4 <= c <= MAX_CHANNELS and c % 4 == 0, f"emer_voxel_select: {c} channels")
    _require(_addr(count) and _addr(workspace), "emer_voxel_select: NULL pointer")
    if n == 0:
        return
    _require(ld_feat >= c and ld_feat % 4 == 0 and _addr(feat) % 16 == 0,
             "emer_voxel_select: feature rows must be 16-byte aligned")
    dens = [_view(p, 1, n).numpy()[0] for p in (d0, d1, d2)[:k]]
    keep = select_rows(dens, threshold, n)
    f = _view(feat, n, c, ld_feat).numpy()[keep]
    m = _view(reduction, c, 3).numpy()
    lo, hi = _view(cmin, 1, 3).numpy()[0], _view(cmax, 1, 3).numpy()[0]
    cnt = _view(count, 1, 1, ctype=ctypes.c_int64, dtype=np.int64)[0].numpy()
    base, kept = int(cnt[0]), int(keep.sum())
    if kept:
        _view(out_points, base + kept, 3).numpy()[base:] = _view(points, n, 3).numpy()[keep]
        _view(out_colors, base + kept, 3).numpy()[base:] = colours(f, m, lo, hi)
    cnt[0] = base + kept


ENTRY_POINTS = ("emer_voxel_mark", "emer_voxel_compact", "emer_voxel_select")


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: the voxel kernels here, everything else in errormap_emulator."""
    if name not in ENTRY_POINTS:
        return errormap_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib, voxels

    errormap_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(voxels, "_WS", {})

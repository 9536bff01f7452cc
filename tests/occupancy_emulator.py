"""CPU emulator of the few-shot occupancy entry points of the C ABI (emer_occ_accumulate, emer_occ_classify;
csrc/occupancy.cu) -- TEST INFRASTRUCTURE ONLY.

Host restatements in fp64 through the same raw pointers, row strides and sizes the product hands to the library.
``install(monkeypatch)`` installs ``metrics_emulator`` (and through it ``cabi_emulator``, the rest of the ABI) and
routes these two entry points here, so ``emernerf_b200.metrics.collect_centroids`` / ``eval_few_shot_occ`` run on CPU
tensors, with the drop-in field, in the ``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

import cabi_emulator
import metrics_emulator
from cabi_emulator import _addr, _require, _view


def _i64(ptr, n):
    return _view(ptr, 1, n, ctype=ctypes.c_int64, dtype=np.int64)[0]


def _rows(what, feat, ld_feat, c, density, ld_density, labels, n, k, counts, workspace):
    _require(all(_addr(p) for p in (feat, density, labels, counts, workspace)), f"{what}: NULL pointer")
    _require(n >= 0, f"{what}: negative size")
    _require(4 <= c <= 256 and c % 4 == 0, f"{what}: {c} channels (a multiple of 4, at most 256)")
    _require(1 <= k <= 32, f"{what}: {k} classes (1..32)")
    _require(ld_feat >= c and ld_feat % 4 == 0 and _addr(feat) % 16 == 0, f"{what}: feature rows must be 16-byte aligned")
    _require(ld_density >= 1, f"{what}: density stride {ld_density}")
    q = _view(feat, n, c, ld_feat).double()
    d = _view(density, n, 1, ld_density)[:, 0]
    lab = _i64(labels, n)
    return q, d, lab


def emer_occ_accumulate(feat, ld_feat, c, density, ld_density, labels, n, k, threshold, sums, counts, workspace,
                        stream):
    q, d, lab = _rows("emer_occ_accumulate", feat, ld_feat, c, density, ld_density, labels, n, k, counts, workspace)
    _require(_addr(sums), "emer_occ_accumulate: NULL pointer")
    keep = (d > np.float32(threshold)) & (lab >= 0) & (lab < k)
    s = _view(sums, k, c, ctype=ctypes.c_double, dtype=np.float64)
    cnt = _i64(counts, k)
    for j in range(k):
        m = keep & (lab == j)
        s[j] += q[m].sum(0)
        cnt[j] += int(m.sum())


def emer_occ_classify(feat, ld_feat, c, density, ld_density, labels, n, centroids, k, label_bank, threshold, counts,
                      workspace, stream):
    q, d, lab = _rows("emer_occ_classify", feat, ld_feat, c, density, ld_density, labels, n, k, counts, workspace)
    _require(_addr(centroids) and _addr(label_bank), "emer_occ_classify: NULL pointer")
    cen = _view(centroids, k, c).double()
    bank = _i64(label_bank, k)
    cnt = _i64(counts, 2 * k + 2)
    measured = d > np.float32(threshold)
    inside = measured & (lab >= 0) & (lab < k)
    chat = cen / (cen.norm(dim=-1, keepdim=True) + 1e-7)
    pred = bank[torch.argmax(q[inside] @ chat.T, dim=-1)] if bool(inside.any()) else bank[:0]  # first maximum wins
    true = lab[inside]
    for j in range(k):
        cnt[j] += int((true == j).sum())
        cnt[k + j] += int(((true == j) & (pred == j)).sum())
    cnt[2 * k] += int(measured.sum())
    cnt[2 * k + 1] += int((measured & ~inside).sum())


ENTRY_POINTS = ("emer_occ_accumulate", "emer_occ_classify")


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: the occupancy kernels here, everything else in the other emulators."""
    if name not in ENTRY_POINTS:
        return metrics_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib, metrics

    metrics_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(metrics, "_OCC_WS", {})

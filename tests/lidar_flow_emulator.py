"""CPU emulator of the lidar scene-flow entry point of the C ABI (emer_lidar_flow_accumulate; csrc/metrics.cu) -- TEST
INFRASTRUCTURE ONLY.

A host restatement through the same raw pointers, row stride and size the product hands to the library: the
flow-class and ground filters, the fp32 gate ``pred *= 0`` where the dynamic density is below the fp32 threshold, and
the NSFP terms in fp64 from ``oracle.metrics_ref.scene_flow_metrics``.  ``install(monkeypatch)`` installs
``metrics_emulator`` (and through it ``cabi_emulator``, the rest of the ABI) and routes this entry point here, so
``emernerf_b200.metrics.eval_lidar_flow`` runs on CPU tensors, with the drop-in field, in the ``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import numpy as np

import cabi_emulator
import metrics_emulator
from cabi_emulator import _addr, _require, _view
from oracle import metrics_ref

SUMS = 8                     # EMER_LIDAR_FLOW_SUMS


def emer_lidar_flow_accumulate(pred, ld_pred, density, labels, flow_class, ground, n, threshold, sums, workspace,
                               stream):
    inputs = (pred, density, labels, flow_class)
    _require(_addr(sums) and _addr(workspace) and (n == 0 or all(_addr(p) for p in inputs)),
             "emer_lidar_flow_accumulate: NULL pointer")
    _require(n >= 0, "emer_lidar_flow_accumulate: negative size")
    _require(ld_pred >= 3, f"emer_lidar_flow_accumulate: prediction row stride {ld_pred} below 3")
    p = _view(pred, n, 3, ld_pred).numpy().copy()
    d = _view(density, 1, n).numpy()[0]
    lab = _view(labels, n, 3).numpy()
    cls = _view(flow_class, 1, n, ctype=ctypes.c_int64, dtype=np.int64).numpy()[0]
    valid = cls != -1
    counted = valid
    if _addr(ground):
        counted = valid & (_view(ground, 1, n, ctype=ctypes.c_uint8, dtype=np.uint8).numpy()[0] == 0)
    gate = d < np.float32(threshold)                 # NaN is not gated
    p[gate] *= np.float32(0.0)                       # NaN stays NaN, a negative value gives -0
    s = _view(sums, 1, SUMS, ctype=ctypes.c_double, dtype=np.float64).numpy()[0]
    m = int(counted.sum())
    s[7] += int(valid.sum())
    s[6] += m
    if m == 0:
        return
    stats, counts = metrics_ref.scene_flow_metrics(p[counted], lab[counted])
    s[0] += stats["EPE3D"] * m
    s[1] += counts["acc3d_strict"]
    s[2] += counts["acc3d_relax"]
    s[3] += counts["outlier"]
    if counts["angle"]:
        s[4] += stats["angle_error"] * counts["angle"]
    s[5] += counts["angle"]


ENTRY_POINTS = ("emer_lidar_flow_accumulate",)


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: the lidar flow kernel here, everything else in the other emulators."""
    if name not in ENTRY_POINTS:
        return metrics_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib, metrics

    metrics_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(metrics, "_SAMPLERS", type(metrics._SAMPLERS)())

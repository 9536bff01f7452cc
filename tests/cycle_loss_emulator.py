"""CPU emulator of the flow cycle-loss entry points of the C ABI (emer_cycle_loss_fwd / _bwd; csrc/losses.cu) -- TEST
INFRASTRUCTURE ONLY.

Host restatements of the kernels' fp32 arithmetic through the same raw pointers, row strides and sizes the product hands
to the library.  ``install(monkeypatch)`` installs ``loss_emulator`` (the other loss entry points, and through it
``cabi_emulator`` for the rest of the ABI) and routes these two entry points here, so ``loss.flow_cycle_loss`` runs on
CPU tensors in the ``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import torch

import cabi_emulator
import loss_emulator
from cabi_emulator import _addr, _require, _vec, _view
from loss_emulator import _f32


def _cycle_inputs(f, ld_f, b, ld_b, fpb, ld_fpb, bpf, ld_bpf, n, what):
    _require(n >= 1, f"{what}: no rows")
    _require(min(ld_f, ld_b, ld_fpb, ld_bpf) >= 3, f"{what}: row stride below 3")
    return [_view(p, n, 3, ld) for p, ld in ((f, ld_f), (b, ld_b), (fpb, ld_fpb), (bpf, ld_bpf))]


def emer_cycle_loss_fwd(f, ld_f, b, ld_b, fpb, ld_fpb, bpf, ld_bpf, n, coef, out, workspace, stream):
    """0.5 * mean((f + fpb)^2 + (b + bpf)^2) * coef and the four maximum row norms (NaN if any row's is)."""
    _require(all(_addr(p) for p in (f, b, fpb, bpf, out, workspace)), "emer_cycle_loss_fwd: NULL pointer")
    F, B, FP, BP = _cycle_inputs(f, ld_f, b, ld_b, fpb, ld_fpb, bpf, ld_bpf, n, "emer_cycle_loss_fwd")
    with torch.no_grad():
        term = (F + FP) * (F + FP) + (B + BP) * (B + BP)
        cnt = _f32(float(3 * n))
        o = _vec(out, 6)
        o[0] = _f32(0.5) * (term.sum() / cnt) * _f32(coef)
        o[1] = cnt
        for k, x in enumerate((F, B, FP, BP)):
            norms = torch.sqrt(x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1] + x[:, 2] * x[:, 2])
            o[2 + k] = norms.max()             # torch.max propagates NaN, as the kernel's ordered keys do


def emer_cycle_loss_bwd(f, ld_f, b, ld_b, fpb, ld_fpb, bpf, ld_bpf, n, coef, fwd_out, g, d_fpb, d_bpf, stream):
    _require(all(_addr(p) for p in (f, b, fpb, bpf, fwd_out, g)), "emer_cycle_loss_bwd: NULL pointer")
    _require(_addr(d_fpb) or _addr(d_bpf), "emer_cycle_loss_bwd: no gradient requested")
    F, B, FP, BP = _cycle_inputs(f, ld_f, b, ld_b, fpb, ld_fpb, bpf, ld_bpf, n, "emer_cycle_loss_bwd")
    with torch.no_grad():
        gs = _vec(g, 1)[0] * _f32(coef) * _f32(0.5) / _vec(fwd_out, 2)[1]
        if _addr(d_fpb):
            _view(d_fpb, n, 3).copy_(2.0 * (F + FP) * gs)
        if _addr(d_bpf):
            _view(d_bpf, n, 3).copy_(2.0 * (B + BP) * gs)


ENTRY_POINTS = ("emer_cycle_loss_fwd", "emer_cycle_loss_bwd")


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: the cycle loss here, everything else in ``loss_emulator``."""
    if name not in ENTRY_POINTS:
        return loss_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib

    loss_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)

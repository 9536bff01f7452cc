"""CPU emulator of the live line-of-sight entry points (emer_ray_loss_live_*; csrc/losses.cu) -- TEST INFRASTRUCTURE
ONLY.

The kernels read ``[eps, 2 sigma^2, amp, pre]`` from device memory and then run the float entries' arithmetic; here the
four values are read through the pointer the product passes and handed to ``loss_emulator``'s restatement of the float
entries.  ``install(monkeypatch)`` installs ``loss_emulator`` and routes the two live entries here."""
from __future__ import annotations

import ctypes

import cabi_emulator
import loss_emulator
from cabi_emulator import _addr, _require, _vec


def _consts(ptr):
    return [float(v) for v in _vec(ptr, 4)]


def emer_ray_loss_live_fwd(kind, w, t, gt, n_rays, n_samples, consts, post, out, workspace, stream):
    _require(kind in (0, 2), f"emer_ray_loss_live_fwd: kind {kind} has no live constants")
    _require(all(_addr(p) for p in (w, t, gt, consts, out, workspace)), "emer_ray_loss_live_fwd: NULL pointer")
    _require(n_rays >= 0 and n_samples >= 1, "emer_ray_loss_live_fwd: bad shape")
    eps, two_sigma_sq, amp, pre = _consts(consts)
    loss_emulator.emer_ray_loss_fwd(kind, w, t, gt, n_rays, n_samples, eps, two_sigma_sq, amp, pre, post, out,
                                    workspace, stream)


def emer_ray_loss_live_bwd(kind, w, t, gt, n_rays, n_samples, consts, post, fwd_out, g, dw, stream):
    _require(kind in (0, 2), f"emer_ray_loss_live_bwd: kind {kind} has no live constants")
    _require(all(_addr(p) for p in (w, t, gt, consts, fwd_out, g, dw)), "emer_ray_loss_live_bwd: NULL pointer")
    _require(n_rays >= 0 and n_samples >= 1, "emer_ray_loss_live_bwd: bad shape")
    eps, two_sigma_sq, amp, pre = _consts(consts)
    loss_emulator.emer_ray_loss_bwd(kind, w, t, gt, n_rays, n_samples, eps, two_sigma_sq, amp, pre, post, fwd_out, g,
                                    dw, stream)


ENTRY_POINTS = ("emer_ray_loss_live_fwd", "emer_ray_loss_live_bwd")


def call(name: str, *args) -> None:
    if name not in ENTRY_POINTS:
        return loss_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib

    loss_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)

"""CPU emulator of the training-loss entry points of the C ABI (emer_pointwise_loss_*, emer_ray_loss_*;
csrc/losses.cu) -- TEST INFRASTRUCTURE ONLY.

Host restatements of the kernels' fp32 arithmetic through the same raw pointers and arguments the product hands to the
library, alongside ``cabi_emulator`` (the rest of the ABI).  ``install(monkeypatch)`` installs ``cabi_emulator`` and
routes these four entry points here, so ``emernerf_b200.loss`` runs on CPU tensors in the ``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import torch

import cabi_emulator
from cabi_emulator import _addr, _require, _vec, _view

# ----------------------------------------------------------------------------- training losses
def _real_term(base, d):
    if base == 0:
        return d.abs()
    if base == 1:
        return d * d
    z = d.abs()
    return torch.where(z < 1.0, 0.5 * z * z / 1.0, z - 0.5 * 1.0)


def _real_grad(base, d, gs):
    if base == 0:
        return torch.sign(d) * gs
    if base == 1:
        return 2.0 * d * gs
    return torch.where(d <= -1.0, -gs, torch.where(d >= 1.0, gs, d * gs / 1.0))


def _f32(v):
    return torch.tensor(v, dtype=torch.float32)


def _entropy_parts(a, st, k):
    den = a + st + _f32(1e-7)
    r = a / den
    sk = r * r if k == 2.0 else torch.pow(r, _f32(k))
    lo, hi = _f32(1e-6), _f32(1.0 - 1e-6)
    return den, r, sk, torch.minimum(torch.maximum(sk, lo), hi), lo, hi


def emer_pointwise_loss_fwd(kind, a, b, n, p0, p1, pre, post, out, workspace, stream):
    """Each element's term, then its sum over the counted elements divided by their count (the kernel sums per CTA in
    another order: values agree to rounding)."""
    _require(0 <= kind <= 8, f"emer_pointwise_loss_fwd: unknown kind {kind}")
    _require(_addr(a) and _addr(out) and _addr(workspace) and (kind == 7 or _addr(b)), "emer_pointwise_loss_fwd: NULL pointer")
    x = _vec(a, n)
    y = _vec(b, n) if kind != 7 else None
    p0f, pre_f = _f32(p0), _f32(pre)
    with torch.no_grad():
        counted = torch.ones(n, dtype=torch.bool)
        if kind <= 2:
            term = _real_term(kind, x - y) * pre_f
        elif kind <= 5:
            counted = (y > 0.01) & (y < p0f)
            nd = lambda v: torch.clamp(v / p0f, 0.0, 1.0)
            term = _real_term(kind - 3, nd(x) - nd(y))
        elif kind == 6:
            t = 1.0 - y
            term = (t - 1.0) * torch.clamp(torch.log(1.0 - x), min=-100.0) - t * torch.clamp(torch.log(x), min=-100.0)
        elif kind == 7:
            term = x.clone()
        else:
            _, _, _, c, _, _ = _entropy_parts(x, y, p0)
            term = -(c * torch.log(c)) + -(1.0 - c) * torch.log(1.0 - c)
        cnt = _f32(float(int(counted.sum())))
        o = _vec(out, 2)
        o[0] = term[counted].sum() / cnt * _f32(post)
        o[1] = cnt


def emer_pointwise_loss_bwd(kind, a, b, n, p0, p1, pre, post, fwd_out, g, da, db, stream):
    _require(0 <= kind <= 8, f"emer_pointwise_loss_bwd: unknown kind {kind}")
    _require(_addr(a) and _addr(fwd_out) and _addr(g) and (kind == 7 or _addr(b)), "emer_pointwise_loss_bwd: NULL pointer")
    _require(_addr(da) or (kind == 8 and _addr(db)), "emer_pointwise_loss_bwd: no gradient requested")
    if n <= 0:
        return
    x = _vec(a, n)
    y = _vec(b, n) if kind != 7 else None
    p0f = _f32(p0)
    with torch.no_grad():
        gs = _vec(g, 1)[0] * _f32(post) / _vec(fwd_out, 2)[1] * _f32(pre)
        if kind <= 2:
            _vec(da, n).copy_(_real_grad(kind, x - y, gs))
        elif kind <= 5:
            valid = (y > 0.01) & (y < p0f)
            xs = x / p0f
            dl = _real_grad(kind - 3, torch.clamp(xs, 0.0, 1.0) - torch.clamp(y / p0f, 0.0, 1.0), gs)
            keep = valid & (xs >= 0.0) & (xs <= 1.0)
            _vec(da, n).copy_(torch.where(keep, dl / p0f, torch.zeros_like(x)))
        elif kind == 6:
            t = 1.0 - y
            _vec(da, n).copy_(gs * (x - t) / torch.clamp((1.0 - x) * x, min=1e-12))
        elif kind == 7:
            _vec(da, n).fill_(gs)
        else:
            den, r, sk, c, lo, hi = _entropy_parts(x, y, p0)
            dc = gs * torch.log(1.0 - c) - gs * -(1.0 - c) / (1.0 - c) + -gs * torch.log(c) + -gs * c / c
            dsk = torch.where((sk >= lo) & (sk <= hi), dc, torch.zeros_like(dc))
            dr = dsk * (2.0 * r if p0 == 2.0 else p0f * torch.pow(r, _f32(p1)))
            dden = -dr * (r / den)
            if _addr(da):
                _vec(da, n).copy_(dr / den + dden)
            if _addr(db):
                _vec(db, n).copy_(dden)


def _ray_masks(t, gt, eps):
    lo, hi = gt[:, None] - _f32(eps), gt[:, None] + _f32(eps)
    return t < lo, (t > lo) & (t < hi)


def _dirac(t, gt, two_sigma_sq, amp):
    x = t - gt[:, None]
    return _f32(amp) * torch.exp(-(x * x) / _f32(two_sigma_sq))


def emer_ray_loss_fwd(kind, w, t, gt, n_rays, n_samples, eps, two_sigma_sq, amp, pre, post, out, workspace, stream):
    _require(kind in (0, 1, 2), f"emer_ray_loss_fwd: unknown kind {kind}")
    _require(_addr(w) and _addr(gt) and _addr(out) and _addr(workspace) and (kind == 1 or _addr(t)),
             "emer_ray_loss_fwd: NULL pointer")
    _require(n_rays >= 0 and n_samples >= 1, "emer_ray_loss_fwd: bad shape")
    W, G = _view(w, n_rays, n_samples), _vec(gt, n_rays)
    rays = _f32(float(n_rays))
    o = _vec(out, 2)
    with torch.no_grad():
        if kind in (0, 2):
            T = _view(t, n_rays, n_samples)
            empty, near = _ray_masks(T, G, eps)
            e = (W * W * empty).sum(-1)
            nr = ((W - _dirac(T, G, two_sigma_sq, amp)) ** 2 * near).sum(-1)
            cnt = _f32(float(int((G > 0).sum()))) if kind == 0 else rays
            sight = e.sum() / rays + nr.sum() / rays
            o[0] = sight * _f32(pre) * cnt / rays * _f32(post) if kind == 0 else sight * _f32(pre) * _f32(post)
            o[1] = cnt
        else:
            o[0] = ((W * W).sum(-1) * G).sum() / rays * _f32(post)
            o[1] = rays


def emer_ray_loss_bwd(kind, w, t, gt, n_rays, n_samples, eps, two_sigma_sq, amp, pre, post, fwd_out, g, dw, stream):
    _require(kind in (0, 1, 2), f"emer_ray_loss_bwd: unknown kind {kind}")
    _require(_addr(w) and _addr(gt) and _addr(fwd_out) and _addr(g) and _addr(dw) and (kind == 1 or _addr(t)),
             "emer_ray_loss_bwd: NULL pointer")
    if n_rays == 0:
        return
    W, G = _view(w, n_rays, n_samples), _vec(gt, n_rays)
    rays = _f32(float(n_rays))
    with torch.no_grad():
        gg = _vec(g, 1)[0] * _f32(post) / rays
        if kind in (0, 2):
            T = _view(t, n_rays, n_samples)
            if kind == 0:
                gr = gg * _f32(pre) * _vec(fwd_out, 2)[1] / rays
            else:
                gr = _vec(g, 1)[0] * _f32(post) * _f32(pre) / rays
            empty, near = _ray_masks(T, G, eps)
            d = torch.where(empty, 2.0 * W * gr, torch.zeros_like(W))
            d = torch.where(near, 2.0 * (W - _dirac(T, G, two_sigma_sq, amp)) * gr, d)
        else:
            d = 2.0 * W * (gg * G[:, None])
        _view(dw, n_rays, n_samples).copy_(d)


# ----------------------------------------------------------------------------- dispatch
ENTRY_POINTS = ("emer_pointwise_loss_fwd", "emer_pointwise_loss_bwd", "emer_ray_loss_fwd", "emer_ray_loss_bwd")


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: the loss entry points here, everything else in ``cabi_emulator``."""
    if name not in ENTRY_POINTS:
        return cabi_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib, _ops

    cabi_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(_ops, "_LOSS_WS", {})

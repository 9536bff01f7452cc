"""CPU emulator of the flow branch's entry points of the C ABI (emer_flow_warp_fwd / _bwd, emer_flow_field_fwd / _bwd;
csrc/flow_branch.cu, csrc/field_fused.cu) -- TEST INFRASTRUCTURE ONLY.

Host restatements through the same raw pointers, row strides and sizes the product hands to the library, with the
arithmetic of the reference lines (radiance_field.py:449-460) and of ``cabi_emulator``'s single-query chain.
``install(monkeypatch)`` installs ``cabi_emulator`` (the rest of the ABI) and routes these four entry points here, so
``RadianceField.forward`` with ``EMER_FLOW_BRANCH=fused`` runs on CPU tensors in the ``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import torch

import cabi_emulator
from cabi_emulator import _addr, _require, _vec, _view
from oracle import hotpath


def _warp(pos, flow, noise, t, aabb, td, unbounded, n):
    """[2n, 4] rows: the forward warp, then the backward warp (the reference's operation order)."""
    nz = noise[:, None]
    rows = []
    for d, sign in ((0, 1.0), (1, -1.0)):
        x = pos + flow[:, 3 * d:3 * d + 3] * nz
        xyz = hotpath.contract_points(x, aabb, bool(unbounded))
        w_t = torch.clamp(t + (sign * td) * noise, 0, 1.0)
        rows.append(torch.cat([xyz, w_t[:, None]], -1))
    return torch.cat(rows)


def _noise(noise, ld_noise, n):
    return _view(noise, n, 1, ld_noise)[:, 0] if _addr(noise) else torch.ones(n)


def emer_flow_warp_fwd(pos, flow, noise, ld_noise, t, aabb6, time_diff, unbounded, coords, n, stream):
    _require(all(_addr(p) for p in (pos, flow, t, aabb6, time_diff, coords)), "emer_flow_warp_fwd: NULL pointer")
    _require(_addr(coords) % 16 == 0, "emer_flow_warp_fwd: coords must be 16-byte aligned")
    if n == 0:
        return
    with torch.no_grad():
        _view(coords, 2 * n, 4).copy_(_warp(_view(pos, n, 3), _view(flow, n, 6), _noise(noise, ld_noise, n), _vec(t, n),
                                            _vec(aabb6, 6), _vec(time_diff, 1), unbounded, n))


def emer_flow_warp_bwd(pos, flow, noise, ld_noise, aabb6, unbounded, d_coords, d_flow, n, stream):
    _require(all(_addr(p) for p in (pos, flow, aabb6, d_coords, d_flow)), "emer_flow_warp_bwd: NULL pointer")
    if n == 0:
        return
    fl = _view(flow, n, 6).clone().requires_grad_(True)
    with torch.enable_grad():
        out = _warp(_view(pos, n, 3), fl, _noise(noise, ld_noise, n), torch.zeros(n), _vec(aabb6, 6), torch.zeros(1),
                    unbounded, n)
        g = _view(d_coords, 2 * n, 4).clone()
        g[:, 3] = 0.0
        (gf,) = torch.autograd.grad(out, fl, g)
    _view(d_flow, n, 6).copy_(gf)


def _chain(x, wb0, bb0, wb1, bb1, n_feat, n):
    """(hb [3n, 64], feats [n, n_feat]) of the three queries and their blend."""
    hb = torch.relu(x @ wb0.T + bb0)
    F = hb @ wb1.T + bb1
    return hb, (F[:n] + 0.5 * F[n:2 * n] + 0.5 * F[2 * n:]) / 2.0


def emer_flow_field_fwd(enc, ld_enc, k_enc, wb0, bb0, wb1, bb1, n_feat, w0g, ld_w0, w1h, w1g, ld_w1, w2, b2, ray_bias,
                        samples, sigma, rgb, save_hb, save_hg, save_h1, save_sem, n, stream):
    _require(k_enc in (40, 64), f"emer_flow_field_fwd: k_enc={k_enc} must be 40 or 64")
    _require(n_feat in (64, 128) and samples > 0, "emer_flow_field_fwd: bad shape")
    _require(not _addr(rgb) or _addr(ray_bias), "emer_flow_field_fwd: the colour head needs ray_bias")
    _require(_addr(save_hg) and (n_feat == 64 or _addr(save_sem)), "emer_flow_field_fwd: the blend needs save_hg")
    _require(ld_enc % 8 == 0 and cabi_emulator._aligned32(enc, save_hb, save_hg, save_h1, save_sem),
             "emer_flow_field_fwd: rows must be 32-byte aligned")
    if n == 0:
        return
    with torch.no_grad():
        hb, feats = _chain(_view(enc, 3 * n, k_enc, ld_enc), _view(wb0, 64, k_enc), _vec(bb0, 64), _view(wb1, n_feat, 64),
                           _vec(bb1, n_feat), n_feat, n)
        geo = feats[:, :64]
        _vec(sigma, n).copy_(torch.exp(feats[:, 0] - 1.0))
        hg = _view(save_hg, n, 128)
        hg[:, 64:] = geo
        if _addr(save_hb):
            _view(save_hb, 3 * n, 64).copy_(hb)
        if n_feat == 128:
            _view(save_sem, n, 64).copy_(feats[:, 64:])
        if not _addr(rgb):
            return
        n_rays = (n + samples - 1) // samples
        rb = _view(ray_bias, n_rays, 128)[torch.arange(n) // samples]
        h0 = torch.relu(geo @ _view(w0g, 64, 64, ld_w0).T + rb[:, :64])
        h1 = torch.relu(h0 @ _view(w1h, 64, 64, ld_w1).T + geo @ _view(w1g, 64, 64, ld_w1).T + rb[:, 64:])
        _view(rgb, n, 3).copy_(torch.sigmoid(h1 @ _view(w2, 3, 64).T + _vec(b2, 3)))
        hg[:, :64] = h0
        if _addr(save_h1):
            _view(save_h1, n, 64).copy_(h1)


def emer_flow_field_bwd(d_rgb, rgb, d_sigma, sigma, d_geo, d_sem, hb, hg, h1, wb0, k_enc, wb1, n_feat, w0g, ld_w0, w1h,
                        w1g, ld_w1, w2, dz2, dz1, d1, dzb, d_enc, ld_denc, d_ray_bias, d_sem_q, samples, n, stream):
    head = bool(_addr(h1))
    _require(all(_addr(p) for p in (sigma, hb, wb0, wb1, w0g, w1h, w1g, w2, d1, dzb)), "emer_flow_field_bwd: NULL pointer")
    _require(not head or (_addr(rgb) and _addr(hg) and _addr(dz1)), "emer_flow_field_bwd: colour head buffers")
    _require(head or not (_addr(d_rgb) or _addr(d_ray_bias) or _addr(dz2)), "emer_flow_field_bwd: density only")
    _require(not _addr(d_sem) or _addr(d_sem_q), "emer_flow_field_bwd: d_sem needs d_sem_q")
    _require(k_enc in (40, 64) and n_feat in (64, 128) and samples > 0, "emer_flow_field_bwd: bad shape")
    _require(not _addr(d_ray_bias) or samples % 32 == 0, "emer_flow_field_bwd: per-ray sums need samples % 32 == 0")
    if n == 0:
        return
    with torch.no_grad():
        D1 = _view(d1, 3 * n, 128)
        dF = torch.zeros(n, 64)
        if head:
            z2 = torch.zeros(n, 3)
            if _addr(d_rgb):
                y = _view(rgb, n, 3)
                z2 = _view(d_rgb, n, 3) * (y * (1.0 - y))
                if _addr(dz2):
                    _view(dz2, n, 3).copy_(z2)
            z1 = (z2 @ _view(w2, 3, 64)) * (_view(h1, n, 64) > 0)
            _view(dz1, n, 64).copy_(z1)
            z0 = (z1 @ _view(w1h, 64, 64, ld_w1)) * (_view(hg, n, 64, 128) > 0)
            dF = z1 @ _view(w1g, 64, 64, ld_w1) + z0 @ _view(w0g, 64, 64, ld_w0)
            D1[:n, :64] = z0
            if _addr(d_ray_bias):
                acc = _view(d_ray_bias, (n + samples - 1) // samples, 128)
                ray = torch.arange(n) // samples
                acc[:, :64].index_add_(0, ray, z0)
                acc[:, 64:].index_add_(0, ray, z1)
        if _addr(d_geo):
            dF = dF + _view(d_geo, n, 64)
        if _addr(d_sigma):
            dF[:, 0] += _vec(d_sigma, n) * torch.clamp(_vec(sigma, n), max=3269017.25)
        wb1_ = _view(wb1, n_feat, 64)
        for q, s in enumerate((0.5, 0.25, 0.25)):
            rows = slice(q * n, (q + 1) * n)
            D1[rows, 64:] = dF * s
            dhb = (dF * s) @ wb1_[:64]
            if n_feat == 128 and _addr(d_sem):
                ds = _view(d_sem, n, 64) * s
                _view(d_sem_q, 3 * n, 64)[rows] = ds
                dhb = dhb + ds @ wb1_[64:]
            zb = dhb * (_view(hb, 3 * n, 64)[rows] > 0)
            _view(dzb, 3 * n, 64)[rows] = zb
            if _addr(d_enc):
                _view(d_enc, 3 * n, k_enc, ld_denc)[rows] = zb @ _view(wb0, 64, k_enc)


ENTRY = {f.__name__: f for f in (emer_flow_warp_fwd, emer_flow_warp_bwd, emer_flow_field_fwd, emer_flow_field_bwd)}


def install(monkeypatch) -> None:
    """``cabi_emulator.install`` plus the four flow-branch entry points."""
    from emernerf_b200 import _lib

    cabi_emulator.install(monkeypatch)
    rest = _lib.call

    def call(name, *args):
        fn = ENTRY.get(name)
        if fn is None:
            return rest(name, *args)
        cabi_emulator.CALLS.append(name)
        fn(*[a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args])

    monkeypatch.setattr(_lib, "call", call)

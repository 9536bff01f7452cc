"""CPU emulator of the rendering entry points of the C ABI (emer_render_fwd / _bwd; csrc/render.cu) -- TEST
INFRASTRUCTURE ONLY.

Host restatements through the same host structs, raw pointers, row strides and sizes the product hands to the library:
the forward is ``oracle.hotpath.rendering`` (the reference's ``rendering``) on fp32 views of the inputs, the backward
autograd through it.  ``install(monkeypatch)`` installs ``cabi_emulator`` for the rest of the ABI and routes these two
entry points here, so ``render_rays`` with ``EMER_RENDERING=fused`` runs on CPU tensors in the ``-m "not gpu"`` suite.
"""
from __future__ import annotations

import ctypes

import torch

import cabi_emulator
from cabi_emulator import _addr, _require, _view
from oracle import hotpath

# emer_render_in field -> the results key of the reference's query_fn
_RESULT_KEYS = {"sigma": "density", "sigma_s": "static_density", "sigma_d": "dynamic_density", "rgb": "rgb",
                "rgb_s": "static_rgb", "rgb_d": "dynamic_rgb", "shadow": "shadow_ratio", "rgb_sky": "rgb_sky",
                "dino": "dino_feat", "dino_s": "static_dino_feat", "dino_d": "dynamic_dino_feat",
                "dino_sky": "dino_sky_feat", "dino_pe": "dino_pe"}
# emer_render_out field -> the reference's output key
_OUT_KEYS = {"dino": "dino_feat"}
RENDER_MAX_CHANNELS = 32 * 8        # render.cu: RENDER_MAX_PER_LANE = 8


def _struct(ref):
    return ref._obj if hasattr(ref, "_obj") else ref


def _inputs(cin, what):
    """(t0, t1, results dict of [R,S,...] views, R, S) after the library's argument checks."""
    _require(cin.t0 and cin.t1 and cin.sigma, f"{what}: NULL pointer")
    r, s, c = cin.n_rays, cin.n_samples, cin.n_dino
    _require(s >= 1, f"{what}: n_samples must be >= 1")
    _require(bool(cin.sigma_s) == bool(cin.sigma_d), f"{what}: sigma_s and sigma_d come together")
    _require(bool(cin.rgb_s) == bool(cin.rgb_d) and (not cin.rgb_s or cin.sigma_s),
             f"{what}: rgb_s and rgb_d come together, with sigma_s and sigma_d")
    _require(bool(cin.dino_s) == bool(cin.dino_d) and (not cin.dino_s or cin.sigma_s),
             f"{what}: dino_s and dino_d come together, with sigma_s and sigma_d")
    _require(not (cin.dino or cin.dino_s) or 1 <= c <= RENDER_MAX_CHANNELS, f"{what}: feature channels {c} out of range")
    _require(bool(cin.fwd_flow) == bool(cin.bwd_flow) and (not cin.fwd_flow or cin.ld_flow >= 3),
             f"{what}: flows need both directions and a row stride >= 3")
    cols = {"rgb": 3, "rgb_s": 3, "rgb_d": 3, "dino": c, "dino_s": c, "dino_d": c}
    res = {}
    for k, key in _RESULT_KEYS.items():
        p = getattr(cin, k)
        if not p:
            continue
        if k in ("rgb_sky", "dino_sky", "dino_pe"):
            res[key] = _view(p, r, 3 if k == "rgb_sky" else c)
        elif k in cols:
            res[key] = _view(p, r * s, cols[k]).reshape(r, s, cols[k])
        elif k == "shadow":
            res[key] = _view(p, r, s)[..., None]
        else:
            res[key] = _view(p, r, s)
    if cin.fwd_flow:
        res["forward_flow"] = _view(cin.fwd_flow, r * s, 3, cin.ld_flow).reshape(r, s, 3)
        res["backward_flow"] = _view(cin.bwd_flow, r * s, 3, cin.ld_flow).reshape(r, s, 3)
    return _view(cin.t0, r, s), _view(cin.t1, r, s), res, r, s


def _outputs(out, extras):
    """reference output key -> tensor, including the weights and transmittance"""
    got = {_OUT_KEYS.get(k, k): v for k, v in out.items() if k != "extras"}
    got["weights"], got["trans"] = extras["weights"], extras["trans"]
    return got


def emer_render_fwd(cin, cout, stream):
    cin, cout = _struct(cin), _struct(cout)
    if cin.n_rays == 0:
        return
    t0, t1, res, r, s = _inputs(cin, "emer_render_fwd")
    names = [k for k, _ in type(cout)._fields_ if getattr(cout, k)]
    decomp = any(k in names for k in ("static_opacity", "dynamic_opacity", "static_depth", "dynamic_depth",
                                      "static_rgb", "dynamic_rgb", "shadow", "forward_flow", "static_dino",
                                      "dynamic_dino", "shadow_reduced_static_rgb", "shadow_only_static_rgb"))
    _require(not decomp or cin.sigma_s, "emer_render_fwd: the decomposition needs sigma_s and sigma_d")
    with torch.no_grad():
        out = hotpath.rendering(t0, t1, res, return_decomposition=decomp)
    got = _outputs(out, out["extras"])
    for k in names:
        key = _OUT_KEYS.get(k, k)
        _require(key in got, f"emer_render_fwd: {k} asked for, but the inputs do not define it")
        v = got[key]
        _view(getattr(cout, k), r, v[0].numel() if v.dim() > 1 else 1).copy_(v.reshape(r, -1))


def emer_render_bwd(cin, weights, trans, grad, stream):
    cin, g = _struct(cin), _struct(grad)
    if cin.n_rays == 0:
        return
    t0, t1, res, r, s = _inputs(cin, "emer_render_bwd")
    _require(_addr(weights) and _addr(trans), "emer_render_bwd: NULL weights or trans")
    leaves = {}
    for k, key in _RESULT_KEYS.items():
        if key in res and getattr(g, "d_" + k):
            leaves[k] = res[key] = res[key].detach().clone().requires_grad_(True)
    with torch.enable_grad():
        out = hotpath.rendering(t0, t1, res)
        got = _outputs(out, out["extras"])
        outs, grads = [], []
        for k in ("weights", "trans", "opacity", "depth", "rgb", "shadow_ratio", "dino", "dino_pe_free"):
            p = getattr(g, "g_" + k)
            key = _OUT_KEYS.get(k, k)
            if p and key in got:
                v = got[key]
                outs.append(v)
                grads.append(_view(p, r, v.numel() // max(r, 1)).reshape(v.shape))
        ds = torch.autograd.grad(outs, list(leaves.values()), grads, allow_unused=True) if outs and leaves else []
    for (k, leaf), d in zip(leaves.items(), ds):
        dst = _view(getattr(g, "d_" + k), 1, leaf.numel())[0]
        dst.copy_(torch.zeros(leaf.numel()) if d is None else d.reshape(-1))


ENTRY_POINTS = ("emer_render_fwd", "emer_render_bwd")


def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: rendering here, everything else in ``cabi_emulator``."""
    if name not in ENTRY_POINTS:
        return cabi_emulator.call(name, *args)
    cabi_emulator.CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    globals()[name](*plain)


def install(monkeypatch) -> None:
    from emernerf_b200 import _lib

    cabi_emulator.install(monkeypatch)
    monkeypatch.setattr(_lib, "call", call)

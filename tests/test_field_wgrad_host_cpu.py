"""The host side of the one-launch weight gradients of the fused field chain (``emer_field_wgrad``) on CPU: the full-size
training pass of test_host_path_full_cpu.py with that entry point answered by a restatement below (same checks as
csrc/field_wgrad.cu, oracle arithmetic), so its argument list, strides, column-block destinations and gradient sinks
are checked against the vectors the reference's own Python produced (tests/golden/full_static.npz)."""
import os
import types

import numpy as np
import pytest
import torch

import cabi_emulator as em
import full_cases as fc
from helpers import GOLDEN_DIR, Golden, rel_err
from oracle import adapters


def emer_field_wgrad(enc, ld_enc, k_enc, hb, hg, h1, dz2, dz1, d1, dzb, d_sem, n_feat, dwb0, dbb0, dwb1, dbb1, dw0g, ld_w0,
                     dw1h, dw1g, ld_w1, dw2, db2, n, stream):
    if n == 0:
        return
    a = em._addr
    em._require(all(a(p) for p in (enc, hb, d1, dzb, dwb0, dbb0, dwb1, dbb1)), "emer_field_wgrad: NULL pointer")
    em._require(not a(dz2) or all(a(p) for p in (hg, h1, dz1, dw0g, dw1h, dw1g, dw2, db2)),
                "emer_field_wgrad: NULL pointer among the colour head's buffers")
    em._require(k_enc in (32, 40, 64) and n_feat in (64, 128), "emer_field_wgrad: bad shape")
    em._require(not a(d_sem) or n_feat == 128, "emer_field_wgrad: d_sem needs n_feat = 128")
    em._require(ld_enc % 4 == 0 and ld_enc >= k_enc, "emer_field_wgrad: ld_enc")
    em._require(not a(dz2) or (ld_w0 >= 64 and ld_w1 >= 64), "emer_field_wgrad: ld_w0 / ld_w1 shorter than a block")
    em._require(em._aligned16(enc, hb, hg, h1, dz2, dz1, d1, dzb, d_sem), "emer_field_wgrad: row buffers must be 16-byte aligned")
    D1, hb_ = em._view(d1, n, 128), em._view(hb, n, 64)
    em._bwd_weight(em._view(enc, n, k_enc, ld_enc), em._view(dzb, n, 64), em._view(dwb0, 64, k_enc), em._vec(dbb0, 64))
    em._bwd_weight(hb_, D1[:, 64:], em._view(dwb1, 64, 64), em._vec(dbb1, 64))
    if a(d_sem):
        em._bwd_weight(hb_, em._view(d_sem, n, 64), em._view(a(dwb1) + 64 * 64 * 4, 64, 64), em._vec(a(dbb1) + 64 * 4, 64))
    if a(dz2):
        h0, geo, z1 = em._view(hg, n, 64, 128), em._view(a(hg) + 64 * 4, n, 64, 128), em._view(dz1, n, 64)
        em._bwd_weight(geo, D1[:, :64], em._view(dw0g, 64, 64, ld_w0), None)
        em._bwd_weight(h0, z1, em._view(dw1h, 64, 64, ld_w1), None)
        em._bwd_weight(geo, z1, em._view(dw1g, 64, 64, ld_w1), None)
        em._bwd_weight(em._view(h1, n, 64), em._view(dz2, n, 3), em._view(dw2, 3, 64), em._vec(db2, 3))


@pytest.mark.parametrize("sinks", [False, True])
def test_full_size_gradients_through_one_weight_gradient_launch(sinks, monkeypatch):
    """``sinks``: FusedAdam's gradient buffers receive the weight gradients in place (the head's blocks as strided
    column blocks of the w0 / w1 buffers), or autograd gets them as tensors shaped like the parameters."""
    from emernerf_b200 import _ops
    from emernerf_b200.optim import FusedAdam
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder
    from emernerf_b200.radiance_fields.render_utils import render_rays
    from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator

    em.install(monkeypatch)
    monkeypatch.setattr(em, "emer_field_wgrad", emer_field_wgrad, raising=False)
    monkeypatch.setattr(_ops, "_field_wgrad_usable", lambda t: True)
    _ops.clear_grad_sinks()
    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField, build_density_field=build_density_field)
    field, props = fc.build_models(ns, "static")
    g = Golden.__new__(Golden)
    g.case, g.z = "static", np.load(os.path.join(GOLDEN_DIR, "full_static.npz"))
    field.load_state_dict(g.tensors("sd/field"), strict=False)
    [p.load_state_dict(g.tensors(f"sd/prop{i}"), strict=False) for i, p in enumerate(props)]
    if sinks:
        FusedAdam(field.parameters(), lr=1e-3)
    try:
        est = PropNetEstimator(None, None)
        field.train(); est.train()
        [p.train() for p in props]
        est._jitter_override, field._noise_override = g.jitters("train"), g.noise("train")
        out = render_rays(field, est, props, g.tensors("in/pixel"), fc.render_cfg(), proposal_requires_grad=True)
        keep = torch.from_numpy(g.z["train/stable"])
        del em.CALLS[:]
        adapters.parity_loss(fc.mask_rays(out, keep)).backward()
    finally:
        _ops.clear_grad_sinks()
    assert em.CALLS.count("emer_field_wgrad") == 1
    wg, wp = g.tensors("train/grad/field"), g.tensors("train/gradproj/field")
    n = 0
    for k, v in field.named_parameters():
        if k in wg:
            assert rel_err(v.grad, wg[k]) < 2e-5, (k, rel_err(v.grad, wg[k]))
            n += 1
        elif k in wp:
            got = fc.projections(v.grad, n_proj=4)
            assert float((got[:4] - wp[k][:4]).abs().max()) <= 2e-5 * float(wp[k][-1]), k
            assert abs(float(got[-1] - wp[k][-1])) <= 2e-5 * float(wp[k][-1]), k
            n += 1
    assert n == len(wg) + len(wp)

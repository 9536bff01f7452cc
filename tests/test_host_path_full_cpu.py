"""The host side of the product at the BENCHMARKED configuration, on CPU: the drop-in modules, the autograd wrappers
and -- what the miniature fixtures cannot reach, their 16-d grids are outside the fused kernel's shapes -- the FUSED
FIELD CHAIN's host logic (per-ray bias folding, weight column blocks, the backward walk over the saved activations,
ray-bias / embedding gradients through autograd, the one weight-gradient launch after either data path and its
gradient sinks) run through tests/cabi_emulator.py against the vectors the reference's own Python produced for the
full-size model (tests/golden/full_*.npz)."""
import os
import types

import numpy as np
import pytest
import torch

import cabi_emulator
import full_cases as fc
from helpers import GOLDEN_DIR, Golden, rel_err
from oracle import adapters


@pytest.mark.parametrize("sinks", [False, True])
@pytest.mark.parametrize("chain_bwd", ["fused", "layers"])
@pytest.mark.parametrize("variant", ["static"])       # ("dynamic" passes too: two fused launches; 60+ s of CPU time)
def test_full_size_training_pass_through_the_emulator(variant, chain_bwd, sinks, monkeypatch):
    """``chain_bwd``: the field chain's data gradients from emer_field_bwd or layer by layer (EMER_CHAIN_BWD), both
    followed by one emer_field_wgrad launch.  ``sinks``: FusedAdam's gradient buffers receive the weight gradients in
    place (the head's blocks as strided column blocks of the w0 / w1 buffers), or autograd gets them as tensors shaped
    like the parameters."""
    from emernerf_b200 import _ops
    from emernerf_b200.optim import FusedAdam
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder
    from emernerf_b200.radiance_fields.render_utils import render_rays
    from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator

    cabi_emulator.install(monkeypatch)
    monkeypatch.setattr(_ops, "CHAIN_BWD", chain_bwd)
    _ops.clear_grad_sinks()
    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField, build_density_field=build_density_field)
    field, props = fc.build_models(ns, variant)
    g = Golden.__new__(Golden)
    g.case, g.z = variant, np.load(os.path.join(GOLDEN_DIR, f"full_{variant}.npz"))
    field.load_state_dict(g.tensors("sd/field"), strict=False)
    [p.load_state_dict(g.tensors(f"sd/prop{i}"), strict=False) for i, p in enumerate(props)]
    # static branch and (without a flow field) the dynamic branch are one fused chain each
    n_chain = 1 if variant == "static" else 2
    if sinks:
        FusedAdam(field.parameters(), lr=1e-3)
    try:
        est = PropNetEstimator(None, None)
        field.train(); est.train()
        [p.train() for p in props]
        est._jitter_override, field._noise_override = g.jitters("train"), g.noise("train")
        out = render_rays(field, est, props, g.tensors("in/pixel"), fc.render_cfg(), proposal_requires_grad=True)
        assert cabi_emulator.CALLS.count("emer_field_fwd") == n_chain
        assert "emer_field_tail_fwd" not in cabi_emulator.CALLS
        want = g.nested("train/out")
        for k in ("rgb", "depth", "opacity", "shadow_ratio"):
            if k in want:
                assert rel_err(out[k], want[k]) < 2e-6, (k, rel_err(out[k], want[k]))
        for k in ("density", "static_density", "dynamic_density", "weights"):
            if k in want["extras"]:
                assert rel_err(out["extras"][k], want["extras"][k]) < 2e-6, k
        keep = torch.from_numpy(g.z["train/stable"])
        loss = adapters.parity_loss(fc.mask_rays(out, keep))
        assert abs(loss.item() - g.scalar("train/loss")) < 1e-6
        del cabi_emulator.CALLS[:]
        loss.backward()
    finally:
        _ops.clear_grad_sinks()
    assert cabi_emulator.CALLS.count("emer_field_bwd") == (n_chain if chain_bwd == "fused" else 0)
    assert cabi_emulator.CALLS.count("emer_field_wgrad") == n_chain
    wg, wp = g.tensors("train/grad/field"), g.tensors("train/gradproj/field")
    n = 0
    for k, v in field.named_parameters():
        if k in wg:
            assert rel_err(v.grad, wg[k]) < 2e-5, (k, rel_err(v.grad, wg[k]))
            n += 1
        elif k in wp:
            got = fc.projections(v.grad, n_proj=4)              # (the first 4 of the fixture's 16: CPU time)
            assert float((got[:4] - wp[k][:4]).abs().max()) <= 2e-5 * float(wp[k][-1]), k
            assert abs(float(got[-1] - wp[k][-1])) <= 2e-5 * float(wp[k][-1]), k
            n += 1
    assert n == len(wg) + len(wp)

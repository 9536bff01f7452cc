"""Golden vectors of the BENCHMARKED configuration (full_cases.py) from the REFERENCE's own Python on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_full.py [variant ...]

Same procedure as make_golden.py -- unmodified reference modules with the stand-ins of ``oracle.ref_shims``,
cross-checked against ``oracle.hotpath`` -- on 256 Waymo-shape rays x 64 samples with the 2^20 / 2^18-entry
tables, proposal samples [128, 64].  Writes ``tests/golden/full_<variant>.npz``: inputs, every parameter except
the hash tables (those are regenerated from the portable hash of full_cases.py; a checksum is stored), the
random draws, the reference's outputs for a train pass (with proposal loss, parity-loss gradients of the MLPs and
projections of the table gradients), an eval pass with decomposition and a lidar pass.
"""
from __future__ import annotations

import os
import sys
import time
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

warnings.filterwarnings("ignore", category=FutureWarning)

from oracle import ref_shims  # noqa: E402

ref_shims.install()

import full_cases as fc  # noqa: E402
from make_golden import check, flat  # noqa: E402
from oracle import adapters, hotpath  # noqa: E402
from radiance_fields import RadianceField, build_density_field  # noqa: E402  (reference)
from radiance_fields.encodings import HashEncoder  # noqa: E402  (reference)
from radiance_fields.render_utils import render_rays  # noqa: E402  (reference)
from third_party.nerfacc_prop_net import PropNetEstimator  # noqa: E402  (reference)

REF = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                            build_density_field=build_density_field)
SEED_RENDER = 777


def stable_rays(field, props, batch, training, prefix, base_t_vals, jitters=None, noise=None):
    """hotpath.sample_stability for one pass (same weights, same random draws)."""
    fsd = adapters.cpu_state_dict(field)
    psd = [adapters.cpu_state_dict(p) for p in props]
    fspec, pspec = adapters.spec_from_module(field), [adapters.spec_from_module(p) for p in props]

    def render(scale):
        with torch.no_grad():
            return hotpath.render_rays(fsd, fspec, psd, pspec, batch, num_samples=fc.NUM_SAMPLES,
                                       prop_samples=fc.PROP_SAMPLES, near_plane=fc.NEAR, far_plane=fc.FAR,
                                       training=training, prefix=prefix, jitters=jitters, noise=noise,
                                       prop_sigma_scale=scale)[0]

    return hotpath.sample_stability(render, base_t_vals)


def oracle_render(field, props, batch, training, prg, decomp, prefix, rec=None):
    fsd = adapters.cpu_state_dict(field, requires_grad=training)
    psd = [adapters.cpu_state_dict(p, requires_grad=training) for p in props]
    out, cache = hotpath.render_rays(
        fsd, adapters.spec_from_module(field), psd, [adapters.spec_from_module(p) for p in props], batch,
        num_samples=fc.NUM_SAMPLES, prop_samples=fc.PROP_SAMPLES, near_plane=fc.NEAR, far_plane=fc.FAR,
        training=training, proposal_requires_grad=prg, return_decomposition=decomp, prefix=prefix, rng_record=rec)
    return out, cache, fsd, psd


def table_keys(m):
    return [k for k, _ in m.named_parameters() if k.endswith("tcnn_encoding.params")]


def run(variant: str):
    t_start = time.time()
    store = {}
    field, props = fc.build_models(REF, variant)
    est = PropNetEstimator(torch.optim.Adam([q for p in props for q in p.parameters()], lr=0.01), None)
    cfg = fc.render_cfg()
    flat("sd/field", fc.small_state(field), store)
    for i, p in enumerate(props):
        flat(f"sd/prop{i}", fc.small_state(p), store)
    for k in table_keys(field):
        v = dict(field.named_parameters())[k].detach()
        store[f"table_check/field/{k}"] = np.array([v.double().sum().item(), v.double().abs().sum().item(),
                                                     float(v[12345]), float(v[-1])])

    # ---------------- train pass
    batch = fc.make_batch(variant)
    flat("in/pixel", batch, store)
    field.train(); [p.train() for p in props]; est.train()
    torch.manual_seed(SEED_RENDER)
    ref = render_rays(field, est, props, batch, cfg, proposal_requires_grad=True)
    rec = {}
    torch.manual_seed(SEED_RENDER)
    orc, cache, fsd, psd = oracle_render(field, props, batch, True, True, False, "", rec)
    check(f"{variant}/train", ref, orc)
    # the scalar losses (and their gradients) are taken over the rays whose samples are well-conditioned
    # (hotpath.sample_stability): on the others no two implementations place the samples alike
    keep = stable_rays(field, props, batch, True, "", ref["extras"]["t_vals"].detach(), rec["jitters"], rec.get("noise"))
    store["train/stable"] = keep.numpy()
    fc.mask_prop_cache(est.prop_cache, keep)
    prop_loss = est.compute_loss(ref["extras"]["trans"][keep], 1024.0)
    pnames = [(i, k) for i, p in enumerate(props) for k, _ in p.named_parameters()]
    pg = torch.autograd.grad(prop_loss, [q for p in props for q in p.parameters()], allow_unused=True)
    loss = adapters.parity_loss(fc.mask_rays(ref, keep))
    names = [k for k, _ in field.named_parameters()]
    fg = torch.autograd.grad(loss, [v for _, v in field.named_parameters()], allow_unused=True)

    fc.mask_prop_cache(cache, keep)
    o_prop_loss = hotpath.proposal_loss(cache, orc["extras"]["trans"][keep], (0.03, 0.003), 1024.0)
    assert abs(o_prop_loss.item() - prop_loss.item()) <= 1e-5 * max(1.0, abs(prop_loss.item()))
    o_loss = adapters.parity_loss(fc.mask_rays(orc, keep))
    ofg = torch.autograd.grad(o_loss, [fsd[k] for k in names], allow_unused=True)
    for k, a, b in zip(names, fg, ofg):
        if a is None:
            assert b is None or b.abs().max() == 0, k
            continue
        err = (a - b).abs().max().item() / max(1e-12, a.abs().max().item())
        assert err < 1e-4, f"oracle grad {k}: {err}"

    flat("train/out", ref, store)
    store["train/prop_loss"] = np.float32(prop_loss.item())
    store["train/loss"] = np.float32(loss.item())
    for k, g in zip(names, fg):
        if g is None:
            continue
        if k.endswith("tcnn_encoding.params"):
            store[f"train/gradproj/field/{k}"] = fc.projections(g).numpy()
        else:
            store[f"train/grad/field/{k}"] = g.numpy()
    for (i, k), g in zip(pnames, pg):
        if g is None:
            continue
        if k.endswith("tcnn_encoding.params"):
            store[f"train/gradproj/prop{i}/{k}"] = fc.projections(g).numpy()
        else:
            store[f"train/grad/prop{i}/{k}"] = g.numpy()
    for i, jt in enumerate(rec["jitters"]):
        store[f"train/jitter{i}"] = jt.numpy()
    if "noise" in rec:
        store["train/noise"] = rec["noise"].detach().numpy()

    # ---------------- eval pass with decomposition
    field.eval(); [p.eval() for p in props]; est.eval()
    with torch.no_grad():
        ref = render_rays(field, est, props, batch, cfg, return_decomposition=True)
        orc, _, _, _ = oracle_render(field, props, batch, False, False, True, "")
    check(f"{variant}/eval", ref, orc)
    flat("eval/out", ref, store)
    store["eval/stable"] = stable_rays(field, props, batch, False, "", ref["extras"]["t_vals"]).numpy()

    # ---------------- lidar pass (density only), training mode, no proposal grads
    lb = fc.make_batch(variant, seed=7, lidar=True)
    flat("in/lidar", lb, store)
    field.train(); [p.train() for p in props]; est.train()
    torch.manual_seed(SEED_RENDER + 1)
    ref = render_rays(field, est, props, lb, cfg, proposal_requires_grad=False, prefix="lidar_")
    rec = {}
    torch.manual_seed(SEED_RENDER + 1)
    orc, _, _, _ = oracle_render(field, props, lb, True, False, False, "lidar_", rec)
    check(f"{variant}/lidar", ref, orc)
    flat("lidar/out", ref, store)
    for i, jt in enumerate(rec["jitters"]):
        store[f"lidar/jitter{i}"] = jt.numpy()
    if "noise" in rec:
        store["lidar/noise"] = rec["noise"].detach().numpy()
    store["lidar/stable"] = stable_rays(field, props, lb, True, "lidar_", ref["extras"]["t_vals"].detach(),
                                        rec["jitters"], rec.get("noise")).numpy()
    print(f"  stable rays: train {int(store['train/stable'].sum())} eval {int(store['eval/stable'].sum())} "
          f"lidar {int(store['lidar/stable'].sum())} of {fc.N_RAYS}")

    path = os.path.join(HERE, f"full_{variant}.npz")
    np.savez_compressed(path, **store)
    print(f"full_{variant}: {len(store)} arrays, {os.path.getsize(path) / 1e6:.2f} MB, {time.time() - t_start:.0f} s")


if __name__ == "__main__":
    assert ref_shims.reference_available(), "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
    torch.set_num_threads(min(os.cpu_count() or 1, 16))
    for v in (sys.argv[1:] or fc.VARIANTS):
        run(v)

"""Generate the golden vectors by running the REFERENCE's own Python hot path on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden.py

For every case of ``cases.py`` this imports the unmodified reference modules
(``radiance_fields/*``, ``third_party/nerfacc_prop_net.py``) with the stand-ins of
``oracle.ref_shims`` for tiny-cuda-nn / nerfacc / omegaconf, renders a train pass
(stratified, proposal grads, parity-loss gradients), an eval pass with
decomposition and a lidar pass, cross-checks the functional oracle
(``oracle.hotpath``) against them, and writes ``tests/golden/<case>.npz`` holding
inputs, state-dicts, the random draws (jitter / temporal-aggregation noise) and the
reference outputs.  The tcnn / nerfacc arithmetic inside both comes from
``oracle.tcnn_ref`` / ``oracle.nerfacc_ref`` (parity unpinned, see ``oracle/__init__.py``).
"""
from __future__ import annotations

import os
import sys
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

import cases  # noqa: E402
from oracle import adapters, hotpath  # noqa: E402
from radiance_fields import RadianceField, build_density_field  # noqa: E402  (reference)
from radiance_fields.encodings import HashEncoder  # noqa: E402  (reference)
from radiance_fields.render_utils import render_rays  # noqa: E402  (reference)
from third_party.nerfacc_prop_net import PropNetEstimator  # noqa: E402  (reference)

REF = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                            build_density_field=build_density_field)
SEED_RENDER = 4242


def flat(prefix, d, store):
    for k, v in d.items():
        if isinstance(v, dict):
            flat(f"{prefix}/{k}", v, store)
        elif torch.is_tensor(v):
            store[f"{prefix}/{k}"] = v.detach().cpu().numpy()


def check(name, a, b, tol=2e-6):
    for k in a:
        if k == "extras":
            check(name + "/extras", a[k], b[k], tol)
            continue
        x, y = a[k].detach(), b[k].detach()
        assert x.shape == y.shape, (name, k, x.shape, y.shape)
        err = (x - y).abs().max().item() / max(1.0, x.abs().max().item())
        assert err <= tol, f"oracle != reference for {name}/{k}: {err}"
    assert set(a) == set(b), (name, set(a) ^ set(b))


def oracle_render(field, props, batch, training, prg, decomp, prefix, rec=None, jitters=None, noise=None):
    fsd = adapters.cpu_state_dict(field, requires_grad=training)
    psd = [adapters.cpu_state_dict(p, requires_grad=training) for p in props]
    out, cache = hotpath.render_rays(
        fsd, adapters.spec_from_module(field), psd, [adapters.spec_from_module(p) for p in props],
        batch, num_samples=cases.NUM_SAMPLES, prop_samples=cases.PROP_SAMPLES, near_plane=cases.NEAR,
        far_plane=cases.FAR, training=training, proposal_requires_grad=prg,
        return_decomposition=decomp, prefix=prefix, rng_record=rec, jitters=jitters, noise=noise)
    return out, cache, fsd, psd


def run_case(case: str):
    store = {}
    field, props = cases.build_models(REF, case)
    est = PropNetEstimator(torch.optim.Adam([q for p in props for q in p.parameters()], lr=0.01), None)
    cfg = cases.render_cfg()
    flat("sd/field", dict(field.state_dict()), store)
    for i, p in enumerate(props):
        flat(f"sd/prop{i}", dict(p.state_dict()), store)
    store["meta/time_diff"] = np.float32(field.time_diff if hasattr(field, "time_diff") else 0.0)

    # ---------------- train pass (pixel rays)
    batch = cases.make_batch(case)
    flat("in/pixel", batch, store)
    field.train(); [p.train() for p in props]; est.train()
    torch.manual_seed(SEED_RENDER)
    ref = render_rays(field, est, props, batch, cfg, proposal_requires_grad=True)
    prop_loss = est.compute_loss(ref["extras"]["trans"], 1024.0)
    pg = torch.autograd.grad(prop_loss, [q for p in props for q in p.parameters()], allow_unused=True)
    loss = adapters.parity_loss(ref)
    names = [k for k, v in field.named_parameters()]
    fg = torch.autograd.grad(loss, [v for _, v in field.named_parameters()], allow_unused=True)

    rec = {}
    torch.manual_seed(SEED_RENDER)
    orc, cache, fsd, psd = oracle_render(field, props, batch, True, True, False, "", rec)
    check(f"{case}/train", ref, orc)
    o_prop_loss = hotpath.proposal_loss(cache, orc["extras"]["trans"], (0.03, 0.003), 1024.0)
    assert abs(o_prop_loss.item() - prop_loss.item()) <= 1e-5 * max(1.0, abs(prop_loss.item()))
    o_loss = adapters.parity_loss(orc)
    ofg = torch.autograd.grad(o_loss, [fsd[k] for k in names], allow_unused=True)
    for k, a, b in zip(names, fg, ofg):
        if a is None:
            assert b is None or b.abs().max() == 0, k
            continue
        err = (a - b).abs().max().item() / max(1e-12, a.abs().max().item())
        assert err < 1e-4, f"grad {k}: {err}"

    flat("train/out", ref, store)
    store["train/prop_loss"] = np.float32(prop_loss.item())
    store["train/loss"] = np.float32(loss.item())
    for k, g in zip(names, fg):
        if g is not None:
            store[f"train/grad/field/{k}"] = g.numpy()
    j = 0
    for i, p in enumerate(props):
        for k, _ in p.named_parameters():
            if pg[j] is not None:
                store[f"train/grad/prop{i}/{k}"] = pg[j].numpy()
            j += 1
    for i, jt in enumerate(rec["jitters"]):
        store[f"train/jitter{i}"] = jt.numpy()
    if "noise" in rec:
        store["train/noise"] = rec["noise"].detach().numpy()

    # ---------------- eval pass with decomposition
    field.eval(); [p.eval() for p in props]; est.eval()
    with torch.no_grad():
        ref = render_rays(field, est, props, batch, cfg, return_decomposition=True)
        orc, _, _, _ = oracle_render(field, props, batch, False, False, True, "")
    check(f"{case}/eval", ref, orc)
    flat("eval/out", ref, store)

    # ---------------- lidar pass (density only), training mode, no proposal grads
    lb = cases.make_batch(case, seed=7, lidar=True)
    flat("in/lidar", lb, store)
    field.train(); [p.train() for p in props]; est.train()
    torch.manual_seed(SEED_RENDER + 1)
    ref = render_rays(field, est, props, lb, cfg, proposal_requires_grad=False, prefix="lidar_")
    rec = {}
    torch.manual_seed(SEED_RENDER + 1)
    orc, _, _, _ = oracle_render(field, props, lb, True, False, False, "lidar_", rec)
    check(f"{case}/lidar", ref, orc)
    flat("lidar/out", ref, store)
    for i, jt in enumerate(rec["jitters"]):
        store[f"lidar/jitter{i}"] = jt.numpy()
    if "noise" in rec:
        store["lidar/noise"] = rec["noise"].detach().numpy()

    path = os.path.join(HERE, f"{case}.npz")
    np.savez_compressed(path, **store)
    print(f"{case}: {len(store)} arrays, {os.path.getsize(path) / 1e6:.2f} MB")


def run_raygen():
    """raygen.npz: the reference's get_rays (datasets/base/pixel_source.py:39-76, executed from its source file) on
    seeded rays, per-ray and shared camera matrices (test_live_reference_variants.py)."""
    src = open(os.path.join(ref_shims.REFERENCE_ROOT, "datasets", "base", "pixel_source.py")).read()
    ns = {}
    exec("from torch import Tensor\nfrom typing import Tuple\nimport torch\n"
         + src[src.index("def get_rays("):src.index("class ScenePixelSource")], ns)
    g = torch.Generator().manual_seed(0)
    x, y = torch.randint(0, 960, (777,), generator=g).float(), torch.randint(0, 640, (777,), generator=g).float()
    c2w = torch.eye(4).repeat(777, 1, 1) + torch.randn(777, 4, 4, generator=g) * 0.3
    K = torch.tensor([[1030.0, 0, 480], [0, 1030, 320], [0, 0, 1]]).repeat(777, 1, 1)
    out = {"x": x, "y": y, "c2w": c2w, "K": K}
    for tag, (c, k) in (("per_ray", (c2w, K)), ("shared", (c2w[0], K[0]))):
        out.update({f"{tag}/{i}": t for i, t in enumerate(ns["get_rays"](x, y, c, k))})
    np.savez_compressed(os.path.join(HERE, "raygen.npz"), **{k: v.numpy() for k, v in out.items()})


if __name__ == "__main__":
    assert ref_shims.reference_available(), "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
    for c in (sys.argv[1:] or list(cases.CASES) + ["raygen"]):
        run_raygen() if c == "raygen" else run_case(c)

"""Option variants of the field / estimator: the DROP-IN against the REFERENCE's own classes.

Run by tests/test_live_reference_variants.py in a subprocess (C ABI answered by tests/cabi_emulator.py).  Built with the
reference's constructor arguments and seeds, the drop-in holds the reference's weights exactly; the maximum relative
error of every output, proposal loss and gradient against the reference's results stored in tests/golden/variants.npz
(shapes and SAMPLE seeded positions per tensor) is printed as JSON.  Covers the constructor options and data-dict shapes
of SURVEY.md section 8b that the shipped configs do not exercise.

    python tests/live_reference_variants.py [variant ...]
    EMER_REFERENCE_ROOT=<checkout of NVlabs/EmerNeRF> python tests/live_reference_variants.py --write [variant ...]

``--write`` runs the reference's own classes (with the oracle stand-ins for tiny-cuda-nn / nerfacc, oracle/ref_shims.py)
and stores what they compute.
"""
from __future__ import annotations

import json
import os
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(HERE, "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)
warnings.filterwarnings("ignore")
FIXTURES = os.path.join(HERE, "golden", "variants.npz")
WRITE = "--write" in sys.argv[1:]

if WRITE:
    from oracle import ref_shims

    ref_shims.install()
    from radiance_fields import RadianceField as RefField, build_density_field as ref_build_density  # noqa: E402
    from radiance_fields.encodings import HashEncoder as RefEncoder  # noqa: E402
    from radiance_fields.render_utils import render_rays as ref_render_rays  # noqa: E402
    from third_party.nerfacc_prop_net import PropNetEstimator as RefEstimator  # noqa: E402

import cabi_emulator  # noqa: E402
import cases  # noqa: E402
from emernerf_b200.radiance_fields import RadianceField, build_density_field  # noqa: E402
from emernerf_b200.radiance_fields.encodings import HashEncoder  # noqa: E402
from emernerf_b200.radiance_fields.render_utils import render_rays  # noqa: E402
from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator  # noqa: E402


class _Patch:
    """monkeypatch-like object for cabi_emulator.install outside pytest."""

    def setattr(self, obj, name, value):
        setattr(obj, name, value)


cabi_emulator.install(_Patch())

OURS = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                             build_density_field=build_density_field, render_rays=render_rays,
                             PropNetEstimator=PropNetEstimator)
if WRITE:
    REF = types.SimpleNamespace(HashEncoder=RefEncoder, RadianceField=RefField, build_density_field=ref_build_density,
                                render_rays=ref_render_rays, PropNetEstimator=RefEstimator)

BASE = dict(geometry_feature_dim=64, base_mlp_layer_width=64, head_mlp_layer_width=64, enable_cam_embedding=False,
            enable_img_embedding=True, num_cams=cases.N_CAMS, appearance_embedding_dim=16, semantic_feature_dim=64,
            feature_mlp_layer_width=64, feature_embedding_dim=64, enable_sky_head=True, enable_shadow_head=False,
            enable_feature_head=False, num_train_timesteps=cases.N_TIMESTEPS, interpolate_xyz_encoding=True,
            enable_learnable_pe=True, enable_temporal_interpolation=False, unbounded=True)

# name -> (field kwargs, dynamic grid?, flow grid?, batch edits, render cfg edits, estimator kwargs, mode)
VARIANTS = {
    "cam_embedding": (dict(enable_cam_embedding=True, enable_img_embedding=False), False, False, "cam_idx", {}, {}, "eval"),
    "no_embedding": (dict(enable_img_embedding=False), False, False, None, {}, {}, "eval"),
    "mean_embedding": ({}, False, False, "drop_idx", {}, {}, "eval"),          # novel view: no img_idx in the batch
    "bounded_aabb": (dict(unbounded=False), False, False, None, {}, {}, "eval"),
    "no_sky_head": (dict(enable_sky_head=False), False, False, None, {}, {}, "eval"),
    "narrow_widths": (dict(geometry_feature_dim=32, base_mlp_layer_width=32, head_mlp_layer_width=32,
                           appearance_embedding_dim=8), False, False, None, {}, {}, "eval"),
    "odd_geometry_width": (dict(geometry_feature_dim=15), False, False, None, {}, {}, "eval"),   # the class default
    "dynamic_no_shadow": ({}, True, False, None, {}, {}, "eval"),
    "feature_head_no_pe": (dict(enable_feature_head=True, enable_learnable_pe=False), True, True, "features", {}, {},
                           "eval"),
    "wide_embedding": (dict(appearance_embedding_dim=48), False, False, None, {}, {}, "train"),   # > 32: generic tail
    "wide_heads": (dict(head_mlp_layer_width=256, base_mlp_layer_width=256, geometry_feature_dim=128), True, False,
                   None, {}, {}, "train"),                 # layers the tensor-core kernels cannot hold -> CUDA-core path
    "wide_feature_head": (dict(enable_feature_head=True, feature_mlp_layer_width=256, feature_embedding_dim=384,
                               semantic_feature_dim=32), True, True, "features384", {}, {}, "train"),
    "dynamic_model_no_time": ({}, True, False, "drop_time", {}, {}, "eval"),      # no timestamps: static branch only
    "one_proposal": ({}, False, False, None, dict(num_samples_per_prop=[24], n_props=1), {}, "train"),
    "three_proposals": ({}, False, False, None, dict(num_samples_per_prop=[40, 24, 16], n_props=3), {}, "eval"),
    "many_samples": ({}, False, False, None, dict(num_samples_per_prop=[300, 280], num_samples=270), {}, "eval"),
    "sampling_lindisp": ({}, False, False, None, dict(sampling_type="lindisp"), {}, "eval"),
    "sampling_uniform": ({}, False, False, None, dict(sampling_type="uniform", far_plane=120.0), {}, "eval"),
    "train_stratified": ({}, True, False, None, {}, {}, "train"),
    "train_plain_pdf_loss": ({}, False, False, None, {}, dict(enable_anti_aliasing_loss=False), "train"),
}


def build(ns, kwargs, dynamic, flow, seed=0):
    torch.manual_seed(seed)
    enc = ns.HashEncoder(verbose=False, **cases.ENC_STATIC)
    dyn = ns.HashEncoder(verbose=False, **cases.ENC_DYN) if dynamic else None
    flw = ns.HashEncoder(verbose=False, **cases.ENC_FLOW) if flow else None
    kw = dict(BASE)
    kw.update(kwargs)
    field = ns.RadianceField(xyz_encoder=enc, dynamic_xyz_encoder=dyn, flow_xyz_encoder=flw, aabb=cases.AABB, **kw)
    field.register_normalized_training_timesteps(torch.linspace(0, 1, cases.N_TIMESTEPS),
                                                 time_diff=1.0 / cases.N_TIMESTEPS)
    props = []
    for e in cases.ENC_PROP:
        p = ns.build_density_field(n_input_dims=3, n_levels=e["n_levels"], max_resolution=e["max_resolution"],
                                   log2_hashmap_size=e["log2_hashmap_size"],
                                   n_features_per_level=e["n_features_per_level"], unbounded=kw["unbounded"])
        p.set_aabb(cases.AABB)
        props.append(p)
    return field, props


def randomise(field, props, seed=1):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in [field] + props:
            for k, v in m.named_parameters():
                if k.endswith("tcnn_encoding.params"):
                    v.copy_(torch.randn(v.shape, generator=g) * 0.5)


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()


def flatten(d, prefix, out):
    for k, v in d.items():
        if isinstance(v, dict):
            flatten(v, prefix + k + "/", out)
        else:
            out[prefix + k] = v


def run_side(ns, name):
    """Build the variant from ``ns`` (the reference's classes or the drop-in's), render, and in training mode take the
    proposal loss and the parameter gradients.  Returns {key: tensor}, or {"raises": "<type>: <message>"} when the
    render refuses the input (the same refusal on both sides is parity too)."""
    kwargs, dynamic, flow, edit, cfg_edit, est_kw, mode = VARIANTS[name]
    field, props = build(ns, kwargs, dynamic, flow)
    randomise(field, props)
    case = "flow_feat" if edit in ("features", "features384") else "static"
    batch = cases.make_batch(case)
    if edit == "features384":
        batch["features"] = torch.rand(batch["origins"].shape[0], 384, generator=torch.Generator().manual_seed(5))
    if edit == "cam_idx":
        batch["cam_idx"] = batch.pop("img_idx") % cases.N_CAMS
    elif edit == "drop_idx":
        batch.pop("img_idx")
    elif edit == "drop_time":
        batch.pop("normed_timestamps")
    cfg = cases.render_cfg()
    cfg_edit = dict(cfg_edit)
    n_props = cfg_edit.pop("n_props", None)
    if "num_samples" in cfg_edit:
        cfg.nerf.sampling.num_samples = cfg_edit.pop("num_samples")
    for k, v in cfg_edit.items():
        setattr(cfg.nerf.propnet, k, v)
    if n_props is not None:
        # drop one network, or append a third built like the second
        props = props[:n_props]
        while len(props) < n_props:
            e = cases.ENC_PROP[-1]
            torch.manual_seed(9)
            p = ns.build_density_field(n_input_dims=3, n_levels=e["n_levels"], max_resolution=e["max_resolution"],
                                       log2_hashmap_size=e["log2_hashmap_size"],
                                       n_features_per_level=e["n_features_per_level"], unbounded=True)
            p.set_aabb(cases.AABB)
            randomise(p, [], seed=3)
            props = props + [p]
    train = mode == "train"
    est = ns.PropNetEstimator(torch.optim.Adam([q for p in props for q in p.parameters()], lr=0.01), None, **est_kw)
    for m in (field, est, *props):
        m.train(train)
    with torch.set_grad_enabled(train):
        torch.manual_seed(77)
        try:
            out = ns.render_rays(field, est, props, dict(batch), cfg, proposal_requires_grad=train,
                                 return_decomposition=not train)
        except (AssertionError, ValueError, KeyError) as e:
            return {"raises": f"{type(e).__name__}: {e}"}
    res = {}
    flatten(out, "out/", res)
    if train:
        ploss = est.compute_loss(out["extras"]["trans"], 1024.0)
        res["prop_loss"] = ploss.detach().reshape(1)
        loss = (out["rgb"] - batch["pixels"]).square().mean() + out["depth"].mean() * 1e-2
        (loss + ploss).backward()
        for k, v in field.named_parameters():
            if v.grad is not None:
                res["grad/" + k] = v.grad
        for i, p in enumerate(props):
            for k, v in p.named_parameters():
                if v.grad is not None:
                    res[f"grad/prop{i}/" + k] = v.grad
    return res


SAMPLE = 256


def sample(res):
    """{key: tensor} -> {key: values at SAMPLE fixed seeded positions (all of them for smaller tensors), shape/key: shape}"""
    out = {}
    for k, v in res.items():
        if isinstance(v, str):
            out[k] = v
            continue
        flat = v.detach().reshape(-1)
        if flat.numel() > SAMPLE:
            flat = flat[torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:SAMPLE]]
        out[k] = flat
        out["shape/" + k] = torch.tensor(v.shape, dtype=torch.int64)
    return out


def compare_variant(name):
    """Errors of the drop-in against the stored reference results of one variant."""
    z = np.load(FIXTURES)
    want = {k[len(name) + 1:]: (str(z[k]) if z[k].dtype.kind == "U" else torch.from_numpy(z[k]))
            for k in z.files if k.startswith(name + "/")}
    got = sample(run_side(OURS, name))
    if "raises" in want or "raises" in got:
        assert str(want.get("raises")) == got.get("raises"), (name, want.get("raises"), got.get("raises"))
        return {"raises:" + got["raises"].split(":")[0]: 0.0}
    assert set(got) == set(want), (name, sorted(set(got) ^ set(want)))
    errs = {}
    for k, w in want.items():
        g = got[k]
        assert g.shape == w.shape, (name, k, g.shape, w.shape)
        if k.startswith("shape/"):
            assert torch.equal(g, w), (name, k, g, w)
        elif k == "prop_loss":
            errs[k] = abs(g.item() - w.item()) / max(1.0, abs(w.item()))
        else:
            errs[k[len("out/"):] if k.startswith("out/") else k] = rel(g, w)
    return errs


if __name__ == "__main__":
    names = [a for a in sys.argv[1:] if a != "--write"] or list(VARIANTS)
    if WRITE:
        assert ref_shims.reference_available(), "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
        arrays = dict(np.load(FIXTURES)) if os.path.exists(FIXTURES) else {}
        for name in names:
            for k, v in sample(run_side(REF, name)).items():
                arrays[f"{name}/{k}"] = np.array(v) if isinstance(v, str) else v.numpy()
        np.savez_compressed(FIXTURES, **arrays)
        sys.exit(0)
    out = {}
    for name in names:
        del cabi_emulator.CALLS[:]
        out[name] = {"errors": compare_variant(name), "calls": sorted(set(cabi_emulator.CALLS))}
    print("JSON:" + json.dumps(out))

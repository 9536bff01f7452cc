"""The drop-in claim, end to end, at the REAL configuration (needs a reference checkout in EMER_REFERENCE_ROOT).

The reference's own ``builders.py`` (unmodified, imported from EMER_REFERENCE_ROOT) builds the model and the
proposal estimator from the reference's own ``configs/default_config.yaml`` twice:

  ref   <file>   with the reference's classes (oracle stand-ins for tiny-cuda-nn / nerfacc)
                 -> saves the state-dicts, a ray batch and the rendered outputs
  ours  <file>   after ``emernerf_b200.install_dropin()`` (C ABI answered by tests/cabi_emulator.py)
                 -> loads them, renders the same rays through the reference's import names, prints the errors

Only ``omegaconf`` (annotation only) and ``datasets.base`` (annotation only; its real import chain needs timm) are
stubbed.  The configuration is default_config.yaml with every branch switched on (dynamic, flow, shadow, feature
head) so that every config key the builders read is exercised; table sizes are the real ones (203 MB of grids).
"""
from __future__ import annotations

import json
import os
import re
import sys
import types
import warnings

import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ["EMER_REFERENCE_ROOT"]
for p in (ROOT, HERE, os.path.join(HERE, "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)
warnings.filterwarnings("ignore")

N_RAYS, T = 40, 12


class Cfg(dict):
    """attribute-style access like OmegaConf's DictConfig (what builders.py / render_rays do with cfg)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


def to_cfg(o):
    if isinstance(o, dict):
        return Cfg({k: to_cfg(v) for k, v in o.items()})
    if isinstance(o, list):
        return [to_cfg(v) for v in o]
    if isinstance(o, str) and re.fullmatch(r"[+-]?\d+(\.\d*)?[eE][+-]?\d+", o):
        return float(o)                     # "1e-5": a float to OmegaConf (YAML 1.2), a string to PyYAML (YAML 1.1)
    return o


def load_cfg():
    with open(os.path.join(REF, "configs", "default_config.yaml")) as f:
        cfg = to_cfg(yaml.safe_load(f))
    head = cfg.nerf.model.head
    head.enable_dynamic_branch = True
    head.enable_flow_branch = True
    head.enable_shadow_head = True
    head.enable_feature_head = True
    # what train_emernerf.py:130-133 copies into the model section before calling the builders
    cfg.nerf.model.num_cams = cfg.data.pixel_source.num_cams
    cfg.nerf.model.unbounded = cfg.nerf.unbounded
    cfg.nerf.model.resume_from = cfg.resume_from
    return cfg


def dataset_stub():
    px = types.SimpleNamespace(features=None)
    return types.SimpleNamespace(num_train_timesteps=T, test_pixel_set=None, num_img_timesteps=T,
                                 unique_normalized_training_timestamps=torch.linspace(0, 1, T),
                                 aabb=torch.tensor([-25.0, -35.0, -2.0, 90.0, 45.0, 25.0]), pixel_source=px)


def stub_annotation_only_modules():
    if "omegaconf" not in sys.modules:
        m = types.ModuleType("omegaconf")
        m.OmegaConf = type("OmegaConf", (), {})
        sys.modules["omegaconf"] = m
    ds = types.ModuleType("datasets")
    ds.__path__ = []
    base = types.ModuleType("datasets.base")
    base.SceneDataset = type("SceneDataset", (), {})
    sys.modules["datasets"], sys.modules["datasets.base"] = ds, base


def make_batch():
    import cases

    b = cases.make_batch("flow_feat", seed=3, n_rays=N_RAYS)
    b["img_idx"] = torch.randint(0, T * 3, (N_RAYS,), generator=torch.Generator().manual_seed(8))
    return b


def build_with_reference_builders(cfg):
    """builders.py, verbatim: whatever ``radiance_fields`` / ``third_party`` resolve to builds the model."""
    import builders

    ds = dataset_stub()
    model = builders.build_model_from_cfg(cfg.nerf.model, ds, torch.device("cpu"))
    est, props = builders.build_estimator_and_propnet_from_cfg(cfg.nerf, cfg.optim, ds, torch.device("cpu"))
    return model, est, props


def render(model, est, props, batch, cfg):
    from radiance_fields.render_utils import render_rays          # the name train_emernerf.py imports

    for m in (model, est, *props):
        m.eval()
    with torch.no_grad():
        return render_rays(radiance_field=model, proposal_estimator=est, proposal_networks=props, data_dict=batch,
                           cfg=cfg, proposal_requires_grad=False, return_decomposition=True)


def flatten(d, prefix=""):
    out = {}
    for k, v in d.items():
        if isinstance(v, dict):
            out.update(flatten(v, prefix + k + "/"))
        else:
            out[prefix + k] = v
    return out


def main():
    mode, path = sys.argv[1], sys.argv[2]
    cfg = load_cfg()
    stub_annotation_only_modules()
    sys.path.insert(0, REF)
    if mode == "ref":
        from oracle import ref_shims

        ref_shims.install()
        torch.manual_seed(0)
        model, est, props = build_with_reference_builders(cfg)
        g = torch.Generator().manual_seed(1)
        with torch.no_grad():                       # give the scene structure (tcnn's own init is ~1e-4)
            for m in [model] + props:
                for k, v in m.named_parameters():
                    if k.endswith("tcnn_encoding.params"):
                        v.copy_(torch.randn(v.shape, generator=g) * 0.5)
        assert type(model).__module__ == "radiance_fields.radiance_field", type(model).__module__
        batch = make_batch()
        out = render(model, est, props, dict(batch), cfg)
        torch.save({"model": model.state_dict(), "props": [p.state_dict() for p in props], "batch": batch,
                    "out": flatten(out)}, path)
        print("JSON:" + json.dumps({"keys": sorted(flatten(out)), "n_params": sum(p.numel() for p in model.parameters())}))
    else:
        import cabi_emulator
        import emernerf_b200

        emernerf_b200.install_dropin()
        cabi_emulator.install(types.SimpleNamespace(setattr=setattr))
        blob = torch.load(path)
        model, est, props = build_with_reference_builders(cfg)
        assert type(model).__module__.startswith("emernerf_b200."), type(model).__module__
        assert type(est).__module__.startswith("emernerf_b200.") and type(props[0]).__module__.startswith("emernerf_b200.")
        model.load_state_dict(blob["model"])                       # strict: same keys, same shapes
        for p, sd in zip(props, blob["props"]):
            p.load_state_dict(sd)
        got = flatten(render(model, est, props, dict(blob["batch"]), cfg))
        want = blob["out"]
        assert set(got) == set(want), sorted(set(got) ^ set(want))
        errs = {}
        for k in want:
            a, b = got[k].double(), want[k].double()
            assert a.shape == b.shape, (k, a.shape, b.shape)
            errs[k] = ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()
        print("JSON:" + json.dumps({"errors": errs, "calls": sorted(set(cabi_emulator.CALLS))}))


if __name__ == "__main__":
    main()

"""INTEGRATION.md's two-line claim, executed on the reference's ENTRY SCRIPT (needs EMER_REFERENCE_ROOT).

After ``emernerf_b200.install_dropin()`` the import block of the reference's unmodified ``train_emernerf.py``
(lines 1-27: builders, loss, datasets, radiance_fields.render_utils, radiance_fields.video_utils,
third_party.nerfacc_prop_net, utils.*) is executed verbatim.  Third-party packages that this image does not have
(imageio, omegaconf, wandb, timm, skimage, plotly, matplotlib, ...) are answered by empty stand-in modules -- they
are dependencies of the reference's driver, not of the hot path; ``nerfacc`` and ``tinycudann`` are NOT stubbed:
the drop-in has to answer for them.

Checks: the overridden names resolve to this package, the non-overridden submodules
(``radiance_fields.video_utils``, ``third_party.feature_extractor``) still resolve to the reference's files, and
``loss/base.py``'s ``from nerfacc import accumulate_along_rays`` is answered (compute_line_of_sight_loss runs).
"""
from __future__ import annotations

import importlib.abc
import importlib.machinery
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ["EMER_REFERENCE_ROOT"]

# packages of the reference's driver / data / visualisation layers that are absent from this image
ABSENT_OK = ("imageio", "omegaconf", "wandb", "timm", "skimage", "plotly", "matplotlib", "cv2", "lpips", "open3d",
             "tensorflow", "waymo_open_dataset", "nuscenes", "pyquaternion", "xformers", "PIL", "sklearn", "kornia",
             "torchvision", "seaborn", "gdown", "trimesh", "scipy")


class _Anything(types.ModuleType):
    """A stand-in module: any attribute is a dummy class (usable as a base class, decorator or annotation)."""

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        obj = type(name, (), {"__init__": lambda self, *a, **k: None, "__call__": lambda self, *a, **k: None})
        setattr(self, name, obj)
        return obj


class StubFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def __init__(self):
        self.stubbed = []

    def find_spec(self, name, path=None, target=None):
        top = name.split(".")[0]
        if top in ABSENT_OK:
            try:
                real = importlib.machinery.PathFinder.find_spec(top)
            except Exception:
                real = None
            if real is None:
                return importlib.machinery.ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _Anything(spec.name)
        m.__path__ = []
        self.stubbed.append(spec.name)
        return m

    def exec_module(self, module):
        pass


def main():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    sys.path.insert(0, REF)
    finder = StubFinder()
    sys.meta_path.append(finder)               # last: only consulted for modules nothing else can find

    import cabi_emulator
    import emernerf_b200

    emernerf_b200.install_dropin()
    cabi_emulator.install(types.SimpleNamespace(setattr=setattr))

    with open(os.path.join(REF, "train_emernerf.py")) as f:
        lines = f.read().splitlines()
    end = next(i for i, l in enumerate(lines) if l.startswith("logger = "))
    block = "\n".join(lines[:end])
    assert "from radiance_fields.video_utils import render_pixels, save_videos" in block
    scope = {"__name__": "train_emernerf_imports"}
    exec(compile(block, os.path.join(REF, "train_emernerf.py"), "exec"), scope)

    import torch

    def origin(obj):
        return sys.modules[obj.__module__].__file__

    res = {
        "RadianceField": origin(scope["RadianceField"]),
        "DensityField": origin(scope["DensityField"]),
        "render_rays": origin(scope["render_rays"]),
        "PropNetEstimator": origin(scope["PropNetEstimator"]),
        "render_pixels": origin(scope["render_pixels"]),
        "builders": scope["builders"].__file__,
        "loss": scope["loss"].__file__,
        "nerfacc": sys.modules["nerfacc"].__file__,
        "stubbed": sorted(set(n.split(".")[0] for n in finder.stubbed)),
    }
    import third_party.feature_extractor as fe

    res["feature_extractor"] = fe.__file__
    # video_utils and builders must hold the DROP-IN's classes
    import radiance_fields.video_utils as vu

    assert vu.RadianceField is scope["RadianceField"] and vu.render_rays is scope["render_rays"]
    assert scope["builders"].PropNetEstimator is scope["PropNetEstimator"]

    # loss/base.py's nerfacc import is answered: the line-of-sight loss runs (host side through the emulator)
    from loss.base import compute_line_of_sight_loss

    g = torch.Generator().manual_seed(0)
    w = torch.rand(6, 16, generator=g) * 0.1
    t = torch.sort(torch.rand(6, 16, generator=g) * 50, dim=-1).values
    gt = torch.rand(6, 1, generator=g) * 40 + 2
    got = compute_line_of_sight_loss(gt, w, t)
    eps = 2.0
    gd = gt.squeeze().unsqueeze(-1)
    dirac = (1 / (2 * torch.pi * (eps / 3) ** 2) ** 0.5) * torch.exp(-((t - gd) ** 2) / (2 * (eps / 3) ** 2))
    want = ((w.square() * (t < gd - eps)).sum(-1, keepdim=True).mean()
            + ((w - dirac).square() * ((t > gd - eps) & (t < gd + eps))).sum(-1, keepdim=True).mean()) * (gt.squeeze() > 0)
    res["los_err"] = float((got - want).abs().max())
    print("JSON:" + json.dumps(res))


if __name__ == "__main__":
    main()

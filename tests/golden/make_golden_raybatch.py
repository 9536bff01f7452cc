"""Generate tests/golden/raybatch.npz by running the REFERENCE's own ``ScenePixelSource.get_train_rays`` and
``SceneLidarSource.get_train_rays`` on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_raybatch.py

The reference's modules are loaded unmodified (their data-loading imports -- omegaconf, PIL, tqdm, the feature
extractor -- are stood in for by empty modules, as sampling never reaches them).  Each case of ``raybatch_cases``
fills a bare instance of the reference's class (``__abstractmethods__`` cleared, ``__init__`` not run) and calls
``get_train_rays`` under ``torch.manual_seed`` for its calls in turn; the file keeps every output of every call and
eight ``torch.rand`` draws taken after the last call, which pin where the reference leaves the generator.
"""
from __future__ import annotations

import importlib.machinery
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import raybatch_cases as rc  # noqa: E402

REFERENCE_ROOT = os.environ.get("EMER_REFERENCE_ROOT", "")


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, None)
    m.__dict__.update(attrs)
    sys.modules.setdefault(name, m)
    return sys.modules[name]


def load_reference(rel: str, name: str):
    _stub("omegaconf", OmegaConf=type("OmegaConf", (), {}))
    _stub("third_party").__path__ = []
    _stub("third_party.feature_extractor", delete_features=None, extract_and_save_features=None)
    _stub("utils").__path__ = []
    _stub("utils.misc", get_robust_pca=None)
    for opt, attr in (("PIL", "Image"), ("tqdm", "tqdm")):
        if importlib.util.find_spec(opt) is None:
            _stub(opt, **{attr: None})
    spec = importlib.util.spec_from_file_location(name, os.path.join(REFERENCE_ROOT, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def bare(cls):
    cls.__abstractmethods__ = frozenset()
    return object.__new__(cls)


def main():
    assert os.path.isfile(os.path.join(REFERENCE_ROOT, "datasets", "base", "pixel_source.py")), \
        "set EMER_REFERENCE_ROOT to a checkout of the reference"
    ps = load_reference("datasets/base/pixel_source.py", "reference_pixel_source")
    ls = load_reference("datasets/base/lidar_source.py", "reference_lidar_source")
    out = {}
    for case, (_, _, _, _, rays, calls, seed) in rc.PIXEL_CASES.items():
        src = rc.fill_pixel(bare(ps.ScenePixelSource), case)
        torch.manual_seed(seed)
        for c in range(calls):
            batch = src.get_train_rays(rays, candidate_indices=rc.pixel_candidates(case))
            out[f"pixel/{case}/{c}/keys"] = np.array(list(batch))
            for k, v in batch.items():
                out[f"pixel/{case}/{c}/{k}"] = v.numpy()
        out[f"pixel/{case}/after"] = torch.rand(8).numpy()
    for case, (sets, rays, seed) in rc.LIDAR_CASES.items():
        src = rc.fill_lidar(bare(ls.SceneLidarSource), case)
        torch.manual_seed(seed)
        for c in range(len(sets)):
            batch = src.get_train_rays(rays, candidate_indices=rc.lidar_candidates(case, c))
            out[f"lidar/{case}/{c}/keys"] = np.array(list(batch))
            for k, v in batch.items():
                out[f"lidar/{case}/{c}/{k}"] = v.numpy()
        out[f"lidar/{case}/after"] = torch.rand(8).numpy()
    path = os.path.join(HERE, "raybatch.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()

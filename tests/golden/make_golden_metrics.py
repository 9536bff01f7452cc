"""Generate tests/golden/metrics.npz by running the REFERENCE's own datasets/metrics.py on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_metrics.py

Loads the unmodified ``datasets/metrics.py`` file with stand-ins for its ``skimage`` import (its compute_ssim is not
part of the fixture: the SSIM yardstick is ``oracle.metrics_ref``) and its ``radiance_fields`` import (a type used only
by the kNN evaluation), runs every case of ``metric_cases.py`` and writes the inputs and each returned value.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import metric_cases as mc  # noqa: E402

REFERENCE_ROOT = os.environ.get("EMER_REFERENCE_ROOT", "")


def load_reference_metrics():
    def unavailable(*a, **k):
        raise RuntimeError("skimage stand-in: structural_similarity is not part of this fixture")

    sk = types.ModuleType("skimage")
    sk.__path__ = []
    skm = types.ModuleType("skimage.metrics")
    skm.structural_similarity = unavailable
    rf = types.ModuleType("radiance_fields")
    rf.RadianceField = type("RadianceField", (), {})
    sys.modules.update({"skimage": sk, "skimage.metrics": skm, "radiance_fields": rf})
    spec = importlib.util.spec_from_file_location("reference_metrics",
                                                  os.path.join(REFERENCE_ROOT, "datasets", "metrics.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    torch.set_num_threads(1)                       # a fixed CPU reduction order
    ref = load_reference_metrics()
    x = mc.make_inputs()
    store = {f"in/{k}": v.numpy() for k, v in x.items()}
    for case, fn, keys in mc.CASES:
        got = getattr(ref, fn)(*(x[k] for k in keys))
        if isinstance(got, dict):
            for k in mc.FLOW_KEYS:
                store[f"{case}/{k}"] = np.array(got[k], np.float64)
        else:
            store[f"{case}/value"] = np.array(got, np.float64)
        print(f"{case:16s} {got}")
    path = os.path.join(HERE, "metrics.npz")
    np.savez_compressed(path, **store)
    print(f"metrics: {len(store)} arrays, {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    assert os.path.isfile(os.path.join(REFERENCE_ROOT, "datasets", "metrics.py")), \
        "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
    main()

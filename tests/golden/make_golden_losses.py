"""Generate tests/golden/losses.npz by running the REFERENCE's own loss/base.py on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_losses.py

Imports the unmodified ``loss`` package with the stand-ins of ``oracle.ref_shims`` (nerfacc's accumulate_along_rays),
runs every case of ``loss_cases.py`` with autograd and writes, per case, the returned key and value and the gradient of
the value w.r.t. each input that takes one; plus a digest of the seeded inputs (the tests regenerate them), the
line-of-sight helper's [R] result, and the parameter
names and defaults of every class's constructor and ``__call__`` (so that the tests never read the reference).
"""
from __future__ import annotations

import inspect
import json
import os
import sys
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

import loss_cases as lc  # noqa: E402
import loss as ref_loss  # noqa: E402  (reference)


def _default(v):
    return None if v is inspect.Parameter.empty else v


def signatures():
    out = {}
    for name in lc.CLASSES:
        cls = getattr(ref_loss, name)
        out[name] = {fn: [(p.name, _default(p.default)) for p in inspect.signature(getattr(cls, fn)).parameters.values()
                          if p.name != "self"] for fn in ("__init__", "__call__")}
    for name in lc.FUNCTIONS:
        out[name] = [(p.name, _default(p.default)) for p in inspect.signature(getattr(ref_loss, name)).parameters.values()]
    return out


def main():
    torch.set_num_threads(1)                       # a fixed CPU reduction order
    x = lc.make_inputs()
    store = {f"in_digest/{k}": v.numpy() for k, v in lc.digest(x).items()}
    keys = {}
    for c in lc.CASES:
        case = c[0]
        key, value, grads = lc.run_case(ref_loss, x, c)
        keys[case] = key
        store[f"{case}/value"] = value.detach().numpy()
        for a, gr in grads.items():
            store[f"{case}/grad/{a}"] = gr.numpy()
        print(f"{case:22s} {key:28s} {value.item():.8g}")
    for eps in (6.0, 2.5):
        w = x["weights"].clone().requires_grad_()
        v = ref_loss.compute_line_of_sight_loss(x["lidar_ranges"], w, x["t_vals"], eps)
        store[f"fn/los_{eps}/value"] = v.detach().numpy()
        store[f"fn/los_{eps}/grad/weights"] = torch.autograd.grad(v.sum(), w)[0].numpy()
    store["meta/keys"] = np.array(json.dumps(keys))
    store["meta/signatures"] = np.array(json.dumps(signatures()))
    path = os.path.join(HERE, "losses.npz")
    np.savez_compressed(path, **store)
    print(f"losses: {len(store)} arrays, {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    assert ref_shims.reference_available(), "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
    main()

"""Generate tests/golden/errormap.npz by running the REFERENCE's own ``ScenePixelSource.get_render_rays`` and
``update_pixel_error_maps`` on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_errormap.py

The reference's module is loaded unmodified, as make_golden_raybatch.py loads it.  Each source of
``errormap_cases`` fills a bare instance of the reference's class; ``get_render_rays`` runs for a few images at every
downscale, and ``update_pixel_error_maps`` on every set of render results.  The file keeps every output.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import errormap_cases as ec  # noqa: E402
from make_golden_raybatch import REFERENCE_ROOT, bare, load_reference  # noqa: E402


def main():
    assert os.path.isfile(os.path.join(REFERENCE_ROOT, "datasets", "base", "pixel_source.py")), \
        "set EMER_REFERENCE_ROOT to a checkout of the reference"
    ps = load_reference("datasets/base/pixel_source.py", "reference_pixel_source")
    out = {}
    for case in ec.SOURCES:
        for name, d in ec.DOWNSCALES.items():
            src = ec.fill(bare(ps.ScenePixelSource), case, d)
            for i in ec.IMAGES[name]:
                rays = src.get_render_rays(i)
                out[f"rays/{case}/{name}/{i}/keys"] = np.array(list(rays))
                for k, v in rays.items():
                    out[f"rays/{case}/{name}/{i}/{k}"] = v.numpy()
    for case in ec.UPDATES:
        src = ec.fill(bare(ps.ScenePixelSource), "full")
        src.update_pixel_error_maps(ec.render_results(case))
        out[f"update/{case}"] = src.pixel_error_maps.numpy()
    path = os.path.join(HERE, "errormap.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()

"""Generate tests/golden/trajectory.npz: the items ``trajectory_cases.golden_items`` picks of every case, with the
pose interpolated in fp64 by oracle/trajectory_ref.py and the rays from the REFERENCE's own ``get_rays`` on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_trajectory.py

The reference's module is loaded unmodified, as make_golden_raybatch.py loads it.  The reference has no trajectory
code: what the file pins is that the frames are the reference's rays of the interpolated poses.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import trajectory_cases as tc  # noqa: E402
from make_golden_raybatch import REFERENCE_ROOT, load_reference  # noqa: E402
from oracle import trajectory_ref  # noqa: E402


def main():
    assert os.path.isfile(os.path.join(REFERENCE_ROOT, "datasets", "base", "pixel_source.py")), \
        "set EMER_REFERENCE_ROOT to a checkout of the reference"
    ps = load_reference("datasets/base/pixel_source.py", "reference_pixel_source")
    out = {}
    for case, (name, d, m, offset) in tc.CASES.items():
        src = tc.source(name, d)
        for k in tc.golden_items(case):
            a, b, i, c = tc.segment(name, m, k)
            rays = trajectory_ref.frame_rays(src, a, b, i, m, c, offset, get_rays=ps.get_rays)
            out[f"{case}/{k}/keys"] = np.array(list(rays))
            for key, v in rays.items():
                out[f"{case}/{k}/{key}"] = v.numpy()
    path = os.path.join(HERE, "trajectory.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()

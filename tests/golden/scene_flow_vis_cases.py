"""The fixture of the scene-flow figure (tests/golden/scene_flow_vis.npz, written by make_golden_scene_flow_vis.py from
the reference's own ``visualize_scene_flow``, ``get_valid_lidar_mask`` and ``scene_flow_to_rgb``).

It is built on ``lidar_flow_cases``: its ``flow_feat`` field with the density shift of tests/golden/lidar_flow.npz (so
the dynamic densities straddle the 0.2 gate, with the points near the gate already dropped there), its scans and its
sources.  The labels are that fixture's, with every seventh point's replaced in turn by a zero flow, a flow on the
x axis, a flow at the atan2 branch cut (y = +0 or -0 with x < 0) and a flow longer than the colour radius 2.  A
``pixel_source`` adds ``NUM_CAMS`` cameras per split position with intrinsics, poses, ``WIDTH`` and ``HEIGHT``; the
poses depend on the position in the split (the reference's camera index), not on the scan.  The split repeats the
scans so that positions 0, 10 and 20 are drawn; position 10 of the "drive" source is its scan without labels.

The generator drops the points within ``MARGIN`` relative of an image edge or of depth 0 in any camera; the fixture
stores which candidates each scan keeps.
"""
from __future__ import annotations

import math
import types
from typing import Dict

import numpy as np
import torch

import lidar_flow_cases as lc

NUM_CAMS = 3
WIDTH, HEIGHT = 160, 60
FOCAL = 80.0
YAWS = (0.0, 1.2, 3.3)           # camera headings (radians): cameras 0 and 1 overlap, the rest of the circle is unseen
MARGIN = 1e-4
CASES = {"drive": "drive", "unsorted": "unsorted"}     # case -> lidar_flow_cases source
SPLIT = [s % lc.N_SCANS for s in range(24)]
SPLIT[10], SPLIT[20] = 3, 5


def cam_to_world(i: int, c: int) -> torch.Tensor:
    """OpenCV axes (x right, y down, z forward) of camera c at split position i, as columns, and its centre."""
    scan = SPLIT[i]
    yaw = YAWS[c] + 0.05 * i
    fwd = torch.tensor([math.cos(yaw), math.sin(yaw), -0.05 * (c - 1)], dtype=torch.float64)
    fwd = fwd / fwd.norm()
    up = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
    right = torch.linalg.cross(fwd, up)
    right = right / right.norm()
    down = torch.linalg.cross(fwd, right)
    m = torch.eye(4, dtype=torch.float64)
    m[:3, 0], m[:3, 1], m[:3, 2] = right, down, fwd
    m[:3, 3] = torch.tensor([1.5 * scan + 0.1 * c, 0.2 * c, 2.0 + 0.01 * i], dtype=torch.float64)
    return m.float()


def intrinsics(i: int, c: int) -> torch.Tensor:
    f = FOCAL * (1.0 + 0.1 * c)
    return torch.tensor([[f, 0.0, WIDTH / 2 + 3.0 * c], [0.0, f, HEIGHT / 2 - 2.0 * c], [0.0, 0.0, 1.0]])


class PixelSource:
    def __init__(self, device="cpu"):
        n = len(SPLIT)
        self.num_cams, self.WIDTH, self.HEIGHT = NUM_CAMS, WIDTH, HEIGHT
        self.intrinsics = torch.stack([intrinsics(i, c) for i in range(n) for c in range(NUM_CAMS)]).to(device)
        self.cam_to_worlds = torch.stack([cam_to_world(i, c) for i in range(n) for c in range(NUM_CAMS)]).to(device)


def special_labels(labels: torch.Tensor) -> torch.Tensor:
    """Every seventh label replaced in turn by the flows whose colours sit on an edge of the formula."""
    out = labels.clone()
    j = torch.arange(len(out))
    kinds = [(0, torch.tensor([0.0, 0.0, 0.0])), (1, torch.tensor([0.7, 0.0, 0.1])),
             (2, torch.tensor([-0.4, 0.0, 0.0])), (3, torch.tensor([-0.9, -0.0, 0.2])),
             (4, torch.tensor([-1.3, 0.0, -0.1]))]
    for k, v in kinds:
        out[(j % 35) == 7 * k] = v
    big = (j % 7) == 5
    out[big] = out[big] * 6.0 + torch.sign(out[big]) * 2.5
    return out


def base_scans(z, source: str):
    keeps = {s: torch.from_numpy(z[f"{source}/scan{s}/keep"]) for s in range(lc.N_SCANS)}
    labels = {s: special_labels(torch.from_numpy(z[f"{source}/scan{s}/labels"])) for s in range(lc.N_SCANS)}
    return keeps, labels


def drop(keeps: Dict[int, torch.Tensor], labels: Dict[int, torch.Tensor], firm: Dict[int, np.ndarray]):
    """The scans without the candidates the generator found too near an image edge (``firm`` per kept candidate)."""
    k2, l2 = {}, {}
    for s in keeps:
        idx = torch.nonzero(keeps[s]).squeeze(1)
        f = torch.from_numpy(firm[s])
        k = keeps[s].clone()
        k[idx[~f]] = False
        k2[s], l2[s] = k, labels[s][f]
    return k2, l2


def load(zl, zs, case: str, device="cpu"):
    """The fixture's dataset: (dataset with ``full_lidar_set`` and ``pixel_source``, the lidar source)."""
    source = CASES[case]
    keeps, labels = base_scans(zl, source)
    firm = {s: zs[f"{case}/scan{s}/firm"] for s in range(lc.N_SCANS)}
    keeps, labels = drop(keeps, labels, firm)
    src = lc.fill(lc.LidarSource(), source, keeps, labels, device=device)
    ds = types.SimpleNamespace(full_lidar_set=lc.SplitSet(src, SPLIT), pixel_source=PixelSource(device))
    return ds, src

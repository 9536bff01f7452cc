"""Lidar sources, split sets and the field of the lidar scene-flow fixture (tests/golden/lidar_flow.npz, written by
make_golden_lidar_flow.py from the reference's own ``get_render_rays``, ``SplitWrapper``, ``query_flow`` and
``compute_scene_flow_metrics``).

The field is ``occ_cases``' miniature flow model (``flow_feat``: static, dynamic and flow branches), seeded by
``occ_cases.seed_parameters``, its density band widened and shifted so that the dynamic densities of the scans straddle
the 0.2 gate; the fixture stores only the shift.  Each scan has ``POINTS`` seeded candidate points (origin, direction,
range, flow class, ground flag); the generator composes the labels from the reference field's gated flows plus noise at
several scales, drops the points near a threshold, and stores which candidates a scan keeps and their labels.
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

import cases
import occ_cases as oc
from oracle import lidar_flow_ref

MODEL = "flow_feat"
N_SCANS = 6                  # scans 0..5 (the field has cases.N_TIMESTEPS = 10 training timesteps)
POINTS = 400                 # candidate points per scan
ABSENT = 8                   # a time index no scan has: an empty frame
THRESHOLD = 0.2              # the dynamic-density gate
MARGIN = 1e-4                # points within MARGIN relative of a threshold are dropped, so every count is well defined
NOISE_SCALES = (0.004, 0.02, 0.07, 0.25, 1.0)

# source -> (seed, {scan: what is special about it}, shuffled point order)
SOURCES = {
    "drive": (0, {3: "invalid"}, False),           # scan 3: every point has flow class -1
    "all_ground": (1, {1: "all_ground"}, False),   # scan 1: every labelled point is ground
    "static_labels": (2, {2: "static"}, False),    # scan 2: no label norm above 0.1
    "unsorted": (3, {}, True),                     # the scans' points interleaved
}
# case -> (source, remove_ground, split indices)
CASES = {
    "drive": ("drive", True, [0, 1, 2, 3, 4, 5, ABSENT]),
    "drive_keep_ground": ("drive", False, [0, 1, 2, 3, 4, 5, ABSENT]),
    "all_ground": ("all_ground", True, [0, 1, 2]),
    "static_labels": ("static_labels", True, [0, 1, 2, 3]),
    "unsorted": ("unsorted", True, [5, 0, 3, 1, 2, 4]),
}
FRAME_KEYS = ("lidar_origins", "lidar_viewdirs", "lidar_ranges", "lidar_normed_timestamps", "lidar_flow",
              "lidar_flow_class", "lidar_ground")
ATTRS = {"lidar_origins": "origins", "lidar_viewdirs": "directions", "lidar_ranges": "ranges",
         "lidar_normed_timestamps": "normalized_timestamps", "lidar_flow": "flows", "lidar_flow_class": "flow_classes",
         "lidar_ground": "grounds"}


def fixture_field(ns, shift: float):
    """The field of the fixture, from any namespace with the reference's class names; in eval mode."""
    return oc.fixture_field(ns, MODEL, shift)


def candidates(source: str, scan: int) -> Dict[str, torch.Tensor]:
    """The seeded candidate points of one scan: origins, unit directions, ranges [P, 1], int64 flow classes (-1 for
    about one point in five), bool ground flags, and the label noise (unit direction x scale) the generator adds."""
    seed, special, _ = SOURCES[source]
    g = torch.Generator().manual_seed(700 + 37 * seed + scan)
    p = POINTS
    origins = torch.tensor([1.5 * scan, 0.0, 2.0]) + 0.1 * torch.randn(p, 3, generator=g)
    dirs = torch.nn.functional.normalize(torch.randn(p, 3, generator=g) * torch.tensor([1.0, 1.0, 0.25]), dim=-1)
    ranges = 3.0 + 37.0 * torch.rand(p, 1, generator=g)
    classes = torch.randint(0, 4, (p,), generator=g)
    classes[torch.rand(p, generator=g) < 0.2] = -1
    ground = torch.rand(p, generator=g) < 0.3
    scale = torch.tensor(NOISE_SCALES)[torch.randint(0, len(NOISE_SCALES), (p,), generator=g)]
    noise = torch.nn.functional.normalize(torch.randn(p, 3, generator=g), dim=-1) * \
        (scale * (0.5 + torch.rand(p, generator=g)))[:, None]
    kind = special.get(scan)
    if kind == "invalid":
        classes[:] = -1
    elif kind == "all_ground":
        ground = classes != -1
    elif kind == "static":
        noise = noise / noise.norm(dim=-1, keepdim=True) * (0.09 * torch.rand(p, 1, generator=g))
    return {"origins": origins, "directions": dirs, "ranges": ranges, "flow_classes": classes, "grounds": ground,
            "noise": noise, "static": torch.tensor(kind == "static")}


def normed_time(scan: int, n: int) -> torch.Tensor:
    return oc.normed_time(scan, n)


class LidarSource:
    """The attributes of WaymoLiDARSource that the flow evaluation reads, and the reference's boolean-index
    ``get_render_rays`` (oracle.lidar_flow_ref).  ``flows`` and the rest are None on a source without flow labels."""
    timesteps = property(lambda self: self._timesteps)
    normalized_timestamps = property(lambda self: self._normalized_timestamps)
    flows = flow_classes = grounds = None

    def get_render_rays(self, time_idx: int):
        return lidar_flow_ref.get_render_rays(self, time_idx)


class SplitSet:
    """The part of the reference's SplitWrapper (split "full") that the evaluation reads."""

    def __init__(self, datasource, split_indices: List[int]):
        self.datasource, self.split_indices = datasource, list(split_indices)

    def __getitem__(self, idx):
        return self.datasource.get_render_rays(self.split_indices[idx])

    def __len__(self):
        return len(self.split_indices)


def fill(src, source: str, keeps: Dict[int, torch.Tensor], labels: Dict[int, torch.Tensor], with_flows=True,
         device="cpu"):
    """Set the source's tensors: the kept candidates of every scan, concatenated in scan order (interleaved by a
    seeded permutation for a shuffled source), with their labels."""
    parts: Dict[str, list] = {k: [] for k in ("origins", "directions", "ranges", "flow_classes", "grounds", "t")}
    for scan in range(N_SCANS):
        c, keep = candidates(source, scan), keeps[scan]
        for k in ("origins", "directions", "ranges", "flow_classes", "grounds"):
            parts[k].append(c[k][keep])
        parts["t"].append(torch.full((int(keep.sum()),), scan, dtype=torch.int64))
    arrays = {k: torch.cat(v) for k, v in parts.items()}
    arrays["flows"] = torch.cat([labels[s] for s in range(N_SCANS)])
    if SOURCES[source][2]:
        perm = torch.randperm(len(arrays["t"]), generator=torch.Generator().manual_seed(4242))
        arrays = {k: v[perm] for k, v in arrays.items()}
    ts = arrays.pop("t")
    src.device = torch.device(device)
    src.origins, src.directions, src.ranges = (arrays[k].to(device) for k in ("origins", "directions", "ranges"))
    src._timesteps = ts.to(device)
    src._normalized_timestamps = (ts.float() / (cases.N_TIMESTEPS + 1e-6 - 1)).to(device)
    if with_flows:
        src.flows, src.flow_classes, src.grounds = (arrays[k].to(device) for k in ("flows", "flow_classes", "grounds"))
    return src


def load(z, source: str, with_flows=True, device="cpu"):
    keeps = {s: torch.from_numpy(z[f"{source}/scan{s}/keep"]) for s in range(N_SCANS)}
    labels = {s: torch.from_numpy(z[f"{source}/scan{s}/labels"]) for s in range(N_SCANS)}
    return fill(LidarSource(), source, keeps, labels, with_flows, device)


def rows(z, source: str, t: int) -> torch.Tensor:
    """The source rows the reference's get_render_rays returns for time index t, in its order."""
    return torch.from_numpy(z[f"{source}/rows{t}"]).to(torch.int64)


def counts_of(frame_sums: np.ndarray) -> np.ndarray:
    """The integer columns of the per-frame sums: strict, relaxed, outlier, angle count, counted, valid."""
    return np.rint(frame_sums[:, [1, 2, 3, 5, 6, 7]]).astype(np.int64)

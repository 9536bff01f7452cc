"""Models, frames and the dataset object of the few-shot occupancy fixture (tests/golden/occupancy.npz, written by
make_golden_occ.py from the reference's own ``collect_centroids`` / ``eval_few_shot_occ``).

Two miniature fields: ``flow_feat`` of ``cases.build_models`` (static + dynamic + flow with temporal aggregation and
the feature head) and ``static_feat``, the same static field with the feature head and nothing else.  Their
parameters are seeded here (``seed_parameters``), so the fixture stores none: only the density shift the generator
chose (``shift_density``).  Frames are Occ3D-like voxel lists with 15 classes; the generator draws candidate voxels per
frame (``candidates``) and composes the frames from the reference field's own values at them, so the fixture stores
which candidates a frame keeps and their labels.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch

import cases

MODELS = ("flow_feat", "static_feat")
LABEL_MAPPING = {0: "general_obj", 1: "vehicle", 2: "pedestrian", 3: "sign", 4: "cyclist", 5: "traffic_light",
                 6: "pole", 7: "construction_cone", 8: "bicyle", 9: "motorcycle", 10: "building", 11: "vegetation",
                 12: "tree_trunck", 13: "road", 14: "walkable"}          # datasets/waymo.py:560-576
N_CLASSES = len(LABEL_MAPPING)
TRAIN = (0, 3, 6)
TEST = (1, 4, 7, 8)
EMPTY_TEST = 8               # no voxel of this test frame passes the density filter
MISSING_TRAIN = 5            # no train voxel: a zero centroid
MISSING_TEST = 9             # no test voxel
OUTSIDE = 15                 # a label outside the mapping (Occ3D's free space)
CANDIDATES = 1200            # candidate voxels per frame
THRESHOLD = 0.2
MARGIN = 1e-4                # densities within MARGIN * 0.2 of the threshold, and best-two cosine gaps within MARGIN,
                             # are dropped, so that every count is well defined


def build_field(ns, model: str, seed: int = 0):
    """The field of ``model`` from any namespace with the reference's class names (the reference or the drop-in)."""
    if model == "flow_feat":
        return cases.build_models(ns, "flow_feat", seed)[0]
    torch.manual_seed(seed)
    field = ns.RadianceField(
        xyz_encoder=ns.HashEncoder(verbose=False, **cases.ENC_STATIC), dynamic_xyz_encoder=None,
        flow_xyz_encoder=None, aabb=cases.AABB, unbounded=True, geometry_feature_dim=64, base_mlp_layer_width=64,
        head_mlp_layer_width=64, enable_cam_embedding=False, enable_img_embedding=True, num_cams=cases.N_CAMS,
        appearance_embedding_dim=16, semantic_feature_dim=64, feature_mlp_layer_width=64, feature_embedding_dim=64,
        enable_sky_head=True, enable_shadow_head=False, enable_feature_head=True,
        num_train_timesteps=cases.N_TIMESTEPS, interpolate_xyz_encoding=True, enable_learnable_pe=True,
        enable_temporal_interpolation=False)
    g = torch.Generator().manual_seed(seed + 1)       # the table rescale of cases.build_models
    with torch.no_grad():
        for k, v in field.named_parameters():
            if k.endswith("tcnn_encoding.params"):
                v.copy_(torch.randn(v.shape, generator=g) * 0.5)
    return field


def seed_parameters(field, seed: int = 0) -> None:
    """Every parameter from one seeded stream, in sorted name order (the reference and the drop-in share the names):
    hash tables N(0, 0.5^2) as cases.build_models rescales them, everything else U(-1, 1) / sqrt(fan-in), biases and
    other vectors U(-0.1, 0.1)."""
    g = torch.Generator().manual_seed(9000 + seed)
    params = dict(field.named_parameters())
    with torch.no_grad():
        for name in sorted(params):
            v = params[name]
            if name.endswith("tcnn_encoding.params"):
                v.copy_(torch.randn(v.shape, generator=g) * 0.5)
            elif v.dim() >= 2:
                v.copy_((torch.rand(v.shape, generator=g) * 2 - 1) / v.shape[1] ** 0.5)
            else:
                v.copy_((torch.rand(v.shape, generator=g) * 2 - 1) * 0.1)


DENSITY_ROWS = ("base_mlp.2", "dynamic_base_mlp.2")   # the layers whose output column 0 is the density's exponent


def widen_density(field) -> None:
    """x4 on the density row of the last base-MLP layer(s): the miniature fields' densities sit in a narrow band."""
    params = dict(field.named_parameters())
    with torch.no_grad():
        for k in DENSITY_ROWS:
            if f"{k}.weight" in params:
                params[f"{k}.weight"][0] *= 4.0


def shift_density(field, shift: float) -> None:
    """One shared bias shift of the density's exponent, which the generator picks to centre the band on 0.2."""
    params = dict(field.named_parameters())
    with torch.no_grad():
        for k in DENSITY_ROWS:
            if f"{k}.bias" in params:
                params[f"{k}.bias"][0] -= shift


def fixture_field(ns, model: str, shift: float):
    """The field of the fixture: built, seeded, widened and shifted by the stored ``shift``; in eval mode."""
    field = build_field(ns, model)
    seed_parameters(field)
    widen_density(field)
    shift_density(field, shift)
    return field.eval()


def normed_time(index: int, n: int) -> torch.Tensor:
    """datasets/waymo.py:631-635 with the miniature's timestep count."""
    return torch.ones(n) * index / (cases.N_TIMESTEPS + 1e-6 - 1)


def candidates(index: int) -> torch.Tensor:
    """Seeded voxel centres of frame ``index`` on a 0.4 m grid in front of the ego car."""
    g = torch.Generator().manual_seed(500 + index)
    ijk = torch.stack([torch.randint(0, 100, (CANDIDATES,), generator=g), torch.randint(0, 100, (CANDIDATES,), generator=g),
                       torch.randint(0, 16, (CANDIDATES,), generator=g)], -1).float()
    return ijk * 0.4 + torch.tensor([0.2, -19.8, 0.2])


class OccDataset:
    """The part of the reference's WaymoDataset the occupancy evaluation reads: ``get_occ(i)`` -> (world voxel
    centres [N, 3], int64 labels [N], normed timestamps [N]) on ``device``, and ``label_mapping``."""

    def __init__(self, frames: Dict[int, Tuple[torch.Tensor, torch.Tensor, torch.Tensor]], device="cpu"):
        self.frames = frames
        self.device = device
        self.label_mapping = dict(LABEL_MAPPING)

    def get_occ(self, index: int):
        return tuple(x.to(self.device) for x in self.frames[index])


def frame(index: int, keep: torch.Tensor, labels: torch.Tensor):
    """(coords, int64 labels, normed time) of the candidates of frame ``index`` that ``keep`` selects."""
    coords = candidates(index)[keep]
    return coords, labels.to(torch.int64), normed_time(index, len(coords))


def load_frames(z, model: str) -> Dict[int, Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
    """The frames of ``model`` stored in occupancy.npz (kept candidates and their labels)."""
    return {i: frame(i, torch.from_numpy(z[f"{model}/frame{i}/keep"]), torch.from_numpy(z[f"{model}/frame{i}/labels"]))
            for i in TRAIN + TEST}

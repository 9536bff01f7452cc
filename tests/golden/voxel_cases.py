"""Models, rays and the dataset object of the voxel-lifting fixture (tests/golden/voxels.npz, written by
make_golden_voxels.py from the reference's own ``visualize_voxels``).

Two miniature fields with the feature head and the two proposal networks of ``cases``: ``static_feat`` (static field
only) and ``flow_feat`` (static + dynamic + flow).  Every parameter comes from one seeded stream
(``occ_cases.seed_parameters``), so the fixture stores none: only the density shifts the generator chose.  Each image
is a seeded [H, W] grid of rays with the keys of the reference's ``get_render_rays``; some cameras sit just outside the
box, so rays leave it and cross the band just below its minimum (where ``.long()`` truncates into voxel 0).  The
miniature fields are dense everywhere, so rendered depths stay far below 80: the depth filter is pinned by the kernel
tests on given depths instead.

Cases (name -> model, cameras, images, dynamic shift): one static field with one camera, a dynamic field with three
cameras and 34 images (11 groups: groups 0 and 10 are queried, and the last image is dropped), and a dynamic field
with one camera whose dynamic density is shifted so far down that no voxel passes the 0.1 gate.
"""
from __future__ import annotations

import math
import types
from typing import Dict

import torch

import cases
import occ_cases

H, W = 8, 12
VOXEL_SIZE = 2.0
CASES = {
    "static_1cam": dict(model="static_feat", cams=1, images=12, dynamic=False),
    "dynamic_3cam": dict(model="flow_feat", cams=3, images=34, dynamic=True),
    "dynamic_1cam_closed": dict(model="flow_feat", cams=1, images=12, dynamic=True),
}
STATIC_DENSITY_ROWS = ("base_mlp.2",)
DYNAMIC_DENSITY_ROWS = ("dynamic_base_mlp.2",)
CLOSED_SHIFT = 40.0          # dynamic density exp(raw - 1 - 40): nothing passes 0.1
MARGIN = 1e-4                # q within MARGIN of an integer, depth within MARGIN * 80 of 80, density within
                             # MARGIN relative of its threshold: outcomes the fixture does not pin


def render_cfg(voxel_size: float = VOXEL_SIZE):
    cfg = cases.render_cfg()
    cfg.render.vis_voxel_size = voxel_size
    return cfg


def build_models(ns, model: str, shifts):
    """(field, proposal networks) of ``model`` from any namespace with the reference's class names, seeded, with the
    density of the last base-MLP layer widened and shifted by ``shifts`` = (static, dynamic); in eval mode."""
    c = dict(dynamic=model == "flow_feat", flow=model == "flow_feat", shadow=model == "flow_feat", feature=True)
    torch.manual_seed(0)
    enc = ns.HashEncoder(verbose=False, **cases.ENC_STATIC)
    dyn = ns.HashEncoder(verbose=False, **cases.ENC_DYN) if c["dynamic"] else None
    flw = ns.HashEncoder(verbose=False, **cases.ENC_FLOW) if c["flow"] else None
    field = ns.RadianceField(
        xyz_encoder=enc, dynamic_xyz_encoder=dyn, flow_xyz_encoder=flw, aabb=cases.AABB, unbounded=True,
        geometry_feature_dim=64, base_mlp_layer_width=64, head_mlp_layer_width=64, enable_cam_embedding=False,
        enable_img_embedding=True, num_cams=cases.N_CAMS, appearance_embedding_dim=16, semantic_feature_dim=64,
        feature_mlp_layer_width=64, feature_embedding_dim=64, enable_sky_head=True, enable_shadow_head=c["shadow"],
        enable_feature_head=True, num_train_timesteps=cases.N_TIMESTEPS, interpolate_xyz_encoding=True,
        enable_learnable_pe=True, enable_temporal_interpolation=False)
    field.register_normalized_training_timesteps(torch.linspace(0, 1, cases.N_TIMESTEPS),
                                                 time_diff=1.0 / cases.N_TIMESTEPS)
    occ_cases.seed_parameters(field)
    props = []
    for k, e in enumerate(cases.ENC_PROP):
        p = ns.build_density_field(n_input_dims=3, n_levels=e["n_levels"], max_resolution=e["max_resolution"],
                                   log2_hashmap_size=e["log2_hashmap_size"],
                                   n_features_per_level=e["n_features_per_level"], unbounded=True)
        p.set_aabb(cases.AABB)
        occ_cases.seed_parameters(p, seed=1 + k)
        props.append(p.eval())
    params = dict(field.named_parameters())
    with torch.no_grad():
        for rows, shift in ((STATIC_DENSITY_ROWS, shifts[0]), (DYNAMIC_DENSITY_ROWS, shifts[1])):
            for k in rows:
                if f"{k}.weight" in params:
                    params[f"{k}.weight"][0] *= 4.0
                    params[f"{k}.bias"][0] -= shift
    return field.eval(), props


def image_rays(case: str, i: int) -> Dict[str, torch.Tensor]:
    """Image ``i`` of ``case``: camera i % cams at timestep i // cams, [H, W] rays with the reference's keys.  The
    centre cycles with i over two points inside the box and one just below its x minimum."""
    c = CASES[case]
    cams, n = c["cams"], c["images"]
    cam, step = i % cams, i // cams
    steps = (n + cams - 1) // cams
    g = torch.Generator().manual_seed(7000 + 97 * i + len(case))
    place = i % 3
    centre = [torch.tensor([5.0, 0.0, 2.0]), torch.tensor([-21.3, 3.0, 1.0]), torch.tensor([40.0, 10.0, 5.0])][place]
    centre = centre + torch.tensor([0.7 * step, 0.0, 0.0]) + (torch.rand(3, generator=g) - 0.5)
    yaw0 = [0.0, math.pi, 0.2][place]
    yaw = yaw0 + torch.linspace(-1.0, 1.0, W)[None, :].expand(H, W) + 0.01 * torch.rand(H, W, generator=g)
    pitch = torch.linspace(-0.35, 0.25, H)[:, None].expand(H, W) + 0.01 * torch.rand(H, W, generator=g)
    d = torch.stack([torch.cos(pitch) * torch.cos(yaw), torch.cos(pitch) * torch.sin(yaw), torch.sin(pitch)], -1)
    d = d / d.norm(dim=-1, keepdim=True)
    y, x = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    return {
        "origins": centre.expand(H, W, 3).contiguous(),
        "viewdirs": d.contiguous(),
        "direction_norm": torch.ones(H, W, 1),
        "pixel_coords": torch.stack([y / H, x / W], -1),
        "normed_timestamps": torch.full((H, W), step / max(steps - 1, 1)),
        "img_idx": torch.full((H, W), i % (cases.N_TIMESTEPS * cases.N_CAMS), dtype=torch.long),
        "cam_idx": torch.full((H, W), cam, dtype=torch.long),
        "pixels": torch.rand(H, W, 3, generator=g),
    }


def unique_timestamps(case: str) -> torch.Tensor:
    c = CASES[case]
    steps = (c["images"] + c["cams"] - 1) // c["cams"]
    return torch.arange(steps).float() / max(steps - 1, 1)


class Dataset:
    """What ``visualize_voxels`` reads of the reference's SceneDataset: ``full_pixel_set`` (items are fresh ray
    dicts), ``num_cams`` and ``pixel_source.unique_normalized_timestamps``."""

    def __init__(self, case: str, device="cpu"):
        c = CASES[case]
        self.num_cams = c["cams"]
        self.full_pixel_set = [{k: v.to(device) for k, v in image_rays(case, i).items()} for i in range(c["images"])]
        self.pixel_source = types.SimpleNamespace(unique_normalized_timestamps=unique_timestamps(case).to(device))


class _Items(list):
    """A list whose items are copies, so a caller that adds keys to an item does not change the dataset."""

    def __getitem__(self, i):
        return dict(super().__getitem__(i))


def dataset(case: str, device="cpu") -> Dataset:
    ds = Dataset(case, device)
    ds.full_pixel_set = _Items(ds.full_pixel_set)
    return ds

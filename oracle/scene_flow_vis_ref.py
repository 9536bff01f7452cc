"""The reference's scene-flow figure (``visualize_scene_flow``, utils/visualization_tools.py:729-821 of
NVlabs/EmerNeRF@8c051d7, with ``get_valid_lidar_mask`` from datasets/waymo.py:638-668 and ``scene_flow_to_rgb`` from
utils/visualization_tools.py:159-275), restated op for op as it runs on the GPU -- TEST INFRASTRUCTURE ONLY, the
baseline of tools/bench_scene_flow_vis.py and of tests/test_gpu_scene_flow_vis.py.

Per sampled frame: the frame's boolean indexes (``get_render_rays``), seven on ``lidar_flow_class != -1``, the empty
check, the camera mask (per camera ``pad(intrinsics) @ cam_to_worlds.inverse()`` and the matmul projection), seven
more boolean indexes, ``query_flow``, the in-place gate, ``scene_flow_to_rgb`` of the prediction and of the label, and
three ``.cpu().numpy()`` copies; then the box.  The figures are left out: the result is the keyword arguments of the
two ``vis_occ_plotly`` calls.  Never run on NaN flows: the wheel index of a NaN is out of range.
"""
from __future__ import annotations

import logging
from collections import namedtuple
from itertools import accumulate
from typing import Dict, Optional

import numpy as np
import torch
from torch import Tensor

logger = logging.getLogger()
TRANSITIONS = (15, 6, 4, 11, 13, 6)


def make_wheel() -> Tensor:
    """The 55-hue wheel, each transition an ``np.linspace(..., endpoint=False)`` stored as uint8, then the first hue
    again (the cyclic wheel): [56, 3] fp32."""
    hues = [np.array(h) for h in ([255, 0, 0], [255, 255, 0], [0, 255, 0], [0, 255, 255], [0, 0, 255],
                                  [255, 0, 255], [255, 0, 0])]
    wheel = np.zeros((sum(TRANSITIONS), 3), dtype="uint8")
    start = 0
    for t, end in enumerate(accumulate(TRANSITIONS)):
        wheel[start:end] = np.linspace(hues[t], hues[t + 1], end - start, endpoint=False)
        start = end
    w = torch.FloatTensor(wheel)
    return torch.vstack((w, w[0]))


WHEEL = make_wheel()
N_COLS = len(WHEEL) - 1


def scene_flow_to_rgb(flow: Tensor, flow_max_radius: Optional[float] = None, background: str = "dark") -> Tensor:
    if background not in ("bright", "dark"):
        raise ValueError(f"background should be one the following: {('bright', 'dark')}, not {background}.")
    complex_flow = flow[..., 0] + 1j * flow[..., 1]
    radius, angle = torch.abs(complex_flow), torch.angle(complex_flow)
    if flow_max_radius is None:
        flow_max_radius = torch.quantile(radius, 0.99)
    if flow_max_radius > 0:
        radius /= flow_max_radius
    angle[angle < 0] += 2 * np.pi
    angle = angle * ((N_COLS - 1) / (2 * np.pi))
    frac, lo, hi = torch.fmod(angle, 1), angle.trunc(), torch.ceil(angle)
    frac = frac.unsqueeze(-1)
    wheel = WHEEL.to(lo.device)
    hue = wheel[lo.long()] * (1 - frac) + wheel[hi.long()] * frac
    Args = namedtuple("Args", ["valid", "oversized"])

    def v_axis(hues, factors):
        return hues * factors.unsqueeze(-1)

    def s_axis(hues, factors):
        return 255.0 - factors.unsqueeze(-1) * (255.0 - hues)

    move = Args(v_axis, s_axis) if background == "dark" else Args(s_axis, v_axis)
    colors = move.valid(hue, radius)
    over = radius > 1
    colors[over] = move.oversized(hue[over], 1 / radius[over])
    return colors / 255.0


def get_valid_lidar_mask(pixel_source, lidar_timestep: int, data: Dict[str, Tensor]) -> Tensor:
    points = data["lidar_origins"] + data["lidar_ranges"] * data["lidar_viewdirs"]
    valid = torch.zeros_like(points[:, 0]).bool()
    for c in range(pixel_source.num_cams):
        img = lidar_timestep * pixel_source.num_cams + c
        k4 = torch.nn.functional.pad(pixel_source.intrinsics[img], (0, 1, 0, 1))
        k4[3, 3] = 1.0
        l2i = k4 @ pixel_source.cam_to_worlds[img].inverse()
        proj = (l2i[:3, :3] @ points.T + l2i[:3, 3:4]).T
        depth = proj[:, 2]
        cam = proj[:, :2] / (depth.unsqueeze(-1) + 1e-6)
        valid = valid | ((cam[:, 0] >= 0) & (cam[:, 0] < pixel_source.WIDTH) & (cam[:, 1] >= 0)
                         & (cam[:, 1] < pixel_source.HEIGHT) & (depth > 0))
    return valid


def visualize_scene_flow(cfg, model, dataset, device="cuda") -> Dict[str, Dict[str, object]]:
    pred_colors, gt_colors, coords = [], [], []
    for i in range(0, len(dataset.full_lidar_set) - 1, 10):
        data = dataset.full_lidar_set[i].copy()
        cls = data["lidar_flow_class"]
        for k, v in data.items():
            data[k] = v[cls != -1]
        if data[k].shape[0] == 0:
            logger.info("no valid points, skipping...")
            continue
        mask = get_valid_lidar_mask(dataset.pixel_source, i, data)
        for k, v in data.items():
            data[k] = v[mask]
        points = data["lidar_origins"] + data["lidar_ranges"] * data["lidar_viewdirs"]
        with torch.no_grad():
            pred = model.query_flow(positions=points, normed_timestamps=data["lidar_normed_timestamps"])
        flow = pred["forward_flow"]
        flow[pred["dynamic_density"] < 0.2] *= 0
        pred_colors.append(scene_flow_to_rgb(flow, flow_max_radius=2.0, background="bright").cpu().numpy())
        gt_colors.append(scene_flow_to_rgb(data["lidar_flow"], flow_max_radius=2.0, background="bright").cpu().numpy())
        coords.append(points.cpu().numpy())
    box = torch.tensor(model.aabb, device=device)
    box[1:3] -= 1
    box[3:] += 1
    lo, hi = torch.split(box, 3, dim=-1)
    length = hi - lo
    common = {"vis_aabb": box.cpu().numpy().tolist(), "dynamic_coords": coords, "x_ratio": 1,
              "y_ratio": (length[1] / length[0]).item(), "z_ratio": (length[2] / length[0]).item()}
    return {"pred": dict(common, dynamic_colors=pred_colors), "gt": dict(common, dynamic_colors=gt_colors)}

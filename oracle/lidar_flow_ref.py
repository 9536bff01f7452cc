"""The reference's lidar scene-flow evaluation (train_emernerf.py:237-281 of NVlabs/EmerNeRF@8c051d7, with
``WaymoLiDARSource.get_render_rays`` from datasets/waymo.py:341-356 and ``compute_scene_flow_metrics`` from
datasets/metrics.py:73-128), restated op for op as it runs on the GPU -- TEST INFRASTRUCTURE ONLY, the baseline of
tools/bench_lidar_flow.py.

Per frame: seven boolean indexes on ``timesteps == t``, seven on ``lidar_flow_class != -1``, the empty check, seven on
the ground, ``query_flow`` on the kept points, the in-place gate ``pred[dynamic_density < 0.2] *= 0`` and the NSFP
statistics with their two ``.cpu()`` copies and fp32 ``.item()`` means; then ``np.mean`` per key over the frames.  The
progress bar, the JSON file and wandb are left out.
"""
from __future__ import annotations

import logging
from typing import Dict, List, Optional

import numpy as np
import torch
from torch import Tensor

logger = logging.getLogger()
KEYS = ("EPE3D", "acc3d_strict", "acc3d_relax", "angle_error", "outlier")


def get_render_rays(source, time_idx: int) -> Dict[str, Tensor]:
    """The Waymo source's frame: the base class's four keys, plus the flows, flow classes and ground flags when the
    source has them."""
    keys = {"lidar_origins": "origins", "lidar_viewdirs": "directions", "lidar_ranges": "ranges",
            "lidar_normed_timestamps": "normalized_timestamps"}
    if all(getattr(source, k, None) is not None for k in ("flows", "flow_classes", "grounds")):
        keys.update(lidar_flow="flows", lidar_flow_class="flow_classes", lidar_ground="grounds")
    return {k: getattr(source, a)[source.timesteps == time_idx] for k, a in keys.items()}


def scene_flow_metrics(pred: Tensor, labels: Tensor) -> Dict[str, float]:
    """compute_scene_flow_metrics of [1, N, 3] flows: fp32 on the device, then the statistics on the host."""
    l2 = torch.sqrt(torch.sum((pred - labels) ** 2, 2)).cpu()
    ln = torch.sqrt(torch.sum(labels * labels, 2)).cpu()
    rel = l2 / (ln + 1e-20)
    out = {"EPE3D": torch.mean(l2).item(),
           "acc3d_strict": torch.mean(((l2 < 0.05) | (rel < 0.05)).float()).item(),
           "acc3d_relax": torch.mean(((l2 < 0.1) | (rel < 0.1)).float()).item(),
           "outlier": torch.mean(((l2 > 0.3) | (rel > 0.1)).float()).item()}
    unit_label = labels / (labels.norm(dim=-1, keepdim=True) + 1e-7)
    unit_pred = pred / (pred.norm(dim=-1, keepdim=True) + 1e-7)
    moving = ln > 0.1
    dot = (unit_label[moving] * unit_pred[moving]).sum(-1).clamp(min=-1 + 1e-7, max=1 - 1e-7)
    dot[dot != dot] = 0
    out["angle_error"] = torch.acos(dot).mean().item()
    return out


def eval_lidar_flow(lidar_set, model, remove_ground: bool = True, flow_metrics=None,
                    frames: Optional[List[dict]] = None) -> Dict[str, np.float64]:
    """The driver's loop over the frames of ``lidar_set`` (a SplitWrapper: iterating it calls its source's
    ``get_render_rays`` for each split index).  ``flow_metrics(pred, labels)`` defaults to the restatement above (the
    golden generator passes the reference's own); ``frames``, when given, receives per frame {"valid", "counted",
    "metrics"} ("metrics" is None for a skipped frame)."""
    flow_metrics = flow_metrics or scene_flow_metrics
    per_frame = {k: [] for k in KEYS}
    with torch.no_grad():
        for data in lidar_set:
            cls = data["lidar_flow_class"]
            for k, v in data.items():
                data[k] = v[cls != -1]
            valid = data["lidar_ground"].shape[0]
            if valid == 0:
                logger.info("no valid points, skipping...")
                if frames is not None:
                    frames.append({"valid": 0, "counted": 0, "metrics": None})
                continue
            if remove_ground:
                for k, v in data.items():
                    data[k] = v[~data["lidar_ground"]]
            points = data["lidar_origins"] + data["lidar_ranges"] * data["lidar_viewdirs"]
            pred = model.query_flow(positions=points, normed_timestamps=data["lidar_normed_timestamps"])
            flow = pred["forward_flow"]
            flow[pred["dynamic_density"] < 0.2] *= 0
            got = flow_metrics(flow[None, ...], data["lidar_flow"][None, ...])
            if frames is not None:
                frames.append({"valid": valid, "counted": int(points.shape[0]), "metrics": dict(got)})
            for k, v in got.items():
                per_frame[k].append(v)
    return {k: np.mean(v) for k, v in per_frame.items()}

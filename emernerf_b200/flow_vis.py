"""The scene-flow figure of the reference's ``visualize_scene_flow`` (utils/visualization_tools.py:729-821) on the
device (csrc/flow_vis.cu), and a drop-in ``scene_flow_to_rgb`` (utils/visualization_tools.py:204-275).

    kw = flow_vis.visualize_scene_flow(cfg, model, dataset, device=device)
    pred_figure = vis_occ_plotly(**kw["pred"], size=2, black_bg=True, title="Predicted Flow")   # the reference's code
    gt_figure = vis_occ_plotly(**kw["gt"], size=2, black_bg=True, title="GT Flow")

``visualize_scene_flow`` returns ``{"pred": kw, "gt": kw}``, each ``kw`` the keyword arguments the reference hands to
``vis_occ_plotly``: ``vis_aabb``, ``dynamic_coords`` (a list of [n_f, 3] float32 arrays, the same list in both),
``dynamic_colors``, ``x_ratio``, ``y_ratio`` and ``z_ratio``.  Per sampled frame, one ``emer_flow_vis_select`` launch
keeps the labelled points some camera sees and writes their label colours; after one host sync for the frames' counts
and the box, ``model.query_flow`` runs on each frame's kept points, in chunks of ``metrics.FLOW_CHUNK_POINTS``, with one
``emer_flow_vis_color`` launch per chunk for the gated prediction's colours; one device-to-host copy brings back a
[total, 9] buffer (coordinates, prediction colour, label colour).  So a call syncs the host twice, plus the frame
table's two when the lidar source's timesteps are new.  Everything runs under ``no_grad``; the model's mode is not
changed.

The reference's behaviour that is kept on purpose:
  * frames: the positions ``i in range(0, len(dataset.full_lidar_set) - 1, 10)`` of the split;
  * camera index: image ``i * num_cams + c`` for camera c, with ``i`` the position in the split, not the timestep
    ``split_indices[i]``;
  * skipped frames: a frame without a labelled point (``lidar_flow_class != -1``) is skipped and logged ("no valid
    points, skipping..."), and this check comes before the camera mask;
  * camera mask: ``get_valid_lidar_mask``'s ``pad(intrinsics) @ cam_to_worlds.inverse()`` per image (here
    ``torch.linalg.inv_ex``, the same kernel without the error check's sync), the fp32 projection, and a point kept
    when ``0 <= u < WIDTH``, ``0 <= v < HEIGHT`` and ``depth > 0`` for any camera;
  * box: ``vis_aabb[1:3] -= 1`` and ``vis_aabb[3:] += 1`` on ``model.aabb`` in fp32 (``voxels.grown_box``), the ratios
    fp32 quotients of its extents;
  * gate: ``pred_flow[dynamic_density < 0.2] *= 0``: NaN stays NaN, ``inf`` becomes NaN, a NaN density does not gate;
  * points: ``lidar_origins + lidar_ranges * lidar_viewdirs`` with two fp32 roundings; these are the coordinates;
  * colours: ``scene_flow_to_rgb(..., flow_max_radius=2.0, background="bright")`` of the prediction and of the label.

Deliberate differences:
  * a frame with labelled points of which no camera sees any gives empty (0, 3) arrays; the reference's
    ``query_flow`` fails on zero rows there;
  * a NaN flow gets NaN colours, where the reference's wheel index asserts on the device;
  * frames larger than ``metrics.FLOW_CHUNK_POINTS`` points are queried in chunks of that many; only such frames can
    differ in the layer kernels' choice by row count.

``scene_flow_to_rgb(flow, flow_max_radius=None, background="dark")`` is one launch without a host sync for a given
radius.  With ``None`` the radius is the reference's ``torch.quantile(radius, 0.99)`` over a device buffer of radii
written by the same device formula, and the kernel applies the reference's ``> 0`` test to that 0-d device tensor
itself, so the call does not sync the host either.
"""
from __future__ import annotations

import logging
from typing import Dict, List, Optional, Union

import torch
from torch import Tensor

from . import _lib, _ops, metrics, voxels

__all__ = ["visualize_scene_flow", "scene_flow_to_rgb"]
logger = logging.getLogger()

FRAME_STRIDE = 10                # every tenth frame of the split is drawn
FLOW_MAX_RADIUS = 2.0            # the reference's colour scale for both figures
GATE = 0.2                       # flows count only on dynamic points
MAX_ROWS = 1 << 24               # EMER_FLOW_VIS_MAX_ROWS: points per frame
MAX_CAMS = 16                    # EMER_FLOW_VIS_MAX_CAMS
SELECT_WORKSPACE_BYTES = 131080  # EMER_FLOW_VIS_WORKSPACE_BYTES
SCALE_NONE, SCALE_HOST, SCALE_DEVICE = 0, 1, 2   # EMER_FLOW_SCALE_*
BACKGROUNDS = ("bright", "dark")
_WS: Dict[object, Tensor] = {}


def _need_device(*ts: Optional[Tensor]) -> None:
    for t in ts:
        if t is not None and not _ops.on_device(t):
            raise ValueError("scene flow visualisation: tensors must be CUDA tensors")


def color(flow: Tensor, colors: Optional[Tensor], density: Optional[Tensor] = None, threshold: float = GATE,
          scale_mode: int = SCALE_HOST, radius: float = FLOW_MAX_RADIUS, device_radius: Optional[Tensor] = None,
          bright: bool = True, radii: Optional[Tensor] = None) -> None:
    """One ``emer_flow_vis_color`` launch over the rows of ``flow`` (x and y first, read in place): their colours
    into ``colors`` (rows of 3, any row stride), gated by ``density`` when given; or, with ``colors`` None, the
    unscaled radii into ``radii`` (dense)."""
    f, ld = _ops._rows(flow, flow.shape[-1])
    n = f.shape[0]
    if flow.shape[-1] < 2:
        raise ValueError(f"scene flow colours: flows of {flow.shape[-1]} components (x and y at least)")
    dens = None if density is None else _ops._f32c(density.reshape(-1))
    if dens is not None and dens.numel() != n:
        raise ValueError(f"scene flow colours: {dens.numel()} densities for {n} flows")
    ld_c = 0
    if colors is not None:
        if colors.dtype != torch.float32 or colors.dim() != 2 or colors.shape[0] != n or colors.shape[1] != 3 \
                or colors.stride(1) != 1:
            raise ValueError("scene flow colours: colours must be fp32 rows of 3 with unit inner stride")
        ld_c = colors.stride(0) if n > 1 else 3
    _ops._need_cuda(f, dens, colors, device_radius, radii)
    p = _ops._ptr
    _lib.call("emer_flow_vis_color", p(f), ld, p(dens), threshold, n, scale_mode, radius, p(device_radius),
              int(bright), p(colors), ld_c, p(radii), _ops._stream())


def scene_flow_to_rgb(flow: Tensor, flow_max_radius: Union[None, float, Tensor] = None,
                      background: Optional[str] = "dark") -> Tensor:
    """The reference's ``scene_flow_to_rgb``: the RGB colours [..., 3] (fp32, on the flow's device) of the flows
    [..., >= 2] (x and y), normalised by ``flow_max_radius`` (when > 0) or, for None, by the 0.99 quantile of the
    radii; zero flow is white for "bright" and black for "dark".  No host sync; a NaN flow gives NaN colours."""
    if background not in BACKGROUNDS:
        raise ValueError(f"background should be one the following: {BACKGROUNDS}, not {background}.")
    _need_device(flow)
    if flow.dim() < 1 or flow.shape[-1] < 2:
        raise ValueError(f"scene_flow_to_rgb: a flow of shape {tuple(flow.shape)} (x and y in the last dimension)")
    bright = background == "bright"
    out = torch.empty(*flow.shape[:-1], 3, dtype=torch.float32, device=flow.device)
    rows = out.view(-1, 3)
    if flow_max_radius is None:
        radii = torch.empty(rows.shape[0], dtype=torch.float32, device=flow.device)
        color(flow, None, scale_mode=SCALE_NONE, radii=radii)
        q = torch.quantile(radii, 0.99)                       # the reference's own call, on the same radii
        color(flow, rows, scale_mode=SCALE_DEVICE, device_radius=q, bright=bright)
    elif isinstance(flow_max_radius, Tensor) and _ops.on_device(flow_max_radius):
        q = _ops._f32c(flow_max_radius.reshape(()))           # a 0-d device divisor: a true division when > 0
        color(flow, rows, scale_mode=SCALE_DEVICE, device_radius=q, bright=bright)
    else:
        r = float(flow_max_radius)                            # a host scalar (a CPU tensor is one to torch as well)
        color(flow, rows, scale_mode=SCALE_HOST if r > 0 else SCALE_NONE, radius=r, bright=bright)
    return out


def lidar2img(pixel_source, i: int, num_cams: int) -> Tensor:
    """[num_cams, 4, 4] fp32: ``get_valid_lidar_mask``'s ``pad(intrinsics) @ cam_to_worlds.inverse()`` for the images
    ``i * num_cams + c``, one image at a time (``torch.linalg.inv_ex`` is ``inverse()``'s kernel without its sync)."""
    mats = []
    for c in range(num_cams):
        img = i * num_cams + c
        k4 = torch.nn.functional.pad(pixel_source.intrinsics[img], (0, 1, 0, 1))
        k4[3, 3].fill_(1.0)                              # `k4[3, 3] = 1.0` copies a host scalar: a sync
        mats.append(k4 @ torch.linalg.inv_ex(pixel_source.cam_to_worlds[img]).inverse)
    return torch.stack(mats).to(torch.float32).contiguous()


def select(frame: Dict[str, Tensor], l2i: Tensor, width: float, height: float, points: Tensor, times: Tensor,
           rows9: Tensor, count: Tensor, frame_counts: Tensor) -> None:
    """One ``emer_flow_vis_select`` launch for one frame of ``LidarRaySampler.get_render_rays`` (read in place): its
    labelled points that a camera sees, appended at ``count`` (int64 [1], advanced) to ``points``, ``times`` and
    ``rows9`` (coordinates and label colours); ``frame_counts`` (int64 [2]) += (labelled, kept)."""
    o, ld_o = _ops._rows(frame["lidar_origins"], 3)
    d, ld_d = _ops._rows(frame["lidar_viewdirs"], 3)
    r, ld_r = _ops._rows(frame["lidar_ranges"], 1)
    t, ld_t = _ops._rows(frame["lidar_normed_timestamps"], 1)
    f, ld_f = _ops._rows(frame["lidar_flow"], 3)
    cls = frame["lidar_flow_class"].reshape(-1, 1)
    if cls.dtype != torch.int64:
        cls = cls.to(torch.int64)
    if cls.stride(1) != 1 or (cls.shape[0] > 1 and cls.stride(0) < 1):
        cls = cls.contiguous()
    ld_c = cls.stride(0) if cls.shape[0] > 1 else 1
    n = o.shape[0]
    if any(x.shape[0] != n for x in (d, r, t, f, cls)):
        raise ValueError(f"scene flow visualisation: a frame of {n} origins and "
                         f"{[x.shape[0] for x in (d, r, t, f, cls)]} other rows")
    if n > MAX_ROWS:
        raise ValueError(f"scene flow visualisation: a frame of {n} points (at most {MAX_ROWS})")
    cams = l2i.shape[0]
    if not 1 <= cams <= MAX_CAMS:
        raise ValueError(f"scene flow visualisation: {cams} cameras (1..{MAX_CAMS})")
    ws = _ops._workspace(_WS, o.device, SELECT_WORKSPACE_BYTES, "scene flow visualisation")
    _ops._need_cuda(o, d, r, t, f, cls, l2i, points, times, rows9, count, frame_counts)
    p = _ops._ptr
    _lib.call("emer_flow_vis_select", p(o), ld_o, p(d), ld_d, p(r), ld_r, p(t), ld_t, p(f), ld_f, p(cls), ld_c, n,
              p(l2i), cams, float(width), float(height), p(points), p(times), p(rows9), p(count), p(frame_counts),
              p(ws), _ops._stream())


def visualize_scene_flow(cfg, model, dataset, device: str = "cuda") -> Dict[str, Dict[str, object]]:
    """The reference's ``visualize_scene_flow`` up to its two ``vis_occ_plotly`` calls: returns those calls' keyword
    arguments as ``{"pred": kw, "gt": kw}``.  ``cfg`` and ``device`` are the reference's arguments; the figures and
    their files stay with the caller, and the model's device is used."""
    lidar_set = dataset.full_lidar_set
    source = getattr(lidar_set, "datasource", None)
    split = getattr(lidar_set, "split_indices", None)
    if source is None or split is None:
        raise ValueError("scene flow visualisation: the lidar set needs `datasource` and `split_indices`")
    if getattr(model, "flow_xyz_encoder", None) is None:
        raise ValueError("scene flow visualisation: the model has no flow branch")
    _need_device(model.aabb)
    split = list(split)
    pix = dataset.pixel_source
    num_cams = int(pix.num_cams)
    frames = list(range(0, len(lidar_set) - 1, FRAME_STRIDE))
    sampler = metrics._lidar_sampler(source)
    table, _ = sampler._frame_table()
    cap = sum(table.get(int(split[i]), (0, 0))[1] for i in frames)
    dev = model.aabb.device
    rows9 = torch.empty(cap, 9, dtype=torch.float32, device=dev)
    points = torch.empty(cap, 3, dtype=torch.float32, device=dev)
    times = torch.empty(cap, dtype=torch.float32, device=dev)
    counts = torch.zeros(2 * len(frames) + 1, dtype=torch.int64, device=dev)   # per frame (labelled, kept), then all
    with torch.no_grad():
        for f, i in enumerate(frames):
            frame = sampler.get_render_rays(split[i])
            if "lidar_flow" not in frame:
                raise ValueError("scene flow visualisation: the lidar source has no flows and flow classes")
            select(frame, lidar2img(pix, i, num_cams), pix.WIDTH, pix.HEIGHT, points, times, rows9,
                   counts[2 * len(frames):], counts[2 * f:2 * f + 2])
        vis_aabb, length = voxels.grown_box(model.aabb)
        got = torch.cat([counts[:2 * len(frames)].double(), vis_aabb.double(), length.double()]).tolist()   # sync 1
        per_frame = [(int(got[2 * f]), int(got[2 * f + 1])) for f in range(len(frames))]
        live: List[tuple] = []
        start = 0
        for labelled, kept in per_frame:
            if labelled == 0:
                logger.info("no valid points, skipping...")
                continue
            live.append((start, kept))
            for s in range(start, start + kept, metrics.FLOW_CHUNK_POINTS):
                e = min(s + metrics.FLOW_CHUNK_POINTS, start + kept)
                out = model.query_flow(positions=points[s:e], normed_timestamps=times[s:e])
                color(out["forward_flow"], rows9[s:e, 3:6], density=out["dynamic_density"])
                out = None                              # free this chunk before the next query
            start += kept
        host = rows9[:start].cpu().numpy()              # the one copy back (sync 2)
    dynamic_coords = [host[s:s + k, 0:3].copy() for s, k in live]
    pred = [host[s:s + k, 3:6].copy() for s, k in live]
    gt = [host[s:s + k, 6:9].copy() for s, k in live]
    box = [float(v) for v in got[2 * len(frames):2 * len(frames) + 6]]
    x_ratio, y_ratio, z_ratio = voxels.box_ratios(got[2 * len(frames) + 6:])
    common = {"vis_aabb": box, "dynamic_coords": dynamic_coords, "x_ratio": x_ratio, "y_ratio": y_ratio,
              "z_ratio": z_ratio}
    return {"pred": dict(common, dynamic_colors=pred), "gt": dict(common, dynamic_colors=gt)}

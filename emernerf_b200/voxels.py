"""The voxel lifting of the reference's ``visualize_voxels`` (utils/visualization_tools.py:456-726) on the device
(csrc/voxels.cu): the 2-D foundation features lifted into a 3-D point cloud, coloured by a robust PCA.

    kw = voxels.visualize_voxels(cfg, model, proposal_estimator, proposal_networks, dataset, device=device,
                                 is_dynamic=cfg.nerf.model.head.enable_dynamic_branch)
    figure = vis_occ_plotly(**kw, size=3, black_bg=True, title=...)          # the reference's own figure code

``visualize_voxels`` returns the keyword arguments the reference hands to ``vis_occ_plotly``: ``vis_aabb``, ``coords``
and ``colors`` (numpy), ``dynamic_coords`` and ``dynamic_colors`` (lists of numpy arrays, or None), and ``x_ratio``,
``y_ratio``, ``z_ratio``.  It is built from three phases:

  1. marking: per image of ``dataset.full_pixel_set`` a lidar-mode ``render_rays`` and one ``emer_voxel_mark`` launch
     into bit grids; the first ``num_cams`` images are also rendered in full for the PCA features.  No host sync with
     ``raygen.PixelRaySampler`` bound as the source's ``get_render_rays``.
  2. ``robust_pca``: the reference's ``get_robust_pca``, the same torch calls in the same order.
  3. query: the occupied voxels of every grid listed by ``emer_voxel_compact`` (one sync for the counts), then per
     chunk one field pass with the feature head, the proposal networks' densities and one ``emer_voxel_select``;
     one device-to-host copy at the end.

A call syncs the host three times (the box, the voxel counts, the result) plus the syncs inside ``robust_pca``,
whatever the number of images, groups and chunks.  Everything runs under ``no_grad``.

The reference's behaviour that is kept on purpose:
  * the box grows by 1 on y_min, z_min and every maximum (``aabb[1:3] -= 1``, ``aabb[3:] += 1``), not on x_min;
  * resolutions are ``ceil(extent / vis_voxel_size)`` and, dynamic, ``ceil(extent / vis_voxel_size * 0.8)``, computed
    on the model's device with its arithmetic; points go to voxel ``trunc((p - min) / ((max - min) / res))``, and a
    voxel comes back as its minimum corner ``min + index * voxel_size``;
  * static rays count when their depth is below 80 (``depth`` for a static field, ``static_depth`` for a dynamic one);
    dynamic rays have no depth test;
  * a dynamic group is closed after image i when ``i % num_cams == 0 and i > 0`` (so group 0 holds num_cams + 1
    images), the images after the last close are dropped, and only the groups j with ``j % 10 == 0`` are queried, at
    ``pixel_source.unique_normalized_timestamps[j]``, with ``dynamic_density > 0.1`` and ``dynamic_dino_feat``; a
    group where no voxel passes is left out of the lists;
  * the static query runs the field without timestamps (static density and the static head's ``dino_feat``) and
    keeps the voxels whose mean density over the proposal networks and the field is above 0.5, chunk by chunk of
    2^18 voxels, with torch's CUDA mean;
  * no kept static voxel raises ``RuntimeError``, as the reference's ``torch.cat`` of an empty list does.

Deliberate differences: one field pass per chunk with the feature head (the density does not depend on it) where the
reference runs a density pass and a feature pass over the kept voxels; dynamic groups are queried in chunks of 2^18
voxels (the gate is one density per voxel, so chunking changes nothing); the PCA colour's dot product is fp64, rounded
once; and the figure and its files stay with the caller.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib, _ops

__all__ = ["visualize_voxels", "robust_pca", "VoxelGeometry"]

MAX_DEPTH = 80.0                 # the reference's static depth filter
STATIC_THRESHOLD = 0.5
DYNAMIC_THRESHOLD = 0.1
CHUNK = 1 << 18                  # the reference's static chunk: torch's mean factor depends on the chunk's length
GROUP_STRIDE = 10                # every tenth dynamic group is queried
MAX_VOXELS = 1 << 32             # per grid (EMER voxel index range)
MAX_CHANNELS = 256               # EMER_VOXEL_MAX_CHANNELS
MAX_GRIDS = 32                   # EMER_VOXEL_MAX_GRIDS
BLOCK_WORDS = 2048               # EMER_VOXEL_BLOCK_WORDS
SELECT_WORKSPACE_BYTES = 65600   # EMER_VOXEL_SELECT_WORKSPACE_BYTES
_WS: Dict[object, Tensor] = {}


def grown_box(aabb: Tensor) -> Tuple[Tensor, Tensor]:
    """The reference's figure box on ``aabb``'s device, fp32: (vis_aabb [6], its extent [3]).  The box grows by 1 on
    y_min, z_min and every maximum, not on x_min.  No host sync."""
    vis_aabb = aabb.detach().reshape(-1).to(torch.float32).clone()
    vis_aabb[1:3] -= 1
    vis_aabb[3:] += 1
    aabb_min, aabb_max = torch.split(vis_aabb, 3, dim=-1)
    return vis_aabb, aabb_max - aabb_min


def box_ratios(length) -> Tuple[float, float, float]:
    """The figure's x, y and z ratios: 1 and the fp32 quotients of the box's extents, as the reference's ``.item()``."""
    l0, l1, l2 = np.asarray(length, np.float32)
    return 1, float(l1 / l0), float(l2 / l0)


class VoxelGeometry:
    """The box, resolutions and voxel sizes of the reference, computed on ``device`` with its torch ops (one sync)."""

    def __init__(self, aabb: Tensor, vis_voxel_size: float):
        vis_aabb, length = grown_box(aabb)
        res_s = torch.ceil(length / vis_voxel_size).long()
        res_d = torch.ceil(length / vis_voxel_size * 0.8).long()
        packed = torch.cat([vis_aabb, length, length / res_s, length / res_d]).double()
        vals = torch.cat([packed, res_s.double(), res_d.double()]).tolist()     # the one sync
        self.vis_aabb = vals[0:6]
        self.min = vals[0:3]
        self.length = np.array(vals[6:9], np.float32)
        self.static_size, self.dynamic_size = vals[9:12], vals[12:15]
        self.static_res = [int(v) for v in vals[15:18]]
        self.dynamic_res = [int(v) for v in vals[18:21]]
        for res in (self.static_res, self.dynamic_res):
            if min(res) < 1 or int(np.prod(res, dtype=np.float64)) > MAX_VOXELS:
                raise ValueError(f"voxel lifting: a {res[0]} x {res[1]} x {res[2]} grid (1 to 2^32 voxels)")

    def ratios(self) -> Tuple[float, float, float]:
        return box_ratios(self.length)


class BitGrid:
    """One bit grid on the device and its ``emer_voxel_grid`` host struct."""

    def __init__(self, origin, size, res, device):
        n = res[0] * res[1] * res[2]
        self.bits = torch.zeros((n + 31) // 32, dtype=torch.int32, device=device)
        self.words = self.bits.numel()
        self.c = _lib.EmerVoxelGrid((ctypes.c_float * 3)(*origin), (ctypes.c_float * 3)(*size),
                                    (ctypes.c_int64 * 3)(*res), _ops._ptr(self.bits), 0)


def _need_device(*ts: Tensor) -> None:
    for t in ts:
        if t is not None and not _ops.on_device(t):
            raise ValueError("voxel lifting: tensors must be CUDA tensors")


def mark(grid: BitGrid, origins: Tensor, viewdirs: Tensor, depth: Tensor, dynamic: Optional[BitGrid] = None,
         dynamic_depth: Optional[Tensor] = None) -> None:
    """One ``emer_voxel_mark`` launch for one image's rays: any shapes ending in 3 (origins, viewdirs) and 1 (depths),
    read in place when their rows are strided."""
    _need_device(origins, viewdirs, depth, dynamic_depth)
    o, ld_o = _ops._rows(origins, 3)
    d, ld_d = _ops._rows(viewdirs, 3)
    t, ld_t = _ops._rows(depth, 1)
    dd, ld_dd = (None, 1) if dynamic is None else _ops._rows(dynamic_depth, 1)
    n = o.shape[0]
    if d.shape[0] != n or t.shape[0] != n or (dd is not None and dd.shape[0] != n):
        raise ValueError(f"voxel lifting: {n} origins, {d.shape[0]} directions and {t.shape[0]} depths")
    _ops._need_cuda(o, d, t, dd, grid.bits)
    p = _ops._ptr
    _lib.call("emer_voxel_mark", p(o), ld_o, p(d), ld_d, p(t), ld_t, p(dd), ld_dd, n, MAX_DEPTH,
              ctypes.byref(grid.c), None if dynamic is None else ctypes.byref(dynamic.c), _ops._stream())


def _compact_workspace(grids: List[BitGrid], dev) -> Tensor:
    blocks = sum((g.words + BLOCK_WORDS - 1) // BLOCK_WORDS for g in grids)
    return torch.zeros(1 + blocks, dtype=torch.int64, device=dev)


def compact(grids: List[BitGrid]) -> Tuple[Tensor, List[int]]:
    """The set voxels of every grid as world coordinates in linear-index order, one [total, 3] tensor, and each grid's
    count.  One host sync, for the counts."""
    dev = grids[0].bits.device
    _ops._need_cuda(*(g.bits for g in grids))
    counts = torch.empty(len(grids), dtype=torch.int64, device=dev)
    batches = [grids[s:s + MAX_GRIDS] for s in range(0, len(grids), MAX_GRIDS)]
    spaces = []
    p = _ops._ptr
    for b, batch in enumerate(batches):
        ws = _compact_workspace(batch, dev)
        arr = (_lib.EmerVoxelGrid * len(batch))(*(g.c for g in batch))
        _lib.call("emer_voxel_compact", arr, len(batch), p(counts[b * MAX_GRIDS:]), None, p(ws), _ops._stream())
        spaces.append((arr, ws))
    got = counts.tolist()                                                    # the one sync
    coords = torch.empty((sum(got), 3), dtype=torch.float32, device=dev)
    row = 0
    for b, (arr, ws) in enumerate(spaces):
        for j in range(len(arr)):
            arr[j].first_row = row
            row += got[b * MAX_GRIDS + j]
        _lib.call("emer_voxel_compact", arr, len(arr), p(counts[b * MAX_GRIDS:]), p(coords), p(ws), _ops._stream())
    return coords, got


def _select_workspace(dev) -> Tensor:
    return _ops._workspace(_WS, dev, SELECT_WORKSPACE_BYTES, "voxels")


def select(densities: List[Tensor], threshold: float, points: Tensor, feat: Tensor, reduction: Tensor,
           color_min: Tensor, color_max: Tensor, out_points: Tensor, out_colors: Tensor, count: Tensor) -> None:
    """One ``emer_voxel_select`` launch: the voxels of ``points`` whose mean of ``densities`` (1 to 3 columns, torch's
    CUDA mean) is above ``threshold`` are appended with their PCA colours at ``count`` (int64 [1], advanced)."""
    n = points.shape[0]
    if not 1 <= len(densities) <= 3:
        raise ValueError(f"voxel lifting: {len(densities)} density columns (1..3)")
    c = feat.shape[-1]
    if c % 4 != 0 or not 4 <= c <= MAX_CHANNELS:
        raise ValueError(f"voxel lifting: {c} feature channels (a multiple of 4, at most {MAX_CHANNELS})")
    cols = [_ops._f32c(d.reshape(-1)) for d in densities]
    f, ld = _ops._rows(feat, c)
    if ld % 4 != 0 or f.data_ptr() % 16 != 0:
        f, ld = f.contiguous(), c
    if f.shape[0] != n or any(x.numel() != n for x in cols):
        raise ValueError(f"voxel lifting: {f.shape[0]} feature rows and densities of "
                         f"{[x.numel() for x in cols]} for {n} voxels")
    pts, m = _ops._f32c(points), _ops._f32c(reduction)
    if tuple(m.shape) != (c, 3):
        raise ValueError(f"voxel lifting: a {tuple(m.shape)} reduction for {c} channels")
    lo, hi = _ops._f32c(color_min.reshape(-1)), _ops._f32c(color_max.reshape(-1))
    _ops._need_cuda(pts, f, m, lo, hi, out_points, out_colors, count, *cols)
    cols += [None] * (3 - len(cols))
    p = _ops._ptr
    _lib.call("emer_voxel_select", p(cols[0]), p(cols[1]), p(cols[2]), len(densities), threshold, p(pts), p(f), ld,
              c, p(m), p(lo), p(hi), n, p(out_points), p(out_colors), p(count), p(_select_workspace(pts.device)),
              _ops._stream())


def robust_pca(features: Tensor, m: float = 2.5) -> Tuple[Tensor, Tensor, Tensor]:
    """A 3-channel PCA basis of ``features`` [N, C] and the per-channel colour range of its inliers: the reference's
    ``get_robust_pca`` (utils/misc.py:23-47).  ``pca_lowrank(q=3, niter=20)``, the projection, then per channel the
    points whose distance to the median is below ``m`` median absolute deviations; the minimum and maximum of those
    give the range.  Returns (basis [C, 3], minimum [3], maximum [3]) on the features' device."""
    if features.dim() != 2:
        raise ValueError("robust_pca: features must be [N, C]")
    basis = torch.pca_lowrank(features, q=3, niter=20)[2]
    proj = features @ basis
    spread = torch.abs(proj - torch.median(proj, dim=0).values)
    score = spread / torch.median(spread, dim=0).values
    inliers = [proj[score[:, a] < m, a] for a in range(3)]
    lo = torch.stack([x.min() for x in inliers])
    hi = torch.stack([x.max() for x in inliers])
    return basis, lo.to(basis), hi.to(basis)


def _eval(model, proposal_estimator, proposal_networks) -> None:
    model.eval()
    if proposal_estimator is not None:
        proposal_estimator.eval()
    for p in proposal_networks or ():
        p.eval()


def group_of(i: int, num_cams: int) -> int:
    """The dynamic group image ``i`` falls in (group 0 holds images 0..num_cams)."""
    return 0 if i == 0 else (i - 1) // num_cams


def queried_groups(n_images: int, num_cams: int) -> List[int]:
    """The groups the reference queries: closed after an image i > 0 with i % num_cams == 0, every tenth."""
    closed = (n_images - 1) // num_cams if n_images > 0 else 0
    return [j for j in range(closed) if j % GROUP_STRIDE == 0]


def mark_images(cfg, model, proposal_estimator, proposal_networks, dataset, geo: VoxelGeometry, is_dynamic: bool):
    """Phase 1: (static grid, {group: dynamic grid}, PCA feature rows).  No host sync of its own."""
    from .radiance_fields.render_utils import render_rays

    _eval(model, proposal_estimator, proposal_networks)
    dev = model.aabb.device
    static = BitGrid(geo.min, geo.static_size, geo.static_res, dev)
    pixel_set = dataset.full_pixel_set
    n_images, num_cams = len(pixel_set), dataset.num_cams
    groups = {j: BitGrid(geo.min, geo.dynamic_size, geo.dynamic_res, dev)
              for j in queried_groups(n_images, num_cams)} if is_dynamic else {}
    patches = []
    with torch.no_grad():
        for i in range(n_images):
            data = dict(pixel_set[i])
            _need_device(data["origins"])
            if i < num_cams:
                out = render_rays(radiance_field=model, proposal_estimator=proposal_estimator,
                                  proposal_networks=proposal_networks, data_dict=data, cfg=cfg,
                                  proposal_requires_grad=False)
                f = out["dino_pe_free"] if "dino_pe_free" in out else out["dino_feat"]
                patches.append(f.reshape(-1, f.shape[-1]))
            data["lidar_origins"] = data["origins"]
            data["lidar_viewdirs"] = data["viewdirs"]
            data["lidar_normed_timestamps"] = data["normed_timestamps"]
            out = render_rays(radiance_field=model, proposal_estimator=proposal_estimator,
                              proposal_networks=proposal_networks, data_dict=data, cfg=cfg,
                              proposal_requires_grad=False, prefix="lidar_", return_decomposition=True)
            dyn = groups.get(group_of(i, num_cams)) if is_dynamic else None
            mark(static, data["origins"], data["viewdirs"], out["static_depth"] if is_dynamic else out["depth"],
                 dyn, out["dynamic_depth"] if dyn is not None else None)
    return static, groups, patches


def query(model, proposal_networks, grids: List[Tuple[Optional[int], Tensor]], timestamps: Optional[Tensor], pca,
          out_points: Tensor, out_colors: Tensor, counts: Tensor) -> None:
    """Phase 3 after the compaction, for ``grids`` = [(None, static candidates), (group j, its candidates), ...]:
    the static candidates gated over the proposal networks and the field (0.5), a group's over its dynamic density
    (0.1).  Grid g's kept voxels and colours go to ``out_points`` / ``out_colors`` from the row where its candidates
    start, ``counts[g]`` (int64, zeroed) the kept count.  No host sync."""
    props = list(proposal_networks or ())
    if len(props) > 2:
        raise ValueError(f"voxel lifting: {len(props)} proposal networks (the gate takes at most 2)")
    row = 0
    with torch.no_grad():
        for g, (j, pts_all) in enumerate(grids):
            for s in range(0, pts_all.shape[0], CHUNK):
                pts = pts_all[s:s + CHUNK]
                if j is None:
                    res = model.forward(pts, query_feature_head=True, query_pe_head=False)
                    dens = [p(pts)["density"].squeeze(-1) for p in props] + [res["density"]]
                    feat, thr = res["dino_feat"], STATIC_THRESHOLD
                else:
                    ts = timestamps[j].repeat(pts.shape[0], 1)
                    res = model.forward(pts, data_dict={"normed_timestamps": ts}, query_feature_head=True,
                                        query_pe_head=False)
                    dens, feat, thr = [res["dynamic_density"]], res["dynamic_dino_feat"], DYNAMIC_THRESHOLD
                n = pts_all.shape[0]
                select(dens, thr, pts, feat, *pca, out_points[row:row + n], out_colors[row:row + n],
                       counts[g:g + 1])
                res = feat = dens = None                # free this chunk before the next forward
            row += pts_all.shape[0]


def visualize_voxels(cfg, model, proposal_estimator=None, proposal_networks=None, dataset=None, device="cuda",
                     is_dynamic: bool = False) -> Dict[str, object]:
    """The reference's ``visualize_voxels`` up to its ``vis_occ_plotly`` call: returns that call's keyword arguments
    (``vis_aabb``, ``coords``, ``colors``, ``dynamic_coords``, ``dynamic_colors``, ``x_ratio``, ``y_ratio``,
    ``z_ratio``).  The model's device is used; ``device`` is the reference's argument and only names it."""
    vs = getattr(getattr(cfg, "render", None), "vis_voxel_size", None)
    if vs is None:
        raise ValueError("voxel lifting: cfg.render.vis_voxel_size is not set")
    _need_device(model.aabb)
    geo = VoxelGeometry(model.aabb, float(vs))
    static, groups, patches = mark_images(cfg, model, proposal_estimator, proposal_networks, dataset, geo,
                                          is_dynamic)
    pca = robust_pca(torch.cat(patches, dim=0), m=2.5)
    if pca[0].shape[0] % 4 != 0 or not 4 <= pca[0].shape[0] <= MAX_CHANNELS:
        raise ValueError(f"voxel lifting: {pca[0].shape[0]} feature channels (a multiple of 4, at most "
                         f"{MAX_CHANNELS})")
    order = sorted(groups)
    coords, got = compact([static] + [groups[j] for j in order])
    dev, total, n_grids = coords.device, coords.shape[0], len(got)
    # one buffer for everything that comes back: kept counts, then points and colours per grid from its first row
    buf = torch.empty(8 * n_grids + 24 * total, dtype=torch.uint8, device=dev)
    counts = buf[:8 * n_grids].view(torch.int64)
    counts.zero_()
    out_points = buf[8 * n_grids:8 * n_grids + 12 * total].view(torch.float32).view(total, 3)
    out_colors = buf[8 * n_grids + 12 * total:].view(torch.float32).view(total, 3)
    starts = np.cumsum([0] + got).tolist()
    grids = [(j, coords[starts[g]:starts[g + 1]]) for g, j in enumerate([None] + order)]
    timestamps = dataset.pixel_source.unique_normalized_timestamps.to(dev) if order else None
    query(model, proposal_networks, grids, timestamps, pca, out_points, out_colors, counts)
    host = buf.cpu()                                                          # the one copy back
    kept = host[:8 * n_grids].view(torch.int64).tolist()
    pts = host[8 * n_grids:8 * n_grids + 12 * total].view(torch.float32).view(total, 3).numpy()
    cols = host[8 * n_grids + 12 * total:].view(torch.float32).view(total, 3).numpy()
    if kept[0] == 0:
        raise RuntimeError("torch.cat(): expected a non-empty list of Tensors (no voxel passed the static density "
                           "threshold, as in the reference)")
    dynamic_coords = dynamic_colors = None
    if is_dynamic:
        live = [g for g in range(1, n_grids) if kept[g] > 0]
        dynamic_coords = [pts[starts[g]:starts[g] + kept[g]].copy() for g in live]
        dynamic_colors = [cols[starts[g]:starts[g] + kept[g]].copy() for g in live]
    x_ratio, y_ratio, z_ratio = geo.ratios()
    return {"vis_aabb": geo.vis_aabb, "coords": pts[:kept[0]].copy(), "colors": cols[:kept[0]].copy(),
            "dynamic_coords": dynamic_coords, "dynamic_colors": dynamic_colors, "x_ratio": x_ratio, "y_ratio": y_ratio, "z_ratio": z_ratio}

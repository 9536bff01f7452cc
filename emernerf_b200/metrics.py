"""The evaluation metrics of the reference on the device (csrc/metrics.cu): ``datasets/metrics.py``'s ``compute_psnr``,
``compute_ssim``, ``compute_valid_depth_rmse`` and ``compute_scene_flow_metrics`` with the same signatures, return types
and keys, plus the per-image metric block of ``radiance_fields/video_utils.py:render`` and its aggregation.

    from emernerf_b200 import metrics
    per_image.append(metrics.image_metrics(rgb, pixels, dynamic_mask, dino_feat, features))   # no host sync
    results = metrics.summarize(per_image)                                                   # one sync

Every function is one library launch.  ``image_metrics`` returns 0-d fp64 device tensors and can be captured in a CUDA
graph; the functions that return Python floats sync once, for that float.

Differences from the reference, all deliberate:
  * SSIM's window moments and map are fp64 (skimage computes them in the images' dtype, float32 here); the results
    agree with skimage's float32 path to its own rounding, about 1e-6.
  * PSNRs, RMSE and the flow statistics accumulate in fp64, so they are the fp64 values of the reference's formulas.
  * Inputs are cast to fp32 on the device; numpy arrays are moved to the current CUDA device first.  Any other
    non-CUDA tensor is an error, as everywhere in this package.

The few-shot occupancy evaluation (csrc/occupancy.cu), ``collect_centroids`` and ``eval_few_shot_occ``, keeps the
reference's signatures, return types and keys:

    centroids_bank, label_bank = metrics.collect_centroids(train_indices, dataset, model, device)   # no host sync
    occ = metrics.eval_few_shot_occ(test_indices, dataset, model, device, centroids_bank, label_bank)  # one sync

Per frame it runs the field once, in chunks of ``OCC_CHUNK_POINTS`` voxels, and launches one kernel per chunk.
Deliberate differences from the reference:
  * One field pass with the feature head, where the reference runs a density pass, keeps the voxels with
    density > 0.2 by boolean indexing and runs a second pass over them for the features.  The field is
    row-independent, so the kept voxels get the same features, up to the layer kernels' choice by row count.
  * Frames are evaluated in chunks, so memory does not grow with a frame's size, and the centroids come from fp64
    per-class sums, not from a concatenation of every kept feature row of every train frame.
  * Cosine similarities are fp64, and an exact tie goes to the lowest class index (the reference's ``topk`` leaves
    the order of ties unspecified).
  * Neither function switches the model to eval mode; the reference's driver does that before it calls them.

The lidar scene-flow evaluation (``emer_lidar_flow_accumulate``, csrc/metrics.cu) replaces the flow block of the
reference's driver (train_emernerf.py:237-281) with one call:

    avg_flow_metrics = metrics.eval_lidar_flow(dataset.full_lidar_set, model, remove_ground=True)   # one sync

Per frame it runs ``model.query_flow`` over every point of the frame, in chunks of ``FLOW_CHUNK_POINTS``, and launches
one kernel per chunk, which applies the flow-class filter, the ground filter and the dynamic-density gate itself.
Deliberate differences from the reference:
  * The field runs on every point of the frame, where the reference first compacts the frame by boolean indexing.
    The field is row-independent, so the counted points get the same flows, up to the layer kernels' choice by row
    count.
  * The per-frame statistics are fp64 sums, where the reference's are fp32 means; a point whose error lies within
    fp32 rounding of a threshold may count differently.
"""
from __future__ import annotations

import logging
import weakref
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from . import _lib, _ops

__all__ = ["compute_psnr", "compute_ssim", "compute_valid_depth_rmse", "compute_scene_flow_metrics", "image_metrics",
           "summarize", "collect_centroids", "eval_few_shot_occ", "eval_lidar_flow"]
logger = logging.getLogger()

WORKSPACE_BYTES = 81920          # EMER_METRICS_WORKSPACE_BYTES
MAX_CHANNELS = 4                 # image channels
MAX_FEATURE_CHANNELS = 256
WINDOW = 7                       # SSIM window: images need at least 7 x 7 pixels
IMAGE_OUT = ("psnr", "ssim", "masked_psnr", "masked_ssim", "feat_psnr", "masked_feat_psnr", "mask_count",
             "pred_min", "pred_max", "target_min", "target_max")         # EMER_METRIC_* order
FLOW_KEYS = ("EPE3D", "acc3d_strict", "acc3d_relax", "outlier", "angle_error")
SUMMARY_KEYS = ("psnr", "ssim", "feat_psnr", "masked_psnr", "masked_ssim", "masked_feat_psnr")
_WS: Dict[object, Tensor] = {}
OCC_WORKSPACE_BYTES = 16912640   # EMER_OCC_WORKSPACE_BYTES
OCC_MAX_CHANNELS = 256           # EMER_OCC_MAX_CHANNELS
OCC_MAX_CLASSES = 32             # EMER_OCC_MAX_CLASSES
OCC_CHUNK_POINTS = 1 << 20       # voxels per field pass: bounds the memory of a frame of any size
OCC_DENSITY_THRESHOLD = 0.2      # the reference's filter of the voxels the cameras see
OCC_FEATURE_DIM = 64             # the reference's width of a centroid when no frame produced a feature
_OCC_WS: Dict[object, Tensor] = {}
FLOW_CHUNK_POINTS = 1 << 20      # lidar points per query_flow call: bounds the memory of a frame of any size
FLOW_DENSITY_THRESHOLD = 0.2     # the reference's gate: flows count only on dynamic points
FLOW_SUMS = 8                    # EMER_LIDAR_FLOW_SUMS
FLOW_EVAL_KEYS = ("EPE3D", "acc3d_strict", "acc3d_relax", "angle_error", "outlier")   # the driver's key order


def _numpy_device() -> torch.device:
    return torch.device("cuda", torch.cuda.current_device())


def _tensor(x: Union[Tensor, np.ndarray]) -> Tensor:
    """numpy arrays go to the current CUDA device (the reference's compute_psnr / compute_ssim accept them)."""
    if isinstance(x, Tensor):
        return x
    return torch.as_tensor(np.asarray(x)).to(_numpy_device())


def _image_launch(pred: Tensor, target: Tensor, mask: Optional[Tensor] = None, feat_pred: Optional[Tensor] = None,
                  feat_target: Optional[Tensor] = None) -> Tensor:
    """One emer_image_metrics launch; returns its fp64 out[11] on the device."""
    _ops._need_cuda(pred, target, mask, feat_pred, feat_target)
    if pred.dim() != 3 or pred.shape != target.shape:
        raise ValueError(f"image metrics: prediction {tuple(pred.shape)} and target {tuple(target.shape)} must be the "
                         "same [H, W, C]")
    h, w, c = pred.shape
    if not 1 <= c <= MAX_CHANNELS:
        raise ValueError(f"image metrics: {c} channels (1..{MAX_CHANNELS})")
    if h < WINDOW or w < WINDOW:
        raise ValueError(f"image metrics: a {h}x{w} image is smaller than the {WINDOW}x{WINDOW} SSIM window")
    x, y = _ops._f32c(pred), _ops._f32c(target)
    m = None
    if mask is not None:
        if mask.numel() != h * w:
            raise ValueError(f"image metrics: mask {tuple(mask.shape)} for a {h}x{w} image")
        m = _ops._f32c(mask.reshape(-1))
    fx = fy = None
    ld_x = ld_y = cf = 0
    if feat_pred is not None and feat_target is not None:
        if feat_pred.dim() != 3 or feat_pred.shape != feat_target.shape or tuple(feat_pred.shape[:2]) != (h, w):
            raise ValueError(f"image metrics: features {tuple(feat_pred.shape)} and {tuple(feat_target.shape)} must "
                             f"be the same [{h}, {w}, Cf]")
        cf = feat_pred.shape[-1]
        if not 1 <= cf <= MAX_FEATURE_CHANNELS:
            raise ValueError(f"image metrics: {cf} feature channels (1..{MAX_FEATURE_CHANNELS})")
        fx, ld_x = _ops._rows(feat_pred, cf)
        fy, ld_y = _ops._rows(feat_target, cf)
    out = torch.empty(len(IMAGE_OUT), dtype=torch.float64, device=x.device)
    ws = _ops._workspace(_WS, x.device, WORKSPACE_BYTES, "metrics")
    _lib.call("emer_image_metrics", _ops._ptr(x), _ops._ptr(y), h, w, c, _ops._ptr(m), _ops._ptr(fx), ld_x,
              _ops._ptr(fy), ld_y, cf, _ops._ptr(out), _ops._ptr(ws), _ops._stream())
    return out


def _pair_launch(name: str, pred: Tensor, target: Tensor, n_out: int) -> Tensor:
    _ops._need_cuda(pred, target)
    p, t = _ops._f32c(pred), _ops._f32c(target)
    out = torch.empty(n_out, dtype=torch.float64, device=p.device)
    n = p.numel() // 3 if name == "emer_scene_flow_metrics" else p.numel()
    ws = _ops._workspace(_WS, p.device, WORKSPACE_BYTES, "metrics")
    _lib.call(name, _ops._ptr(p), _ops._ptr(t), n, _ops._ptr(out), _ops._ptr(ws), _ops._stream())
    return out


def compute_valid_depth_rmse(prediction: Tensor, target: Tensor) -> float:
    """RMSE between predicted and target depths over the rays with target > 0 (NaN when there is none)."""
    prediction, target = prediction.squeeze(), target.squeeze()
    if prediction.shape != target.shape:
        raise ValueError(f"depth RMSE: {tuple(prediction.shape)} vs {tuple(target.shape)}")
    return _pair_launch("emer_depth_rmse", prediction, target, 3)[0].item()


def compute_psnr(prediction: Union[Tensor, np.ndarray], target: Union[Tensor, np.ndarray]) -> float:
    """-10 log10(mean squared error) over all elements of two tensors of one shape."""
    prediction, target = _tensor(prediction), _tensor(target)
    if prediction.shape != target.shape:
        raise ValueError(f"PSNR: {tuple(prediction.shape)} vs {tuple(target.shape)}")
    return _pair_launch("emer_depth_rmse", prediction, target, 3)[2].item()


def compute_ssim(prediction: Union[Tensor, np.ndarray], target: Union[Tensor, np.ndarray]) -> float:
    """skimage's structural_similarity(target, prediction, data_range=1.0, channel_axis=-1) of two [H, W, C] images,
    after the reference's range assertions (target first), which read the extrema of the same launch."""
    prediction, target = _tensor(prediction), _tensor(target)
    out = _image_launch(prediction, target).tolist()
    o = dict(zip(IMAGE_OUT, out))
    assert o["target_max"] <= 1.0 and o["target_min"] >= 0.0, "target must be in range [0, 1]"
    assert o["pred_max"] <= 1.0 and o["pred_min"] >= 0.0, "prediction must be in range [0, 1]"
    return o["ssim"]


def compute_scene_flow_metrics(pred: Tensor, labels: Tensor) -> Dict[str, float]:
    """The NSFP statistics (EPE3D, acc3d_strict, acc3d_relax, outlier, angle_error) of [..., N, 3] flows."""
    if pred.shape != labels.shape or pred.dim() != 3 or pred.shape[-1] != 3:
        raise ValueError(f"scene flow metrics: pred {tuple(pred.shape)} and labels {tuple(labels.shape)} must be the "
                         "same [B, N, 3]")
    out = _pair_launch("emer_scene_flow_metrics", pred, labels, 7).tolist()
    return dict(zip(FLOW_KEYS, out[:5]))


def image_metrics(rgb: Tensor, pixels: Tensor, dynamic_mask: Optional[Tensor] = None,
                  dino_feat: Optional[Tensor] = None, features: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """The metric block of ``video_utils.render`` for one image, as 0-d fp64 device tensors, in one launch and with no
    host sync: ``psnr`` and ``ssim``; with a mask, ``masked_psnr``, ``masked_ssim`` and ``mask_count`` (the masked
    metrics are NaN when the mask is empty); with both feature maps, ``feat_psnr`` and, with a mask,
    ``masked_feat_psnr``.  ``summarize`` aggregates a list of these as the reference does."""
    have_feat = dino_feat is not None and features is not None
    out = _image_launch(rgb, pixels, dynamic_mask, dino_feat if have_feat else None, features if have_feat else None)
    keys = ["psnr", "ssim"]
    if dynamic_mask is not None:
        keys += ["masked_psnr", "masked_ssim", "mask_count"]
    if have_feat:
        keys += ["feat_psnr"] + (["masked_feat_psnr"] if dynamic_mask is not None else [])
    return {k: out[IMAGE_OUT.index(k)] for k in keys}


def summarize(per_image: List[Dict[str, Tensor]]) -> Dict[str, float]:
    """The reference's aggregation (``video_utils.py:45-47,421-428``): per metric, the mean over the images that
    produced it, or -1 where none did.  The masked metrics count for an image whose mask is not empty, as the
    reference's ``dynamic_mask.sum() > 0``.  One host sync for the whole list."""
    flat = [v for d in per_image for v in d.values()]
    values = torch.stack(flat).tolist() if flat else []
    lists: Dict[str, List[float]] = {k: [] for k in SUMMARY_KEYS}
    i = 0
    for d in per_image:
        got = dict(zip(d.keys(), values[i:i + len(d)]))
        i += len(d)
        for k in SUMMARY_KEYS:
            if k not in got or (k.startswith("masked_") and not got.get("mask_count", 0.0) > 0):
                continue
            lists[k].append(got[k])
    return {k: sum(v) / len(v) if len(v) > 0 else -1 for k, v in lists.items()}


# ---------------------------------------------------------------------------------------------- few-shot occupancy
def _occ_workspace(dev: torch.device) -> Tensor:
    return _ops._workspace(_OCC_WS, dev, OCC_WORKSPACE_BYTES, "occupancy")


def _occ_limits(n_classes: int, channels: int) -> None:
    if not 1 <= n_classes <= OCC_MAX_CLASSES:
        raise ValueError(f"occupancy evaluation: {n_classes} classes (1..{OCC_MAX_CLASSES})")
    if channels % 4 != 0 or not 4 <= channels <= OCC_MAX_CHANNELS:
        raise ValueError(f"occupancy evaluation: {channels} feature channels (a multiple of 4, at most "
                         f"{OCC_MAX_CHANNELS})")


def _occ_field(dataset, index: int, model, device):
    """One frame of ``dataset.get_occ``: yields, per chunk of at most OCC_CHUNK_POINTS voxels, the field's dino
    features as 16-byte aligned rows, their row stride, the densities and the int64 labels, from ONE forward pass with
    the feature head.  The frame's voxel count comes first."""
    coords, labels, t = dataset.get_occ(index)
    coords, labels, t = coords.to(device), labels.to(device), t.to(device)
    labels = labels.reshape(-1).to(torch.int64).contiguous()
    n = labels.numel()
    yield n
    for s in range(0, n, OCC_CHUNK_POINTS):
        e = min(s + OCC_CHUNK_POINTS, n)
        with torch.no_grad():
            out = model.forward(positions=coords[s:e], data_dict={"normed_timestamps": t[s:e]},
                                combine_static_dynamic=True, query_feature_head=True, query_pe_head=False)
        c = out["dino_feat"].shape[-1]
        feat, ld = _ops._rows(out["dino_feat"], c)
        if ld % 4 != 0 or feat.data_ptr() % 16 != 0:
            feat, ld = feat.contiguous(), c
        density = _ops._f32c(out["density"].reshape(-1))
        if feat.shape[0] != e - s or density.numel() != e - s:
            raise ValueError(f"occupancy evaluation: the field returned {feat.shape[0]} feature rows and "
                             f"{density.numel()} densities for {e - s} voxels")
        yield feat, ld, density, labels[s:e]
        out = feat = density = None                 # free this chunk before the next forward


def collect_centroids(train_indices, dataset, model, device) -> Tuple[Tensor, Tensor]:
    """The per-class mean dino feature of the voxels with density > 0.2 over the train frames, as the reference's
    ``collect_centroids``: (centroids_bank fp32 [len(dataset.label_mapping), C] with zero rows for the classes no
    such voxel has, label_bank int64 arange).  Labels outside the mapping are skipped.  No host sync."""
    sums = counts = None
    for i in train_indices:
        frame = _occ_field(dataset, i, model, device)
        next(frame)
        k = len(dataset.label_mapping)              # the reference's Occ3D dataset sets it in get_occ
        for feat, ld, density, labels in frame:
            c = feat.shape[1]
            if sums is None:
                _occ_limits(k, c)
                sums = torch.zeros(k, c, dtype=torch.float64, device=feat.device)
                counts = torch.zeros(k, dtype=torch.int64, device=feat.device)
            if tuple(sums.shape) != (k, c):
                raise ValueError(f"occupancy evaluation: {k} classes x {c} channels after {tuple(sums.shape)}")
            _ops._need_cuda(feat, density, labels, sums)
            ws = _occ_workspace(feat.device)
            _lib.call("emer_occ_accumulate", _ops._ptr(feat), ld, c, _ops._ptr(density), 1, _ops._ptr(labels),
                      feat.shape[0], k, OCC_DENSITY_THRESHOLD, _ops._ptr(sums), _ops._ptr(counts), _ops._ptr(ws),
                      _ops._stream())
    k = len(dataset.label_mapping)
    if sums is None:
        return torch.zeros(k, OCC_FEATURE_DIM, device=device), torch.arange(k, device=device)
    centroids = (sums / counts.clamp_min(1)[:, None].to(torch.float64)).to(torch.float32)
    return centroids, torch.arange(k, device=centroids.device)


def eval_few_shot_occ(test_indices, dataset, model, device, centroids_bank: Tensor,
                      label_bank: Tensor) -> Dict[str, object]:
    """Nearest-centroid (cosine) classification of the voxels with density > 0.2 over the test frames, as the
    reference's ``eval_few_shot_occ``: ``micro_accuracy``, ``macro_accuracy`` (over the classes with voxels),
    ``per_class_accuracy`` keyed by class name, ``cover_rate``, ``num_measured_points`` and ``num_total_points``, as
    Python numbers.  One host sync, at the end.  Raises ZeroDivisionError when no test voxel passes the filter and
    KeyError when a voxel that does has a label outside ``dataset.label_mapping``, as the reference does."""
    mapping = dataset.label_mapping
    k = len(mapping)
    if sorted(mapping) != list(range(k)):
        raise ValueError("occupancy evaluation: label_mapping must map the class ids 0..K-1 to names")
    if centroids_bank.dim() != 2 or centroids_bank.shape[0] != k or label_bank.numel() != k:
        raise ValueError(f"occupancy evaluation: centroids {tuple(centroids_bank.shape)} and label bank "
                         f"{tuple(label_bank.shape)} for {k} classes")
    c = centroids_bank.shape[1]
    _occ_limits(k, c)
    centroids = _ops._f32c(centroids_bank)
    bank = label_bank.reshape(-1).to(torch.int64).contiguous()
    counts = torch.zeros(2 * k + 2, dtype=torch.int64, device=centroids.device)
    num_total_points = 0
    for i in test_indices:
        frame = _occ_field(dataset, i, model, device)
        num_total_points += next(frame)
        for feat, ld, density, labels in frame:
            if feat.shape[1] != c:
                raise ValueError(f"occupancy evaluation: {feat.shape[1]}-channel features for {c}-channel centroids")
            _ops._need_cuda(feat, density, labels, centroids, bank, counts)
            ws = _occ_workspace(feat.device)
            _lib.call("emer_occ_classify", _ops._ptr(feat), ld, c, _ops._ptr(density), 1, _ops._ptr(labels),
                      feat.shape[0], _ops._ptr(centroids), k, _ops._ptr(bank), OCC_DENSITY_THRESHOLD,
                      _ops._ptr(counts), _ops._ptr(ws), _ops._stream())
    got = counts.tolist()                           # the one host sync
    total, correct, measured, outside = got[:k], got[k:2 * k], got[2 * k], got[2 * k + 1]
    if outside:
        raise KeyError(f"{outside} measured voxels have labels outside label_mapping")
    micro = sum(correct) / measured                 # ZeroDivisionError when no voxel is measured, as the reference
    accs, non_zero = 0, 0
    for label in mapping:
        if total[label] != 0:
            accs += correct[label] / total[label]
            non_zero += 1
    return {
        "micro_accuracy": micro,
        "macro_accuracy": accs / non_zero,
        "per_class_accuracy": {name: correct[cid] / (total[cid] + 1e-10) for cid, name in mapping.items()},
        "cover_rate": measured / num_total_points,
        "num_measured_points": measured,
        "num_total_points": num_total_points,
    }


# ---------------------------------------------------------------------------------------------- lidar scene flow
_SAMPLERS: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()


def _lidar_sampler(source):
    """The LidarRaySampler whose frame table serves ``source``: the one bound as ``source.get_render_rays`` if there
    is one, else one kept per source (it holds the source by a weak proxy, so the cache does not keep it alive)."""
    from .raygen import LidarRaySampler

    bound = getattr(getattr(source, "get_render_rays", None), "__self__", None)
    if isinstance(bound, LidarRaySampler) and bound.source is source:
        return bound
    try:
        sampler = _SAMPLERS.get(source)
        if sampler is None:
            sampler = _SAMPLERS[source] = LidarRaySampler(weakref.proxy(source))
        return sampler
    except TypeError:                               # not weakly referenceable: a table per call
        return LidarRaySampler(source)


def eval_lidar_flow(lidar_set, model, remove_ground: bool = True) -> Dict[str, np.float64]:
    """The lidar scene-flow evaluation of the reference's driver (train_emernerf.py:237-281) over
    ``dataset.full_lidar_set`` (anything with ``datasource`` and ``split_indices``): per frame, the points with a
    flow label (``lidar_flow_class != -1``), without the ground points when ``remove_ground``, the model's forward
    flow zeroed where its dynamic density is below 0.2, and the NSFP statistics against ``lidar_flow``; then the mean
    of each statistic over the frames, as ``np.float64`` under the driver's keys and in its order.

    As there, a frame without a labelled point is skipped (and logged), the check comes before the ground removal, a
    frame without a label norm above 0.1 gives a NaN angle error, and no frame at all gives NaN.  A frame whose
    labelled points are all ground gives NaN for every statistic, what the reference's statistics give for an empty
    frame (the reference's ``query_flow`` itself fails on zero points).  Runs under ``no_grad``; one host sync, at the
    end, and the frame table's two when the source's timesteps are new."""
    rows = _lidar_flow_sums(lidar_set, model, remove_ground).cpu().tolist()     # the one host sync
    per_frame: Dict[str, List[np.float64]] = {k: [] for k in FLOW_EVAL_KEYS}
    for r in rows:
        if r[7] == 0:                                   # EMER_LIDAR_FLOW_VALID
            logger.info("no valid points, skipping...")
            continue
        counted = np.float64(r[6])
        with np.errstate(divide="ignore", invalid="ignore"):
            got = {"EPE3D": r[0] / counted, "acc3d_strict": r[1] / counted, "acc3d_relax": r[2] / counted,
                   "angle_error": np.float64(r[4]) / np.float64(r[5]), "outlier": r[3] / counted}
        for k in FLOW_EVAL_KEYS:
            per_frame[k].append(got[k])
    return {k: np.mean(v) for k, v in per_frame.items()}


def _lidar_flow_sums(lidar_set, model, remove_ground: bool) -> Tensor:
    """The fp64 [frames, EMER_LIDAR_FLOW_SUMS] rows of ``eval_lidar_flow``, on the device; no host sync once the frame table
    exists."""
    source = getattr(lidar_set, "datasource", None)
    indices = getattr(lidar_set, "split_indices", None)
    if source is None or indices is None:
        raise ValueError("lidar flow evaluation: the set needs `datasource` and `split_indices` (a SplitWrapper)")
    if getattr(model, "flow_xyz_encoder", None) is None:
        raise ValueError("lidar flow evaluation: the model has no flow branch")
    indices = list(indices)
    dev = source.origins.device
    sums = torch.zeros(len(indices), FLOW_SUMS, dtype=torch.float64, device=dev)
    _ops._need_cuda(sums)
    ws = _ops._workspace(_WS, dev, WORKSPACE_BYTES, "metrics")
    sampler = _lidar_sampler(source)
    p = _ops._ptr
    with torch.no_grad():
        for f, t in enumerate(indices):
            d = sampler.get_render_rays(t)
            if "lidar_flow" not in d:
                raise ValueError("lidar flow evaluation: the source has no flows, flow_classes and grounds")
            points = d["lidar_origins"] + d["lidar_ranges"] * d["lidar_viewdirs"]
            times, labels, classes = d["lidar_normed_timestamps"], d["lidar_flow"], d["lidar_flow_class"]
            ground = d["lidar_ground"] if remove_ground else None
            n = points.shape[0]
            for s in range(0, n, FLOW_CHUNK_POINTS):
                e = min(s + FLOW_CHUNK_POINTS, n)
                out = model.query_flow(positions=points[s:e], normed_timestamps=times[s:e])
                pred, ld = _ops._rows(out["forward_flow"], 3)      # in place in the [n, 6] flow output
                density = _ops._f32c(out["dynamic_density"].reshape(-1))
                lab = _ops._f32c(labels[s:e])
                cls = classes[s:e].to(torch.int64).contiguous()
                g = None
                if ground is not None:
                    g = ground[s:e]
                    g = (g if g.dtype == torch.bool else g != 0).contiguous().view(torch.uint8)
                if pred.shape[0] != e - s or density.numel() != e - s:
                    raise ValueError(f"lidar flow evaluation: the field returned {pred.shape[0]} flows and "
                                     f"{density.numel()} densities for {e - s} points")
                _ops._need_cuda(pred, density, lab, cls, g, sums)
                _lib.call("emer_lidar_flow_accumulate", p(pred), ld, p(density), p(lab), p(cls), p(g), e - s,
                          FLOW_DENSITY_THRESHOLD, p(sums[f]), p(ws), _ops._stream())
                out = pred = density = None             # free this chunk before the next query
    return sums

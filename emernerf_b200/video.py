"""The evaluation videos of the reference's ``render_pixels`` + ``save_videos`` pair (radiance_fields/video_utils.py:
50-627) in one call, with every frame composed on the device (csrc/video.cu) and handed to the writer as it finishes.

    results, vis_frame_dict = video.render_videos(
        cfg, model, proposal_estimator, proposal_networks, dataset, save_pth, num_timestamps,
        keys, num_cams, save_seperate_video=False, save_images=False, fps=10, verbose=True,
        compute_metrics=False, vis_indices=None, return_decomposition=True)

``results`` holds ``render_pixels``' six metrics (``psnr``, ``ssim``, ``feat_psnr``, ``masked_psnr``, ``masked_ssim``,
``masked_feat_psnr``; -1 where the reference gives -1), from ``metrics.image_metrics`` per image and one
``metrics.summarize``, and the same log lines.  ``vis_frame_dict`` is what ``save_videos`` returns: the uint8 frame
of timestep ``num_timestamps // 2`` as ``{"concatenated_frame": frame}``, or one per key in separate mode.  Files,
names, writer modes and fps are the reference's.

Per image, with no host sync of its own: ``render_rays`` on ``dataset[i]``; the products of the reference's ``render``
as its own torch expressions on the device (the green screen, the PCA colours, the first image's ``robust_pca`` fits
for the positional-embedding branch, ``flow_vis.scene_flow_to_rgb`` for the flows); then one ``emer_video_compose``
launch writes every row of this image into its camera's column of the frame: ``to8b`` of the RGB products, the turbo
depth colours, the two blends and the sky masks.  After a timestep's last camera, the frame is copied asynchronously
into one of two pinned host buffers, and one writer thread waits for that copy, appends the frame and releases the
buffer, so encoding overlaps the next timestep's rendering.  A writer exception is raised in the caller; the thread
is joined and the writers closed on every exit path.  The host holds two frames, whatever the number of timesteps.

The reference's behaviour that is kept on purpose:
  * rows follow ``keys``; a key is skipped when the reference skips it: absent or empty, or a depth key whose
    ``depths -> opacities`` key does not exist (``median_depths`` uses ``opacities``); ``sky_masks`` is ``1 -
    opacities``; ``gt_sky_masks`` the dataset's masks;
  * the dtype of ``to8b``'s product: a frame with a depth row is float64 (the turbo colours are), so every tile of it
    gets ``255 * x`` in float64; otherwise in float32.  In separate mode the rule holds per key;
  * the depth colours: ``visualize_depth(lo=4, hi=120, curve -log(x + 1e-6))``, clip, ``nan_to_num``, ``*= opacity``
    and matplotlib's ``min(int(v * 256), 255)`` on the turbo map, read from matplotlib at the first call
    (``load_turbo_lut``), as the reference reads it at import;
  * the separate mode's ``_{key}.mp4`` / ``_{key}.png`` names and its PNGs ``_{i*3 + j:03d}.png`` (a literal 3);
    ``mode="I"`` without fps for a single timestamp.

Deliberate differences:
  * render products never reach host memory: the call returns metrics and frames, not ``render_results`` lists;
  * ``len(indices) != num_timestamps * num_cams`` raises ``ValueError`` (the reference writes short frames), and so
    does ``num_cams == 5`` (``resize_five_views`` resizes with scipy's cubic-spline ``ndimage.zoom``);
  * a depth pixel may take the neighbouring turbo entry where ``v * 256`` lies within 1e-4 of an integer: numpy 1.x
    colours in float32, numpy 2 in float64, and this module in float64 from the float32 curve;
  * separate mode writes no file for an absent key (the reference opens, and never closes, a writer for it), and
    treats depth keys as concatenated mode does: ``median_depths`` is coloured with ``opacities`` and a depth key
    without opacities is skipped, where the reference's separate mode raises ``KeyError``.
"""
from __future__ import annotations

import ctypes
import logging
import os
import queue
import threading
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib, _ops, flow_vis, metrics, voxels

__all__ = ["render_videos", "load_turbo_lut", "plan_rows"]
logger = logging.getLogger()

RGB, DEPTH, BLEND, GRAY = 0, 1, 2, 3     # EMER_VIDEO_*
MAX_TILES = 32                           # EMER_VIDEO_MAX_TILES
MAX_PIXELS = 1 << 26                     # EMER_VIDEO_MAX_PIXELS
FLOW_MAX_RADIUS = 1.0                    # flow_visualizer, video_utils.py:35-43
PCA_M = 2.5
BLENDS = ("dynamic_rgb_on_static_dinos", "dynamic_dino_on_static_rgbs")
# the lists render() returns whether or not they are empty (video_utils.py:429-437)
ALWAYS = ("rgbs", "static_rgbs", "dynamic_rgbs", "depths", "opacities", "static_depths", "static_opacities",
          "dynamic_depths", "dynamic_opacities")
OPACITY = {"opacities": "opacity", "static_opacities": "static_opacity", "dynamic_opacities": "dynamic_opacity"}
_LUT: Dict[object, Tensor] = {}


def load_turbo_lut() -> np.ndarray:
    """matplotlib's turbo map as the reference reads it (``matplotlib.colormaps["turbo"]``, or ``cm.get_cmap`` on older
    versions), as the [256, 3] uint8 table ``to8b`` makes of it: trunc(255 * colour) in float64."""
    import matplotlib

    try:
        cmap = matplotlib.colormaps["turbo"]
    except (AttributeError, KeyError):
        from matplotlib import cm

        cmap = cm.get_cmap("turbo")
    rgba = np.asarray(cmap(np.arange(256)), np.float64)
    return (255 * np.clip(rgba[:, :3], 0, 1)).astype(np.uint8)


def _lut(dev: torch.device) -> Tensor:
    lut = _LUT.get(dev)
    if lut is None:
        table = np.ascontiguousarray(load_turbo_lut(), np.uint8)
        if table.shape != (256, 3):
            raise ValueError(f"video frames: a turbo table of shape {table.shape} (256 x 3)")
        lut = torch.from_numpy(table).to(dev, non_blocking=True)
        _LUT[dev] = lut
    return lut


def _host_frame(shape: Tuple[int, ...]) -> Tensor:
    """One of the two host frames: pinned, so the device-to-host copy is asynchronous."""
    return torch.empty(shape, dtype=torch.uint8, pin_memory=True)


def _record(dev: torch.device):
    """An event after the frame's copy on the device's current stream."""
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(dev))
    return ev


def _wait(ev) -> None:
    """The writer thread's wait for one frame's copy."""
    ev.synchronize()


def _get_writer(path: str, **kw):
    import imageio

    return imageio.get_writer(path, **kw)


def _imwrite(path: str, image: np.ndarray) -> None:
    import imageio

    imageio.imwrite(path, image)


# ------------------------------------------------------------------------------------------------------------- rows
def plan_rows(keys: Sequence[str], produced: Sequence[str], separate: bool = False
              ) -> List[Tuple[str, int, Optional[str]]]:
    """The frame's rows as (key, kind, opacity key) in ``keys`` order, for the non-empty lists ``produced`` of the
    reference's ``render``: ``save_concatenated_videos``' skipping rules (video_utils.py:525-553).  Separate mode
    skips ``sky_masks``, a key ``render`` never returns (video_utils.py:587-588)."""
    present = set(ALWAYS) | set(produced)
    rows = []
    for key in keys:
        if key == "sky_masks" and not separate:         # 1 - opacities; opacities are always rendered
            rows.append((key, GRAY, "opacities"))
            continue
        if key not in produced:
            continue
        if key == "gt_sky_masks":
            rows.append((key, GRAY, None))
        elif "depth" in key:
            okey = key.replace("depths", "opacities")
            if okey not in present:
                if "median" not in key:
                    continue
                okey = "opacities"
            rows.append((key, DEPTH, okey))
        elif key in BLENDS:
            rows.append((key, BLEND, None))
        else:
            rows.append((key, RGB, None))
    return rows


def produced_keys(results: Dict[str, Tensor], data: Dict[str, Tensor]) -> List[str]:
    """The lists the reference's ``render`` fills for an image with these render results and data
    (video_utils.py:161-418)."""
    out = ["rgbs", "depths", "opacities"]
    if "pixels" in data:
        out.append("gt_rgbs")
    for k in ("static_rgb", "shadow_reduced_static_rgb", "shadow_only_static_rgb", "forward_flow", "backward_flow"):
        if k in results:
            out.append(k + "s")
    if "dynamic_rgb" in results:
        out.append("dynamic_rgbs")
    if "static_depth" in results:
        out += ["static_depths", "static_opacities"]
    if "dynamic_depth" in results:
        out += ["dynamic_depths", "dynamic_opacities"]
    elif "median_depth" in results:
        out.append("median_depths")
    if "sky_masks" in data:
        out.append("gt_sky_masks")
    if "dino_feat" in results:
        out.append("dino_feats")
        if "features" in data:
            out.append("gt_dino_feats")
        if "dino_pe_free" in results:
            out += ["dino_feats_pe_free", "dino_pe"]
        if "static_dino" in results:
            out += ["static_dino_feats", "dynamic_rgb_on_static_dinos"]
        if "dynamic_dino" in results:
            out += ["dynamic_dino_feats", "dynamic_dino_on_static_rgbs"]
    return out


# --------------------------------------------------------------------------------------------------------- products
class _Products:
    """The reference's per-image products (video_utils.py:161-418) as its own torch expressions, computed on demand
    and kept for one image.  The positional-embedding branch's PCA is fitted on the first image that has it."""

    def __init__(self, model, green: Tensor):
        self.model, self.green = model, green
        self.pca = None

    def image(self, results: Dict[str, Tensor], data: Dict[str, Tensor]) -> None:
        self.r, self.d, self.cache = results, data, {}
        if "dino_feat" in results and "dino_pe_free" in results and self.pca is None:
            # video_utils.py:272-301, at the same point of the image loop, so the CUDA generator is consumed alike
            pe_free = results["dino_pe_free"]
            non_sky = pe_free * (~data["sky_masks"].bool().unsqueeze(-1)).to(pe_free)
            self.pca = (voxels.robust_pca(non_sky.reshape(-1, pe_free.shape[-1]), m=PCA_M),
                        voxels.robust_pca(results["dino_pe"].reshape(-1, results["dino_pe"].shape[-1]), m=PCA_M))

    def release(self) -> None:
        self.r = self.d = self.cache = None

    def _model_pca(self, x: Tensor, like: Tensor) -> Tensor:
        m = self.model
        return (x - m.feat_color_min.to(like)) / (m.feat_color_max.to(like) - m.feat_color_min.to(like))

    def _pred(self) -> Tensor:
        """pred_dino_feat after the model's PCA, before its clamp (video_utils.py:252-260)."""
        if "pred" not in self.cache:
            pred = self.r["dino_feat"]
            pred = pred @ self.model.feats_reduction_mat.to(pred)
            self.cache["pred"] = self._model_pca(pred, pred)
        return self.cache["pred"]

    def get(self, key: str) -> Tensor:
        if key not in self.cache:
            self.cache[key] = self._compute(key)
        return self.cache[key]

    def _compute(self, key: str) -> Tensor:
        r, d = self.r, self.d
        if key == "rgbs":
            return r["rgb"]
        if key == "gt_rgbs":
            return d["pixels"]
        if key in ("static_rgbs", "shadow_reduced_static_rgbs", "shadow_only_static_rgbs"):
            return r[key[:-1]]
        if key == "dynamic_rgbs":                                     # :168-174, the green screen
            return r["dynamic_rgb"] * r["dynamic_opacity"] + self.green * (1 - r["dynamic_opacity"])
        if key in ("forward_flows", "backward_flows"):                # :184-187
            return flow_vis.scene_flow_to_rgb(r[key[:-1]], flow_max_radius=FLOW_MAX_RADIUS, background="bright")
        if key in ("depths", "static_depths", "dynamic_depths", "median_depths"):
            return r[key[:-1]]
        if key in OPACITY:
            return r[OPACITY[key]]
        if key == "gt_sky_masks":
            return d["sky_masks"]
        if key == "dino_feats":                                       # :413
            return torch.clamp(self._pred(), 0, 1)
        if key == "gt_dino_feats":                                    # :263-271, :417
            pred = self._pred()
            gt = d["features"] @ self.model.feats_reduction_mat.to(pred)
            return torch.clamp(self._model_pca(gt, pred), 0, 1)
        pred = self._pred()
        if "dino_pe_free" in r:
            (mat, lo, hi), (pe_mat, pe_lo, pe_hi) = self.pca
            if key == "dino_feats_pe_free":                           # :302-312
                x = r["dino_pe_free"] @ mat
                x = (x - lo.to(pred)) / (hi.to(pred) - lo.to(pred))
                x = torch.clamp(x, 0, 1)
                x *= r["opacity"]
                return x
            if key == "dino_pe":                                      # :314-319
                x = r["dino_pe"] @ pe_mat
                x = (x - pe_lo.to(pred)) / (pe_hi - pe_lo).to(pred)
                return torch.clamp(x, 0, 1)
            if key == "static_dino_feats":                            # :321-332
                x = r["static_dino"] @ mat
                x = (x - lo.to(pred)) / (hi - lo).to(pred)
                return torch.clamp(x, 0, 1)
            if key == "dynamic_dino_feats":                           # :344-356
                x = r["dynamic_dino"] @ mat
                x = (x - lo.to(pred)) / (hi - lo).to(pred)
                x = torch.clamp(x, 0, 1)
                x *= r["dynamic_opacity"]
                return x
        else:
            if key == "static_dino_feats":                            # :368-379
                x = r["static_dino"] @ self.model.feats_reduction_mat.to(pred)
                return torch.clamp(self._model_pca(x, pred), 0, 1)
            if key == "dynamic_dino_feats":                           # :390-401
                x = r["dynamic_dino"] @ self.model.feats_reduction_mat
                return torch.clamp(self._model_pca(x, pred), 0, 1)
        raise ValueError(f"video frames: no product {key!r}")

    def inputs(self, key: str, kind: int, okey: Optional[str]) -> Tuple[Tensor, ...]:
        """The float32 inputs of one tile, as the kernel reads them."""
        if kind == DEPTH:
            return self.get(key), self.get(okey)
        if kind == GRAY:
            return (self.get(okey if key == "sky_masks" else key),)
        if key == "dynamic_rgb_on_static_dinos":                      # :334-342
            return self.r["dynamic_rgb"], self.r["dynamic_opacity"], self.get("static_dino_feats")
        if key == "dynamic_dino_on_static_rgbs":                      # :358-366
            return self.get("dynamic_dino_feats"), self.r["dynamic_opacity"], self.get("static_rgbs")
        return (self.get(key),)


# ---------------------------------------------------------------------------------------------------------- compose
def _checked(t: Tensor, h: int, w: int, c: int, what: str, dev) -> Tensor:
    """A tile input as the kernel reads it: a contiguous float32 CUDA tensor of [h, w, c] ([h, w] for c = 1)."""
    if not isinstance(t, Tensor) or not _ops.on_device(t):
        raise ValueError(f"video frames: {what} must be a CUDA tensor")
    if t.device != dev:
        raise ValueError(f"video frames: {what} is on {t.device}, the frame on {dev}")
    if t.dtype != torch.float32:
        raise ValueError(f"video frames: {what} is {t.dtype}, not float32")
    if not t.is_contiguous():
        raise ValueError(f"video frames: {what} is not contiguous")
    shape = tuple(t.shape)
    if shape != (h, w, c) and not (c == 1 and shape == (h, w)):
        raise ValueError(f"video frames: {what} of shape {shape} for a {h} x {w} x {c} tile")
    return t


def compose(frame: Tensor, tiles: Sequence[Tuple[int, Sequence[Tensor], int, bool, bool]], h: int, w: int,
            col: int, lut: Optional[Tensor]) -> None:
    """One ``emer_video_compose`` launch: ``tiles`` = [(kind, inputs, row, invert, f64)] of one [h, w] image into
    column ``col`` of ``frame`` (uint8 [rows * h, cams * w, 3] on the device).  Every input, the frame and the tile
    count are checked here; a mismatch is a ``ValueError`` and nothing is launched."""
    if not isinstance(frame, Tensor) or not _ops.on_device(frame) or frame.dtype != torch.uint8 \
            or frame.dim() != 3 or frame.shape[2] != 3 or not frame.is_contiguous():
        raise ValueError("video frames: the frame must be a contiguous uint8 CUDA tensor [rows * H, cams * W, 3]")
    if h < 1 or w < 1 or h * w > MAX_PIXELS:
        raise ValueError(f"video frames: a {h} x {w} tile (1 to {MAX_PIXELS} pixels)")
    if frame.shape[0] % h != 0:
        raise ValueError(f"video frames: a frame of {frame.shape[0]} rows for tiles of {h}")
    rows = frame.shape[0] // h
    if not 0 <= col or (col + 1) * w > frame.shape[1]:
        raise ValueError(f"video frames: column {col} of {w} pixels in a frame {frame.shape[1]} wide")
    if not 1 <= len(tiles) <= MAX_TILES:
        raise ValueError(f"video frames: {len(tiles)} tiles (1..{MAX_TILES})")
    dev = frame.device
    arr = (_lib.EmerVideoTile * len(tiles))()
    keep = []
    for i, (kind, inputs, row, invert, f64) in enumerate(tiles):
        if kind not in (RGB, DEPTH, BLEND, GRAY):
            raise ValueError(f"video frames: tile {i} of kind {kind}")
        if not 0 <= row < rows:
            raise ValueError(f"video frames: tile {i} at row {row} of a frame of {rows} rows")
        chans = {RGB: (3,), DEPTH: (1, 1), BLEND: (3, 1, 3), GRAY: (1,)}[kind]
        if len(inputs) != len(chans):
            raise ValueError(f"video frames: tile {i} has {len(inputs)} inputs, its kind takes {len(chans)}")
        ins = [_checked(t, h, w, c, f"input {k} of tile {i}", dev) for k, (t, c) in enumerate(zip(inputs, chans))]
        keep += ins
        arr[i].inputs = (ctypes.c_void_p * 3)(*([t.data_ptr() for t in ins] + [None] * (3 - len(ins))))
        arr[i].kind, arr[i].row, arr[i].invert, arr[i].f64 = kind, row, int(bool(invert)), int(bool(f64))
    if any(t[0] == DEPTH for t in tiles):
        if lut is None or lut.dtype != torch.uint8 or tuple(lut.shape) != (256, 3) or not lut.is_contiguous() \
                or lut.device != dev:
            raise ValueError("video frames: depth tiles need the turbo table as a contiguous uint8 [256, 3] tensor "
                             "on the frame's device")
    _ops._need_cuda(frame, lut, *keep)
    p = _ops._ptr
    _lib.call("emer_video_compose", p(frame), frame.shape[1], arr, len(tiles), h, w, col, p(lut), _ops._stream())


# ----------------------------------------------------------------------------------------------------------- writer
class _Stream:
    """The frame, the two pinned host frames and the writer thread of one call."""

    def __init__(self, rows, h: int, w: int, num_cams: int, num_timestamps: int, separate: bool, save_pth: str,
                 fps: int, save_images: bool, dev: torch.device):
        self.rows, self.h, self.w, self.num_cams = rows, h, w, num_cams
        self.separate, self.save_images, self.dev = separate, save_images, dev
        self.return_id = num_timestamps // 2
        any_depth = any(kind == DEPTH for _, kind, _ in rows)
        self.f64 = [kind == DEPTH if separate else any_depth for _, kind, _ in rows]
        shape = (len(rows) * h, num_cams * w, 3)
        self.frame = torch.empty(shape, dtype=torch.uint8, device=dev)
        self.host = [_host_frame(shape) for _ in range(2)]
        self.free = [threading.Semaphore(1) for _ in range(2)]
        self.queue: "queue.Queue" = queue.Queue(maxsize=1)
        self.returned: Dict[str, np.ndarray] = {}
        self.error: Optional[BaseException] = None
        kw = {"mode": "I"} if num_timestamps == 1 else {"mode": "I", "fps": fps}
        if separate:
            self.paths = [save_pth.replace(".mp4", f"_{key}.mp4").replace(".png", f"_{key}.png")
                          for key, _, _ in rows]
        else:
            self.paths = [save_pth]
        self.writers = []
        try:
            for path in self.paths:
                self.writers.append(_get_writer(path, **kw))
        except BaseException:
            self._close_writers()
            raise
        self.thread = threading.Thread(target=self._run, name="emernerf-video-writer")
        self.thread.start()

    def compose(self, tiles_of, col: int, lut) -> None:
        tiles = [(kind, tiles_of(key, kind, okey), r, key == "sky_masks", self.f64[r])
                 for r, (key, kind, okey) in enumerate(self.rows)]
        compose(self.frame, tiles, self.h, self.w, col, lut)

    def flush(self, t: int) -> None:
        """Timestep t is composed: copy it into a free host frame and hand that to the writer."""
        b = t % 2
        while not self.free[b].acquire(timeout=0.1):
            if not self.thread.is_alive():
                raise RuntimeError("video frames: the writer thread stopped")
        self.raise_error()
        self.host[b].copy_(self.frame, non_blocking=True)
        self.queue.put((t, b, _record(self.dev)))

    def _run(self) -> None:
        while True:
            item = self.queue.get()
            if item is None:
                return
            t, b, ev = item
            try:
                if self.error is None:
                    _wait(ev)
                    self._write(t, self.host[b].numpy())
            except BaseException as e:                 # raised in the caller; keep draining the queue
                self.error = e
            finally:
                self.free[b].release()

    def _write(self, t: int, frame: np.ndarray) -> None:
        if not self.separate:
            out = frame.copy()
            self.writers[0].append_data(out)
            if t == self.return_id:
                self.returned["concatenated_frame"] = out
            return
        h, w = self.h, self.w
        for r, (key, _, _) in enumerate(self.rows):
            out = frame[r * h:(r + 1) * h].copy()
            path = self.paths[r]
            if self.save_images:                        # video_utils.py:609-616
                if t == 0:
                    os.makedirs(path.replace(".mp4", ""), exist_ok=True)
                for j in range(self.num_cams):
                    _imwrite(path.replace(".mp4", f"_{t*3 + j:03d}.png"), out[:, j * w:(j + 1) * w].copy())
            self.writers[r].append_data(out)
            if t == self.return_id:
                self.returned[key] = out

    def raise_error(self) -> None:
        if self.error is not None:
            raise self.error

    def _close_writers(self) -> None:
        for wr in self.writers:
            try:
                wr.close()
            except BaseException as e:
                if self.error is None:
                    self.error = e
        self.writers = []

    def close(self) -> None:
        """Join the writer thread after the frames it holds, and close the writers.  Never raises."""
        if self.thread.is_alive():
            self.queue.put(None)
        self.thread.join()
        self._close_writers()


# ------------------------------------------------------------------------------------------------------------- call
def _device_dict(data) -> Dict[str, object]:
    out = dict(data)
    for k, v in out.items():
        if isinstance(v, Tensor) and not _ops.on_device(v):
            out[k] = v.cuda(non_blocking=True)
    return out


def _tile_input(t: Tensor) -> Tensor:
    return _ops._f32c(t)


def render_videos(cfg, model, proposal_estimator, proposal_networks, dataset, save_pth: str, num_timestamps: int,
                  keys: Sequence[str] = ("gt_rgbs", "rgbs", "depths"), num_cams: int = 3,
                  save_seperate_video: bool = False, save_images: bool = False, fps: int = 10, verbose: bool = True,
                  compute_metrics: bool = False, vis_indices: Optional[Sequence[int]] = None,
                  return_decomposition: bool = True) -> Tuple[Dict[str, float], Dict[str, np.ndarray]]:
    """``render_pixels(cfg, model, proposal_estimator, dataset, proposal_networks, compute_metrics, vis_indices,
    return_decomposition)`` followed by ``save_videos(render_results, save_pth, num_timestamps, keys, num_cams,
    save_seperate_video, save_images, fps, verbose)``: returns (the six metrics, the returned frames)."""
    from .radiance_fields.render_utils import render_rays

    indices = list(vis_indices) if vis_indices is not None else list(range(len(dataset)))
    if num_cams == 5:
        raise ValueError("video frames: five cameras need resize_five_views (scipy's ndimage.zoom), which is not "
                         "restated")
    if num_cams < 1 or num_timestamps < 1 or len(indices) != num_timestamps * num_cams:
        raise ValueError(f"video frames: {len(indices)} images for {num_timestamps} timestamps of {num_cams} "
                         "cameras")
    keys = list(keys)
    voxels._eval(model, proposal_estimator, proposal_networks)
    products = _Products(model, None)
    per_image: List[Dict[str, Tensor]] = []
    stream: Optional[_Stream] = None
    lut = None
    with torch.no_grad():
        try:
            for p, i in enumerate(indices):
                data = _device_dict(dataset[i])
                results = render_rays(radiance_field=model, proposal_estimator=proposal_estimator,
                                      proposal_networks=proposal_networks, data_dict=data, cfg=cfg,
                                      return_decomposition=return_decomposition)
                rgb = results["rgb"]
                if stream is None:
                    if not _ops.on_device(rgb):
                        raise ValueError("video frames: the model must render on a CUDA device")
                    rows = plan_rows(keys, produced_keys(results, data), save_seperate_video)
                    if not rows:
                        raise ValueError(f"video frames: none of the keys {keys} has a product to show")
                    if len(rows) > MAX_TILES:
                        raise ValueError(f"video frames: {len(rows)} rows (at most {MAX_TILES})")
                    if rgb.dim() != 3:
                        raise ValueError(f"video frames: rendered images of shape {tuple(rgb.shape)}, not [H, W, 3]")
                    h, w = int(rgb.shape[0]), int(rgb.shape[1])
                    # the green screen, built as video_utils.py:170-171 builds it, once
                    products.green = (torch.tensor([0.0, 177, 64]) / 255.0).to(rgb.device, non_blocking=True)
                    if any(kind == DEPTH for _, kind, _ in rows):
                        lut = _lut(rgb.device)
                    stream = _Stream(rows, h, w, num_cams, num_timestamps, save_seperate_video, save_pth, fps,
                                     save_images, rgb.device)
                products.image(results, data)
                if compute_metrics:                   # video_utils.py:205-247
                    have_feat = "dino_feat" in results and "features" in data
                    per_image.append(metrics.image_metrics(
                        rgb, data["pixels"], data.get("dynamic_masks"),
                        results["dino_feat"] if have_feat else None, data["features"] if have_feat else None))

                def tile_inputs(key, kind, okey):
                    try:
                        return tuple(_tile_input(t) for t in products.inputs(key, kind, okey))
                    except KeyError as e:
                        raise ValueError(f"video frames: image {i} has no {e} for the row {key!r}") from None

                stream.compose(tile_inputs, p % num_cams, lut)
                products.release()
                results = data = rgb = None             # this image's products are freed here
                if p % num_cams == num_cams - 1:
                    stream.flush(p // num_cams)
        finally:
            if stream is not None:
                stream.close()
    stream.raise_error()
    out = metrics.summarize(per_image) if compute_metrics else {k: -1 for k in metrics.SUMMARY_KEYS}
    if compute_metrics:                               # render_pixels, video_utils.py:91-99
        logger.info(f"Eval over {len(dataset) if vis_indices is None else len(vis_indices)} images:")
        logger.info(f"\tPSNR: {out['psnr']:.4f}")
        logger.info(f"\tSSIM: {out['ssim']:.4f}")
        logger.info(f"\tFeature PSNR: {out['feat_psnr']:.4f}")
        logger.info(f"\tMasked PSNR: {out['masked_psnr']:.4f}")
        logger.info(f"\tMasked SSIM: {out['masked_ssim']:.4f}")
        logger.info(f"\tMasked Feature PSNR: {out['masked_feat_psnr']:.4f}")
    if verbose:
        for path in stream.paths:
            logger.info(f"saved video to {path}")
    results_dict = {k: out[k] for k in ("psnr", "ssim", "feat_psnr", "masked_psnr", "masked_ssim",
                                        "masked_feat_psnr")}
    return results_dict, dict(stream.returned)

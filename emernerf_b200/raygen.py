"""Ray generation on the device (SURVEY.md section 8 f3): the producer side of ``render_rays``' ``data_dict``.

``get_rays`` keeps the reference's signature and outputs (datasets/base/pixel_source.py:39-76); ``train_rays`` is the
part of ``ScenePixelSource.get_train_rays`` (:666-731) that turns sampled (image, y, x) indices into the ray entries of
the batch -- origins, unit view directions, direction norms, pixel coordinates (y/H, x/W), normalised timestamps and
the image index -- in ONE launch (``emer_gen_rays``, csrc/raygen.cu) straight from the per-image camera tables, without
the gathered [R, 4, 4] / [R, 3, 3] copies.  A training batch then needs 3 integers per ray from the host instead of
15 floats.

``PixelRaySampler`` and ``LidarRaySampler`` replace the sources' ``get_train_rays`` whole: the reference's random
draws, made on the device's generator in the reference's order, and the batch assembled from them without a host sync
(``emer_topk_ratio`` and ``emer_pixel_batch``, csrc/raybatch.cu; INTEGRATION.md section 11).  ``PixelRaySampler`` also
replaces ``get_render_rays`` and ``update_pixel_error_maps``, and with ``refresh_pixel_error_maps`` the whole error-map
refresh of the training loop (``emer_image_rays``, ``emer_error_map`` and ``emer_error_map_normalize``,
csrc/errormap.cu; INTEGRATION.md section 12).  ``LidarRaySampler`` also replaces the lidar sources' ``get_render_rays``
with a frame table (INTEGRATION.md section 10).

``CameraTrajectory`` renders the scene from cameras moving between the source's poses: a dataset for the reference's
``render_pixels`` whose items come from one ``emer_trajectory_rays`` launch each (INTEGRATION.md section 14).
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib, _ops


def _launch(img_idx, x, y, c2w, intrinsic, per_ray, timestamps, height, width, want_coords):
    _ops._need_cuda(x, y, c2w, intrinsic)
    n = x.shape[0]
    f32 = dict(dtype=torch.float32, device=x.device)
    x, y = _ops._f32c(x), _ops._f32c(y)
    c2w, intrinsic = _ops._f32c(c2w).reshape(-1, 16), _ops._f32c(intrinsic).reshape(-1, 9)
    origins, viewdirs, norms = torch.empty((n, 3), **f32), torch.empty((n, 3), **f32), torch.empty((n, 1), **f32)
    coords = torch.empty((n, 2), **f32) if want_coords else None
    ts = None if timestamps is None else _ops._f32c(timestamps)
    times = torch.empty(n, **f32) if ts is not None else None
    idx = None if img_idx is None else img_idx.to(torch.int64).contiguous()
    p = _ops._ptr
    _lib.call("emer_gen_rays", p(idx), p(x), p(y), p(c2w), p(intrinsic), int(per_ray), p(ts), int(height), int(width),
              p(origins), p(viewdirs), p(norms), p(coords), p(times), n, _ops._stream())
    return origins, viewdirs, norms, coords, times


@torch.no_grad()
def get_rays(x: Tensor, y: Tensor, c2w: Tensor, intrinsic: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """(origins [R,3], viewdirs [R,3], direction_norm [R,1]) for pixel centres (x, y); ``c2w`` [R or 1, 4, 4] (or
    [4,4]), ``intrinsic`` [R or 1, 3, 3] (or [3,3]) -- pixel_source.py:39-76."""
    c2w = c2w if c2w.dim() == 3 else c2w[None]
    intrinsic = intrinsic if intrinsic.dim() == 3 else intrinsic[None]
    n = x.shape[0]
    if c2w.shape[0] != intrinsic.shape[0]:
        c2w, intrinsic = c2w.expand(n, 4, 4), intrinsic.expand(n, 3, 3)
    if c2w.shape[0] not in (1, n):
        raise ValueError(f"get_rays: {c2w.shape[0]} camera matrices for {n} rays")
    o, d, nrm, _, _ = _launch(None, x, y, c2w, intrinsic, c2w.shape[0] == n and n > 1, None, 0, 0, False)
    return o, d, nrm


@torch.no_grad()
def train_rays(img_idx: Tensor, y: Tensor, x: Tensor, cam_to_worlds: Tensor, intrinsics: Tensor, height: int, width: int,
               normalized_timestamps: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """The ray entries of ``get_train_rays``' batch from sampled indices and the per-IMAGE camera tables
    (``cam_to_worlds`` [M,4,4], ``intrinsics`` [M,3,3], ``normalized_timestamps`` [M])."""
    o, d, nrm, coords, times = _launch(img_idx, x.float(), y.float(), cam_to_worlds, intrinsics, False,
                                       normalized_timestamps, height, width, True)
    out = {"origins": o, "viewdirs": d, "direction_norms": nrm, "pixel_coords": coords,
           "img_idx": img_idx.to(torch.int64)}
    if times is not None:
        out["normed_timestamps"] = times
    return out


# ----------------------------------------------------------------------------- training batches
RAYBATCH_WORKSPACE_BYTES = 141376    # EMER_RAYBATCH_WORKSPACE_BYTES
TOPK_MAX_K = 16384                   # EMER_TOPK_MAX_K
PIXEL_BATCH_MAX_FEATURES = 256       # EMER_PIXEL_BATCH_MAX_FEATURES
_MAX_CATEGORIES = 1 << 24            # torch.multinomial's limit on the number of weights
_WS: Dict[object, Tensor] = {}


def _workspace(dev: torch.device) -> Tensor:
    return _ops._workspace(_WS, dev, RAYBATCH_WORKSPACE_BYTES, "PixelRaySampler")


ERRORMAP_WORKSPACE_BYTES = 16        # EMER_ERRORMAP_WORKSPACE_BYTES
_MAP_WS: Dict[object, Tensor] = {}
# get_render_rays' entries with a trailing dimension ([h, w, k]); the others are [h, w]
_TRAILING = ("origins", "viewdirs", "direction_norm", "pixel_coords", "pixels", "features")


def _map_workspace(dev: torch.device) -> Tensor:
    return _ops._workspace(_MAP_WS, dev, ERRORMAP_WORKSPACE_BYTES, "PixelRaySampler error map")


def _dense(t: Optional[Tensor], name: str, dtype=torch.float32) -> Optional[Tensor]:
    if t is None:
        return None
    if t.dtype != dtype or not t.is_contiguous():
        raise TypeError(f"PixelRaySampler: source.{name} must be a contiguous {dtype} tensor, got {t.dtype}"
                        f"{'' if t.is_contiguous() else ' (not contiguous)'}")
    return t


def _candidate_key(candidate_indices):
    """What identifies a candidate set without device work: a list's contents, a tensor's identity and version."""
    if candidate_indices is None:
        return ("all",)
    if isinstance(candidate_indices, Tensor):
        return ("tensor", id(candidate_indices), candidate_indices._version)
    return ("list", tuple(int(i) for i in candidate_indices))


class _Candidates:
    """The device copy of the candidate image indices, rebuilt only when ``_candidate_key`` changes.  None means
    every image, as in the reference."""

    def __init__(self):
        self.key, self.tensor, self._held = None, None, None

    def get(self, candidate_indices, n_images: int, dev: torch.device) -> Tuple[Tensor, tuple]:
        key = _candidate_key(candidate_indices) + (n_images,)
        if key == self.key:
            return self.tensor, key
        if key[0] == "all":
            t = torch.arange(n_images, device=dev)
        elif key[0] == "list":
            if key[1] and not (min(key[1]) >= 0 and max(key[1]) < n_images):
                raise IndexError(f"candidate indices out of range for {n_images} images")
            t = torch.tensor(key[1], dtype=torch.int64).to(dev)
        else:
            t = candidate_indices
            if t.device != dev or t.dim() != 1:
                raise ValueError(f"candidate indices must be a 1-D tensor on {dev}")
            t = t.to(torch.int64)
            if t.numel() and not bool(((t >= 0) & (t < n_images)).all()):     # one sync per candidate tensor
                raise IndexError(f"candidate indices out of range for {n_images} images")
        # a tensor's key holds its id: keep the tensor alive, so the id cannot be reused by another one
        self.key, self.tensor, self._held = key, t, candidate_indices
        return t, key


class PixelRaySampler:
    """``ScenePixelSource.get_train_rays`` (datasets/base/pixel_source.py:666-731) on the device, bound to a source:
    ``source.get_train_rays = PixelRaySampler(source).get_train_rays``.

    It makes the reference's random draws on the same generator, in the same order and with the same shapes:
    ``randint`` for the uniform rays' image, column and row, then, when the error map is live
    (``buffer_ratio > 0 and pixel_error_buffered``), the ``Exp(1)`` draw of ``torch.multinomial`` over the candidate
    images' weights and ``randint`` for the importance rays' row and column offsets.  So the batch is the reference's:
    the same pixels, the same gathered values, the same keys, uniform rays first.  The one permitted difference is the
    order of equal top-k keys, which the kernel breaks by ascending index.  Selection and batch assembly are
    ``emer_topk_ratio`` and ``emer_pixel_batch`` (csrc/raybatch.cu).

    No host sync in steady state: the error map is validated as torch.multinomial validates it (finite, non-negative,
    positive sum over the candidate images) once per map state -- a different tensor, a moved ``_version`` or another
    candidate set -- with one sync, and a candidate list is copied to the device once per distinct list.  Every table
    of the source must live on one CUDA device (the reference's ``to()`` puts them there).
    """

    def __init__(self, source):
        self.source = source
        self._cand = _Candidates()
        self._valid = None                   # (error maps, their _version, candidate key) last validated
        self._resized = None                 # (images, their _version, d, the images resized by d)

    def _validate(self, maps: Tensor, cand: Tensor, cand_key) -> None:
        v = self._valid
        if v is not None and v[0] is maps and v[1] == maps._version and v[2] == cand_key:
            return
        if maps.is_cuda and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("PixelRaySampler: the error map changed since the last call; run one call outside "
                               "graph capture first, so it is validated before capture")
        w = maps[cand]
        finite_nonneg, zero_sum = torch.stack([(w.max() < float("inf")) & (w.min() >= 0), w.sum() == 0]).tolist()
        if not finite_nonneg:
            raise RuntimeError("probability tensor contains either `inf`, `nan` or element < 0")
        if zero_sum:
            raise RuntimeError("invalid multinomial distribution (sum of probabilities <= 0)")
        self._valid = (maps, maps._version, cand_key)

    def get_train_rays(self, num_rays: int, candidate_indices=None) -> Dict[str, Tensor]:
        s = self.source
        H, W = int(s.HEIGHT), int(s.WIDTH)
        c2w, intr = _dense(s.cam_to_worlds, "cam_to_worlds"), _dense(s.intrinsics, "intrinsics")
        images = _dense(s.images, "images")
        sky, dyn = _dense(s.sky_masks, "sky_masks"), _dense(s.dynamic_masks, "dynamic_masks")
        feats = _dense(s.features, "features")
        times = _dense(s.normalized_timestamps, "normalized_timestamps")
        cam_ids = _dense(s.cam_ids, "cam_ids", torch.int64)
        if cam_ids is None:
            raise ValueError("PixelRaySampler: the batch's cam_idx needs source.cam_ids")
        n_images = len(images) if images is not None else len(c2w)
        dev = c2w.device
        _ops._need_cuda(c2w, intr, images, sky, dyn, feats, times, cam_ids)
        cand, cand_key = self._cand.get(candidate_indices, n_images, dev)

        importance = s.buffer_ratio > 0 and s.pixel_error_buffered
        n_i = int(num_rays * s.buffer_ratio) if importance else 0
        n_u = num_rays - n_i
        # the reference's draws, in its order (sample_uniform_rays, then sample_important_rays)
        u_pick = torch.randint(0, len(cand), size=(n_u,), device=dev)
        u_x = torch.randint(0, W, size=(n_u,), device=dev)
        u_y = torch.randint(0, H, size=(n_u,), device=dev)
        sel = i_dy = i_dx = maps = None
        map_h = map_w = ds = 0
        if importance:
            maps = _dense(s.pixel_error_maps, "pixel_error_maps")
            _ops._need_cuda(maps)
            _, map_h, map_w = maps.shape
            ds = int(s.buffer_downscale)
            m = len(cand) * map_h * map_w
            # torch.multinomial's argument checks, in its order and with its messages
            if n_i <= 0:
                raise RuntimeError("cannot sample n_sample <= 0 samples")
            if n_i > m:
                raise RuntimeError("cannot sample n_sample > prob_dist.size(-1) samples without replacement")
            if m > _MAX_CATEGORIES:
                raise RuntimeError("number of categories cannot exceed 2^24")
            if n_i > TOPK_MAX_K:
                raise ValueError(f"PixelRaySampler: {n_i} importance rays; the selection kernel takes at most "
                                 f"{TOPK_MAX_K}")
            self._validate(maps, cand, cand_key)
            q = torch.empty(m, dtype=torch.float32, device=dev).exponential_(1)
            sel = torch.empty(n_i, dtype=torch.int64, device=dev)
            p = _ops._ptr
            _lib.call("emer_topk_ratio", p(maps), map_h * map_w, p(cand), len(cand), p(q), n_i, p(sel),
                      p(_workspace(dev)), _ops._stream())
            i_dy = torch.randint(0, ds, (n_i,), device=dev)
            i_dx = torch.randint(0, ds, (n_i,), device=dev)
        return self._assemble(n_u, n_i, cand, u_pick, u_x, u_y, sel, i_dy, i_dx, map_h, map_w, ds, H, W, images, sky,
                              dyn, feats, times, cam_ids, c2w, intr)

    def _assemble(self, n_u, n_i, cand, u_pick, u_x, u_y, sel, i_dy, i_dx, map_h, map_w, ds, H, W, images, sky, dyn,
                  feats, times, cam_ids, c2w, intr) -> Dict[str, Tensor]:
        n, dev = n_u + n_i, c2w.device
        f32 = dict(dtype=torch.float32, device=dev)
        out = {"origins": torch.empty((n, 3), **f32), "viewdirs": torch.empty((n, 3), **f32),
               "direction_norms": torch.empty((n, 1), **f32), "pixel_coords": torch.empty((n, 2), **f32)}
        if times is not None:
            out["normed_timestamps"] = torch.empty(n, **f32)
        out["img_idx"] = torch.empty(n, dtype=torch.int64, device=dev)
        out["cam_idx"] = torch.empty(n, dtype=torch.int64, device=dev)
        if images is not None:
            out["pixels"] = torch.empty((n, 3), **f32)
        if sky is not None:
            out["sky_masks"] = torch.empty(n, **f32)
        if dyn is not None:
            out["dynamic_masks"] = torch.empty(n, **f32)
        fh = fw = fc = 0
        fsy = fsx = 0.0
        if feats is not None:
            _, fh, fw, fc = feats.shape
            if fc > PIXEL_BATCH_MAX_FEATURES:
                raise ValueError(f"PixelRaySampler: {fc} feature channels; at most {PIXEL_BATCH_MAX_FEATURES}")
            scale = self.source.featmap_downscale_factor
            fsy, fsx = (scale, scale) if isinstance(scale, (int, float)) else scale
            out["features"] = torch.empty((n, fc), **f32)
        p = _ops._ptr
        src = dict(cand=cand, u_pick=u_pick, u_x=u_x, u_y=u_y, i_sel=sel, i_dy=i_dy, i_dx=i_dx, images=images,
                   sky_masks=sky, dynamic_masks=dyn, features=feats, timestamps=times, cam_ids=cam_ids, c2w=c2w,
                   intrinsics=intr)
        args_in = _lib.EmerPixelBatchIn(
            *(p(src[k]) for k in _lib.PIXEL_BATCH_IN_PTRS), n_u, n_i, H, W, map_h, map_w, ds, fh, fw, fc,
            float(fsy), float(fsx))
        names = dict(pixels="pixels", sky_masks="sky_masks", dynamic_masks="dynamic_masks", features="features",
                     timestamps="normed_timestamps", origins="origins", viewdirs="viewdirs", norms="direction_norms",
                     pixel_coords="pixel_coords", img_idx="img_idx", cam_idx="cam_idx")
        args_out = _lib.EmerPixelBatchOut(*(p(out.get(names[k])) for k in _lib.PIXEL_BATCH_OUT_PTRS))
        _lib.call("emer_pixel_batch", ctypes.byref(args_in), ctypes.byref(args_out), _ops._stream())
        return out

    # ------------------------------------------------------------------------- render rays and the error map
    def _images_at(self, images: Tensor, d: float) -> Tensor:
        """Every image resized by d, [N, h, w, 3], as get_render_rays resizes one: torch's bicubic antialiased
        ``interpolate`` with ``scale_factor=d``, run once over all images (each image is its own batch entry) and kept
        while the images tensor and its ``_version`` stay the same."""
        if d == 1.0:
            return images
        r = self._resized
        if r is not None and r[0] is images and r[1] == images._version and r[2] == d:
            return r[3]
        out = torch.nn.functional.interpolate(images.permute(0, 3, 1, 2), scale_factor=d, mode="bicubic",
                                              antialias=True).permute(0, 2, 3, 1).contiguous()
        self._resized = (images, images._version, d, out)
        return out

    def _image_rays(self, first: int, count: int, d: float) -> Tuple[Dict[str, Tensor], int, int]:
        """get_render_rays' entries for the images [first, first + count) at downscale d, flat ([count * h * w, ...]),
        in the reference's key order; and (h, w)."""
        s = self.source
        H, W = int(s.HEIGHT), int(s.WIDTH)
        c2w, intr = _dense(s.cam_to_worlds, "cam_to_worlds"), _dense(s.intrinsics, "intrinsics")
        images = _dense(s.images, "images")
        sky, dyn = _dense(s.sky_masks, "sky_masks"), _dense(s.dynamic_masks, "dynamic_masks")
        feats = _dense(s.features, "features")
        times = _dense(s.normalized_timestamps, "normalized_timestamps")
        cam_ids = _dense(s.cam_ids, "cam_ids", torch.int64)
        if images is None or cam_ids is None:
            raise ValueError("PixelRaySampler: render rays need source.images and source.cam_ids")
        _ops._need_cuda(c2w, intr, images, sky, dyn, feats, times, cam_ids)
        if first < 0 or first + count > len(images):
            raise IndexError(f"images [{first}, {first + count}) out of range for {len(images)} images")
        resized = self._images_at(images, d)
        h, w = resized.shape[1:3]
        n, dev = count * h * w, c2w.device
        f32 = dict(dtype=torch.float32, device=dev)
        out = {"origins": torch.empty((n, 3), **f32), "viewdirs": torch.empty((n, 3), **f32),
               "direction_norm": torch.empty((n, 1), **f32), "pixel_coords": torch.empty((n, 2), **f32)}
        if times is not None:
            out["normed_timestamps"] = torch.empty(n, **f32)
        out["img_idx"] = torch.empty(n, dtype=torch.int64, device=dev)
        out["cam_idx"] = torch.empty(n, dtype=torch.int64, device=dev)
        out["pixels"] = resized[first:first + count].reshape(n, 3)
        if sky is not None:
            out["sky_masks"] = torch.empty(n, **f32)
        if dyn is not None:
            out["dynamic_masks"] = torch.empty(n, **f32)
        fh = fw = fc = 0
        fsy = fsx = 0.0
        if feats is not None:
            _, fh, fw, fc = feats.shape
            if fc > PIXEL_BATCH_MAX_FEATURES:
                raise ValueError(f"PixelRaySampler: {fc} feature channels; at most {PIXEL_BATCH_MAX_FEATURES}")
            # get_features(downscale=(featmap_downscale_factor[0] / d, featmap_downscale_factor[1] / d))
            fsy, fsx = (v / d for v in self.source.featmap_downscale_factor)
            out["features"] = torch.empty((n, fc), **f32)
        p = _ops._ptr
        src = dict(sky_masks=sky, dynamic_masks=dyn, features=feats, timestamps=times, cam_ids=cam_ids, c2w=c2w,
                   intrinsics=intr)
        # interpolate(scale_factor=d, mode="nearest") reads source row floor(y * (float)(1 / d))
        args_in = _lib.EmerImageRaysIn(*(p(src[k]) for k in _lib.IMAGE_RAYS_IN_PTRS), first, count, H, W, h, w,
                                       float(d), 1.0 / d, 1.0 / d, fh, fw, fc, float(fsy), float(fsx))
        names = dict(origins="origins", viewdirs="viewdirs", norms="direction_norm", pixel_coords="pixel_coords",
                     timestamps="normed_timestamps", img_idx="img_idx", cam_idx="cam_idx", sky_masks="sky_masks",
                     dynamic_masks="dynamic_masks", features="features")
        args_out = _lib.EmerImageRaysOut(*(p(out.get(names[k])) for k in _lib.IMAGE_RAYS_OUT_PTRS))
        _lib.call("emer_image_rays", ctypes.byref(args_in), ctypes.byref(args_out), _ops._stream())
        return out, h, w

    @torch.no_grad()
    def get_render_rays(self, img_idx: int) -> Dict[str, Tensor]:
        """``ScenePixelSource.get_render_rays`` (pixel_source.py:733-846) at ``source.downscale_factor``: the
        reference's keys, in its order, with its ``[h, w, ...]`` shapes and dtypes, every entry on the device.  The
        image is resized by torch's own bicubic ``interpolate``; the rest is one ``emer_image_rays`` launch."""
        return self._render_rays_at(int(img_idx), float(self.source.downscale_factor))

    def _render_rays_at(self, img_idx: int, d: float) -> Dict[str, Tensor]:
        out, h, w = self._image_rays(img_idx, 1, d)
        return {k: v.reshape(h, w, *v.shape[1:]) if k in _TRAILING else v.reshape(h, w) for k, v in out.items()}

    def _fold_error(self, gt: Tensor, rgb: Tensor, opacity: Optional[Tensor], rows: Tensor) -> None:
        n = rows.numel()
        if gt.numel() != 3 * n or rgb.numel() != 3 * n or (opacity is not None and opacity.numel() != n):
            raise ValueError(f"PixelRaySampler: {n} error-map pixels, got gt {tuple(gt.shape)}, rgb "
                             f"{tuple(rgb.shape)}" + ("" if opacity is None else f", opacity {tuple(opacity.shape)}"))
        gt, rgb = _ops._f32c(gt), _ops._f32c(rgb)
        opacity = None if opacity is None else _ops._f32c(opacity)
        _ops._need_cuda(gt, rgb, opacity, rows)
        p = _ops._ptr
        _lib.call("emer_error_map", p(gt), p(rgb), p(opacity), n, p(rows), p(_map_workspace(rows.device)),
                  _ops._stream())

    def _publish(self, maps: Tensor) -> None:
        p = _ops._ptr
        _ops._need_cuda(maps)
        _lib.call("emer_error_map_normalize", p(maps), maps.numel(), p(_map_workspace(maps.device)), _ops._stream())
        self.source.pixel_error_maps = maps
        self.source.pixel_error_buffered = True

    @torch.no_grad()
    def update_pixel_error_maps(self, render_results) -> None:
        """``ScenePixelSource.update_pixel_error_maps`` (pixel_source.py:491-517): ``render_results`` holds lists,
        one entry per image, of numpy arrays (what ``render_pixels`` returns) or of device tensors under "gt_rgbs",
        "rgbs" and optionally "dynamic_opacities".  The new map is a new tensor, computed and normalised in two
        launches with the reference's arithmetic; the next ``get_train_rays`` validates it."""
        s = self.source
        if s.pixel_error_maps is None:
            return
        dev = s.pixel_error_maps.device

        def stacked(items):
            if isinstance(items[0], np.ndarray):
                return torch.from_numpy(np.stack(items, axis=0)).to(dev)
            return torch.stack(list(items)).to(dev)

        gt, rgb = stacked(render_results["gt_rgbs"]), stacked(render_results["rgbs"])
        assert gt.shape[:-1] == s.pixel_error_maps.shape
        dyn = render_results.get("dynamic_opacities")
        opacity = stacked(dyn) if dyn is not None and len(dyn) > 0 else None
        maps = torch.empty(s.pixel_error_maps.shape, dtype=torch.float32, device=dev)
        self._fold_error(gt, rgb, opacity, maps)
        self._publish(maps)

    @torch.no_grad()
    def refresh_pixel_error_maps(self, model, proposal_estimator, proposal_networks, cfg) -> None:
        """The error-map refresh of the training loop (train_emernerf.py:889-904 of the reference): every image of
        the source rendered at ``1 / buffer_downscale`` through ``render_rays``, one call per image, and its error
        written straight into a new map, which is then normalised and set on the source.  No numpy and no host sync
        of its own; the source's ``downscale_factor`` is not touched.  The decomposition is asked for only when the
        field has a dynamic branch, the one case where the reference's map uses it."""
        from .radiance_fields.render_utils import render_rays

        s = self.source
        if s.pixel_error_maps is None:
            return
        model.eval()
        if proposal_estimator is not None:
            proposal_estimator.eval()
        for p in proposal_networks or ():
            p.eval()
        decomposition = getattr(model, "dynamic_xyz_encoder", None) is not None
        d = 1 / s.buffer_downscale
        maps = torch.empty(s.pixel_error_maps.shape, dtype=torch.float32, device=s.pixel_error_maps.device)
        for i in range(len(maps)):
            data = self._render_rays_at(i, d)
            assert data["pixels"].shape[:2] == maps.shape[1:]
            out = render_rays(radiance_field=model, proposal_estimator=proposal_estimator,
                              proposal_networks=proposal_networks, data_dict=data, cfg=cfg,
                              return_decomposition=decomposition)
            self._fold_error(data["pixels"], out["rgb"], out.get("dynamic_opacity") if decomposition else None,
                             maps[i])
        self._publish(maps)


class CameraTrajectory:
    """Render rays of cameras moving between the source's own poses: a dataset the reference's ``render_pixels`` and
    ``render`` (radiance_fields/video_utils.py:50-468) take as it is, for new-view videos.

    For each camera in ``cams`` (default: every camera of ``source.cam_ids``, in the order they first appear there),
    the keyframes are that camera's images in increasing image index, the reference's timestep-major order.  With T
    keyframes per camera and m = ``frames_per_keyframe``, each camera has ``num_frames = (T - 1) m + 1`` frames: frame
    j lies in segment j // m at fraction (j % m) / m, so every m-th frame is a keyframe.  Item k is frame
    k // len(cams) of camera cams[k % len(cams)], the layout of ``save_videos(..., num_timestamps=num_frames,
    num_cams=len(cams))``.

    ``traj[k]`` holds ``get_render_rays``' ray keys, in its order and with its ``[h, w, ...]`` shapes and dtypes, at the
    source's current ``downscale_factor``: origins, viewdirs, direction_norm, pixel_coords, normed_timestamps (when the
    source has timestamps), img_idx, cam_idx, and all-zero sky_masks when the source has sky masks (``render`` reads
    them for the feature PCA).  The pose slerps the keyframes' rotations and lerps their origins, then moves the origin
    by ``offset`` along the camera's own axes; the time is lerped.  ``img_idx`` is the nearer keyframe's, so the
    per-image appearance embedding stays defined.  A keyframe with a zero offset is ``get_render_rays`` of that image
    on every shared key.  Each item is one ``emer_trajectory_rays`` launch (csrc/errormap.cu) without a host sync; the
    keyframes are found with one sync at construction."""

    split = "trajectory"

    def __init__(self, sampler: PixelRaySampler, cams=None, frames_per_keyframe: int = 1,
                 offset=(0.0, 0.0, 0.0)):
        if int(frames_per_keyframe) != frames_per_keyframe or frames_per_keyframe < 1:
            raise ValueError(f"CameraTrajectory: frames_per_keyframe must be an integer >= 1, "
                             f"got {frames_per_keyframe}")
        offset = tuple(float(v) for v in offset)
        if len(offset) != 3 or not all(np.isfinite(offset)):
            raise ValueError(f"CameraTrajectory: the offset must be 3 finite numbers, got {offset}")
        s = sampler.source
        cam_ids = _dense(s.cam_ids, "cam_ids", torch.int64)
        if cam_ids is None:
            raise ValueError("CameraTrajectory: the keyframes need source.cam_ids")
        _ops._need_cuda(cam_ids)
        ids = cam_ids.tolist()                           # the one host sync
        known = list(dict.fromkeys(ids))
        n_cams = getattr(s, "num_cams", None)
        cams = known if cams is None else [int(c) for c in cams]
        keyframes = []
        for c in cams:
            if c not in known and not (n_cams is not None and 0 <= c < n_cams):
                raise ValueError(f"CameraTrajectory: the source has no camera {c} (cameras {known})")
            keys = [i for i, v in enumerate(ids) if v == c]
            if not keys:
                raise ValueError(f"CameraTrajectory: camera {c} has no image")
            keyframes.append(keys)
        if len({len(k) for k in keyframes}) > 1:
            raise ValueError("CameraTrajectory: the cameras have different numbers of images: "
                             + ", ".join(f"{c}: {len(k)}" for c, k in zip(cams, keyframes)))
        self.sampler, self.cams, self.keyframes = sampler, cams, keyframes
        self.frames_per_keyframe, self.offset = int(frames_per_keyframe), offset
        self.num_frames = (len(keyframes[0]) - 1) * self.frames_per_keyframe + 1

    def __len__(self) -> int:
        return self.num_frames * len(self.cams)

    def segment(self, k: int) -> Tuple[int, int, int, int]:
        """(image a, image b, i, m) of item k: the frame lies between keyframes a and b at fraction i / m."""
        frame, c = divmod(k, len(self.cams))
        keys, m = self.keyframes[c], self.frames_per_keyframe
        seg, i = divmod(frame, m)
        if seg == len(keys) - 1:                        # the last keyframe
            return keys[seg], keys[seg], 0, m
        return keys[seg], keys[seg + 1], i, m

    @torch.no_grad()
    def __getitem__(self, k: int) -> Dict[str, Tensor]:
        k = int(k)
        if not -len(self) <= k < len(self):
            raise IndexError(f"CameraTrajectory: item {k} out of range for {len(self)} items")
        k %= len(self)
        s = self.source
        c2w, intr = _dense(s.cam_to_worlds, "cam_to_worlds"), _dense(s.intrinsics, "intrinsics")
        times, sky = _dense(s.normalized_timestamps, "normalized_timestamps"), _dense(s.sky_masks, "sky_masks")
        images = _dense(s.images, "images")
        if images is None:
            raise ValueError("CameraTrajectory: the frame size needs source.images")
        _ops._need_cuda(c2w, intr, times, images)
        d = float(s.downscale_factor)
        h, w = self.sampler._images_at(images, d).shape[1:3]
        a, b, i, m = self.segment(k)
        f32, dev = dict(dtype=torch.float32, device=c2w.device), c2w.device
        out = {"origins": torch.empty((h, w, 3), **f32), "viewdirs": torch.empty((h, w, 3), **f32),
               "direction_norm": torch.empty((h, w, 1), **f32), "pixel_coords": torch.empty((h, w, 2), **f32)}
        if times is not None:
            out["normed_timestamps"] = torch.empty((h, w), **f32)
        out["img_idx"] = torch.empty((h, w), dtype=torch.int64, device=dev)
        out["cam_idx"] = torch.empty((h, w), dtype=torch.int64, device=dev)
        if sky is not None:
            out["sky_masks"] = torch.empty((h, w), **f32)
        p = _ops._ptr
        args_in = _lib.EmerTrajectoryRaysIn(p(c2w), p(intr), p(times), len(c2w), a, b, self.cams[k % len(self.cams)],
                                            (ctypes.c_double * 3)(*self.offset), i, m, h, w, d)
        names = dict(norms="direction_norm", timestamps="normed_timestamps")
        args_out = _lib.EmerTrajectoryRaysOut(*(p(out.get(names.get(n, n))) for n in _lib.TRAJECTORY_RAYS_OUT_PTRS))
        _lib.call("emer_trajectory_rays", ctypes.byref(args_in), ctypes.byref(args_out), _ops._stream())
        return out

    @property
    def source(self):
        return self.sampler.source


class LidarRaySampler:
    """``SceneLidarSource.get_train_rays`` (datasets/base/lidar_source.py:223-308) without its per-step
    ``torch.tensor`` and ``torch.equal``: the points of the candidate scans are gathered once per candidate set (a
    host compare of the list; a tensor by identity and version), then each step is the reference's one ``randint`` and
    four gathers.  ``torch.isin`` gives the reference's mask, in point order.  ``candidate_indices=None`` samples every
    point (the reference then indexes whatever it cached last).

    ``get_render_rays(time_idx)`` replaces the sources' ``get_render_rays`` (lidar_source.py:310-327 and the Waymo
    override, datasets/waymo.py:341-356) without their seven boolean indexes, each a scan of every point of the drive
    and a host sync.  A frame table is built once per state of ``source.timesteps`` (its identity and ``_version``)
    with two host syncs; after that a frame costs no sync."""

    def __init__(self, source):
        self.source = source
        self._key, self._cached, self._held = None, None, None
        self._frames = None                  # (timesteps, its _version, {time index: (start, count)}, order or None)

    def get_train_rays(self, num_rays: int, candidate_indices=None) -> Dict[str, Tensor]:
        s = self.source
        key = _candidate_key(candidate_indices)
        if key != self._key:
            arrays = (s.origins, s.directions, s.ranges, s.normalized_timestamps)
            if candidate_indices is None:
                self._cached = arrays
            else:
                ts = s.timesteps
                cand = candidate_indices if key[0] == "tensor" else torch.tensor(key[1], dtype=ts.dtype)
                mask = torch.isin(ts, cand.to(ts.device))
                self._cached = tuple(a[mask] for a in arrays)
            self._key, self._held = key, candidate_indices
        origins, directions, ranges, times = self._cached
        idx = torch.randint(0, len(origins), size=(num_rays,), device=s.device)
        return {"lidar_origins": origins[idx], "lidar_viewdirs": directions[idx], "lidar_ranges": ranges[idx],
                "lidar_normed_timestamps": times[idx]}

    def _frame_table(self):
        """(table {time index: (start, count)}, order): the points of frame t are ``order[start:start + count]``, or
        the rows ``[start, start + count)`` when order is None.  When every timestep is one contiguous run (the Waymo
        loader concatenates the scans in order) each frame is a slice; otherwise a stable argsort keeps the points of
        a frame in their order, as the reference's boolean index does."""
        ts = self.source.timesteps
        f = self._frames
        if f is not None and f[0] is ts and f[1] == ts._version:
            return f[2], f[3]
        values, counts = torch.unique_consecutive(ts, return_counts=True)     # sizes its output: one sync
        values, counts = torch.stack([values.to(torch.int64), counts]).tolist()   # the second
        order = None
        if len(set(values)) == len(values):
            starts = np.cumsum([0] + counts[:-1]).tolist()
            table = {v: (s, c) for v, s, c in zip(values, starts, counts)}
        else:
            totals: Dict[int, int] = {}
            for v, c in zip(values, counts):
                totals[v] = totals.get(v, 0) + c
            keys = sorted(totals)
            starts = np.cumsum([0] + [totals[k] for k in keys[:-1]]).tolist()
            table = {k: (s, totals[k]) for k, s in zip(keys, starts)}
            order = torch.argsort(ts, stable=True)
        self._frames = (ts, ts._version, table, order)
        return table, order

    @torch.no_grad()
    def get_render_rays(self, time_idx: int) -> Dict[str, Tensor]:
        """Every point of the scan at ``time_idx``, in the source's point order: the reference's four keys, plus
        ``lidar_flow``, ``lidar_flow_class`` and ``lidar_ground`` when the source has ``flows``, ``flow_classes`` and
        ``grounds`` (the Waymo source).  Each value is ``torch.equal`` to the reference's; an absent index gives empty
        tensors, as there.  Slices of the source's tensors when its timesteps are contiguous runs, gathers
        otherwise."""
        s = self.source
        table, order = self._frame_table()
        start, count = table.get(int(time_idx), (0, 0))
        arrays = {"lidar_origins": s.origins, "lidar_viewdirs": s.directions, "lidar_ranges": s.ranges,
                  "lidar_normed_timestamps": s.normalized_timestamps}
        if all(getattr(s, k, None) is not None for k in ("flows", "flow_classes", "grounds")):
            arrays.update(lidar_flow=s.flows, lidar_flow_class=s.flow_classes, lidar_ground=s.grounds)
        if order is None:
            return {k: v[start:start + count] for k, v in arrays.items()}
        rows = order[start:start + count]
        return {k: v[rows] for k, v in arrays.items()}

"""The reference's evaluation videos, ``render`` + ``save_videos`` (radiance_fields/video_utils.py:104-627), restated
op for op with the package's ``render_rays`` on the caller's device: every product copied to host numpy as the
reference's ``get_numpy`` does, then the host loop of ``save_concatenated_videos`` / ``save_seperate_videos`` with
``visualize_depth`` (utils/visualization_tools.py:79-156) and ``to8b``.  The oracle of tests/test_gpu_videos.py and
the baseline of tools/bench_videos.py.

``Colormap`` restates matplotlib 3.6.1's ``Colormap.__call__`` on a given RGBA table, for the turbo map the reference
reads from matplotlib (the table itself is the caller's).  ``resize_five_views`` is not restated: five cameras raise.
"""
from __future__ import annotations

import logging
import os
from typing import Callable, Dict, List, Optional

import numpy as np
import torch
from torch import Tensor

logger = logging.getLogger()


class Colormap:
    """matplotlib 3.6.1's ``Colormap.__call__`` (colors.py) for a listed map of N RGBA entries: under and over take
    the first and last colour, "bad" (NaN) is (0, 0, 0, 0)."""

    def __init__(self, rgba: np.ndarray):
        rgba = np.asarray(rgba, np.float64)
        self.N = len(rgba)
        self._i_under, self._i_over, self._i_bad = self.N, self.N + 1, self.N + 2
        self._lut = np.concatenate([rgba, rgba[:1], rgba[-1:], np.zeros((1, 4))], axis=0)

    def __call__(self, X, alpha=None, bytes=False):
        xa = np.array(X, copy=True)
        if not xa.dtype.isnative:
            xa = xa.byteswap().newbyteorder()
        if xa.dtype.kind == "f":
            with np.errstate(invalid="ignore"):
                xa *= self.N
                xa[xa < 0] = -1
                xa[xa == self.N] = self.N - 1
                np.clip(xa, -1, self.N, out=xa)
                xa = xa.astype(int)
        mask_bad = np.isnan(X) if np.asarray(X).dtype.kind == "f" else np.zeros(np.shape(X), bool)
        xa[xa > self.N - 1] = self._i_over
        xa[xa < 0] = self._i_under
        xa[mask_bad] = self._i_bad
        lut = self._lut
        if bytes:
            lut = (lut * 255).astype(np.uint8)
        return lut.take(xa, axis=0, mode="clip")


def to8b(x):                                                  # visualization_tools.py:30-33
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    return (255 * np.clip(x, 0, 1)).astype(np.uint8)


def visualize_depth(x, acc, cmap, lo=4.0, hi=120, curve_fn=lambda x: -np.log(x + 1e-6)):
    """visualize_cmap (visualization_tools.py:79-141) as depth_visualizer calls it: given lo and hi, no matte."""
    value, lo, hi = [curve_fn(v) for v in [x, lo, hi]]
    value = np.nan_to_num(np.clip((value - np.minimum(lo, hi)) / np.abs(hi - lo), 0, 1))
    value *= acc
    return cmap(value)[..., :3]


def _numpy(x: Tensor) -> np.ndarray:                          # get_numpy, video_utils.py:44
    return x.squeeze().cpu().numpy()


@torch.no_grad()
def render(dataset, render_func: Callable, model, robust_pca: Callable, indices: List[int],
           scene_flow_to_rgb: Callable) -> Dict[str, list]:
    """video_utils.py:104-468 without the metrics: the lists ``render`` returns."""
    names = ("rgbs", "gt_rgbs", "static_rgbs", "dynamic_rgbs", "shadow_reduced_static_rgbs", "shadow_only_static_rgbs",
             "depths", "median_depths", "static_depths", "static_opacities", "dynamic_depths", "dynamic_opacities",
             "opacities", "gt_sky_masks", "dino_feats", "gt_dino_feats", "dino_feats_pe_free", "dino_pe",
             "static_dino_feats", "dynamic_dino_feats", "dynamic_dino_on_static_rgbs", "dynamic_rgb_on_static_dinos",
             "forward_flows", "backward_flows")
    L = {k: [] for k in names}
    computed = False
    flow = lambda f: scene_flow_to_rgb(f, flow_max_radius=1.0, background="bright").cpu().numpy()  # noqa: E731
    for i in indices:
        data = dict(dataset[i])
        for k, v in data.items():
            if isinstance(v, Tensor):
                data[k] = v.cuda(non_blocking=True)
        r = render_func(data)
        L["rgbs"].append(_numpy(r["rgb"]))
        if "pixels" in data:
            L["gt_rgbs"].append(_numpy(data["pixels"]))
        if "static_rgb" in r:
            L["static_rgbs"].append(_numpy(r["static_rgb"]))
        if "dynamic_rgb" in r:
            green = (torch.tensor([0.0, 177, 64]) / 255.0).to(r["dynamic_rgb"].device)
            L["dynamic_rgbs"].append(_numpy(r["dynamic_rgb"] * r["dynamic_opacity"]
                                            + green * (1 - r["dynamic_opacity"])))
        for k in ("shadow_reduced_static_rgb", "shadow_only_static_rgb"):
            if k in r:
                L[k + "s"].append(_numpy(r[k]))
        if "forward_flow" in r:
            L["forward_flows"].append(flow(r["forward_flow"]))
        if "backward_flow" in r:
            L["backward_flows"].append(flow(r["backward_flow"]))
        L["depths"].append(_numpy(r["depth"]))
        L["opacities"].append(_numpy(r["opacity"]))
        if "static_depth" in r:
            L["static_depths"].append(_numpy(r["static_depth"]))
            L["static_opacities"].append(_numpy(r["static_opacity"]))
        if "dynamic_depth" in r:
            L["dynamic_depths"].append(_numpy(r["dynamic_depth"]))
            L["dynamic_opacities"].append(_numpy(r["dynamic_opacity"]))
        elif "median_depth" in r:
            L["median_depths"].append(_numpy(r["median_depth"]))
        if "sky_masks" in data:
            L["gt_sky_masks"].append(_numpy(data["sky_masks"]))
        if "dino_feat" not in r:
            continue
        m = model
        pred = r["dino_feat"]
        gt = data["features"] if "features" in data else None
        pred = pred @ m.feats_reduction_mat.to(pred)
        pred = (pred - m.feat_color_min.to(pred)) / (m.feat_color_max.to(pred) - m.feat_color_min.to(pred))
        if gt is not None:
            gt = gt @ m.feats_reduction_mat.to(pred)
            gt = (gt - m.feat_color_min.to(pred)) / (m.feat_color_max.to(pred) - m.feat_color_min.to(pred))
        if "dino_pe_free" in r:
            if not computed:
                computed = True
                non_sky = r["dino_pe_free"] * (~data["sky_masks"].bool().unsqueeze(-1)).to(r["dino_pe_free"])
                mat, lo, hi = robust_pca(non_sky.reshape(-1, r["dino_pe_free"].shape[-1]), m=2.5)
                pe_mat, pe_lo, pe_hi = robust_pca(r["dino_pe"].reshape(-1, r["dino_pe"].shape[-1]), m=2.5)
            x = r["dino_pe_free"] @ mat
            x = (x - lo.to(pred)) / (hi.to(pred) - lo.to(pred))
            x = torch.clamp(x, 0, 1)
            x *= r["opacity"]
            L["dino_feats_pe_free"].append(_numpy(x))
            x = r["dino_pe"] @ pe_mat
            x = (x - pe_lo.to(pred)) / (pe_hi - pe_lo).to(pred)
            L["dino_pe"].append(_numpy(torch.clamp(x, 0, 1)))
            if "static_dino" in r:
                x = r["static_dino"] @ mat
                x = torch.clamp((x - lo.to(pred)) / (hi - lo).to(pred), 0, 1)
                L["static_dino_feats"].append(_numpy(x))
                a = L["dynamic_opacities"][-1][..., None]
                L["dynamic_rgb_on_static_dinos"].append(np.clip(_numpy(r["dynamic_rgb"]) * a
                                                                + L["static_dino_feats"][-1] * (1 - a), 0, 1))
            if "dynamic_dino" in r:
                x = r["dynamic_dino"] @ mat
                x = torch.clamp((x - lo.to(pred)) / (hi - lo).to(pred), 0, 1)
                x *= r["dynamic_opacity"]
                L["dynamic_dino_feats"].append(_numpy(x))
                a = L["dynamic_opacities"][-1][..., None]
                L["dynamic_dino_on_static_rgbs"].append(np.clip(L["dynamic_dino_feats"][-1] * a
                                                                + L["static_rgbs"][-1] * (1 - a), 0, 1))
        else:
            if "static_dino" in r:
                x = r["static_dino"] @ m.feats_reduction_mat.to(pred)
                x = (x - m.feat_color_min.to(pred)) / (m.feat_color_max.to(pred) - m.feat_color_min.to(pred))
                L["static_dino_feats"].append(_numpy(torch.clamp(x, 0, 1)))
                a = L["dynamic_opacities"][-1][..., None]
                L["dynamic_rgb_on_static_dinos"].append(np.clip(_numpy(r["dynamic_rgb"]) * a
                                                                + L["static_dino_feats"][-1] * (1 - a), 0, 1))
            if "dynamic_dino" in r:
                x = r["dynamic_dino"] @ m.feats_reduction_mat
                x = (x - m.feat_color_min.to(pred)) / (m.feat_color_max.to(pred) - m.feat_color_min.to(pred))
                L["dynamic_dino_feats"].append(_numpy(torch.clamp(x, 0, 1)))
                a = L["dynamic_opacities"][-1][..., None]
                L["dynamic_dino_on_static_rgbs"].append(np.clip(L["dynamic_dino_feats"][-1] * a
                                                                + L["static_rgbs"][-1] * (1 - a), 0, 1))
        L["dino_feats"].append(_numpy(torch.clamp(pred, 0, 1)))
        if gt is not None:
            L["gt_dino_feats"].append(_numpy(torch.clamp(gt, 0, 1)))
    keep = ("rgbs", "static_rgbs", "dynamic_rgbs", "depths", "opacities", "static_depths", "static_opacities",
            "dynamic_depths", "dynamic_opacities")
    return {k: v for k, v in L.items() if k in keep or len(v) > 0}


def save_videos(render_results, save_pth: str, num_timestamps: int, keys, num_cams: int, save_seperate_video: bool,
                save_images: bool, fps: int, verbose: bool, cmap, get_writer: Callable, imwrite: Callable):
    """video_utils.py:471-627 with the writer factory and ``imwrite`` given; five cameras are refused."""
    if num_cams == 5:
        raise ValueError("resize_five_views is not restated")
    depth = lambda f, o: visualize_depth(f, o, cmap)  # noqa: E731
    R = render_results
    if not save_seperate_video:
        if num_timestamps == 1:
            writer, ret_id = get_writer(save_pth, mode="I"), 0
        else:
            ret_id, writer = num_timestamps // 2, get_writer(save_pth, mode="I", fps=fps)
        for i in range(num_timestamps):
            merged = []
            for key in keys:
                if key == "sky_masks":
                    frames = R["opacities"][i * num_cams:(i + 1) * num_cams]
                else:
                    if key not in R or len(R[key]) == 0:
                        continue
                    frames = R[key][i * num_cams:(i + 1) * num_cams]
                if key == "gt_sky_masks":
                    frames = [np.stack([f, f, f], axis=-1) for f in frames]
                elif key == "sky_masks":
                    frames = [1 - np.stack([f, f, f], axis=-1) for f in frames]
                elif "depth" in key:
                    try:
                        ops = R[key.replace("depths", "opacities")][i * num_cams:(i + 1) * num_cams]
                    except KeyError:
                        if "median" in key:
                            ops = R[key.replace("median_depths", "opacities")][i * num_cams:(i + 1) * num_cams]
                        else:
                            continue
                    frames = [depth(f, o) for f, o in zip(frames, ops)]
                merged.append(np.concatenate(frames, axis=1))
            frame = to8b(np.concatenate(merged, axis=0))
            if i == ret_id:
                ret = frame
            writer.append_data(frame)
        writer.close()
        if verbose:
            logger.info(f"saved video to {save_pth}")
        return {"concatenated_frame": ret}
    ret_id, out = num_timestamps // 2, {}
    for key in keys:
        path = save_pth.replace(".mp4", f"_{key}.mp4").replace(".png", f"_{key}.png")
        if key not in R or len(R[key]) == 0:
            continue                                # (the reference opens a writer first)
        writer = get_writer(path, mode="I") if num_timestamps == 1 else get_writer(path, mode="I", fps=fps)
        for i in range(num_timestamps):
            frames = R[key][i * num_cams:(i + 1) * num_cams]
            if key == "gt_sky_masks":
                frames = [np.stack([f, f, f], axis=-1) for f in frames]
            elif "depth" in key:
                okey = key.replace("depths", "opacities")
                if okey not in R and "median" in key:
                    okey = "opacities"                  # (the reference raises KeyError here)
                ops = R[okey][i * num_cams:(i + 1) * num_cams]
                frames = [depth(f, o) for f, o in zip(frames, ops)]
            if save_images:
                if i == 0:
                    os.makedirs(path.replace(".mp4", ""), exist_ok=True)
                for j, f in enumerate(frames):
                    imwrite(path.replace(".mp4", f"_{i*3 + j:03d}.png"), to8b(f))
            frame = to8b(np.concatenate(frames, axis=1))
            writer.append_data(frame)
            if i == ret_id:
                out[key] = frame
        writer.close()
        if verbose:
            logger.info(f"saved video to {path}")
    return out


def render_videos(cfg, model, proposal_estimator, proposal_networks, dataset, save_pth, num_timestamps, keys,
                  num_cams, save_seperate_video=False, save_images=False, fps=10, verbose=True, vis_indices=None,
                  return_decomposition=True, *, render_rays, robust_pca, scene_flow_to_rgb, cmap, get_writer,
                  imwrite=None):
    """``render_pixels`` (without metrics) and ``save_videos`` as the driver calls them; returns the frame dict."""
    model.eval()
    for p in proposal_networks or ():
        p.eval()
    if proposal_estimator is not None:
        proposal_estimator.eval()
    func = lambda d: render_rays(radiance_field=model, proposal_estimator=proposal_estimator,  # noqa: E731
                                 proposal_networks=proposal_networks, data_dict=d, cfg=cfg,
                                 return_decomposition=return_decomposition)
    indices = list(vis_indices) if vis_indices is not None else list(range(len(dataset)))
    results = render(dataset, func, model, robust_pca, indices, scene_flow_to_rgb)
    return save_videos(results, save_pth, num_timestamps, keys, num_cams, save_seperate_video, save_images, fps,
                       verbose, cmap, get_writer, imwrite)

"""``render_rays`` / ``rendering`` with the reference's signatures and output dictionaries
(radiance_fields/render_utils.py of NVlabs/EmerNeRF), on the sm_90a kernels:

  transmittance / alpha / weights / opacity / depth / median depth -> emer_composite_fwd/bwd
  every accumulate_along_rays                                      -> emer_accumulate_fwd/bwd
  proposal sampling                                                -> PropNetEstimator (emer_pdf_resample)

With ``EMER_RENDERING=fused`` the whole body of ``rendering`` (blend, accumulations, sky / PE terms, decomposition) is
one emer_render_fwd launch and one emer_render_bwd launch instead (csrc/render.cu); the default is ``torch``.

Two behaviours of the reference are preserved on purpose:
  * the per-level proposal closures all bind the LAST proposal network (render_utils.py:357-359
    builds ``[lambda *args: prop_sigma_fn(*args, p) for p in proposal_networks]``; Python closes over
    the loop variable, so every level evaluates ``proposal_networks[-1]``);
  * ``query_fn`` hands the field one value per SAMPLE for every per-ray entry (render_utils.py:332-336).
    Here those are stride-0 ``expand`` views instead of ``repeat_interleave`` copies -- same values,
    no HBM traffic.
"""
from __future__ import annotations

import os
from typing import Callable, Dict, List, Optional, Tuple

import torch
from torch import Tensor

from .. import _ops
from ..third_party.nerfacc_prop_net import FusedProposalLevel, PropNetEstimator
from .radiance_field import DensityField, RadianceField


def _weights_opacity_depth(t_starts: Tensor, t_ends: Tensor, density: Tensor):
    """render_weights_opacity_depth_from_density (render_utils.py:19-45)."""
    weights, _, opacity, depth, _, _ = _ops.composite(t_starts, t_ends, density)
    return weights, opacity, depth


def render_weights_opacity_depth_from_density(t_starts: Tensor, t_ends: Tensor, density: Tensor):
    return _weights_opacity_depth(t_starts, t_ends, density)


_FLOW_KEYS = ("forward_flow", "backward_flow", "forward_pred_backward_flow", "backward_pred_forward_flow")


# "fused": the body of ``rendering`` as one emer_render_fwd launch (and one emer_render_bwd), csrc/render.cu;
# "torch": emer_composite_* and one emer_accumulate_* per accumulated quantity, with the blend in torch ops
RENDERING = os.environ.get("EMER_RENDERING", "torch")

# results key -> emer_render input
_RENDER_KEYS = {"density": "sigma", "static_density": "sigma_s", "dynamic_density": "sigma_d", "rgb": "rgb",
                "static_rgb": "rgb_s", "dynamic_rgb": "rgb_d", "shadow_ratio": "shadow", "rgb_sky": "rgb_sky",
                "dino_feat": "dino", "static_dino_feat": "dino_s", "dynamic_dino_feat": "dino_d",
                "dino_sky_feat": "dino_sky", "dino_pe": "dino_pe"}


def _fused_rendering(t_starts: Tensor, t_ends: Tensor, results: Dict[str, Tensor],
                     return_decomposition: bool) -> Optional[Dict[str, Tensor]]:
    """``rendering``'s outputs from ``_ops.render``, or None where the kernel does not cover the field's results (more
    than 256 feature channels, the decomposition under grad, results with neither colours nor features): the caller
    then takes the op-by-op path."""
    decomposed = "static_density" in results and "dynamic_density" in results
    has_rgb = "rgb" in results or (decomposed and "static_rgb" in results and "dynamic_rgb" in results)
    plain_dino = "dino_feat" in results
    has_dino = plain_dino or (decomposed and "static_dino_feat" in results and "dynamic_dino_feat" in results)
    if not (has_rgb or has_dino):
        return None
    if has_dino and results["dino_feat" if plain_dino else "static_dino_feat"].shape[-1] > _ops.RENDER_MAX_CHANNELS:
        return None
    ins = {"sigma": results["density"].squeeze(-1)}
    for k, name in _RENDER_KEYS.items():
        if k == "density" or k not in results:
            continue
        if name in ("sigma_s", "sigma_d") and not decomposed:
            continue
        if name in ("rgb_s", "rgb_d", "shadow") and ("rgb" in results or not has_rgb):
            continue                       # the reference blends (and reads the shadow) only without a plain rgb
        if name in ("dino_s", "dino_d") and (plain_dino or not has_dino):
            continue
        if name in ("dino_sky", "dino_pe") and not has_dino:
            continue
        if name == "rgb_sky" and not has_rgb:
            continue
        ins[name] = results[k]
    decomp = return_decomposition and decomposed
    if decomp and torch.is_grad_enabled() and any(v.requires_grad for v in ins.values()):
        return None
    flows = None
    if decomp and "forward_flow" in results and "rgb_s" in ins:
        flows = (results["forward_flow"], results["backward_flow"])
    r = _ops.render(t_starts, t_ends, ins, flows=flows, decomposition=decomp)
    out = {"density": ins["sigma"], "depth": r["depth"], "opacity": r["opacity"], "median_depth": r["median_depth"]}
    names = {"dino": "dino_feat"}
    for k in ("rgb", "shadow_ratio", "dino", "dino_pe_free") + _ops.RENDER_DECOMPOSITION:
        if k in r:
            out[names.get(k, k)] = r[k]
    if "dino_pe" in ins:
        out["dino_pe"] = results["dino_pe"]
    out["extras"] = {"weights": r["weights"], "trans": r["trans"]}
    return out


def rendering(t_starts: Tensor, t_ends: Tensor, query_fn: Optional[Callable] = None,
              return_decomposition: bool = False) -> Dict[str, Tensor]:
    results = query_fn(t_starts, t_ends)
    if RENDERING == "fused":
        out = _fused_rendering(t_starts, t_ends, results, return_decomposition)
        if out is not None:
            extras = out["extras"]
            extras.update({"t_vals": (t_starts + t_ends) / 2.0, "t_dist": (t_ends - t_starts)})
            for k in _FLOW_KEYS:
                if k in results:
                    extras[k] = results[k]
            if "static_density" in results and "dynamic_density" in results:
                extras["static_density"] = results["static_density"]
                extras["dynamic_density"] = results["dynamic_density"]
            return out
    density = results["density"].squeeze(-1)
    weights, trans, opacity, depth, median_depth, _ = _ops.composite(t_starts, t_ends, density)
    acc = _ops.accumulate

    extras = {"weights": weights, "trans": trans, "t_vals": (t_starts + t_ends) / 2.0,
              "t_dist": (t_ends - t_starts)}
    for k in _FLOW_KEYS:
        if k in results:
            extras[k] = results[k]

    out = {"density": density, "depth": depth, "opacity": opacity, "median_depth": median_depth}

    decomposed = "static_density" in results and "dynamic_density" in results
    if decomposed:
        extras["static_density"] = results["static_density"]
        extras["dynamic_density"] = results["dynamic_density"]
        static_ratio = results["static_density"] / (results["density"] + 1e-6)
        dynamic_ratio = results["dynamic_density"] / (results["density"] + 1e-6)
        if return_decomposition:
            static_w, out["static_opacity"], out["static_depth"] = _weights_opacity_depth(
                t_starts, t_ends, results["static_density"])
            dynamic_w, out["dynamic_opacity"], out["dynamic_depth"] = _weights_opacity_depth(
                t_starts, t_ends, results["dynamic_density"])

    if "rgb" in results:
        out["rgb"] = acc(weights, results["rgb"])
    elif "static_rgb" in results and "dynamic_rgb" in results:
        shadow = 0.0
        if "shadow_ratio" in results:
            shadow = results["shadow_ratio"]
            out["shadow_ratio"] = acc(weights, shadow.square())          # squared, as the reference (Q6)
        blended = (static_ratio[..., None] * results["static_rgb"] * (1 - shadow)
                   + dynamic_ratio[..., None] * results["dynamic_rgb"])
        out["rgb"] = acc(weights, blended)
        if return_decomposition:
            out["static_rgb"] = acc(static_w, results["static_rgb"])
            if "shadow_ratio" in results:
                out["shadow_reduced_static_rgb"] = acc(static_w, results["static_rgb"] * (1 - shadow))
                shadow_only = acc(static_w, results["static_rgb"] * shadow)
                acc_shadow = acc(weights, shadow)
                out["shadow_only_static_rgb"] = shadow_only + (1 - acc_shadow)
                out["shadow"] = acc_shadow
            out["dynamic_rgb"] = acc(dynamic_w, results["dynamic_rgb"])
            if "forward_flow" in results:
                out["forward_flow"] = acc(dynamic_w, results["forward_flow"])
                out["backward_flow"] = acc(dynamic_w, results["backward_flow"])

    if "rgb_sky" in results:
        out["rgb"] = out["rgb"] + results["rgb_sky"] * (1.0 - out["opacity"])
        if "static_rgb" in out:
            out["static_rgb"] = out["static_rgb"] + results["rgb_sky"] * (1.0 - out["static_opacity"])

    def add_sky_and_pe():
        if "dino_sky_feat" in results:
            out["dino_feat"] = out["dino_feat"] + results["dino_sky_feat"] * (1.0 - out["opacity"])
        if "dino_pe" in results:
            out["dino_pe_free"] = out["dino_feat"].clone()
            out["dino_pe"] = results["dino_pe"]
            out["dino_feat"] = out["dino_feat"] + results["dino_pe"]

    if "dino_feat" in results:
        out["dino_feat"] = acc(weights, results["dino_feat"])
        add_sky_and_pe()
    elif "static_dino_feat" in results and "dynamic_dino_feat" in results:
        blended = (static_ratio[..., None] * results["static_dino_feat"]
                   + dynamic_ratio[..., None] * results["dynamic_dino_feat"])
        out["dino_feat"] = acc(weights, blended)
        add_sky_and_pe()
        if return_decomposition:
            out["static_dino"] = acc(static_w, results["static_dino_feat"])
            out["dynamic_dino"] = acc(dynamic_w, results["dynamic_dino_feat"])
            if "dino_sky_feat" in results:
                out["static_dino"] = out["static_dino"] + results["dino_sky_feat"] * (1.0 - out["opacity"])

    out["extras"] = extras
    return out


def _per_sample(v: Tensor, n_samples: int) -> Tensor:
    """[R, ...] -> [R, ..., S] view with stride 0 along the new sample axis."""
    return v.unsqueeze(-1).expand(*v.shape, n_samples)


def render_rays(
    radiance_field: RadianceField = None,
    proposal_estimator: PropNetEstimator = None,
    proposal_networks: Optional[List[DensityField]] = None,
    data_dict: Dict[str, Tensor] = None,
    cfg=None,
    proposal_requires_grad: bool = False,
    return_decomposition: bool = False,
    prefix="",
) -> Dict[str, Tensor]:
    """Render a batch of rays ([R, 3] or [H, W, 3] origins / viewdirs under ``prefix``)."""
    rays_shape = data_dict[prefix + "origins"].shape
    if len(rays_shape) == 3:
        num_rays = rays_shape[0] * rays_shape[1]
        flat = {k: v.reshape(num_rays, -1).squeeze() for k, v in data_dict.items()}
    else:
        num_rays = rays_shape[0]
        flat = data_dict.copy()
    assert proposal_networks is not None, "proposal_networks is required."
    key_o, key_d = prefix + "origins", prefix + "viewdirs"

    results: List[Dict[str, Tensor]] = []
    extras = None
    chunk = 2 ** 24 if radiance_field.training else cfg.render.render_chunk_size
    for start in range(0, num_rays, chunk):
        rays = {k: v[start:start + chunk] for k, v in flat.items()}
        origins = rays[key_o][..., None, :]
        dirs = rays[key_d][..., None, :]

        def prop_sigma_fn(t_starts, t_ends, proposal_network):
            positions = origins + dirs * (t_starts + t_ends)[..., None] / 2.0
            times = {k: _per_sample(v, t_starts.shape[-1]) for k, v in rays.items() if "time" in k}
            return proposal_network(positions, times)

        def query_fn(t_starts, t_ends):
            n_samples = t_starts.shape[-1]
            t_dirs = dirs.expand(-1, n_samples, -1)
            sub = {k: _per_sample(v, n_samples) for k, v in rays.items()
                   if k not in (key_d, key_o, "pixel_coords")}
            sub["t_starts"], sub["t_ends"] = t_starts, t_ends
            if "pixel_coords" in rays:
                sub["pixel_coords"] = rays["pixel_coords"]
            positions = origins + t_dirs * (t_starts + t_ends)[..., None] / 2.0
            res = radiance_field(positions, t_dirs, sub, return_density_only=(prefix == "lidar_"))
            res["density"] = res["density"].squeeze(-1)
            return res

        # late binding on purpose: every level evaluates proposal_networks[-1] (see module docstring)
        last_prop = proposal_networks[-1]
        level_fns = []
        for _ in proposal_networks:
            fn = lambda *args: prop_sigma_fn(*args, last_prop)     # noqa: E731
            # lets sampling() run the level as one fused kernel when no proposal gradients are needed
            fn.emer_fused = FusedProposalLevel(rays[key_o], rays[key_d], last_prop)
            level_fns.append(fn)
        t_starts, t_ends = proposal_estimator.sampling(
            prop_sigma_fns=level_fns,
            num_samples=cfg.nerf.sampling.num_samples,
            prop_samples=cfg.nerf.propnet.num_samples_per_prop,
            n_rays=rays[key_o].shape[0],
            near_plane=cfg.nerf.propnet.near_plane,
            far_plane=cfg.nerf.propnet.far_plane,
            sampling_type=cfg.nerf.propnet.sampling_type,
            stratified=radiance_field.training,
            requires_grad=proposal_requires_grad,
        )
        rendered = rendering(t_starts, t_ends, query_fn=query_fn, return_decomposition=return_decomposition)
        extras = rendered.pop("extras")
        results.append(rendered)

    merged = results[0] if len(results) == 1 else {k: torch.cat([r[k] for r in results], 0) for k in results[0]}
    extras["density"] = merged.pop("density")
    for k, v in merged.items():
        merged[k] = v.reshape(list(rays_shape[:-1]) + list(v.shape[1:]))
    merged["extras"] = extras
    return merged

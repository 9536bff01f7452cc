"""CPU restatement of EmerNeRF's per-ray-batch hot path as plain functions over a state-dict.

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.  Self-contained (the reference
is not needed to run it): it is what the ``-m gpu`` parity tests, the ``smoke()``
check and the ``cpu_baseline`` leg of ``bench.py`` run.

PINNED against the reference's own Python: ``tests/golden/make_golden.py`` runs
the unmodified reference modules (with ``oracle.ref_shims``) and
``tests/test_oracle_golden.py`` compares this restatement with the committed
vectors.  The hash-grid / nerfacc arithmetic underneath comes from
``oracle.tcnn_ref`` / ``oracle.nerfacc_ref`` (parity unpinned, see there).

Every function cites the reference file:line it follows (NVlabs/EmerNeRF@8c051d7).
State-dict keys are the reference's (SURVEY.md §5): ``xyz_encoder.tcnn_encoding.params``,
``base_mlp.{0,2}.*``, ``rgb_head.layers.{0,1,2}.*``, ...
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

from . import nerfacc_ref as nf
from . import tcnn_ref

SD = Dict[str, Tensor]


# --------------------------------------------------------------------------- specs
def hash_encoder_config(n_levels, base_resolution, max_resolution, log2_hashmap_size,
                        n_features_per_level) -> dict:
    """encodings.py:130-141 -- growth factor in float64 numpy, then the tcnn config dict."""
    growth = np.exp((np.log(max_resolution) - np.log(base_resolution)) / (n_levels - 1))
    return {
        "otype": "HashGrid", "n_levels": n_levels, "n_features_per_level": n_features_per_level,
        "log2_hashmap_size": log2_hashmap_size, "base_resolution": base_resolution,
        "per_level_scale": growth, "interpolation": "linear",
    }


@dataclass
class FieldSpec:
    """Static description of a RadianceField (radiance_field.py:21-217) or, with
    ``density_only=True``, of a proposal DensityField (radiance_field.py:788-812)."""
    xyz: dict
    dynamic: Optional[dict] = None
    flow: Optional[dict] = None
    unbounded: bool = True
    geometry_feature_dim: int = 64
    semantic_feature_dim: int = 0          # already zeroed when the feature head is off (:65-67)
    enable_cam_embedding: bool = False
    enable_img_embedding: bool = False
    appearance_embedding_dim: int = 16
    enable_sky_head: bool = False
    enable_shadow_head: bool = False
    enable_feature_head: bool = False
    enable_learnable_pe: bool = True
    time_diff: float = 0.0
    density_only: bool = False
    geoms: dict = field(default_factory=dict)

    def geom(self, which: str) -> tcnn_ref.GridGeometry:
        if which not in self.geoms:
            cfg = {"xyz": self.xyz, "dynamic": self.dynamic, "flow": self.flow}[which]
            self.geoms[which] = tcnn_ref.grid_geometry(3 if which == "xyz" else 4, cfg)
        return self.geoms[which]


# --------------------------------------------------------------------------- small pieces
class _TruncExp(torch.autograd.Function):
    """nerf_utils.py:59-75: forward exp, backward g * exp(clamp(x, max=15))."""

    @staticmethod
    def forward(ctx, x):
        x = x.to(torch.float32)
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(torch.clamp(x, max=15))


def density_activation(x: Tensor) -> Tensor:
    """radiance_field.py:28,794: trunc_exp(x - 1)."""
    return _TruncExp.apply(x - 1)


def contract(x: Tensor, aabb: Tensor) -> Tensor:
    """nerf_utils.py:13-28 with ord=inf (radiance_field.py:290,830)."""
    lo, hi = torch.split(aabb, 3, dim=-1)
    x = (x - lo) / (hi - lo)
    x = x * 2 - 1
    mag = torch.linalg.norm(x, ord=float("inf"), dim=-1, keepdim=True)
    x = torch.where(mag < 1, x, (2 - 1 / mag) * (x / mag))
    return x / 4 + 0.5


def contract_points(positions: Tensor, aabb: Tensor, unbounded: bool) -> Tensor:
    """radiance_field.py:278-300 / :828-835: contraction, then multiply by the 0/1 in-cube selector."""
    if unbounded:
        p = contract(positions, aabb)
    else:
        lo, hi = torch.split(aabb, 3, dim=-1)
        p = (positions - lo) / (hi - lo)
    sel = ((p > 0.0) & (p < 1.0)).all(dim=-1).to(positions)
    return p * sel.unsqueeze(-1)


def sinusoidal(x: Tensor, min_deg: int = 0, max_deg: int = 4) -> Tensor:
    """encodings.py:86-104 (no_grad; identity first, then sin(x*2^i), then sin(x*2^i + pi/2))."""
    with torch.no_grad():
        scales = torch.tensor([2.0 ** i for i in range(min_deg, max_deg + 1)], dtype=x.dtype)
        xb = (x[..., None, :] * scales[:, None]).reshape(*x.shape[:-1], -1)
        enc = torch.sin(torch.cat([xb, xb + 0.5 * torch.pi], dim=-1))
        return torch.cat([x, enc], dim=-1)


def _lin(sd: SD, name: str, x: Tensor) -> Tensor:
    return F.linear(x, sd[name + ".weight"], sd[name + ".bias"])


def seq_mlp(sd: SD, prefix: str, x: Tensor, idx: Sequence[int]) -> Tensor:
    """nn.Sequential(Linear, ReLU, Linear, ...) with Linear modules at positions ``idx``."""
    for j, i in enumerate(idx):
        x = _lin(sd, f"{prefix}.{i}", x)
        if j < len(idx) - 1:
            x = F.relu(x)
    return x


def skip_mlp(sd: SD, prefix: str, x: Tensor, n_layers: int = 3, skips=(1,)) -> Tensor:
    """mlp.py:38-46: before layer i in ``skips`` the running activation is cat'ed with the input."""
    inp = x
    for i in range(n_layers):
        if i in skips:
            x = torch.cat([x, inp], -1)
        x = _lin(sd, f"{prefix}.layers.{i}", x)
        if i < n_layers - 1:
            x = F.relu(x)
    return x


def encode(sd: SD, key: str, geom: tcnn_ref.GridGeometry, x: Tensor) -> Tensor:
    """encodings.py:159-160 -> tcnn_modules.py:235-263 (pad/cast are no-ops for fp32 here)."""
    shp = x.shape[:-1]
    y = tcnn_ref.grid_forward(x.reshape(-1, x.shape[-1]).to(torch.float32).contiguous(),
                              sd[key + ".tcnn_encoding.params"], geom)
    return y.view(*shp, -1)


# --------------------------------------------------------------------------- fields
def density_field_forward(sd: SD, spec: FieldSpec, positions: Tensor) -> Dict[str, Tensor]:
    """DensityField.forward, radiance_field.py:825-841."""
    p = contract_points(positions, sd["aabb"], spec.unbounded)
    enc = encode(sd, "xyz_encoder", spec.geom("xyz"), p)
    raw = seq_mlp(sd, "base_mlp", enc, (0, 2))
    return {"density": density_activation(raw)}


def _dynamic_hash(sd, spec, normed_pos, t):
    """forward_dynamic_hash, radiance_field.py:320-357 (the live ``if True`` branch)."""
    if t.shape[-1] != 1:
        t = t.unsqueeze(-1)
    enc = encode(sd, "dynamic_xyz_encoder", spec.geom("dynamic"), torch.cat([normed_pos, t], -1))
    return seq_mlp(sd, "dynamic_base_mlp", enc, (0, 2)), enc


def _flow_hash(sd, spec, normed_pos, t):
    """forward_flow_hash, radiance_field.py:359-389 (training / no temporal interpolation branch)."""
    if t.shape[-1] != 1:
        t = t.unsqueeze(-1)
    enc = encode(sd, "flow_xyz_encoder", spec.geom("flow"), torch.cat([normed_pos, t], -1))
    return seq_mlp(sd, "flow_mlp", enc, (0, 2, 4))


def _temporal_aggregation(sd, spec, positions, t, fwd_flow, bwd_flow, dyn_feats, noise):
    """temporal_aggregation, radiance_field.py:553-620.  ``noise`` is [..., 1]."""
    if t.shape[-1] != 1:
        t = t.unsqueeze(-1)
    aabb = sd["aabb"]
    p_f = contract_points(positions + fwd_flow * noise, aabb, spec.unbounded)
    p_b = contract_points(positions + bwd_flow * noise, aabb, spec.unbounded)
    t_f = torch.clamp(t + spec.time_diff * noise, 0, 1.0)
    t_b = torch.clamp(t - spec.time_diff * noise, 0, 1.0)
    f_feats, f_enc = _dynamic_hash(sd, spec, p_f, t_f)
    b_feats, b_enc = _dynamic_hash(sd, spec, p_b, t_b)
    f_flow = _flow_hash(sd, spec, p_f, t_f)
    b_flow = _flow_hash(sd, spec, p_b, t_b)
    agg = (dyn_feats + 0.5 * f_feats + 0.5 * b_feats) / 2.0
    return {
        "dynamic_feats": agg,
        "forward_pred_backward_flow": f_flow[..., 3:],
        "backward_pred_forward_flow": b_flow[..., :3],
        "forward_dynamic_hash_encodings": f_enc,
        "backward_dynamic_hash_encodings": b_enc,
    }


def _appearance(sd, spec, directions, data):
    """radiance_field.py:633-645 / :667-679: embedding by cam_idx / img_idx, else the mean row."""
    if not (spec.enable_cam_embedding or spec.enable_img_embedding):
        return None
    W = sd["appearance_embedding.weight"]
    if "cam_idx" in data and spec.enable_cam_embedding:
        return F.embedding(data["cam_idx"], W)
    if "img_idx" in data and spec.enable_img_embedding:
        return F.embedding(data["img_idx"], W)
    return torch.ones((*directions.shape[:-1], spec.appearance_embedding_dim)) * W.mean(dim=0)


def _query_rgb(sd, spec, directions, geo, dyn_geo, data):
    """query_rgb, radiance_field.py:622-658."""
    d = (directions + 1.0) / 2.0
    h = sinusoidal(d.reshape(-1, d.shape[-1])).view(*d.shape[:-1], -1)
    emb = _appearance(sd, spec, d, data)
    if emb is not None:
        h = torch.cat([h, emb], -1)
    out = {"rgb": torch.sigmoid(skip_mlp(sd, "rgb_head", torch.cat([h, geo], -1)))}
    if spec.dynamic is not None:
        out["dynamic_rgb"] = torch.sigmoid(skip_mlp(sd, "rgb_head", torch.cat([h, dyn_geo], -1)))
    return out


def _query_sky(sd, spec, directions, data):
    """query_sky, radiance_field.py:660-686 (directions are NOT remapped to [0,1] here)."""
    dd = sinusoidal(directions if directions.dim() == 2 else directions[:, 0]).to(directions)
    emb = _appearance(sd, spec, directions, data)
    if emb is not None:
        dd = torch.cat([dd, emb], -1)
    out = {"rgb_sky": torch.sigmoid(skip_mlp(sd, "sky_head", dd))}
    if spec.enable_feature_head:
        out["dino_sky_feat"] = seq_mlp(sd, "dino_sky_head", dd, (0, 2, 4))
    return out


def radiance_field_forward(
    sd: SD, spec: FieldSpec, positions: Tensor, directions: Optional[Tensor] = None,
    data_dict: Optional[Dict[str, Tensor]] = None, *, training: bool,
    return_density_only: bool = False, combine_static_dynamic: bool = False,
    query_feature_head: bool = True, query_pe_head: bool = True,
    noise: Optional[Tensor] = None, rng_record: Optional[dict] = None,
) -> Dict[str, Tensor]:
    """RadianceField.forward, radiance_field.py:391-551."""
    data = data_dict or {}
    res: Dict[str, Tensor] = {}
    G, S_ = spec.geometry_feature_dim, spec.semantic_feature_dim
    normed = contract_points(positions, sd["aabb"], spec.unbounded)          # :302-318
    enc = encode(sd, "xyz_encoder", spec.geom("xyz"), normed)
    feats = seq_mlp(sd, "base_mlp", enc, (0, 2))
    geo, sem = torch.split(feats, [G, S_], dim=-1)
    sigma_s = density_activation(geo[..., 0])

    has_t = "normed_timestamps" in data or "lidar_normed_timestamps" in data
    dynamic_on = spec.dynamic is not None and has_t
    if dynamic_on:
        t = data["normed_timestamps"] if "normed_timestamps" in data else data["lidar_normed_timestamps"]
        dyn_feats, dyn_enc = _dynamic_hash(sd, spec, normed, t)
        if spec.flow is not None:
            flow = _flow_hash(sd, spec, normed, t)
            ff, bf = flow[..., :3], flow[..., 3:]
            res["forward_flow"], res["backward_flow"] = ff, bf
            if noise is None:
                if training:                                                  # :567-570
                    noise = torch.rand_like(ff)[..., 0:1]
                else:
                    noise = torch.ones_like(ff)[..., 0:1]
            if rng_record is not None:
                rng_record["noise"] = noise
            agg = _temporal_aggregation(sd, spec, positions, t, ff, bf, dyn_feats, noise)
            dyn_feats = agg["dynamic_feats"]
            agg["current_dynamic_hash_encodings"] = dyn_enc
            res.update(agg)
        dgeo, dsem = torch.split(dyn_feats, [G, S_], dim=-1)
        sigma_d = density_activation(dgeo[..., 0])
        sigma = sigma_s + sigma_d
        res.update({"density": sigma, "static_density": sigma_s, "dynamic_density": sigma_d})
        if return_density_only:
            return res
        if directions is not None:
            rgbs = _query_rgb(sd, spec, directions, geo, dgeo, data)
            res["dynamic_rgb"] = rgbs["dynamic_rgb"]
            res["static_rgb"] = rgbs["rgb"]
            if combine_static_dynamic:
                rs = sigma_s / (sigma + 1e-6)
                rd = sigma_d / (sigma + 1e-6)
                res["rgb"] = rs[..., None] * res["static_rgb"] + rd[..., None] * res["dynamic_rgb"]
        if spec.enable_shadow_head:
            shadow = torch.sigmoid(seq_mlp(sd, "shadow_head", dgeo, (0, 2)))
            res["shadow_ratio"] = shadow
            if combine_static_dynamic and "rgb" in res:
                res["rgb"] = rs[..., None] * res["rgb"] * (1 - shadow) + rd[..., None] * res["dynamic_rgb"]
    else:
        res["density"] = sigma_s
        if return_density_only:
            return res
        if directions is not None:
            res["rgb"] = _query_rgb(sd, spec, directions, geo, None, data)["rgb"]

    if spec.enable_feature_head and query_feature_head:                        # :508-538
        if spec.enable_learnable_pe and query_pe_head:
            pe = F.grid_sample(sd["learnable_pe_map"], data["pixel_coords"].reshape(1, 1, -1, 2) * 2 - 1,
                               align_corners=False, mode="bilinear")
            pe = pe.squeeze(2).squeeze(0).permute(1, 0)
            res["dino_pe"] = _lin(sd, "pe_head.0", pe)
        dino = seq_mlp(sd, "dino_head", sem, (0, 2, 4))
        if dynamic_on:
            ddino = seq_mlp(sd, "dino_head", dsem, (0, 2, 4))
            res["static_dino_feat"], res["dynamic_dino_feat"] = dino, ddino
            if combine_static_dynamic:
                rs = sigma_s / (sigma + 1e-6)
                rd = sigma_d / (sigma + 1e-6)
                res["dino_feat"] = rs[..., None] * dino + rd[..., None] * ddino
        else:
            res["dino_feat"] = dino

    if spec.enable_sky_head and "lidar_origin" not in data and directions is not None:   # :541-549
        d0 = directions[:, 0]
        red = {k: v[:, 0] for k, v in data.items()}
        res.update(_query_sky(sd, spec, d0, red))
    return res


# --------------------------------------------------------------------------- sampling
def _s_to_t(kind: str, s: Tensor, t_min: float, t_max: float) -> Tensor:
    """_transform_stot + TRANSFROM_DICT, nerfacc_prop_net.py:299-339."""
    fns = {
        "uniform": (lambda x: x, lambda x: x),
        "lindisp": (lambda x: 1 / x, lambda x: 1 / x),
        "sqrt": (lambda x: torch.sqrt(x), lambda x: x ** 2),
        "log": (lambda x: torch.log(x), lambda x: torch.exp(x)),
        "uniform_lindisp": (lambda x: torch.where(x < 200, x / 400, 1 - 1 / (2 * x / 200)),
                            lambda x: torch.where(x < 0.5, x * 400, 200 / (2 - 2 * x))),
        "uniform_lindisp_0": (lambda x: torch.where(x < 1, x / 2, 1 - 1 / (2 * x)),
                              lambda x: torch.where(x < 0.5, 2 * x, 1 / (2 - 2 * x))),
    }
    fwd, inv = fns[kind]
    s_min, s_max = fwd(torch.tensor(float(t_min))), fwd(torch.tensor(float(t_max)))
    return inv(s * s_max + (1 - s) * s_min)


def s_bounds(kind: str, t_min: float, t_max: float) -> Tuple[float, float]:
    """fp32 (s_min, s_max) exactly as _transform_stot computes them."""
    lo = _s_inv_probe(kind, t_min)
    hi = _s_inv_probe(kind, t_max)
    return float(lo), float(hi)


def _s_inv_probe(kind, t):
    x = torch.tensor(float(t))
    if kind == "uniform":
        return x
    if kind == "lindisp":
        return 1 / x
    if kind == "sqrt":
        return torch.sqrt(x)
    if kind == "log":
        return torch.log(x)
    if kind == "uniform_lindisp":
        return torch.where(x < 200, x / 400, 1 - 1 / (2 * x / 200))
    if kind == "uniform_lindisp_0":
        return torch.where(x < 1, x / 2, 1 - 1 / (2 * x))
    raise ValueError(kind)


def sampling(
    prop_sigma_fns: List[Callable], prop_samples: List[int], num_samples: int, n_rays: int,
    near_plane: float, far_plane: float, sampling_type: str = "uniform_lindisp",
    stratified: bool = False, requires_grad: bool = False,
    jitters: Optional[List[Tensor]] = None, rng_record: Optional[dict] = None,
):
    """PropNetEstimator.sampling, nerfacc_prop_net.py:89-179.  Returns (t_starts, t_ends, cache);
    ``cache`` is the prop_cache list the reference keeps on the estimator."""
    cache: list = []
    used_jitters: List[Tensor] = []
    with torch.no_grad():
        cdfs = torch.cat([torch.zeros((n_rays, 1)), torch.ones((n_rays, 1))], dim=-1)
        intervals = nf.RayIntervals(vals=cdfs)

        def resample(intervals, cdfs, n, level):
            j = None
            if stratified:
                j = jitters[level] if jitters is not None else torch.rand(n_rays, 1)
                used_jitters.append(j)
            out, _ = nf.importance_sampling(intervals, cdfs, n, stratified, jitter=j)
            return out

        for i, (fn, n) in enumerate(zip(prop_sigma_fns, prop_samples)):
            intervals = resample(intervals, cdfs, n, i)
            t_vals = _s_to_t(sampling_type, intervals.vals, near_plane, far_plane)
            t0, t1 = t_vals[..., :-1], t_vals[..., 1:]
            with torch.set_grad_enabled(requires_grad):
                sig = fn(t0, t1)["density"].squeeze(-1)
                trans, _ = nf.render_transmittance_from_density(t0, t1, sig)
                cdfs = 1.0 - torch.cat([trans, torch.zeros_like(trans[..., :1])], dim=-1)
                if requires_grad:
                    cache.append((intervals, cdfs, i))
        intervals = resample(intervals, cdfs, num_samples, len(prop_samples))
        t_vals = _s_to_t(sampling_type, intervals.vals, near_plane, far_plane)
        if requires_grad:
            cache.append((intervals, None, None))
    if rng_record is not None:
        rng_record["jitters"] = used_jitters
    return t_vals[..., :-1], t_vals[..., 1:], cache


def blur_stepfun(x, y, r):
    """nerfacc_prop_net.py:22-34."""
    xr, xr_idx = torch.sort(torch.cat([x - r, x + r], dim=-1))
    y1 = (torch.cat([y, torch.zeros_like(y[..., :1])], dim=-1)
          - torch.cat([torch.zeros_like(y[..., :1]), y], dim=-1)) / (2 * r)
    y2 = torch.cat([y1, -y1], dim=-1).take_along_dim(xr_idx[..., :-1], dim=-1)
    yr = torch.cumsum((xr[..., 1:] - xr[..., :-1]) * torch.cumsum(y2, dim=-1), dim=-1).clamp_min(0)
    yr = torch.cat([torch.zeros_like(yr[..., :1]), yr], dim=-1)
    return xr, yr


def sorted_interp_quad(x, xp, fpdf, fcdf):
    """nerfacc_prop_net.py:37-60."""
    mask = x[..., None, :] >= xp[..., :, None]

    def find(v, idx=False):
        v0, i0 = torch.max(torch.where(mask, v[..., None], v[..., :1, None]), -2)
        v1, i1 = torch.min(torch.where(~mask, v[..., None], v[..., -1:, None]), -2)
        return (v0, v1, i0, i1) if idx else (v0, v1)

    c0, c1, i0, i1 = find(fcdf, True)
    p0 = fpdf.take_along_dim(i0, dim=-1)
    p1 = fpdf.take_along_dim(i1, dim=-1)
    x0, x1 = find(xp)
    off = torch.clip(torch.nan_to_num((x - x0) / (x1 - x0), 0), 0, 1)
    return c0 + (x - x0) * (p0 + p1 * off + p0 * (1 - off)) / 2


def proposal_loss(cache: list, trans: Tensor, pulse_width=(0.03, 0.003), loss_scaler: float = 1.0,
                  enable_anti_aliasing_loss: bool = True) -> Tensor:
    """PropNetEstimator.compute_loss, nerfacc_prop_net.py:181-238 (consumes ``cache``)."""
    if len(cache) == 0:
        return torch.zeros(())
    cache = list(cache)
    intervals, _, _ = cache.pop()
    cdfs = (1.0 - torch.cat([trans, torch.zeros_like(trans[..., :1])], dim=-1)).detach()
    loss = 0.0
    if enable_anti_aliasing_loss:
        w_n = (cdfs[..., 1:] - cdfs[..., :-1]) / (intervals.vals[..., 1:] - intervals.vals[..., :-1])
        cs, ws, cds = [], [], []
        for r in pulse_width:
            c, w = blur_stepfun(intervals.vals, w_n, r)
            area = 0.5 * (w[..., 1:] + w[..., :-1]) * (c[..., 1:] - c[..., :-1])
            cs.append(c)
            ws.append(w)
            cds.append(torch.cat([torch.zeros_like(area[..., :1]), torch.cumsum(area, dim=-1)], dim=-1))
        while cache:
            p_int, p_cdfs, pid = cache.pop()
            wp = p_cdfs[..., 1:] - p_cdfs[..., :-1]
            interp = sorted_interp_quad(p_int.vals, cs[pid], ws[pid], cds[pid])
            w_s = torch.diff(interp, dim=-1)
            loss = loss + ((w_s - wp).clamp_min(0) ** 2 / (wp + 1e-5)).mean()
    else:
        while cache:
            p_int, p_cdfs, _ = cache.pop()
            loss = loss + _pdf_loss(intervals, cdfs, p_int, p_cdfs).mean()
    return loss * loss_scaler


def _pdf_loss(seg_q, cdfs_q, seg_k, cdfs_k, eps: float = 1e-7):
    """nerfacc_prop_net.py:342-362, batched branch."""
    il, ir = nf.searchsorted(seg_k, seg_q)
    w = cdfs_q[..., 1:] - cdfs_q[..., :-1]
    il, ir = il[..., :-1], ir[..., 1:]
    w_outer = cdfs_k.gather(-1, ir) - cdfs_k.gather(-1, il)
    return torch.clip(w - w_outer, min=0) ** 2 / (w + eps)


# --------------------------------------------------------------------------- rendering
def _wod(t0, t1, sigma):
    """render_weights_opacity_depth_from_density, render_utils.py:19-45."""
    w, _, _ = nf.render_weight_from_density(t0, t1, sigma)
    op = nf.accumulate_along_rays(w, None).clamp(1e-6, 1.0)
    dep = nf.accumulate_along_rays(w, (t0 + t1)[..., None] / 2.0) / op
    return w, op, dep


def rendering(t0: Tensor, t1: Tensor, results: Dict[str, Tensor], return_decomposition: bool = False):
    """rendering, render_utils.py:48-287 (``results`` = what query_fn returned)."""
    acc = nf.accumulate_along_rays
    trans, alphas = nf.render_transmittance_from_density(t0, t1, results["density"].squeeze(-1))
    weights = trans * alphas
    extras = {"weights": weights, "trans": trans, "t_vals": (t0 + t1) / 2.0, "t_dist": (t1 - t0)}
    for k in ("forward_flow", "backward_flow", "forward_pred_backward_flow", "backward_pred_forward_flow"):
        if k in results:
            extras[k] = results[k]
    opac = acc(weights, None).clamp(1e-6, 1.0)
    steps = (t0 + t1)[..., None] / 2.0
    depth = acc(weights, steps) / opac
    cw = torch.cumsum(weights, dim=-1)
    split = torch.ones((*weights.shape[:-1], 1)) * 0.5
    mi = torch.clamp(torch.searchsorted(cw, split, side="left"), 0, steps.shape[-2] - 1)
    median = torch.gather(steps[..., 0], dim=-1, index=mi)
    out = {"density": results["density"].squeeze(-1), "depth": depth, "opacity": opac, "median_depth": median}

    two = "static_density" in results and "dynamic_density" in results
    if two:
        extras["static_density"] = results["static_density"]
        extras["dynamic_density"] = results["dynamic_density"]
        rs = results["static_density"] / (results["density"] + 1e-6)
        rd = results["dynamic_density"] / (results["density"] + 1e-6)
        if return_decomposition:
            sw, out["static_opacity"], out["static_depth"] = _wod(t0, t1, results["static_density"])
            dw, out["dynamic_opacity"], out["dynamic_depth"] = _wod(t0, t1, results["dynamic_density"])

    if "rgb" in results:
        out["rgb"] = acc(weights, results["rgb"])
    elif "static_rgb" in results and "dynamic_rgb" in results:
        shadow = 0.0
        if "shadow_ratio" in results:
            shadow = results["shadow_ratio"]
            out["shadow_ratio"] = acc(weights, shadow.square())
        rgb = rs[..., None] * results["static_rgb"] * (1 - shadow) + rd[..., None] * results["dynamic_rgb"]
        out["rgb"] = acc(weights, rgb)
        if return_decomposition:
            out["static_rgb"] = acc(sw, results["static_rgb"])
            if "shadow_ratio" in results:
                out["shadow_reduced_static_rgb"] = acc(sw, results["static_rgb"] * (1 - shadow))
                so = acc(sw, results["static_rgb"] * shadow)
                out["shadow_only_static_rgb"] = so + (1 - acc(weights, shadow))
                out["shadow"] = acc(weights, shadow)
            out["dynamic_rgb"] = acc(dw, results["dynamic_rgb"])
            if "forward_flow" in results:
                out["forward_flow"] = acc(dw, results["forward_flow"])
                out["backward_flow"] = acc(dw, results["backward_flow"])

    if "rgb_sky" in results:
        out["rgb"] = out["rgb"] + results["rgb_sky"] * (1.0 - out["opacity"])
        if "static_rgb" in out:
            out["static_rgb"] = out["static_rgb"] + results["rgb_sky"] * (1.0 - out["static_opacity"])

    def finish_dino():
        if "dino_sky_feat" in results:
            out["dino_feat"] = out["dino_feat"] + results["dino_sky_feat"] * (1.0 - out["opacity"])
        if "dino_pe" in results:
            out["dino_pe_free"] = out["dino_feat"].clone()
            out["dino_pe"] = results["dino_pe"]
            out["dino_feat"] = out["dino_feat"] + results["dino_pe"]

    if "dino_feat" in results:
        out["dino_feat"] = acc(weights, results["dino_feat"])
        finish_dino()
    elif "static_dino_feat" in results and "dynamic_dino_feat" in results:
        df = rs[..., None] * results["static_dino_feat"] + rd[..., None] * results["dynamic_dino_feat"]
        out["dino_feat"] = acc(weights, df)
        finish_dino()
        if return_decomposition:
            out["static_dino"] = acc(sw, results["static_dino_feat"])
            out["dynamic_dino"] = acc(dw, results["dynamic_dino_feat"])
            if "dino_sky_feat" in results:
                out["static_dino"] = out["static_dino"] + results["dino_sky_feat"] * (1.0 - out["opacity"])
    out["extras"] = extras
    return out


def render_rays(
    field_sd: SD, field_spec: FieldSpec, prop_sds: List[SD], prop_specs: List[FieldSpec],
    data_dict: Dict[str, Tensor], *, num_samples: int, prop_samples: List[int],
    near_plane: float, far_plane: float, sampling_type: str = "uniform_lindisp",
    training: bool, proposal_requires_grad: bool = False, return_decomposition: bool = False,
    prefix: str = "", render_chunk_size: int = 16384,
    jitters: Optional[List[Tensor]] = None, noise: Optional[Tensor] = None,
    rng_record: Optional[dict] = None, prop_sigma_scale: float = 1.0,
):
    """render_rays, render_utils.py:290-389.  Returns (render_results, prop_cache).

    ``prop_sigma_scale`` (not in the reference; 1.0 = the reference's arithmetic) multiplies the proposal densities:
    the parity tests use 1 +- 1e-6 to measure how far a last-bit difference in the proposal CDFs moves each ray's
    samples (inverse-CDF resampling is ill-conditioned where a CDF is flat), see :func:`sample_stability`."""
    shape = data_dict[prefix + "origins"].shape
    if len(shape) == 3:
        n_rays = shape[0] * shape[1]
        flat = {k: v.reshape(n_rays, -1).squeeze() for k, v in data_dict.items()}
    else:
        n_rays = shape[0]
        flat = dict(data_dict)

    results, cache, extras = [], [], None
    chunk = 2 ** 24 if training else render_chunk_size
    for i in range(0, n_rays, chunk):
        cd = {k: v[i:i + chunk] for k, v in flat.items()}
        o = cd[prefix + "origins"][..., None, :]

        def prop_fn(t0, t1, j):
            d = cd[prefix + "viewdirs"][..., None, :]
            pos = o + d * (t0 + t1)[..., None] / 2.0
            res = density_field_forward(prop_sds[j], prop_specs[j], pos)
            if prop_sigma_scale != 1.0:
                res = {"density": res["density"] * prop_sigma_scale}
            return res

        def query_fn(t0, t1):
            S = t0.shape[-1]
            d = cd[prefix + "viewdirs"][..., None, :].repeat_interleave(S, dim=-2)
            sub = {k: v[..., None].repeat_interleave(S, dim=-1) for k, v in cd.items()
                   if k not in (prefix + "viewdirs", prefix + "origins", "pixel_coords")}
            sub["t_starts"], sub["t_ends"] = t0, t1
            if "pixel_coords" in cd:
                sub["pixel_coords"] = cd["pixel_coords"]
            pos = o + d * (t0 + t1)[..., None] / 2.0
            r = radiance_field_forward(field_sd, field_spec, pos, d, sub, training=training,
                                       return_density_only=(prefix == "lidar_"), noise=noise,
                                       rng_record=rng_record)
            r["density"] = r["density"].squeeze(-1)
            return r

        t0, t1, c = sampling(
            # Q21 (reference quirk): render_utils.py:357-359 builds
            #   [lambda *args: prop_sigma_fn(*args, p) for p in proposal_networks]
            # whose lambdas all close over the comprehension variable `p` (late binding), so EVERY
            # level is evaluated with the LAST proposal network; networks 0..n-2 are never used.
            [lambda a, b: prop_fn(a, b, len(prop_sds) - 1) for _ in range(len(prop_sds))],
            prop_samples, num_samples, cd[prefix + "origins"].shape[0], near_plane, far_plane,
            sampling_type, stratified=training, requires_grad=proposal_requires_grad,
            jitters=jitters, rng_record=rng_record)
        cache.extend(c)
        out = rendering(t0, t1, query_fn(t0, t1), return_decomposition)
        extras = out.pop("extras")
        results.append(out)
    merged = {k: torch.cat([r[k] for r in results], 0) for k in results[0]}
    extras["density"] = merged.pop("density")
    for k, v in merged.items():
        merged[k] = v.reshape(list(shape[:-1]) + list(v.shape[1:]))
    merged["extras"] = extras
    return merged, cache


def sample_stability(render, base_t_vals: Tensor, eps: Sequence[float] = (2e-6, -2e-6, 1e-6, -1e-6, 3e-7, -3e-7, 1e-7, -1e-7),
                     threshold: float = 1e-5) -> Tensor:
    """Which rays have WELL-CONDITIONED samples.  ``render(scale)`` renders with the proposal densities multiplied by
    ``scale`` (``render_rays(..., prop_sigma_scale=scale)``) and returns its results; a ray is stable when none of the
    1 + eps probes -- differences of the size of one expf / summation-order ulp in the proposal CDFs, which no two
    implementations (this oracle, tiny-cuda-nn + nerfacc on a GPU, this repository's kernels) share -- moves any of
    its final sample midpoints by more than ``threshold`` relative.  Where a proposal CDF is flat (transmittance
    already ~0, or empty space), the inverse-CDF resampling amplifies such a difference by orders of magnitude, and
    per-sample quantities and expected depth of that ray are not comparable across implementations.  [R] bool."""
    worst = torch.zeros(base_t_vals.shape[0])
    for e in eps:
        t = render(1.0 + e)["extras"]["t_vals"]
        worst = torch.maximum(worst, ((t - base_t_vals).abs() / base_t_vals.abs()).amax(dim=-1))
    return worst <= threshold

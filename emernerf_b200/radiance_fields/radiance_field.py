"""``RadianceField`` / ``DensityField`` with the reference's constructor arguments, attribute names,
state-dict keys and ``forward`` contracts (radiance_fields/radiance_field.py of NVlabs/EmerNeRF),
evaluated on the sm_90a kernels of libemer_b200.so:

  contract + selector  -> emer_contract_*      (radiance_field.py:278-300,828-835)
  hash grids           -> emer_grid_*          (:314,341,376,836)
  every nn.Linear      -> emer_linear_*        (:74-198,808-812), bias/ReLU/sigmoid fused
  trunc_exp(x - 1)     -> emer_trunc_exp_*     (:28,794)

The ``nn.Sequential`` / ``MLP`` containers exist to own the parameters under the reference's
names (``base_mlp.0.weight`` ...); they are never called as torch modules.
"""
from __future__ import annotations

import logging
from typing import Callable, Dict, List, Literal, Optional, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor

from .. import _ops
from .encodings import HashEncoder, SinusoidalEncoder, build_xyz_encoder_from_cfg
from .mlp import MLP, run_sequential
from .nerf_utils import trunc_exp

logger = logging.getLogger()


def _stack(*widths: int, final: Optional[nn.Module] = None) -> nn.Sequential:
    """Linear/ReLU/.../Linear container: Linear modules land on even indices (0, 2, 4)."""
    mods: List[nn.Module] = []
    for i in range(len(widths) - 1):
        mods.append(nn.Linear(widths[i], widths[i + 1]))
        if i < len(widths) - 2:
            mods.append(nn.ReLU())
    if final is not None:
        mods.append(final)
    return nn.Sequential(*mods)


def _default_density_activation(x: Tensor) -> Tensor:
    return trunc_exp(x - 1)


def _as_aabb(aabb) -> Tensor:
    return aabb if isinstance(aabb, Tensor) else torch.tensor(aabb, dtype=torch.float32)


def _contract_points(positions: Tensor, aabb: Tensor, unbounded: bool) -> Tensor:
    """[..., 3] world -> [..., 3] grid coordinates; points outside (0,1)^3 are sent to the origin
    (the reference multiplies by a 0/1 selector, it does not skip them -- SURVEY.md Q2)."""
    shape = positions.shape
    out = _ops.contract(positions.reshape(-1, 3), aabb, None, unbounded)
    return out.view(shape)


class RadianceField(nn.Module):
    def __init__(
        self,
        xyz_encoder: HashEncoder,
        dynamic_xyz_encoder: Optional[HashEncoder] = None,
        flow_xyz_encoder: Optional[HashEncoder] = None,
        aabb: Union[Tensor, List[float]] = [-1, -1, -1, 1, 1, 1],
        num_dims: int = 3,
        density_activation: Callable = _default_density_activation,
        unbounded: bool = True,
        geometry_feature_dim: int = 15,
        base_mlp_layer_width: int = 64,
        head_mlp_layer_width: int = 64,
        enable_cam_embedding: bool = False,
        enable_img_embedding: bool = False,
        num_cams: int = 3,
        appearance_embedding_dim: int = 16,
        semantic_feature_dim: int = 64,
        feature_mlp_layer_width: int = 256,
        feature_embedding_dim: int = 768,
        enable_sky_head: bool = False,
        enable_shadow_head: bool = False,
        enable_feature_head: bool = False,
        num_train_timesteps: int = 0,
        interpolate_xyz_encoding: bool = False,
        enable_learnable_pe: bool = True,
        enable_temporal_interpolation: bool = False,
    ) -> None:
        super().__init__()
        self.register_buffer("aabb", _as_aabb(aabb))
        self.unbounded = unbounded
        self.num_cams = num_cams
        self.num_dims = num_dims
        self.density_activation = density_activation
        self._fused_density = density_activation is _default_density_activation

        self.enable_cam_embedding = enable_cam_embedding
        self.enable_img_embedding = enable_img_embedding
        self.appearance_embedding_dim = appearance_embedding_dim
        self.geometry_feature_dim = geometry_feature_dim
        self.semantic_feature_dim = semantic_feature_dim if enable_feature_head else 0
        feat_out = self.geometry_feature_dim + self.semantic_feature_dim
        W = base_mlp_layer_width

        # static field
        self.xyz_encoder = xyz_encoder
        self.base_mlp = _stack(xyz_encoder.n_output_dims, W, feat_out)

        # dynamic field (4-D grid over xyz + t)
        self.interpolate_xyz_encoding = interpolate_xyz_encoding
        self.dynamic_xyz_encoder = dynamic_xyz_encoder
        self.enable_temporal_interpolation = enable_temporal_interpolation
        if dynamic_xyz_encoder is not None:
            self.register_buffer("training_timesteps", torch.zeros(num_train_timesteps))
            self.dynamic_base_mlp = _stack(dynamic_xyz_encoder.n_output_dims, W, feat_out)

        # flow field: 3 forward + 3 backward components, no output activation
        self.flow_xyz_encoder = flow_xyz_encoder
        if flow_xyz_encoder is not None:
            self.flow_mlp = _stack(flow_xyz_encoder.n_output_dims, W, W, 6)

        if enable_cam_embedding:
            self.appearance_embedding = nn.Embedding(num_cams, appearance_embedding_dim)
        elif enable_img_embedding:
            self.appearance_embedding = nn.Embedding(num_train_timesteps * num_cams, appearance_embedding_dim)
        else:
            self.appearance_embedding = None
        emb_dim = appearance_embedding_dim if (enable_cam_embedding or enable_img_embedding) else 0

        self.direction_encoding = SinusoidalEncoder(n_input_dims=3, min_deg=0, max_deg=4)
        dir_dim = self.direction_encoding.n_output_dims

        self.rgb_head = MLP(in_dims=geometry_feature_dim + dir_dim + emb_dim, out_dims=3, num_layers=3,
                            hidden_dims=head_mlp_layer_width, skip_connections=[1])

        self.enable_shadow_head = enable_shadow_head
        if enable_shadow_head:
            self.shadow_head = _stack(geometry_feature_dim, W, 1, final=nn.Sigmoid())

        self.enable_sky_head = enable_sky_head
        if enable_sky_head:
            self.sky_head = MLP(in_dims=dir_dim + emb_dim, out_dims=3, num_layers=3,
                                hidden_dims=head_mlp_layer_width, skip_connections=[1])
            if enable_feature_head:
                self.dino_sky_head = _stack(dir_dim + emb_dim, feature_mlp_layer_width, feature_mlp_layer_width,
                                            feature_embedding_dim)

        self.enable_feature_head = enable_feature_head
        if enable_feature_head:
            self.dino_head = _stack(semantic_feature_dim, feature_mlp_layer_width, feature_mlp_layer_width,
                                    feature_embedding_dim)
            self.register_buffer("feats_reduction_mat", torch.zeros(feature_embedding_dim, 3))
            self.register_buffer("feat_color_min", torch.zeros(3, dtype=torch.float32))
            self.register_buffer("feat_color_max", torch.ones(3, dtype=torch.float32))
            self.enable_learnable_pe = enable_learnable_pe
            if enable_learnable_pe:
                self.learnable_pe_map = nn.Parameter(0.05 * torch.randn(1, feature_embedding_dim // 2, 80, 120),
                                                     requires_grad=True)
                self.pe_head = nn.Sequential(nn.Linear(feature_embedding_dim // 2, feature_embedding_dim))

        # test hook: fixed temporal-aggregation noise instead of torch.rand_like (parity runs)
        self._noise_override: Optional[Tensor] = None

    # ------------------------------------------------------------------ registration helpers
    def register_normalized_training_timesteps(self, normalized_timesteps: Tensor, time_diff: float = None) -> None:
        if self.dynamic_xyz_encoder is None:
            return
        self.training_timesteps.copy_(normalized_timesteps)
        self.training_timesteps = self.training_timesteps.to(self.device)
        if time_diff is not None:
            self.time_diff = time_diff
        elif len(self.training_timesteps) > 1:
            self.time_diff = self.training_timesteps[1] - self.training_timesteps[0]
        else:
            self.time_diff = 0

    def set_aabb(self, aabb: Union[Tensor, List[float]]) -> None:
        aabb = _as_aabb(aabb)
        logger.info(f"Set aabb from {self.aabb} to {aabb}")
        self.aabb.copy_(aabb)
        self.aabb = self.aabb.to(self.device)

    def register_feats_reduction_mat(self, feats_reduction_mat: Tensor, feat_color_min: Tensor,
                                     feat_color_max: Tensor) -> None:
        for name, src in (("feats_reduction_mat", feats_reduction_mat), ("feat_color_min", feat_color_min),
                          ("feat_color_max", feat_color_max)):
            buf = getattr(self, name)
            buf.copy_(src)
            setattr(self, name, buf.to(self.device))

    @property
    def device(self) -> torch.device:
        return self.aabb.device

    # ------------------------------------------------------------------ fused field tail
    def _tail_inputs(self, directions, data_dict):
        """(dirs [R,3], idx [R] | None, emb weight | None) when the fused tail applies: default density
        activation, per-ray view directions / embedding indices handed over as stride-0 per-sample views
        (what render_rays builds), CUDA tensors.  None -> the general per-point path."""
        if not (self._fused_density and directions is not None and _ops.on_device(directions) and directions.dim() == 3
                and directions.stride(1) == 0 and self.geometry_feature_dim % 4 == 0):
            return None                                   # (the fused kernel moves 16-byte pieces of the features)
        idx = emb = None
        if self.enable_cam_embedding or self.enable_img_embedding:
            if "cam_idx" in data_dict and self.enable_cam_embedding:
                t = data_dict["cam_idx"]
            elif "img_idx" in data_dict and self.enable_img_embedding:
                t = data_dict["img_idx"]
            else:
                return None                               # mean-embedding case: general path
            if not (t.dim() == 2 and t.stride(1) == 0) or self.appearance_embedding_dim > 32:
                return None
            idx, emb = t[:, 0], self.appearance_embedding.weight
        return directions[:, 0], idx, emb

    def _field_tail(self, feats: Tensor, tail) -> Tuple[Tensor, Tuple[Tensor, Tensor]]:
        """density and the colour head's input; the input rows are laid out behind ``front`` spare columns so
        that they already are the [hidden | input] skip concatenation of the head's second layer."""
        front = self.rgb_head.layers[0].out_features
        if front % 4 or len(self.rgb_head.layers) < 2:
            front = 0
        res = _ops.field_tail(feats, *tail, self.geometry_feature_dim, front=front)
        return res[0], (res[1], res[2] if front else None)

    def _rgb_from_tail(self, tail_out: Tuple[Tensor, Optional[Tensor]]) -> Tensor:
        """rgb head on a [geo | dir | emb] input: the reference order is [dir | emb | geo]
        (radiance_field.py:647), so the weight columns that multiply the input are permuted."""
        rgb_in, catbuf = tail_out
        G = self.geometry_feature_dim
        tail = rgb_in.shape[-1] - G
        key = (G, tail, str(rgb_in.device))
        if getattr(self, "_perm_key", None) != key:
            perm = torch.cat([torch.arange(tail, tail + G), torch.arange(0, tail)]).to(rgb_in.device)
            hid = self.rgb_head.layers[1].weight.shape[1] - (tail + G)
            self._perm0 = perm
            self._perm1 = torch.cat([torch.arange(hid, device=rgb_in.device), hid + perm])
            self._perm_key = key
        l0, l1, l2 = self.rgb_head.layers
        return _ops.mlp_chain(rgb_in, [l0.weight[:, self._perm0], l1.weight[:, self._perm1], l2.weight],
                              [l0.bias, l1.bias, l2.bias], _ops.ACT_SIGMOID, 1, catbuf=catbuf)

    # ------------------------------------------------------------------ fused chain
    def _chain_usable(self, encoder: HashEncoder, base: nn.Sequential) -> bool:
        lin = [m for m in base if isinstance(m, nn.Linear)]
        if len(lin) != 2 or len(self.rgb_head.layers) != 3 or self.rgb_head.skip_connections != [1]:
            return False
        head = [(l.out_features, l.in_features) for l in self.rgb_head.layers]
        return (self.geometry_feature_dim == 64 and lin[0].in_features == encoder.n_output_dims
                and lin[1].in_features == lin[0].out_features
                and _ops.field_chain_usable(encoder.n_output_dims, lin[1].out_features, lin[0].out_features, head))

    def _ray_bias(self, tail) -> Tensor:
        """[R, 128]: what the per-ray input columns of the colour head -- direction encoding and appearance embedding,
        the same for every sample of a ray -- contribute to its first two layers, biases included:
        [b0 + W0[:, :c] v | b1 + W1[:, 64:64+c] v] with v = [sinenc((d+1)/2) | emb[idx]] (radiance_field.py:629-647;
        W1's input is [hidden | v | geo], mlp.py:42-43).  8192 rows instead of 524 288."""
        dirs, idx, emb = tail
        v = self.direction_encoding((dirs + 1.0) / 2.0)
        if emb is not None:
            v = torch.cat([v, _ops.gather_rows(emb, idx)], dim=-1)
        c = v.shape[-1]
        l0, l1, _ = self.rgb_head.layers
        h = l0.out_features
        w = torch.cat([l0.weight[:, :c], l1.weight[:, h:h + c]], dim=0)
        return _ops.linear(_ops.cat_pad4([v]), w, torch.cat([l0.bias, l1.bias]))

    def _chain_params(self, base: nn.Sequential):
        """(base, head) parameter tuples of the fused chains: the base MLP's two nn.Linear layers, (wb0, bb0, wb1, bb1),
        and the colour head's three layers, (w0, w1, w2, b2)."""
        lin = [m for m in base if isinstance(m, nn.Linear)]
        l0, l1, l2 = self.rgb_head.layers
        return (lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias), (l0.weight, l1.weight, l2.weight, l2.bias)

    def _run_chain(self, encoder: HashEncoder, base: nn.Sequential, coords: Tensor, ray_bias: Tensor,
                   want_geo: bool = False):
        """(density [R,S], rgb [R,S,3], geo [R,S,64] | None, sem [R,S,64] | None) for grid coordinates [R,S,D]."""
        r, s_ = coords.shape[:2]
        enc = encoder(coords.reshape(-1, coords.shape[-1]))
        sigma, rgb, geo, sem = _ops.field_chain(enc, ray_bias, s_, *self._chain_params(base), want_geo=want_geo)
        return (sigma.view(r, s_), rgb.view(r, s_, 3), None if geo is None else geo.view(r, s_, -1),
                None if sem is None else sem.view(r, s_, -1))

    # ------------------------------------------------------------------ building blocks
    def contract_points(self, positions: Tensor) -> Tensor:
        return _contract_points(positions, self.aabb, self.unbounded)

    def _density(self, feats: Tensor) -> Tensor:
        """density_activation(feats[..., 0]); the default trunc_exp(x-1) is one fused kernel."""
        raw = feats[..., 0]
        return _ops.density_activation(raw) if self._fused_density else self.density_activation(raw)

    def _encode_mlp(self, encoder: HashEncoder, mlp: nn.Sequential, coords: Tensor):
        lead = coords.shape[:-1]
        enc = encoder(coords.reshape(-1, coords.shape[-1]))
        out = run_sequential(mlp, enc)
        return out.view(*lead, -1), enc.view(*lead, -1)

    def forward_static_hash(self, positions: Tensor) -> Tuple[Tensor, Tensor]:
        normed = self.contract_points(positions)
        feats, _ = self._encode_mlp(self.xyz_encoder, self.base_mlp, normed)
        return feats, normed

    def _space_time(self, normed_positions: Tensor, normed_timestamps: Tensor) -> Tensor:
        if normed_timestamps.shape[-1] != 1:
            normed_timestamps = normed_timestamps.unsqueeze(-1)
        return torch.cat([normed_positions, normed_timestamps.to(normed_positions.dtype)], dim=-1)

    def forward_dynamic_hash(self, normed_positions: Tensor, normed_timestamps: Tensor,
                             return_hash_encodings: bool = False):
        # the reference hard-wires the non-interpolated branch (`if True`, radiance_field.py:337)
        feats, enc = self._encode_mlp(self.dynamic_xyz_encoder, self.dynamic_base_mlp,
                                      self._space_time(normed_positions, normed_timestamps))
        return (feats, enc) if return_hash_encodings else feats

    def forward_flow_hash(self, normed_positions: Tensor, normed_timestamps: Tensor) -> Tensor:
        if not self.training and self.enable_temporal_interpolation:
            raise NotImplementedError("temporal interpolation of the flow field is disabled in every shipped "
                                      "config (default_config.yaml:103) and is not implemented")
        flow, _ = self._encode_mlp(self.flow_xyz_encoder, self.flow_mlp,
                                   self._space_time(normed_positions, normed_timestamps))
        return flow

    # ------------------------------------------------------------------ forward
    def _has_time(self, data_dict) -> bool:
        return "normed_timestamps" in data_dict or "lidar_normed_timestamps" in data_dict

    def forward(
        self,
        positions: Tensor,
        directions: Tensor = None,
        data_dict: Dict[str, Tensor] = {},
        return_density_only: bool = False,
        combine_static_dynamic: bool = False,
        query_feature_head: bool = True,
        query_pe_head: bool = True,
    ) -> Dict[str, Tensor]:
        out: Dict[str, Tensor] = {}
        _ops.join_before_field()               # (multi-GPU: a parameter all-gather may still be running beside the sampling)
        G, S = self.geometry_feature_dim, self.semantic_feature_dim
        tail = None if (return_density_only or positions.dim() != 3) else self._tail_inputs(directions, data_dict)
        # the fused chain (base MLP + density + colour head in one wgmma kernel) when the model has its shape
        chain = tail is not None and self._chain_usable(self.xyz_encoder, self.base_mlp)
        rgb_in_static = static_rgb = None
        if chain:
            ray_bias = self._ray_bias(tail)
            normed = self.contract_points(positions)
            static_density, static_rgb, _, sem = self._run_chain(self.xyz_encoder, self.base_mlp, normed, ray_bias)
        else:
            feats, normed = self.forward_static_hash(positions)
            geo, sem = feats[..., :G], feats[..., G:G + S]
            if tail is not None:
                static_density, rgb_in_static = self._field_tail(feats, tail)
            else:
                static_density = self._density(feats)

        dynamic_on = self.dynamic_xyz_encoder is not None and self._has_time(data_dict)
        if dynamic_on:
            t = data_dict["normed_timestamps"] if "normed_timestamps" in data_dict \
                else data_dict["lidar_normed_timestamps"]
            dynamic_rgb = None
            if chain and self.flow_xyz_encoder is None and self._chain_usable(self.dynamic_xyz_encoder,
                                                                              self.dynamic_base_mlp):
                # no temporal aggregation between the base MLP and the head: the dynamic branch is one chain too
                dynamic_density, dynamic_rgb, dyn_geo, dyn_sem = self._run_chain(
                    self.dynamic_xyz_encoder, self.dynamic_base_mlp, self._space_time(normed, t), ray_bias,
                    want_geo=self.enable_shadow_head)
            elif self._flow_branch_usable(positions, chain, return_density_only):
                # EMER_FLOW_BRANCH=fused: the temporal aggregation inside the three-query chain
                dynamic_density, dynamic_rgb, dyn_geo, dyn_sem, flow_out = self._flow_branch(
                    positions, normed, t, ray_bias if chain else None)
                out.update(flow_out)
            else:
                dyn_feats, dyn_enc = self.forward_dynamic_hash(normed, t, return_hash_encodings=True)
                if self.flow_xyz_encoder is not None:
                    flow = self.forward_flow_hash(normed, t)
                    fwd, bwd = flow[..., :3], flow[..., 3:]
                    out["forward_flow"], out["backward_flow"] = fwd, bwd
                    agg = self.temporal_aggregation(positions, t, fwd, bwd, dyn_feats)
                    dyn_feats = agg["dynamic_feats"]
                    agg["current_dynamic_hash_encodings"] = dyn_enc
                    out.update(agg)
                dyn_geo, dyn_sem = dyn_feats[..., :G], dyn_feats[..., G:G + S]
                if tail is not None:
                    dynamic_density, rgb_in_dynamic = self._field_tail(dyn_feats, tail)
                else:
                    dynamic_density = self._density(dyn_feats)
            density = static_density + dynamic_density
            out.update(density=density, static_density=static_density, dynamic_density=dynamic_density)
            if return_density_only:
                return out
            if tail is not None:
                out["dynamic_rgb"] = dynamic_rgb if dynamic_rgb is not None else self._rgb_from_tail(rgb_in_dynamic)
                out["static_rgb"] = static_rgb if static_rgb is not None else self._rgb_from_tail(rgb_in_static)
            elif directions is not None:
                colours = self.query_rgb(directions, geo, dyn_geo, data_dict=data_dict)
                out["dynamic_rgb"] = colours["dynamic_rgb"]
                out["static_rgb"] = colours["rgb"]
            if "static_rgb" in out and combine_static_dynamic:
                s_ratio = static_density / (density + 1e-6)
                d_ratio = dynamic_density / (density + 1e-6)
                out["rgb"] = s_ratio[..., None] * out["static_rgb"] + d_ratio[..., None] * out["dynamic_rgb"]
            if self.enable_shadow_head:
                shadow = run_sequential(self.shadow_head, dyn_geo)
                out["shadow_ratio"] = shadow
                if combine_static_dynamic and "rgb" in out:
                    out["rgb"] = (s_ratio[..., None] * out["rgb"] * (1 - shadow)
                                  + d_ratio[..., None] * out["dynamic_rgb"])
        else:
            out["density"] = static_density
            if return_density_only:
                return out
            if tail is not None:
                # a dynamic field asked for colour without timestamps fails like the reference's query_rgb
                # (radiance_field.py:651-654)
                assert self.dynamic_xyz_encoder is None, "Dynamic geometry features are not provided."
                out["rgb"] = static_rgb if static_rgb is not None else self._rgb_from_tail(rgb_in_static)
            elif directions is not None:
                out["rgb"] = self.query_rgb(directions, geo, data_dict=data_dict)["rgb"]

        if self.enable_feature_head and query_feature_head:
            if self.enable_learnable_pe and query_pe_head:
                # pixel_coords are (y/H, x/W) while grid_sample reads (x, y): the map is sampled
                # transposed, as in the reference (SURVEY.md Q10)
                grid = data_dict["pixel_coords"].reshape(1, 1, -1, 2) * 2 - 1
                pe = F.grid_sample(self.learnable_pe_map, grid, align_corners=False, mode="bilinear")
                pe = pe.squeeze(2).squeeze(0).permute(1, 0)
                out["dino_pe"] = run_sequential(self.pe_head, pe)
            dino = run_sequential(self.dino_head, sem)
            if dynamic_on:
                dyn_dino = run_sequential(self.dino_head, dyn_sem)
                out["static_dino_feat"], out["dynamic_dino_feat"] = dino, dyn_dino
                if combine_static_dynamic:
                    s_ratio = static_density / (density + 1e-6)
                    d_ratio = dynamic_density / (density + 1e-6)
                    out["dino_feat"] = s_ratio[..., None] * dino + d_ratio[..., None] * dyn_dino
            else:
                out["dino_feat"] = dino

        # sky is a per-RAY quantity: sample 0 of every per-sample tensor (SURVEY.md Q8)
        if self.enable_sky_head and "lidar_origin" not in data_dict and directions is not None:
            first = {k: v[:, 0] for k, v in data_dict.items()}
            out.update(self.query_sky(directions[:, 0], data_dict=first))
        return out

    def _temporal_noise(self, forward_flow: Tensor) -> Optional[Tensor]:
        """The warp's noise as the reference draws it (radiance_field.py:563-568): the same generator call in the same
        place, so the generator state after a step does not depend on the path; None for the eval renders' ones."""
        if self._noise_override is not None:
            return self._noise_override.to(forward_flow)
        if self.training:
            return torch.rand_like(forward_flow)[..., 0:1]
        return None

    def _flow_branch_usable(self, positions: Tensor, chain: bool, density_only: bool) -> bool:
        return (_ops.FLOW_BRANCH == "fused" and self.flow_xyz_encoder is not None and self._fused_density
                and (chain or density_only) and positions.dim() == 3 and _ops.on_device(positions)
                and self.dynamic_xyz_encoder.n_output_dims in _ops.FLOW_K_ENC
                and self._chain_usable(self.dynamic_xyz_encoder, self.dynamic_base_mlp))

    def _flow_branch(self, positions: Tensor, normed: Tensor, t: Tensor, ray_bias: Optional[Tensor]):
        """``forward``'s dynamic + flow branch with the temporal aggregation fused (EMER_FLOW_BRANCH=fused): the flow
        field at the points, both warps in one launch, ONE dynamic-table gather over the stacked [current | forward |
        backward] coordinates, ONE flow-table gather + flow MLP over the 2N warped rows, and the three-query chain.
        ``ray_bias`` None: density only.  Returns (density, rgb | None, geo, sem | None, the flow keys of the
        per-layer path: flows, predicted flows, the three hash encodings and ``dynamic_feats``)."""
        lead = positions.shape[:-1]
        n = positions[..., 0].numel()
        G = self.geometry_feature_dim
        flow = self.forward_flow_hash(normed, t)
        fwd, bwd = flow[..., :3], flow[..., 3:]
        noise = self._temporal_noise(fwd)
        coords_w = _ops.flow_warp(positions, flow, noise, t, self.aabb, self.time_diff, self.unbounded)
        pred, _ = self._encode_mlp(self.flow_xyz_encoder, self.flow_mlp, coords_w)
        enc_d = self.dynamic_xyz_encoder
        enc = _ops.grid_encode_rows(self._space_time(normed, t).reshape(n, -1), coords_w, enc_d.tcnn_encoding.params,
                                    enc_d.desc)
        sigma, rgb, geo, sem = _ops.flow_field_chain(enc, ray_bias, lead[-1], *self._chain_params(self.dynamic_base_mlp))
        k = enc.shape[-1]
        feats = geo if sem is None else torch.cat([geo, sem], dim=-1)
        res = {"forward_flow": fwd, "backward_flow": bwd,
               "forward_dynamic_hash_encodings": enc[n:2 * n].view(*lead, k),
               "forward_pred_backward_flow": pred[:n, 3:].view(*lead, 3),
               "backward_dynamic_hash_encodings": enc[2 * n:].view(*lead, k),
               "backward_pred_forward_flow": pred[n:, :3].view(*lead, 3),
               "dynamic_feats": feats.view(*lead, -1),
               "current_dynamic_hash_encodings": enc[:n].view(*lead, k)}
        return (sigma.view(lead), None if rgb is None else rgb.view(*lead, 3), geo.view(*lead, G),
                None if sem is None else sem.view(*lead, -1), res)

    def temporal_aggregation(self, positions: Tensor, normed_timestamps: Tensor, forward_flow: Tensor,
                             backward_flow: Tensor, dynamic_feats: Tensor) -> Dict[str, Tensor]:
        """Eq. (8) of the paper (radiance_field.py:553-620): re-query the dynamic and flow fields at
        the flow-warped positions / neighbouring times and blend."""
        if normed_timestamps.shape[-1] != 1:
            normed_timestamps = normed_timestamps.unsqueeze(-1)
        noise = self._temporal_noise(forward_flow)
        if noise is None:
            noise = torch.ones_like(forward_flow)[..., 0:1]
        results = {}
        warped_feats = []
        for tag, flow, sign in (("forward", forward_flow, 1.0), ("backward", backward_flow, -1.0)):
            w_pos = self.contract_points(positions + flow * noise)
            w_time = torch.clamp(normed_timestamps + sign * self.time_diff * noise, 0, 1.0)
            feats, enc = self.forward_dynamic_hash(w_pos, w_time, return_hash_encodings=True)
            pred = self.forward_flow_hash(w_pos, w_time)
            warped_feats.append(feats)
            results[f"{tag}_dynamic_hash_encodings"] = enc
            if tag == "forward":
                results["forward_pred_backward_flow"] = pred[..., 3:]
            else:
                results["backward_pred_forward_flow"] = pred[..., :3]
        results["dynamic_feats"] = (dynamic_feats + 0.5 * warped_feats[0] + 0.5 * warped_feats[1]) / 2.0
        return results

    # ------------------------------------------------------------------ heads
    def _embed(self, idx: Tensor) -> Tensor:
        """``self.appearance_embedding(idx)``; on the device through the sort-free gather (``_ops.gather_rows``): the
        backward of nn.Embedding radix-sorts the indices every step."""
        w = self.appearance_embedding.weight
        if not _ops.on_device(w):
            return self.appearance_embedding(idx)
        return _ops.gather_rows(w, idx).reshape(*idx.shape, w.shape[1])

    def _appearance(self, like: Tensor, data_dict) -> Optional[Tensor]:
        if not (self.enable_cam_embedding or self.enable_img_embedding):
            return None
        if "cam_idx" in data_dict and self.enable_cam_embedding:
            return self._embed(data_dict["cam_idx"])
        if "img_idx" in data_dict and self.enable_img_embedding:
            return self._embed(data_dict["img_idx"])
        mean = self.appearance_embedding.weight.mean(dim=0)
        return torch.ones((*like.shape[:-1], self.appearance_embedding_dim), device=like.device) * mean

    def query_rgb(self, directions: Tensor, geo_feats: Tensor, dynamic_geo_feats: Tensor = None,
                  data_dict: Dict[str, Tensor] = None) -> Dict[str, Tensor]:
        data_dict = data_dict or {}
        unit = (directions + 1.0) / 2.0                     # the reference remaps BEFORE encoding (Q1)
        h = self.direction_encoding(unit.reshape(-1, unit.shape[-1])).view(*unit.shape[:-1], -1)
        emb = self._appearance(unit, data_dict)
        if emb is not None:
            h = torch.cat([h, emb], dim=-1)
        results = {"rgb": self.rgb_head(_ops.cat_pad4([h, geo_feats]), out_act=_ops.ACT_SIGMOID)}
        if self.dynamic_xyz_encoder is not None:
            assert dynamic_geo_feats is not None, "Dynamic geometry features are not provided."
            results["dynamic_rgb"] = self.rgb_head(_ops.cat_pad4([h, dynamic_geo_feats]), out_act=_ops.ACT_SIGMOID)
        return results

    def query_sky(self, directions: Tensor, data_dict: Dict[str, Tensor] = None) -> Dict[str, Tensor]:
        data_dict = data_dict or {}
        d = directions if directions.dim() == 2 else directions[:, 0]
        dd = self.direction_encoding(d).to(directions)
        emb = self._appearance(directions, data_dict)
        if emb is not None:
            dd = _ops.cat_pad4([dd, emb])              # 49 columns in 52-float rows: the tensor-core loaders want 16-byte rows
        results = {"rgb_sky": self.sky_head(dd, out_act=_ops.ACT_SIGMOID)}
        if self.enable_feature_head:
            # (the reference evaluates dino_sky_head twice and discards the first result, Q9)
            results["dino_sky_feat"] = run_sequential(self.dino_sky_head, dd)
        return results

    def query_flow(self, positions: Tensor, normed_timestamps: Tensor, query_density: bool = True):
        normed = self.contract_points(positions)
        flow = self.forward_flow_hash(normed, normed_timestamps)
        results = {"forward_flow": flow[..., :3], "backward_flow": flow[..., 3:]}
        if query_density:
            dyn = self.forward_dynamic_hash(normed, normed_timestamps)
            results["dynamic_density"] = self._density(dyn)
        return results

    def query_attributes(self, positions: Tensor, normed_timestamps: Tensor = None,
                         query_feature_head: bool = True):
        out: Dict[str, Tensor] = {}
        G, S = self.geometry_feature_dim, self.semantic_feature_dim
        feats, normed = self.forward_static_hash(positions)
        sem = feats[..., G:G + S]
        static_density = self._density(feats)
        dynamic_on = self.dynamic_xyz_encoder is not None and normed_timestamps is not None
        if dynamic_on:
            dyn_feats, dyn_enc = self.forward_dynamic_hash(normed, normed_timestamps, return_hash_encodings=True)
            if self.flow_xyz_encoder is not None:
                flow = self.forward_flow_hash(normed, normed_timestamps)
                out["forward_flow"], out["backward_flow"] = flow[..., :3], flow[..., 3:]
                agg = self.temporal_aggregation(positions, normed_timestamps, flow[..., :3], flow[..., 3:], dyn_feats)
                dyn_feats = agg["dynamic_feats"]
                agg["current_dynamic_hash_encodings"] = dyn_enc
                out.update(agg)
            dyn_sem = dyn_feats[..., G:G + S]
            dynamic_density = self._density(dyn_feats)
            density = static_density + dynamic_density
            out.update(density=density, static_density=static_density, dynamic_density=dynamic_density)
        else:
            out["density"] = static_density
        if self.enable_feature_head and query_feature_head:
            dino = run_sequential(self.dino_head, sem)
            if dynamic_on:
                dyn_dino = run_sequential(self.dino_head, dyn_sem)
                out["static_dino_feat"], out["dynamic_dino_feat"] = dino, dyn_dino
                out["dino_feat"] = (static_density.unsqueeze(-1) * dino + dynamic_density.unsqueeze(-1) * dyn_dino) \
                    / (density.unsqueeze(-1) + 1e-6)
            else:
                out["dino_feat"] = dino
        return out


class DensityField(nn.Module):
    """Proposal network: contract -> hash grid -> Linear(.,64)-ReLU-Linear(64,1) -> trunc_exp(x-1)
    (radiance_field.py:788-841)."""

    def __init__(self, xyz_encoder: HashEncoder,
                 aabb: Union[Tensor, List[float]] = [[-1.0, -1.0, -1.0, 1.0, 1.0, 1.0]], num_dims: int = 3,
                 density_activation: Callable = _default_density_activation, unbounded: bool = False,
                 base_mlp_layer_width: int = 64) -> None:
        super().__init__()
        self.register_buffer("aabb", _as_aabb(aabb))
        self.num_dims = num_dims
        self.density_activation = density_activation
        self._fused_density = density_activation is _default_density_activation
        self.unbounded = unbounded
        self.xyz_encoder = xyz_encoder
        self.base_mlp = _stack(xyz_encoder.n_output_dims, base_mlp_layer_width, 1)

    @property
    def device(self) -> torch.device:
        return self.aabb.device

    def set_aabb(self, aabb: Union[Tensor, List[float]]) -> None:
        aabb = _as_aabb(aabb)
        logger.info(f"Set propnet aabb from {self.aabb} to {aabb}")
        self.aabb.copy_(aabb)        # a [6] tensor broadcasts into the default [1, 6] buffer (Q18)
        self.aabb = self.aabb.to(self.device)

    def forward(self, positions: Tensor, data_dict: Dict[str, Tensor] = None) -> Dict[str, Tensor]:
        lead = positions.shape[:-1]
        coords = _contract_points(positions, self.aabb, self.unbounded)
        enc = self.xyz_encoder(coords.reshape(-1, self.num_dims))
        raw = run_sequential(self.base_mlp, enc).view(*lead, -1)
        density = _ops.density_activation(raw) if self._fused_density else self.density_activation(raw)
        return {"density": density}


def build_radiance_field_from_cfg(cfg, verbose=True) -> RadianceField:
    head, neck = cfg.head, cfg.neck
    dynamic = build_xyz_encoder_from_cfg(cfg.dynamic_xyz_encoder, verbose=verbose) \
        if head.enable_dynamic_branch else None
    # the flow grid is hard-coded in the reference (radiance_field.py:916-923), not read from cfg
    flow = HashEncoder(n_input_dims=4, n_levels=10, base_resolution=16, max_resolution=4096,
                       log2_hashmap_size=18, n_features_per_level=4) if head.enable_flow_branch else None
    return RadianceField(
        xyz_encoder=build_xyz_encoder_from_cfg(cfg.xyz_encoder, verbose=verbose),
        dynamic_xyz_encoder=dynamic, flow_xyz_encoder=flow, unbounded=cfg.unbounded, num_cams=cfg.num_cams,
        geometry_feature_dim=neck.geometry_feature_dim, base_mlp_layer_width=neck.base_mlp_layer_width,
        head_mlp_layer_width=head.head_mlp_layer_width, enable_cam_embedding=head.enable_cam_embedding,
        enable_img_embedding=head.enable_img_embedding, appearance_embedding_dim=head.appearance_embedding_dim,
        enable_sky_head=head.enable_sky_head, enable_feature_head=head.enable_feature_head,
        semantic_feature_dim=neck.semantic_feature_dim, feature_mlp_layer_width=head.feature_mlp_layer_width,
        feature_embedding_dim=head.feature_embedding_dim, enable_shadow_head=head.enable_shadow_head,
        num_train_timesteps=cfg.num_train_timesteps, interpolate_xyz_encoding=head.interpolate_xyz_encoding,
        enable_learnable_pe=head.enable_learnable_pe,
        enable_temporal_interpolation=head.enable_temporal_interpolation)


def build_density_field(
    aabb: Union[Tensor, List[float]] = [[-1.0, -1.0, -1.0, 1.0, 1.0, 1.0]],
    type: Literal["HashEncoder"] = "HashEncoder",
    n_input_dims: int = 3,
    n_levels: int = 5,
    base_resolution: int = 16,
    max_resolution: int = 128,
    log2_hashmap_size: int = 20,
    n_features_per_level: int = 2,
    unbounded: bool = True,
) -> DensityField:
    if type != "HashEncoder":
        raise NotImplementedError(f"Unknown (xyz_encoder) type: {type}")
    encoder = HashEncoder(n_input_dims=n_input_dims, n_levels=n_levels, base_resolution=base_resolution,
                          max_resolution=max_resolution, log2_hashmap_size=log2_hashmap_size,
                          n_features_per_level=n_features_per_level)
    return DensityField(xyz_encoder=encoder, aabb=aabb, unbounded=unbounded)

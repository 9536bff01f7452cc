"""Position / direction encoders with the reference's class names and constructor arguments
(radiance_fields/encodings.py of NVlabs/EmerNeRF), backed by the sm_90a hash-grid kernels."""
from __future__ import annotations

import json
import logging
import math

import numpy as np
import torch
import torch.nn as nn
from torch import Tensor

from ..third_party import tcnn_modules as tcnn

logger = logging.getLogger()


class XYZ_Encoder(nn.Module):
    encoder_type = "XYZ_Encoder"

    def __init__(self, n_input_dims):
        super().__init__()
        self.n_input_dims = n_input_dims

    @property
    def n_output_dims(self) -> int:
        raise NotImplementedError


class SinusoidalEncoder(XYZ_Encoder):
    """[x, sin(2^i x), sin(2^i x + pi/2)] for i in [min_deg, max_deg]; evaluated without grad
    (encodings.py:60-104).  Only used on unit view directions: 3 -> 33 for degrees 0..4."""
    encoder_type = "SinusoidalEncoder"

    def __init__(self, n_input_dims: int = 3, min_deg: int = 0, max_deg: int = 10, enable_identity: bool = True):
        super().__init__(n_input_dims)
        self.min_deg, self.max_deg, self.enable_identity = min_deg, max_deg, enable_identity
        self.register_buffer("scales", Tensor([2 ** i for i in range(min_deg, max_deg + 1)]))

    @property
    def n_output_dims(self) -> int:
        return (int(self.enable_identity) + (self.max_deg - self.min_deg + 1) * 2) * self.n_input_dims

    @torch.no_grad()
    def forward(self, x: Tensor) -> Tensor:
        if self.max_deg == self.min_deg:
            return x
        n_freq = self.max_deg - self.min_deg + 1
        scaled = (x.unsqueeze(-2) * self.scales.unsqueeze(-1)).flatten(-2)       # [..., n_freq*D]
        assert scaled.shape[-1] == n_freq * self.n_input_dims
        waves = torch.sin(torch.cat([scaled, scaled + 0.5 * torch.pi], dim=-1))
        return torch.cat([x, waves], dim=-1) if self.enable_identity else waves


class SHEncoder(XYZ_Encoder):
    """Present for API parity; the model never builds it (radiance_field.py:126-128 uses the
    sinusoidal encoder) and tcnn's SphericalHarmonics kernel is outside the hot path."""
    encoder_type = "SHEncoder"

    def __init__(self, n_input_dims: int = 3, levels: int = 4) -> None:
        super().__init__(n_input_dims)
        if levels <= 0 or levels > 4:
            raise ValueError(f"Spherical harmonic encoding only supports 1 to 4 levels, requested {levels}")
        raise NotImplementedError("SHEncoder is not on the EmerNeRF hot path (SURVEY.md K5)")


class HashEncoder(XYZ_Encoder):
    """Multi-resolution hash grid (encodings.py:107-160): geometric level growth from
    ``base_resolution`` to ``max_resolution`` (float64 numpy, as the reference computes it)."""
    encoder_type = "HashEncoder"

    def __init__(self, n_input_dims: int = 3, n_levels: int = 16, base_resolution: int = 16,
                 max_resolution: int = 2048, log2_hashmap_size: int = 19, n_features_per_level: int = 2,
                 dtype=torch.float32, verbose: bool = True) -> None:
        super().__init__(n_input_dims)
        self.num_levels = n_levels
        self.base_resolution = base_resolution
        self.max_resolution = max_resolution
        self.log2_hashmap_size = log2_hashmap_size
        self.n_features_per_level = n_features_per_level
        self.growth_factor = np.exp((np.log(max_resolution) - np.log(base_resolution)) / (n_levels - 1))
        self.encoding_config = {
            "otype": "HashGrid",
            "n_levels": n_levels,
            "n_features_per_level": n_features_per_level,
            "log2_hashmap_size": log2_hashmap_size,
            "base_resolution": base_resolution,
            "per_level_scale": self.growth_factor,
            "interpolation": "linear",
        }
        self.tcnn_encoding = tcnn.Encoding(n_input_dims=n_input_dims, encoding_config=self.encoding_config,
                                           dtype=dtype)
        self.num_parameters = self.tcnn_encoding.params.shape
        if verbose:
            logger.info("hash grid config: %s", json.dumps(self.encoding_config))
            logger.info("hash grid params: %.3fM (%s), levels dense->hashed: %s",
                        self.tcnn_encoding.params.numel() / 1e6, self.tcnn_encoding.params.dtype,
                        "".join("h" if h else "d" for h in self.tcnn_encoding.desc.hashed))

    @property
    def n_output_dims(self) -> int:
        return self.tcnn_encoding.n_output_dims

    @property
    def desc(self):
        return self.tcnn_encoding.desc

    def forward(self, in_tensor: Tensor) -> Tensor:
        return self.tcnn_encoding(in_tensor)


def build_xyz_encoder_from_cfg(xyz_encoder_cfg, verbose=True) -> XYZ_Encoder:
    kind = xyz_encoder_cfg.type
    if kind == "HashEncoder":
        return HashEncoder(
            n_input_dims=xyz_encoder_cfg.n_input_dims, n_levels=xyz_encoder_cfg.n_levels,
            n_features_per_level=xyz_encoder_cfg.n_features_per_level,
            base_resolution=xyz_encoder_cfg.base_resolution, max_resolution=xyz_encoder_cfg.max_resolution,
            log2_hashmap_size=xyz_encoder_cfg.log2_hashmap_size, verbose=verbose)
    if kind == "SHEncoder":
        return SHEncoder(n_input_dims=xyz_encoder_cfg.n_input_dims, levels=xyz_encoder_cfg.levels)
    if kind == "SinusoidalEncoder":
        return SinusoidalEncoder(n_input_dims=xyz_encoder_cfg.n_input_dims, min_deg=xyz_encoder_cfg.min_deg,
                                 max_deg=xyz_encoder_cfg.max_deg, enable_identity=xyz_encoder_cfg.enable_identity)
    raise NotImplementedError(f"Unknown nerf encoder type: {kind}")

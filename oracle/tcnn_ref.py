"""Pure-PyTorch restatement of tiny-cuda-nn's ``HashGrid`` encoding (CPU oracle).

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.  **Parity unpinned**: the
tiny-cuda-nn sources are not in the reference tree (the reference installs
them from master, README.md:51); this file restates the published algorithm of
``include/tiny-cuda-nn/encodings/grid.h`` and is anchored on the reference's
call sites ``radiance_fields/encodings.py:130-146,159-160`` and
``third_party/tcnn_modules.py:115-151,235-263,375-423``.

Restated pieces (tiny-cuda-nn names in brackets):
  * level scale      [grid_scale]      scale_l = exp2f(l * log2f(per_level_scale)) * base - 1
  * level resolution [grid_resolution] res_l   = ceil(scale_l) + 1
  * level size       [GridEncodingTemplated ctor]  min(round_up(res^D, 8), 2^log2_hashmap_size)
  * position         [pos_fract]       pos = fmaf(scale, x, 0.5); cell = floor(pos); w = pos - cell
  * index            [grid_index]      dense stride while stride <= size, else coherent-prime hash; % size
  * hash             [coherent_prime_hash]  xor_d cell_d * prime_d (uint32 wrap), primes 1, 2654435761, ...
  * interpolation    [kernel_grid]     sum over 2^D corners of prod_d (w_d or 1-w_d) * table[idx]
  * parameters       level-major flat fp32 vector, F floats per entry, init U(-1e-4, 1e-4)
  * output           [N, L*F], feature index = level*F + f
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List

import numpy as np
import torch
from torch import Tensor

PRIMES = (1, 2654435761, 805459861, 3674653429, 2097192037, 1434869437, 2165219737)
_U32 = 0xFFFFFFFF


@dataclass
class GridGeometry:
    n_dims: int
    n_levels: int
    n_feat: int
    scales: List[float]      # float32 values, one per level
    resolutions: List[int]
    offsets: List[int]       # entries (not floats); len = n_levels + 1
    hashed: List[bool]

    @property
    def n_params(self) -> int:
        return self.offsets[-1] * self.n_feat

    @property
    def n_output_dims(self) -> int:
        return self.n_levels * self.n_feat


def grid_geometry(n_dims: int, cfg: dict) -> GridGeometry:
    """Level table for a tcnn ``HashGrid`` config dict (encodings.py:133-141)."""
    L = int(cfg["n_levels"])
    F = int(cfg["n_features_per_level"])
    log2_T = int(cfg["log2_hashmap_size"])
    base = int(cfg["base_resolution"])
    # json -> float in tcnn; log2 taken in float
    pls = np.float32(cfg.get("per_level_scale", 2.0))
    log2_pls = np.float32(np.log2(pls))
    scales, ress, offs, hashed = [], [], [0], []
    for lvl in range(L):
        s = np.float32(np.exp2(np.float32(lvl) * log2_pls)) * np.float32(base) - np.float32(1.0)
        s = np.float32(s)
        res = int(math.ceil(float(s))) + 1
        dense = res ** n_dims
        max_params = _U32 // 2
        n = max_params if float(res) ** n_dims > float(max_params) else dense
        n = (n + 7) // 8 * 8
        n = min(n, 1 << log2_T)
        scales.append(float(s))
        ress.append(res)
        offs.append(offs[-1] + n)
        # grid_index hashes iff the dense stride product overflows the level size
        stride, h = 1, False
        for _ in range(n_dims):
            if stride > n:
                break
            stride *= res
        hashed.append(n < stride)
    return GridGeometry(n_dims, L, F, scales, ress, offs, hashed)


def _level_indices(cell: Tensor, geom: GridGeometry, lvl: int) -> Tensor:
    """cell: int64 [..., D] holding uint32 values. Returns int64 entry index in level."""
    size = geom.offsets[lvl + 1] - geom.offsets[lvl]
    res = geom.resolutions[lvl]
    D = geom.n_dims
    if geom.hashed[lvl]:
        h = torch.zeros_like(cell[..., 0])
        for d in range(D):
            h = h ^ ((cell[..., d] * PRIMES[d]) & _U32)
        idx = h
    else:
        idx = torch.zeros_like(cell[..., 0])
        stride = 1
        for d in range(D):
            if stride > size:
                break
            idx = (idx + cell[..., d] * stride) & _U32
            stride = (stride * res) & _U32
    return idx % size


def _fma32(a: Tensor, b: Tensor, c: Tensor) -> Tensor:
    """fmaf emulated through float64 (single rounding up to a ~2^-29 double-rounding chance)."""
    return (a.double() * b.double() + c.double()).float()


def corner_indices_and_weights(x: Tensor, geom: GridGeometry, lvl: int):
    """x: [N, D] fp32. Returns (idx int64 [N, 2^D] absolute entry index, w fp32 [N, 2^D], frac [N,D], cell)."""
    scale = torch.tensor(geom.scales[lvl], dtype=torch.float32)
    pos = _fma32(scale.expand_as(x), x, torch.full_like(x, 0.5))
    fl = torch.floor(pos)
    frac = pos - fl
    cell = fl.to(torch.int64) & _U32          # (uint32)(int)floor
    D = geom.n_dims
    idxs, ws = [], []
    for c in range(1 << D):
        w = torch.ones_like(frac[..., 0])
        cc = []
        for d in range(D):
            if (c >> d) & 1:
                w = w * frac[..., d]
                cc.append((cell[..., d] + 1) & _U32)
            else:
                w = w * (1.0 - frac[..., d])
                cc.append(cell[..., d])
        idx = _level_indices(torch.stack(cc, -1), geom, lvl) + geom.offsets[lvl]
        idxs.append(idx)
        ws.append(w)
    return torch.stack(idxs, -1), torch.stack(ws, -1), frac, cell


def grid_forward(x: Tensor, params: Tensor, geom: GridGeometry, fused: bool = True) -> Tensor:
    """[N, D] -> [N, L*F].  Differentiable w.r.t. ``params`` and ``x`` (through the weights,
    matching tcnn's dy_dx: derivative of the D-linear weights times ``scale``)."""
    N = x.shape[0]
    F = geom.n_feat
    table = params.view(-1, F)
    outs = []
    for lvl in range(geom.n_levels):
        idx, w, _, _ = corner_indices_and_weights(x, geom, lvl)
        acc = torch.zeros(N, F, dtype=torch.float32)
        for c in range(idx.shape[-1]):
            v = table[idx[:, c]]
            if fused:
                acc = _fma32(w[:, c : c + 1].expand_as(v), v, acc)
            else:
                acc = acc + w[:, c : c + 1] * v
        outs.append(acc)
    return torch.cat(outs, -1)


class Encoding(torch.nn.Module):
    """Stand-in for ``tcnn.Encoding`` (third_party/tcnn_modules.py:375-423): same ctor
    arguments, ``params`` Parameter (flat fp32, level-major), ``n_output_dims``, ``forward``."""

    def __init__(self, n_input_dims, encoding_config, seed=1337, dtype=None):
        super().__init__()
        if encoding_config.get("otype", "HashGrid") != "HashGrid":
            raise NotImplementedError(encoding_config.get("otype"))
        if encoding_config.get("interpolation", "linear").lower() != "linear":
            raise NotImplementedError("only linear interpolation is on the path")
        self.n_input_dims = n_input_dims
        self.encoding_config = encoding_config
        self.seed = seed
        self.geom = grid_geometry(n_input_dims, encoding_config)
        self.n_output_dims = self.geom.n_output_dims
        g = torch.Generator().manual_seed(seed)
        init = (torch.rand(self.geom.n_params, generator=g, dtype=torch.float32) * 2 - 1) * 1e-4
        self.params = torch.nn.Parameter(init)

    def forward(self, x: Tensor) -> Tensor:
        return grid_forward(x.to(torch.float32).contiguous(), self.params, self.geom)

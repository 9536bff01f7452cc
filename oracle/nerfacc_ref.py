"""Pure-PyTorch restatement of the nerfacc symbols on the EmerNeRF hot path (CPU oracle).

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.  **Parity unpinned** except for
the ``importance_sampling`` docstring example: nerfacc
(8340e19daad4bafe24125150a8c56161838086fa, README.md:50) is not in the
reference tree and is not installed in the build environment.  Call sites this follows:
``third_party/nerfacc_prop_net.py:11-14,148,153,165,172,349``,
``radiance_fields/render_utils.py:4-8,35-42,73-75,103-105,159-282``.

Only the *batched* ([n_rays, n_samples]) code paths are restated -- the reference
never builds packed rays (SURVEY.md F7).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import Tensor


class RayIntervals:
    """nerfacc.data_specs.RayIntervals, batched form: just ``vals`` [n_rays, n_edges]."""

    def __init__(self, vals: Tensor, packed_info=None, is_left=None, is_right=None):
        self.vals = vals
        self.packed_info = packed_info
        self.is_left = is_left
        self.is_right = is_right

    @property
    def device(self):
        return self.vals.device


class RaySamples:
    def __init__(self, vals: Tensor, packed_info=None, ray_indices=None, is_valid=None):
        self.vals = vals
        self.packed_info = packed_info
        self.ray_indices = ray_indices
        self.is_valid = is_valid


class AbstractEstimator(torch.nn.Module):
    """nerfacc.estimators.base.AbstractEstimator: nn.Module with a ``device`` property."""

    def __init__(self) -> None:
        super().__init__()
        self.register_buffer("_dummy", torch.empty(0), persistent=False)

    @property
    def device(self) -> torch.device:
        return self._dummy.device


def exclusive_sum(x: Tensor) -> Tensor:
    """nerfacc.scan.exclusive_sum, batched: cumsum of the right-shifted input."""
    return torch.cumsum(torch.cat([torch.zeros_like(x[..., :1]), x[..., :-1]], dim=-1), dim=-1)


def render_transmittance_from_density(
    t_starts: Tensor, t_ends: Tensor, sigmas: Tensor, packed_info=None, ray_indices=None,
    n_rays=None, prefix_trans=None,
) -> Tuple[Tensor, Tensor]:
    sigmas_dt = sigmas * (t_ends - t_starts)
    alphas = 1.0 - torch.exp(-sigmas_dt)
    trans = torch.exp(-exclusive_sum(sigmas_dt))
    return trans, alphas


def render_weight_from_density(
    t_starts: Tensor, t_ends: Tensor, sigmas: Tensor, packed_info=None, ray_indices=None,
    n_rays=None, prefix_trans=None,
) -> Tuple[Tensor, Tensor, Tensor]:
    trans, alphas = render_transmittance_from_density(t_starts, t_ends, sigmas)
    return trans * alphas, trans, alphas


def accumulate_along_rays(
    weights: Tensor, values: Optional[Tensor] = None, ray_indices=None, n_rays=None
) -> Tensor:
    src = weights[..., None] if values is None else weights[..., None] * values
    return torch.sum(src, dim=-2)


def importance_sampling_bins(cdfs: Tensor, n: int, bias: Tensor):
    """Shared arithmetic of ``importance_sampling``: for every output edge k in [0, n]
    returns (u [R, n+1] fp32, p0, p1 int64) with
        u_k  = cdf_first + (k + (bias - 0.5)) * ((cdf_last - cdf_first) / n)
        p    = first edge index with cdf[p] > u_k  (upper bound; m+1 if none)
        p0   = clamp(p - 1, 0, m),  p1 = clamp(p, 0, m)
    All arithmetic is separate fp32 mul/add (no FMA) in exactly this order."""
    R, m1 = cdfs.shape
    u_floor = cdfs[:, :1]
    u_ceil = cdfs[:, -1:]
    u_step = (u_ceil - u_floor) / float(n)
    k = torch.arange(n + 1, dtype=torch.float32, device=cdfs.device)[None, :]
    u = u_floor + (k + (bias - 0.5)) * u_step
    p = torch.searchsorted(cdfs.contiguous(), u.contiguous(), right=True)
    p0 = (p - 1).clamp(0, m1 - 1)
    p1 = p.clamp(0, m1 - 1)
    return u, p0, p1


def importance_sampling(
    intervals: RayIntervals, cdfs: Tensor, n_intervals_per_ray: int, stratified: bool = False,
    jitter: Optional[Tensor] = None,
):
    """nerfacc.pdf.importance_sampling, batched.  ``jitter`` ([R] or [R,1], U[0,1)) replaces
    the per-ray Philox draw that nerfacc takes from torch's CUDA generator when ``stratified``
    (not reproducible off the GPU, SURVEY.md §7)."""
    vals = intervals.vals
    R = vals.shape[0]
    n = int(n_intervals_per_ray)
    if stratified:
        if jitter is None:
            jitter = torch.rand(R, 1, device=vals.device)
        bias = jitter.reshape(R, 1).to(torch.float32)
    else:
        bias = torch.full((R, 1), 0.5, dtype=torch.float32, device=vals.device)
    u, p0, p1 = importance_sampling_bins(cdfs, n, bias)
    u_lo = cdfs.gather(-1, p0)
    u_hi = cdfs.gather(-1, p1)
    t_lo = vals.gather(-1, p0)
    t_hi = vals.gather(-1, p1)
    du = u_hi - u_lo
    mid = (t_lo + t_hi) * 0.5
    safe = torch.where(du < 1e-10, torch.ones_like(du), du)
    lerp = (u - u_lo) * ((t_hi - t_lo) / safe) + t_lo
    edges = torch.where(du < 1e-10, mid, lerp)
    samples = (edges[..., 1:] + edges[..., :-1]) * 0.5
    return RayIntervals(vals=edges), RaySamples(vals=samples)


def searchsorted(sorted_sequence: RayIntervals, values: RayIntervals):
    """nerfacc.pdf.searchsorted, batched: ids_left = last key edge <= query (clamped),
    ids_right = ids_left + 1 clamped.  Only reached when the anti-aliasing loss is disabled
    (nerfacc_prop_net.py:235-237,349)."""
    key, q = sorted_sequence.vals, values.vals
    hi = torch.searchsorted(key.contiguous(), q.contiguous(), right=True)
    m1 = key.shape[-1]
    ids_left = (hi - 1).clamp(0, m1 - 1)
    ids_right = hi.clamp(0, m1 - 1)
    return ids_left, ids_right

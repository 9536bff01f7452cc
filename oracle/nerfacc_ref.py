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


def warp_sum32(v: Tensor) -> Tensor:
    """The fp32 ray sum of the compositing kernels (csrc/ray_scan.cuh, csrc/composite.cu pass 1), bit for bit: lane l
    adds v[s] for s = l, l + 32, ... in order, then the xor butterfly over 16, 8, 4, 2, 1 lanes.  [R, S] -> [R]."""
    r, s = v.shape
    ch = (s + 31) // 32
    pad = torch.zeros((r, ch * 32), dtype=torch.float32)
    pad[:, :s] = v.float()
    pad = pad.reshape(r, ch, 32)
    acc = torch.zeros((r, 32), dtype=torch.float32)
    for c in range(ch):
        acc = acc + pad[:, c]
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lane ^ o]
    return acc[:, 0]


def composite64(t0: Tensor, t1: Tensor, sigma: Tensor, weights32: Optional[Tensor] = None,
                g_w: Optional[Tensor] = None, g_t: Optional[Tensor] = None, g_o: Optional[Tensor] = None,
                g_d: Optional[Tensor] = None, g_cdf: Optional[Tensor] = None) -> dict:
    """Volume compositing of fp32 rays [R, S] in float64, with the discrete choices of emer_composite_fwd / _bwd.

    The interval length and midpoint are the kernel's fp32 ones, delta = fl(t1 - t0), mid = fl(fl(t0 + t1) / 2); from
    there on everything is float64: x = sigma delta, E_i = sum_{j<i} x_j, T = exp(-E), alpha = 1 - exp(-x), w = T alpha,
    opacity = clamp(sum w, 1e-6, 1), depth = sum w mid / opacity, cdf = 1 - cat(T, 0), the median (first sample whose
    cumulative weight reaches 0.5, else the last).  The opacity clamp is a branch: with ``weights32`` (the kernel's own
    weights) the branch is the kernel's, decided on ``warp_sum32`` of them; otherwise on the float64 sum.

    Given upstream gradients (None for absent ones) the backward runs by autograd on this graph, the weights retaining
    their gradient G (the total gradient reaching w_i).  Returned alongside, for error bounds: ``E``, ``wmid_abs`` =
    sum |w mid|, ``G``, ``gT`` (the gradient reaching T directly: g_t - g_cdf[:, :S]), ``A`` = |G| T exp(-x) and
    ``B`` = sum_{k>i} (|G_k| w_k + |gT_k| T_k)."""
    f64 = torch.float64
    delta32 = t1.float() - t0.float()
    mid = ((t0.float() + t1.float()) / 2.0).to(f64)
    delta = delta32.to(f64)
    sig = sigma.to(f64).clone().requires_grad_(True)
    x = sig * delta
    E = exclusive_sum(x)
    T = torch.exp(-E)
    alpha = 1.0 - torch.exp(-x)
    w = T * alpha
    w.retain_grad()
    sw = w.sum(-1, keepdim=True)
    sw_branch = warp_sum32(weights32)[:, None].to(f64) if weights32 is not None else sw.detach()
    in_range = (sw_branch >= 1e-6) & (sw_branch <= 1.0)
    op = torch.where(in_range, sw, sw_branch.clamp(1e-6, 1.0))
    depth = (w * mid).sum(-1, keepdim=True) / op
    cdf = 1.0 - torch.cat([T, torch.zeros_like(T[:, :1])], -1)
    cw = torch.cumsum(w.detach(), -1)
    S = sigma.shape[-1]
    med_idx = torch.searchsorted(cw, torch.full_like(cw[:, :1], 0.5), side="left").clamp(0, S - 1)
    out = {"weights": w, "trans": T, "opacity": op, "depth": depth, "cdf": cdf, "median_idx": med_idx[:, 0],
           "median_depth": mid.gather(-1, med_idx), "cw": cw, "in_range": in_range[:, 0], "delta": delta, "mid": mid,
           "x": x.detach(), "E": E.detach(), "wmid_abs": (w * mid).abs().sum(-1, keepdim=True).detach()}
    ups = [(w, g_w), (T, g_t), (op, g_o), (depth, g_d), (cdf, g_cdf)]
    ups = [(o, g.to(f64)) for o, g in ups if g is not None]
    if ups:
        torch.autograd.backward([o for o, _ in ups], [g for _, g in ups])
        G = w.grad if w.grad is not None else torch.zeros_like(w)
        gT = torch.zeros_like(T)
        if g_t is not None:
            gT = gT + g_t.to(f64)
        if g_cdf is not None:
            gT = gT - g_cdf[:, :S].to(f64)
        wd, Td = w.detach(), T.detach()
        q = G.abs() * wd + gT.abs() * Td
        out.update(dsigma=sig.grad if sig.grad is not None else torch.zeros_like(sig), G=G, gT=gT,
                   A=G.abs() * Td * torch.exp(-x.detach()),
                   B=torch.flip(exclusive_sum(torch.flip(q, [-1])), [-1]))
    out = {k: v.detach() if isinstance(v, Tensor) else v for k, v in out.items()}
    return out


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

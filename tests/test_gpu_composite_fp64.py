"""Volume compositing (emer_composite_fwd / _bwd, emer_render_fwd / _bwd, emer_accumulate_*) against float64, sample
by sample, on the rays where a transmittance scan goes wrong: empty space in front of a wall, a semi-transparent sample
in front of an opaque one, empty and saturated rays, zero-length intervals, far intervals, an overflowed density and
median ties, mixed across warps and CTAs, at S in {1, 31, 32, 33, 64, 128, 256} and up to 8192 + 5 rays.

Error bounds (u = 2^-24; ``nerfacc_ref.composite64`` makes the kernel's discrete choices, delta = fl(t1 - t0) and
mid = fl(fl(t0 + t1) / 2), and gives every magnitude below; i is a sample, c_i = i // 32 its chunk, n_ch the chunks).

* Transmittance.  The kernel's prefix E_i = carry + (inclusive sum of the lane below) is an fp32 sum of the rounded
  x_j = fl(sigma_j delta_j), j < i: one rounding for x_j, at most 5 Hillis-Steele levels, c_i chunk carries and the
  final add, so |dE_i| <= k_i u E_i with k_i = 7 + c_i -- relative to E_i, not to E_i + x_i: the sample's own term
  never enters.  expf is within 2 ulp (4 u), so |dT_i| <= bT_i = (expm1(k_i u E_i) + 4 u) T_i.
* alpha = 1 - expf(-x) (the reference's form): the error of x and of expf is relative to exp(-x), so it is absolute
  where x is small: |d alpha_i| <= (x_i + 4) u exp(-x_i) + u alpha_i.  w = T alpha rounds once:
  bw_i = alpha_i bT_i + T_i |d alpha_i| + u w_i.  cdf = 1 - T: bT_i + u cdf_i, and every row non-decreasing (the
  kernel's CDF takes the running minimum of T along the ray, which stays within bT_i: it is some T_j, j <= i, with
  E_j <= E_i).
* Ray sums (opacity, sum w mid): per-lane sums over the chunks, then the 5-level butterfly, so
  bop = sum bw + (n_ch + 5) u sum w + u op while the kernel's sum lies in [1e-6, 1]; outside it both sides return the
  clamp's constant (u op apart at 1e-6).  Where the float64 side of the clamp is not the kernel's (the decomposition's
  static and dynamic scans, whose weights the kernel does not write) the first form holds on either side, the clamp
  being non-expansive.
  Depth D / op: (sum bw mid + (n_ch + 5) u sum w mid) / op + |depth| r / (1 - r) + u |depth|, r = bop / op.
* Median: the kernel's cumulative weight at i is off by bcw_i = sum_{j<=i} bw_j + k_i u cw_i; where the fp64 one lies
  within bcw_i of 0.5 the index may move to that sample or the next, elsewhere it is the fp64 index.
* dL/dx_i = G_i T_i exp(-x_i) - sum_{k>i} q_k, q_k = G_k w_k + gT_k T_k (G: the total gradient reaching w, gT the one
  reaching T).  The suffix is the inclusive suffix sum of the lane above plus the carry: each q_k goes through the
  gT fold, its product and fma, 5 levels, n_ch - 1 carries and the final add, (8 + n_ch) u B_i with
  B_i = sum_{k>i} |G_k| w_k + |gT_k| T_k -- again without the sample's own |G_i w_i|.  Widened by the forward:
  sum_{k>i} (|G_k| bw_k + dG_k w_k + |gT_k| bT_k) + A_i (bT_i / T_i + rex_i + 3 u) + dG_i T_i exp(-x_i) + u (A_i + B_i),
  A_i = |G_i| T_i exp(-x_i), rex_i = min(expm1(x_i u), 1) + 4 u.  dG_i, the kernel's error on G = g_w + g_op + g_D mid:
  4 u |terms| (three roundings, and mid's own in the render oracle) + |mid| |g_D| (r' + u)
  + [in range] (u |g_o| + |g_d| sum|w mid| / op^2 (rs + 2 r' + 4 u)), r' = r / (1 - r), rs the relative bound of
  sum w mid.  d sigma = fl(dx delta): delta times that, plus u |d sigma|.
* Render outputs F = sum w v (+ sky (1 - op)) (+ PE): sum (bw + gamma u w) |v| + |sky| (bop + 2 u |1 - op|) + u |F'|
  for each F' an add rounds (after the sky, after the PE), with
  gamma = max(S, n_ch + 5) + 7 (the feature rows accumulate sample by sample; v = r_s c_s (1 - sh) + r_d c_d rounds
  6 times, the fma once).  The two-density ratio terms of d sigma, (d r_s sigma_s + d r_d sigma_d) / den^2,
  d r = w (g.c): bounded by (bw + gamma' u w) (|g|.|c_s| sigma_s + |g|.|c_d| sigma_d) / den^2 with
  gamma' = ceil(C / 32) + 14, and the same magnitude enters dG through g.v.
* Decomposition: shadow and the acc_sh of shadow_only_static_rgb sum over the full weights, shadow_reduced_static_rgb,
  static_dino and the acc_so of shadow_only_static_rgb over the static scan's (composite64 on sigma_s, its own clamp),
  dynamic_dino over the dynamic scan's, each as a render output; shadow_only_static_rgb = acc_so + fl(1 - acc_sh) adds
  u |1 - acc_sh| and u of the result.  static_dino's sky term takes the full opacity and bop (render_utils.py:278-281),
  static_rgb's the static ones.
* Render backward, the other inputs.  w enters as the kernel's fp32 weight: |w~ - w| <= bw, |w~| <= wt = w + bw.
  r_x = fl(sigma_x / fl(sigma + 1e-6f)) is within 3 u of sigma_x / (sigma + 1e-6) (the constant's own rounding, the add,
  the divide); om = fl(1 - sh) and g_F = fl(g_dino + g_dino_pe_free) round once; a dot product g.c over the 3 colour
  channels is an fma chain, within 3 u of |g|.|c|.
  d rgb = fl(w g): (bw + u wt) |g|.  d rgb_s = fl(fl(fl(w g) r_s) om): (bw + 7 u wt) r_s om |g|; d rgb_d: (bw + 5 u wt)
  r_d |g|.  d dino = fl(w g_F): (bw + 2 u wt) |g_F|; d dino_s, d dino_d = fl(fl(w g_F) r_x): (bw + 6 u wt) r_x |g_F|.
  d shadow = fl(2 w g_shr sh - fl(fl(w r_s) g.rgb_s)): the two terms can cancel, so each is bounded on its own,
  2 |g_shr| sh (bw + 3 u wt) + r_s |g|.|rgb_s| (bw + 9 u wt).
  d sigma_x = fl(d r_x / fl(sigma + 1e-6f)), d r_s = fma(w, g_F.dino_s, fl(fl(w g.rgb_s) om)) (d r_d without om): the
  feature dot product is a per-lane fma chain over ceil(C / 32) channels and a 5-level butterfly, on g_F's rounding, so
  (bw + (ceil(C / 32) + 10) u wt) M_x / (sigma + 1e-6), M_s = om |g|.|rgb_s| + |g_F|.|dino_s| (M_d without om); the
  colour chain takes 6 u, the fma 1, the denominator 2 and the divide 1.
  d rgb_sky = fl(g fl(1 - op)) and d dino_sky = fl(g_F fl(1 - op)), against g (1 - op) with composite64's opacity,
  which follows the kernel's side of the clamp: |g| (bop + 2 u (|1 - op| + bop)), 3 u with g_F's rounding.
  d dino_pe = g_dino exactly.
* Accumulate: out and dw are sums of n rounded products, within (n + 1) u sum |terms| (n = S, C); dv = fl(w g) exactly.

Every bound also carries 2^-126 absolute for subnormal results.  A ray whose fp32 opacity sum and float64 sum fall on
different sides of the clamp takes the kernel's branch in composite64; the render backward, whose float64 gradient comes
from ``hotpath.rendering``'s own clamp, leaves those rays to the composite test.

Measured on an H100 80GB HBM3 (700 W power limit): the worst element of each check is at most 0.98 of its bound (the
flow_feat feature sum; 0.64 for transmittance, 0.40 for dsigma, 0.67 for accumulate; in the render backward 0.40 for
d rgb and d dino, at most 0.38 for d rgb_s, d rgb_d, d shadow, d sigma_s, d sigma_d, d dino_s and d dino_d, 0.61 for
d rgb_sky, 0.74 for d dino_sky, d dino_pe exact; in the decomposition 0.30 for shadow, 0.32 for
shadow_reduced_static_rgb, 0.51 for shadow_only_static_rgb, 0.22 for static_dino, 0.33 for dynamic_dino), and the file
runs in about 60 s.  tests/test_render_bounds_cpu.py shows on the CPU that these bounds reject plausible slips.
"""
import math

import pytest
import torch

from oracle import hotpath
from oracle import nerfacc_ref as nf
from test_gpu_rendering import COMBOS, KEYS

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
TINY = 2.0 ** -126
F64 = torch.float64
WORST = {}


def _report(check, ratio):
    WORST[check] = max(WORST.get(check, 0.0), ratio)
    print(f"\n[{check}] worst {WORST[check]:.3g} of its bound")


def _check(check, got, want, bound, mask=None):
    """|got - want| <= bound element by element (where ``mask``), NaN nowhere."""
    got = got.detach().double().cpu()
    want, bound = want.expand_as(got), bound.expand_as(got)
    if mask is not None:
        m = mask.expand_as(got)
        got, want, bound = got[m], want[m], bound[m]
    assert not torch.isnan(got).any(), f"{check}: NaN at {int(torch.isnan(got).sum())} elements"
    err = torch.where(got == want, torch.zeros_like(got), (got - want).abs())
    bad = ~(err <= bound)
    if got.numel():
        _report(check, torch.where(err == 0, torch.zeros_like(err), err / bound).max().item())
    assert not bad.any(), (check, int(bad.sum()), err[bad][:4].tolist(), bound[bad][:4].tolist(),
                           want[bad][:4].tolist(), got[bad][:4].tolist())


# ----------------------------------------------------------------------------------------------- ray families
FAMILIES = ("wall", "two_surfaces", "empty", "faint", "saturated", "zero_length", "far", "inf", "median_tie")


def make_rays(R, S, seed, families=FAMILIES):
    """fp32 t0, t1, sigma [R, S]; ray r is of family families[r % len]; returns the family index per ray too."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *shape: torch.rand(*shape, generator=g, dtype=F64)        # noqa: E731
    fam = torch.arange(R) % len(families)
    delta = rnd(R, S) * 0.02 + 0.01
    t0 = 0.5 + torch.cumsum(delta, -1) - delta
    t1 = t0 + delta
    xd = rnd(R, S) * 1.9 + 0.1                                  # the interior: sigma delta ~ U[0.1, 2]
    wall_lanes = [p for c in sorted({0, (S // 32) // 2 * 32, (S - 1) // 32 * 32}) for p in (c, c + 1, c + 31)]
    wall_lanes = [p for p in wall_lanes if p < S]
    for r in range(R):
        f = families[int(fam[r])]
        k = r // len(families)
        if f in ("wall", "zero_length", "inf"):
            p = wall_lanes[k % len(wall_lanes)]
            empty = rnd(S) * (1e-3 - 1e-7) + 1e-7
            empty[rnd(S) < 0.2] = 0.0
            xd[r, :p] = empty[:p]
            xd[r, p] = (1e2, 3e4, 1e6, 1e8)[k % 4]
            if f == "zero_length":
                zl = rnd(S) < 0.3
                zl[p] = True
                t1[r, zl] = t0[r, zl]
            if f == "inf":
                xd[r, p] = math.inf
        elif f == "two_surfaces":
            p = wall_lanes[k % len(wall_lanes)]
            q = min(p + 1 + k % 3, S - 1)
            xd[r, :] = rnd(S) * 1e-3
            xd[r, p] = 0.3
            if q > p:
                xd[r, q] = 8.0
        elif f == "empty":
            xd[r, :] = 0.0
        elif f == "faint":
            # sum w lands on either side of the 1e-6 clamp
            xd[r, :] = (1e-6 if k % 2 else 4e-9) / S * (0.5 + rnd(S))
        elif f == "saturated":
            xd[r, :] = (20.0 + 180.0 * rnd(1)) / S * (0.5 + rnd(S))
        elif f == "far":
            # uniform_lindisp edges out to t = 1000: linear to 1, then 1 / t-linear
            s = torch.linspace(0.0, 1.0, S + 1, dtype=F64)
            e = torch.where(s < 0.5, 0.1 + 1.8 * s, 1.0 / (1.0 - (s - 0.5) * 1.998))
            t0[r], t1[r] = e[:-1], e[1:]
            xd[r, :] = rnd(S) * 0.2
        elif f == "median_tie":
            # the prefix reaches ln 2 at a sample, so the cumulative weight there is 0.5 up to rounding
            xd[r, :] = rnd(S) * 0.05
            p = wall_lanes[k % len(wall_lanes)]
            if p > 0:
                xd[r, :p] *= math.log(2.0) / xd[r, :p].sum()
            xd[r, p] = 1.0
    t0, t1 = t0.float(), t1.float()
    d32 = (t1 - t0).double()
    sigma = torch.where(d32 > 0, xd / d32.clamp_min(1e-30), xd * 100.0).float()
    return t0.contiguous(), t1.contiguous(), sigma.contiguous(), fam


# ------------------------------------------------------------------------------------------------- bounds
def _safe(a, b):
    """a * b with 0 wherever b is 0 (an infinite error factor on a zero value)."""
    return torch.where(b == 0, torch.zeros_like(a), a * b)


def fwd_bounds(ref, kernel_branch=True):
    """Per-element forward bounds from composite64's output (module docstring); ``kernel_branch``: composite64 had the
    kernel's weights, so it took the kernel's side of the opacity clamp."""
    E, x, T, w, S = ref["E"], ref["x"], ref["trans"], ref["weights"], ref["E"].shape[-1]
    n_ch = (S + 31) // 32
    k = 7 + torch.arange(S, dtype=F64) // 32
    bT = _safe(torch.expm1(k * U * E) + 4 * U, T) + TINY
    ex = torch.exp(-x)
    alpha = 1.0 - ex
    ba = torch.where(torch.isfinite(x), ex * (x + 4) * U, torch.zeros_like(x)) + U * alpha
    bw = alpha * bT + T * ba + U * w + TINY
    sw = w.sum(-1, keepdim=True)
    op = ref["opacity"]
    bop = bw.sum(-1, keepdim=True) + (n_ch + 5) * U * sw + U * op + TINY
    if kernel_branch:
        bop = torch.where(ref["in_range"][:, None], bop, U * op + TINY)
    r = bop / op
    rr = torch.where(r < 0.5, r / (1 - r), torch.full_like(r, math.inf))
    mid = ref["mid"]
    bswm = (bw * mid.abs()).sum(-1, keepdim=True) + (n_ch + 5) * U * ref["wmid_abs"]
    bdep = bswm / op + _safe(rr, ref["depth"].abs()) + U * ref["depth"].abs() + TINY
    bcw = torch.cumsum(bw, -1) + k * U * ref["cw"]
    return {"bT": bT, "bw": bw, "bop": bop, "rr": rr, "bdep": bdep, "bcw": bcw,
            "rs": bswm / ref["wmid_abs"].clamp_min(TINY)}


def dG_bound(ref, fb, gw, go, gd, extra=0.0):
    """The kernel's error on G_i = g_w + g_opraw + g_D mid (+ ``extra``, the render terms' own rounding)."""
    op, mid, rr = ref["opacity"], ref["mid"], fb["rr"]
    go = torch.zeros_like(op) if go is None else go.double()
    gd = torch.zeros_like(op) if gd is None else gd.double()
    gw = torch.zeros_like(mid) if gw is None else gw.double()
    gD = gd.abs() / op
    gop_mag = go.abs() + gd.abs() * ref["wmid_abs"] / op ** 2
    dgop = U * go.abs() + _safe(fb["rs"] + 2 * rr + 4 * U, gd.abs() * ref["wmid_abs"] / op ** 2)
    inr = ref["in_range"][:, None].double()
    return (4 * U * (gw.abs() + inr * gop_mag + gD * mid.abs()) + _safe(rr + U, gD) * mid.abs() + inr * dgop
            + extra)


def dx_bound(ref, fb, dG):
    """Bound on the kernel's dL/dx_i (module docstring)."""
    S = ref["E"].shape[-1]
    n_ch = (S + 31) // 32
    G, gT, T, w, x = ref["G"], ref["gT"], ref["trans"], ref["weights"], ref["x"]
    ex = torch.exp(-x)
    rex = torch.clamp(torch.expm1(x * U), max=1.0) + 4 * U
    A, B = ref["A"], ref["B"]
    per_k = _safe(G.abs(), fb["bw"]) + dG * w + gT.abs() * fb["bT"]
    widen = torch.flip(nf.exclusive_sum(torch.flip(per_k, [-1])), [-1])
    relT = torch.where(T > 0, fb["bT"] / T.clamp_min(TINY), torch.zeros_like(T))
    return A * (relT + rex + 3 * U) + dG * T * ex + widen + (8 + n_ch) * U * B + U * (A + B) + TINY


# ------------------------------------------------------------------------------------------------ composite
SIZES = [1, 31, 32, 33, 64, 128, 256]
RAYS = [1, 37, 8192 + 5]


def _check_forward(t0, t1, sigma, W, T, O, D, M, Cdf, tag):
    ref = nf.composite64(t0, t1, sigma, W.cpu())
    fb = fwd_bounds(ref)
    _check(f"{tag} trans", T, ref["trans"], fb["bT"])
    _check(f"{tag} weights", W, ref["weights"], fb["bw"])
    _check(f"{tag} opacity", O, ref["opacity"], fb["bop"])
    _check(f"{tag} depth", D, ref["depth"], fb["bdep"])
    if Cdf is not None:
        c = Cdf.cpu()
        _check(f"{tag} cdf", c[:, :-1], ref["cdf"][:, :-1], fb["bT"] + U * ref["cdf"][:, :-1])
        assert (c[:, -1] == 1.0).all()
        dec = c[:, 1:] < c[:, :-1]
        assert not dec.any(), (f"{tag}: cdf falls", int(dec.any(-1).sum()), torch.nonzero(dec)[:4].tolist())
    # median: the fp64 index, or a sample at (or just after) one whose cumulative weight is within its bound of 0.5
    amb = (ref["cw"] - 0.5).abs() <= fb["bcw"]
    allowed = amb.clone()
    allowed[:, 1:] |= amb[:, :-1]
    allowed.scatter_(1, ref["median_idx"][:, None], True)
    hit = (M.cpu().double() == ref["mid"]) & allowed
    assert hit.any(-1).all(), (tag, "median", torch.nonzero(~hit.any(-1))[:4].tolist())
    return ref, fb


@pytest.mark.parametrize("R", RAYS)
@pytest.mark.parametrize("S", SIZES)
def test_composite_forward_per_sample(S, R):
    from emernerf_b200 import _ops

    t0, t1, sigma, _ = make_rays(R, S, seed=S * 7 + R)
    W, T, O, D, M, C = _ops.composite(t0.to(DEV), t1.to(DEV), sigma.to(DEV), want_cdf=True)
    torch.cuda.synchronize()
    _check_forward(t0, t1, sigma, W, T, O, D, M, C, "composite")


DROPS = ["none", "weights", "trans", "opacity", "depth", "cdf"]


def _upstream(R, S, seed, drop):
    g = torch.Generator().manual_seed(seed)
    ups = {"weights": torch.randn(R, S, generator=g), "trans": torch.randn(R, S, generator=g),
           "opacity": torch.randn(R, 1, generator=g), "depth": torch.randn(R, 1, generator=g),
           "cdf": torch.randn(R, S + 1, generator=g)}
    for v in ups.values():
        v[torch.rand(v.shape, generator=g) < 0.1] = 0.0       # exact zeros
    if drop != "none":
        ups[drop] = None
    return ups


@pytest.mark.parametrize("drop", DROPS)
@pytest.mark.parametrize("S,R", [(1, 37), (33, 37), (64, 8192 + 5), (128, 37), (256, 8192 + 5)])
def test_composite_backward_per_sample(S, R, drop):
    from emernerf_b200 import _ops

    t0, t1, sigma, _ = make_rays(R, S, seed=S * 11 + R)
    ups = _upstream(R, S, S + R, drop)
    sg = sigma.to(DEV).requires_grad_(True)
    W, T, O, D, M, C = _ops.composite(t0.to(DEV), t1.to(DEV), sg, want_cdf=True)
    outs = [(W, "weights"), (T, "trans"), (O, "opacity"), (D, "depth"), (C, "cdf")]
    pairs = [(o, ups[k].to(DEV)) for o, k in outs if ups[k] is not None]
    torch.autograd.backward([o for o, _ in pairs], [u for _, u in pairs])
    ref = nf.composite64(t0, t1, sigma, W.detach().cpu(), ups["weights"], ups["trans"], ups["opacity"],
                         ups["depth"], ups["cdf"])
    fb = fwd_bounds(ref)
    dG = dG_bound(ref, fb, ups["weights"], ups["opacity"], ups["depth"])
    bdx = dx_bound(ref, fb, dG)
    bound = ref["delta"] * bdx + U * ref["dsigma"].abs() + TINY
    ok = torch.isfinite(ref["dsigma"]) & torch.isfinite(bound)
    _check(f"composite dsigma drop={drop}", sg.grad, ref["dsigma"], bound, ok)
    finite_rays = torch.isfinite(sigma).all(-1, keepdim=True)
    assert (ok | ~finite_rays).all()


# ------------------------------------------------------------------------------------------------- render
CH = [1, 33, 64, 256]


def render_inputs(combo, R, S, C, seed):
    """The families' t0, t1, sigma and the combo's other inputs; sigma_s / sigma_d split sigma, each exactly 0 on some
    samples; shadow exactly 0 and 1 on some; the overflowed density only on the static combo."""
    fams = FAMILIES if combo == "static" else tuple(f for f in FAMILIES if f != "inf")
    t0, t1, sigma, _ = make_rays(R, S, seed, fams)
    g = torch.Generator().manual_seed(seed + 1)
    rnd = lambda *shape: torch.rand(*shape, generator=g)        # noqa: E731
    have = COMBOS[combo]
    ins = {"sigma": sigma}
    if "sigma_s" in have:
        f = rnd(R, S)
        f[rnd(R, S) < 0.1] = 0.0
        f[rnd(R, S) < 0.1] = 1.0
        ins["sigma_s"] = sigma * f
        ins["sigma_d"] = sigma * (1.0 - f)
    for k in have:
        if k in ("rgb", "rgb_s", "rgb_d"):
            ins[k] = rnd(R, S, 3)
        elif k == "shadow":
            sh = rnd(R, S)
            sh[rnd(R, S) < 0.1] = 0.0
            sh[rnd(R, S) < 0.1] = 1.0
            ins[k] = sh
        elif k == "rgb_sky":
            ins[k] = rnd(R, 3)
        elif k in ("dino", "dino_s", "dino_d"):
            ins[k] = torch.randn(R, S, C, generator=g)
        elif k in ("dino_sky", "dino_pe"):
            ins[k] = torch.randn(R, C, generator=g)
    flows = None
    if "flows" in have:
        buf = torch.randn(R, S, 6, generator=g)
        flows = (buf[..., :3], buf[..., 3:])
    return t0, t1, ins, flows


def _hot(t0, t1, ins, flows, decomposition, grad=False):
    """hotpath.rendering in float64 on the kernel's fp32 interval lengths (t1 := t0 + fl(t1 - t0)).  A one-sample ray
    gets a trailing empty sample (zero length, zero density and values: weight exactly 0), because rendering squeezes
    the density's last axis, as the reference does; it changes no output but the median, and the extras keep it."""
    t0d = t0.double()
    t1d = t0d + (t1 - t0).double()
    leaves = {k: v.double().requires_grad_(grad) for k, v in ins.items()}
    res = {KEYS[k]: (v[..., None] if k == "shadow" else v) for k, v in leaves.items()}
    if flows is not None:
        res["forward_flow"], res["backward_flow"] = (f.double() for f in flows)
    if t0.shape[-1] == 1:
        t0d, t1d = torch.cat([t0d, t1d], -1), torch.cat([t1d, t1d], -1)
        res = {k: v if k in ("rgb_sky", "dino_sky_feat", "dino_pe") else torch.cat([v, torch.zeros_like(v)], 1)
               for k, v in res.items()}
    with torch.set_grad_enabled(grad):
        out = hotpath.rendering(t0d, t1d, res, return_decomposition=decomposition)
    return out, leaves


def _vabs(ins, kind):
    """|v| per sample of the values a render output accumulates ([R, S, C])."""
    d = {k: v.double() for k, v in ins.items()}
    sh = d.get("shadow", torch.zeros_like(d["sigma"]))[..., None]
    if "sigma_s" in d:
        den = d["sigma"] + 1e-6
        rs, rd = (d["sigma_s"] / den)[..., None], (d["sigma_d"] / den)[..., None]
    if kind == "rgb":
        return d["rgb"].abs() if "rgb" in d else rs * d["rgb_s"].abs() * (1 - sh) + rd * d["rgb_d"].abs()
    if kind == "dino":
        return d["dino"].abs() if "dino" in d else rs * d["dino_s"].abs() + rd * d["dino_d"].abs()
    if kind == "shadow_ratio":
        return sh.square()
    raise KeyError(kind)


def _acc_bound(w, bw, vabs, S, sky=None, op=None, bop=None, rounded=()):
    """sum w v (+ sky (1 - op)); ``rounded``: the values after each add that follows the sum (sky, PE)."""
    n_ch = (S + 31) // 32
    gamma = max(S, n_ch + 5) + 7
    b = torch.einsum("rs,rsc->rc", bw + gamma * U * w, vabs)
    if sky is not None:
        b = b + sky.double().abs() * (bop + 2 * U * (1 - op).abs())
    for r in rounded:
        b = b + U * r.abs()
    return b + TINY


@pytest.mark.parametrize("C", CH)
@pytest.mark.parametrize("S,R", [(33, 37), (64, 8192 + 5), (256, 37)])
@pytest.mark.parametrize("combo", list(COMBOS))
def test_render_forward_per_sample(combo, S, R, C):
    from emernerf_b200 import _ops

    if C != 64 and not any(k in COMBOS[combo] for k in ("dino", "dino_s")):
        pytest.skip("the channel count only shapes the feature combos")
    t0, t1, ins, flows = render_inputs(combo, R, S, C, seed=S + R + C)
    dev = {k: v.to(DEV) for k, v in ins.items()}
    fl = None if flows is None else tuple(f.to(DEV) for f in flows)
    decomp = "flows" in COMBOS[combo]
    got = _ops.render(t0.to(DEV), t1.to(DEV), dev, flows=fl, decomposition=decomp)
    ref, fb = _check_forward(t0, t1, ins["sigma"], got["weights"], got["trans"], got["opacity"], got["depth"],
                             got["median_depth"], None, f"render {combo}")
    want, _ = _hot(t0, t1, ins, flows, decomp)
    w, bw = ref["weights"], fb["bw"]
    sky = ins.get("rgb_sky")
    op, bop = ref["opacity"], fb["bop"]
    _check(f"render {combo} rgb", got["rgb"], want["rgb"],
           _acc_bound(w, bw, _vabs(ins, "rgb"), S, sky, op, bop, [want["rgb"]] if sky is not None else []))
    if "shadow_ratio" in got:
        _check(f"render {combo} shadow_ratio", got["shadow_ratio"], want["shadow_ratio"],
               _acc_bound(w, bw, _vabs(ins, "shadow_ratio"), S))
    if "dino" in got:
        dsky = ins.get("dino_sky")
        free = want.get("dino_pe_free", want["dino_feat"])
        b = _acc_bound(w, bw, _vabs(ins, "dino"), S, dsky, op, bop, [free] if dsky is not None else [])
        if "dino_pe_free" in got:
            _check(f"render {combo} dino_pe_free", got["dino_pe_free"], want["dino_pe_free"], b)
            b = b + U * want["dino_feat"].abs()
        _check(f"render {combo} dino", got["dino"], want["dino_feat"], b)
    if decomp:
        checks = decomposition_checks(t0, t1, ins, flows, want, ref, fb)
        assert {k for k, _, _ in checks} == {k for k in got if k in _ops.RENDER_DECOMPOSITION}
        for k, v, b in checks:
            _check(f"render {combo} {k}", got[k], v, b)


def decomposition_checks(t0, t1, ins, flows, want, ref, fb):
    """[(output, float64 value, bound)] for every decomposition output; ``ref`` / ``fb``: composite64 on the kernel's
    weights and its forward bounds."""
    S = t0.shape[-1]
    d = {k: v.double() for k, v in ins.items()}
    w, bw, op, bop = ref["weights"], fb["bw"], ref["opacity"], fb["bop"]
    scans = {}
    for part in ("static", "dynamic"):
        sub = nf.composite64(t0, t1, ins["sigma_s" if part == "static" else "sigma_d"])
        scans[part] = sub, fwd_bounds(sub, kernel_branch=False)
    checks = []
    for part, (sub, sb) in scans.items():
        x = "s" if part == "static" else "d"
        checks.append((f"{part}_opacity", want[f"{part}_opacity"], sb["bop"]))
        checks.append((f"{part}_depth", want[f"{part}_depth"], sb["bdep"] + 2 * U * want[f"{part}_depth"].abs()))
        if "rgb_s" in d:
            sky = d.get("rgb_sky") if part == "static" else None
            checks.append((f"{part}_rgb", want[f"{part}_rgb"],
                           _acc_bound(sub["weights"], sb["bw"], d[f"rgb_{x}"].abs(), S, sky, sub["opacity"],
                                      sb["bop"], [want[f"{part}_rgb"]] if sky is not None else [])))
        if part == "dynamic" and flows is not None:
            for k, f in zip(("forward_flow", "backward_flow"), flows):
                checks.append((k, want[k], _acc_bound(sub["weights"], sb["bw"], f.double().abs(), S)))
        if "dino_s" in d:
            # static_dino's sky term takes the full opacity, static_rgb's the static one (render_utils.py:278-281)
            sky = d.get("dino_sky") if part == "static" else None
            checks.append((f"{part}_dino", want[f"{part}_dino"],
                           _acc_bound(sub["weights"], sb["bw"], d[f"dino_{x}"].abs(), S, sky, op, bop,
                                      [want[f"{part}_dino"]] if sky is not None else [])))
    ws, bws = scans["static"][0]["weights"], scans["static"][1]["bw"]
    if "shadow" in d and "rgb_s" in d:
        sh = d["shadow"][..., None]
        checks.append(("shadow", want["shadow"], _acc_bound(w, bw, sh, S)))
        checks.append(("shadow_reduced_static_rgb", want["shadow_reduced_static_rgb"],
                       _acc_bound(ws, bws, d["rgb_s"].abs() * (1 - sh), S)))
        # acc_so (static weights) + fl(1 - acc_sh) (full weights), then the add
        acc_sh = (w[..., None] * sh).sum(1)
        checks.append(("shadow_only_static_rgb", want["shadow_only_static_rgb"],
                       _acc_bound(ws, bws, d["rgb_s"].abs() * sh, S) + _acc_bound(w, bw, sh, S)
                       + U * (1 - acc_sh).abs() + U * want["shadow_only_static_rgb"].abs()))
    return checks


def backward_checks(t0, t1, ins, ups, W):
    """{input: (float64 gradient, bound, mask)} for every input of the render backward, given the kernel's fp32
    weights W and the upstream gradients ``ups`` of every training output (zeros for one the kernel gets as NULL);
    also returns ``_hot``'s leaves and composite64's output."""
    S = ins["sigma"].shape[-1]
    C = ins["dino"].shape[-1] if "dino" in ins else ins["dino_s"].shape[-1] if "dino_s" in ins else 0
    want, leaves = _hot(t0, t1, ins, None, False, grad=True)
    wref = want["extras"]["weights"]
    wref.retain_grad()
    names = {"weights": None, "trans": None, "dino": "dino_feat"}
    outs = [(want["extras"][k][:, :S] if k in ("weights", "trans") else want[names.get(k, k)], u.double())
            for k, u in ups.items()]
    torch.autograd.backward([o for o, _ in outs], [u for _, u in outs])
    ref = nf.composite64(t0, t1, ins["sigma"], W, ups["weights"], ups["trans"], ups["opacity"], ups["depth"])
    # G and its magnitudes from the render graph (composite64's G lacks the colour / feature terms)
    G = wref.grad[:, :S]
    q = G.abs() * ref["weights"] + ref["gT"].abs() * ref["trans"]
    ref.update(G=G, A=G.abs() * ref["trans"] * torch.exp(-ref["x"]),
               B=torch.flip(nf.exclusive_sum(torch.flip(q, [-1])), [-1]))
    fb = fwd_bounds(ref)
    d = {k: v.double() for k, v in ins.items()}
    gmag = torch.zeros_like(ref["weights"])          # sum |g| |v| of the terms g.v in G, and of d r_s, d r_d
    rmag = torch.zeros_like(ref["weights"])
    grgb = ups["rgb"].double().abs()[:, None, :]
    sh = d.get("shadow", torch.zeros_like(d["sigma"]))
    if "rgb" in d:
        gmag = gmag + (grgb * d["rgb"].abs()).sum(-1)
    if "shadow" in d:
        gmag = gmag + ups["shadow_ratio"].double().abs() * sh.square()
    if "sigma_s" in d:
        den = d["sigma"] + 1e-6
        cs = (grgb * d["rgb_s"].abs()).sum(-1) * (1 - sh)
        cd = (grgb * d["rgb_d"].abs()).sum(-1)
        if "dino_s" in d:
            gF = (ups["dino"].double() + (ups["dino_pe_free"].double() if "dino_pe_free" in ups else 0.0)).abs()
            cs = cs + (gF[:, None, :] * d["dino_s"].abs()).sum(-1)
            cd = cd + (gF[:, None, :] * d["dino_d"].abs()).sum(-1)
        gmag = gmag + (d["sigma_s"] * cs + d["sigma_d"] * cd) / den
        rmag = (d["sigma_s"] * cs + d["sigma_d"] * cd) / den ** 2
    elif "dino" in d:
        gF = (ups["dino"].double() + (ups["dino_pe_free"].double() if "dino_pe_free" in ups else 0.0)).abs()
        gmag = gmag + (gF[:, None, :] * d["dino"].abs()).sum(-1)
    gamma_g = math.ceil(C / 32) + 14
    sky_mag = 0.0
    if "rgb_sky" in d:
        sky_mag = (ups["rgb"].double().abs() * d["rgb_sky"].abs()).sum(-1, keepdim=True)
    if "dino_sky" in d:
        gF = (ups["dino"].double() + (ups["dino_pe_free"].double() if "dino_pe_free" in ups else 0.0)).abs()
        sky_mag = sky_mag + (gF * d["dino_sky"].abs()).sum(-1, keepdim=True)
    inr = ref["in_range"][:, None].double()
    dG = dG_bound(ref, fb, ups["weights"], ups["opacity"], ups["depth"],
                  extra=gamma_g * U * gmag + inr * (C + 5) * U * sky_mag)
    bdx = dx_bound(ref, fb, dG)
    bound = (ref["delta"] * bdx + (fb["bw"] + 2 * gamma_g * U * ref["weights"]) * rmag + U * leaves["sigma"].grad.abs()
             + TINY)
    # rays whose fp32 opacity sum and the float64 one sit on different sides of the clamp: hotpath.rendering takes the
    # float64 branch, the kernel its own (composite64 follows the kernel, so the composite backward test covers them)
    sw64 = ref["weights"].sum(-1)
    same = (((sw64 >= 1e-6) & (sw64 <= 1.0)) == ref["in_range"])[:, None]
    ok = same & torch.isfinite(leaves["sigma"].grad) & torch.isfinite(bound)
    checks = {"sigma": (leaves["sigma"].grad, bound, ok)}

    # the other inputs' gradients: w enters each as the kernel's fp32 weight, |w~ - w| <= bw, |w~| <= wt
    w, bw = ref["weights"], fb["bw"]
    wt = w + bw
    grad = lambda k: leaves[k].grad         # noqa: E731
    g = ups["rgb"].double()
    gF = None
    if C:
        gF = ups["dino"].double() + ups.get("dino_pe_free", torch.zeros_like(ups["dino"])).double()
    if "rgb" in d:
        checks["rgb"] = (grad("rgb"), (bw + U * wt)[..., None] * grgb + TINY, None)
    if "sigma_s" in d:
        rs, rd = d["sigma_s"] / den, d["sigma_d"] / den
        checks["rgb_s"] = (grad("rgb_s"), ((bw + 7 * U * wt) * rs * (1 - sh))[..., None] * grgb + TINY, None)
        checks["rgb_d"] = (grad("rgb_d"), ((bw + 5 * U * wt) * rd)[..., None] * grgb + TINY, None)
        if "shadow" in d:
            checks["shadow"] = (grad("shadow"), 2 * ups["shadow_ratio"].double().abs() * sh * (bw + 3 * U * wt)
                                + rs * (grgb * d["rgb_s"].abs()).sum(-1) * (bw + 9 * U * wt) + TINY, None)
        if "dino_s" in d:
            aF = gF.abs()[:, None, :]
            checks["dino_s"] = (grad("dino_s"), ((bw + 6 * U * wt) * rs)[..., None] * aF + TINY, None)
            checks["dino_d"] = (grad("dino_d"), ((bw + 6 * U * wt) * rd)[..., None] * aF + TINY, None)
        gamma_r = math.ceil(C / 32) + 10
        checks["sigma_s"] = (grad("sigma_s"), (bw + gamma_r * U * wt) * cs / den + TINY, None)
        checks["sigma_d"] = (grad("sigma_d"), (bw + gamma_r * U * wt) * cd / den + TINY, None)
    if "dino" in d:
        checks["dino"] = (grad("dino"), (bw + 2 * U * wt)[..., None] * gF.abs()[:, None, :] + TINY, None)
    # the sky terms follow the kernel's side of the opacity clamp, as composite64 on the kernel's weights does
    op, bop = ref["opacity"], fb["bop"]
    if "rgb_sky" in d:
        checks["rgb_sky"] = (g * (1 - op), g.abs() * (bop + 2 * U * ((1 - op).abs() + bop)) + TINY, None)
    if "dino_sky" in d:
        checks["dino_sky"] = (gF * (1 - op), gF.abs() * (bop + 3 * U * ((1 - op).abs() + bop)) + TINY, None)
    if "dino_pe" in d:
        checks["dino_pe"] = (grad("dino_pe"), torch.zeros_like(gF), None)
    assert set(checks) == set(ins)
    return {k: (v.detach(), b, m) for k, (v, b, m) in checks.items()}, leaves, ref


BWD_UPSTREAMS = ("rgb", "shadow_ratio", "dino", "dino_pe_free", "opacity", "depth", "weights", "trans")


@pytest.mark.parametrize("need,drop", [("sigma", None), ("all", None)] + [("all", k) for k in BWD_UPSTREAMS])
@pytest.mark.parametrize("C", CH)
@pytest.mark.parametrize("S,R", [(1, 37), (33, 37), (64, 8192 + 5), (256, 37)])
@pytest.mark.parametrize("combo", list(COMBOS))
def test_render_backward_per_sample(combo, S, R, C, need, drop):
    """``need``: the inputs whose gradient the launch asks for (the others' d_ pointers NULL); ``drop``: the training
    output without an upstream gradient (its g_ pointer NULL)."""
    from emernerf_b200 import _ops

    feat = any(k in COMBOS[combo] for k in ("dino", "dino_s"))
    if C != 64 and not feat:
        pytest.skip("the channel count only shapes the feature combos")
    if C == 256 and R > 37:
        pytest.skip("float64 feature rows of 8197 x 64 x 256 are 1 GB each")
    if need == "sigma" and R > 37:
        pytest.skip("need='all' checks d_sigma at this size; the launch without the other gradients runs at 37 rays")
    if drop is not None and ((S, R) != (33, 37) or C != (33 if feat else 64)):
        pytest.skip("the NULL-upstream branches are per ray: one partial chunk and channel slot covers them")
    t0, t1, ins, _ = render_inputs(combo, R, S, C, seed=3 * S + R + C)
    dev = {k: v.to(DEV).requires_grad_(need == "all" or k == "sigma") for k, v in ins.items()}
    got = _ops.render(t0.to(DEV), t1.to(DEV), dev)
    if drop is not None and drop not in got:
        pytest.skip(f"{combo} has no {drop} output")
    g = torch.Generator().manual_seed(S + R + C)
    ups = {}
    for k, v in got.items():
        if k != "median_depth":
            u = torch.randn(v.shape, generator=g)
            u[torch.rand(v.shape, generator=g) < 0.1] = 0.0
            ups[k] = u
    sent = [k for k in ups if k != drop]
    torch.autograd.backward([got[k] for k in sent], [ups[k].to(DEV) for k in sent])
    if drop is not None:
        ups[drop] = torch.zeros_like(ups[drop])
    for k, v in dev.items():
        assert (v.grad is not None) == (need == "all" or k == "sigma"), k
    checks, _, _ = backward_checks(t0, t1, ins, ups, got["weights"].detach().cpu())
    for k, (want, bound, mask) in checks.items():
        if dev[k].grad is not None:
            _check(f"render {combo} d_{k} C={C}", dev[k].grad, want, bound, mask)


@pytest.mark.parametrize("combo", list(COMBOS))
def test_render_bwd_writes_exactly_what_is_asked(combo):
    """emer_render_bwd through its C ABI: each requested gradient is written (not accumulated) in full and bit for bit
    as the autograd path's, nothing outside it is touched, a NULL d_ pointer is skipped, and a second launch repeats
    the first bit for bit."""
    import ctypes

    from emernerf_b200 import _lib, _ops

    R, S, C = 37, 33, 33
    t0, t1, ins, _ = render_inputs(combo, R, S, C, seed=5)
    t0, t1 = t0.to(DEV), t1.to(DEV)
    dev = {k: v.to(DEV).requires_grad_(True) for k, v in ins.items()}
    got = _ops.render(t0, t1, dev)
    g = torch.Generator().manual_seed(17)
    ups = {k: torch.randn(v.shape, generator=g).to(DEV) for k, v in got.items() if k != "median_depth"}
    torch.autograd.backward([got[k] for k in ups], list(ups.values()))
    cin = _ops._render_in(t0, t1, {k: v.detach() for k, v in dev.items()}, None)
    pick = torch.Generator().manual_seed(23)
    for trial in range(6):
        keep = [k for k in ins if trial == 0 or torch.rand((), generator=pick).item() < 0.5]
        runs = []
        for _ in range(2):
            bufs = {k: torch.full((R + 3, *ins[k].shape[1:]), math.nan, device=DEV) for k in keep}
            grad = _lib.EmerRenderGrad(**{"g_" + k: u.data_ptr() for k, u in ups.items()},
                                       **{"d_" + k: bufs[k][1:R + 1].data_ptr() for k in keep})
            _lib.call("emer_render_bwd", ctypes.byref(cin), _ops._ptr(got["weights"]), _ops._ptr(got["trans"]),
                      ctypes.byref(grad), _ops._stream())
            torch.cuda.synchronize()
            runs.append(bufs)
        for k in keep:
            a, b = runs[0][k], runs[1][k]
            assert torch.equal(a[1:R + 1], dev[k].grad), (combo, trial, k)
            assert torch.equal(a[1:R + 1], b[1:R + 1]), (combo, trial, k)
            assert torch.isnan(a[0]).all() and torch.isnan(a[R + 1:]).all(), (combo, trial, k)


# ----------------------------------------------------------------------------------------------- accumulate
@pytest.mark.parametrize("grads", ["both", "dw", "dv"])
@pytest.mark.parametrize("S", [1, 33, 64])
@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 8, 9, 64, 256, 300])
def test_accumulate_per_element(C, S, grads):
    from emernerf_b200 import _ops

    R = 37 if C >= 256 else 1029
    g = torch.Generator().manual_seed(C * 1000 + S)
    w = torch.rand(R, S, generator=g)
    w[torch.rand(R, S, generator=g) < 0.1] = 0.0
    v = torch.randn(R, S, C, generator=g) * torch.exp(torch.randn(R, S, 1, generator=g) * 4)
    go = torch.randn(R, C, generator=g)
    wg = w.to(DEV).requires_grad_(grads in ("both", "dw"))
    vg = v.to(DEV).requires_grad_(grads in ("both", "dv"))
    out = _ops.accumulate(wg, vg)
    out.backward(go.to(DEV))
    wd, vd = w.double(), v.double()
    _check(f"accumulate out C={C}", out, torch.einsum("rs,rsc->rc", wd, vd),
           (S + 1) * U * torch.einsum("rs,rsc->rc", wd.abs(), vd.abs()) + TINY)
    if grads in ("both", "dw"):
        gd = go.double()
        _check(f"accumulate dw C={C}", wg.grad, torch.einsum("rc,rsc->rs", gd, vd),
               (min(C, 256) + 1) * U * torch.einsum("rc,rsc->rs", gd.abs(), vd.abs()) + TINY)
    else:
        assert wg.grad is None
    if grads in ("both", "dv"):
        assert torch.equal(vg.grad.cpu(), w[..., None] * go[:, None, :])
    else:
        assert vg.grad is None


def test_accumulate_rejects_257_channels():
    from emernerf_b200 import _lib, _ops

    w = torch.rand(3, 4, device=DEV)
    v = torch.rand(3, 4, 257, device=DEV)
    out = torch.empty(3, 257, device=DEV)
    with pytest.raises(RuntimeError, match="channels 257 out of range"):
        _lib.call("emer_accumulate_fwd", _ops._ptr(w), _ops._ptr(v), _ops._ptr(out), 3, 4, 257, _ops._stream())

"""The proposal levels (emer_prop_level, emer_prop_level_bwd) and the interlevel loss (emer_interlevel_loss) against
float64, sample by sample, on the rays where a transmittance scan goes wrong: exact zeros, faint and saturated samples
on one ray, walls at lanes 0, 31, 32 and 63, an overflowed density, zero-length intervals and the NaN that an infinite
density on one gives, at n in {1, 31, 32, 33, 64, 128, 256} and up to 8192 + 5 rays.

Error bounds (u = 2^-24, u' = 2^-53; i, j, k are samples, c_i = i // 32 the chunk of i, n_ch the chunks of a ray).

* Level forward: cdf_i = 1 - min_{j<=i} T_j, T_j = expf(-E_j).  The scan is the composite's (x = fl(sigma fl(t1 - t0)),
  the prefix E_i = carry + the inclusive sum of the lane below), so the bound is the composite's
  (test_gpu_composite_fp64): |dE_i| <= k_i u E_i, k_i = 7 + c_i, relative to the prefix E_i and not to E_i + x_i;
  bT_i = (expm1(k_i u E_i) + 4 u) T_i; and cdf_i within bT_i + u cdf_i of ``nerfacc_ref.composite64``'s 1 - T_i,
  computed from the kernel's own sigma and t edges.  The running minimum is some T_j, j <= i, with E_j <= E_i, so it
  stays within bT_i.  Every row is non-decreasing, cdf[:, 0] = 0 and cdf[:, n] = 1 exactly; where an infinite density
  meets a zero-length interval (inf * 0) the CDF is NaN from the next sample on, exactly where float64's is.
  The s and t edges are bit-exact against ``nerfacc_ref.importance_sampling``, and so are the next level's, drawn from
  this level's rows by ``emer_pdf_resample`` and by a second ``emer_prop_level``; both are non-decreasing.
  sigma cannot be passed to the forward, so the level's inputs program it: W0 rows 0 and 1 are +e_0 and -e_0, b0 = 0,
  w1 = (1, -1, 0, ...), b1 = beta, so raw = fl(beta + enc_0) and sigma = expf(raw - 1); level 0 of the grid is dense
  (base resolution 16) and painted: a random terrain, walls at a plane the rays cross between two chosen samples, and
  cells whose raw is 100 (sigma = +inf).  A previous level with its mass in a zero-width bin gives zero-length
  intervals.

* Level backward: d_raw_j = S_j delta_j min(sigma_j, e^15), S_j = sum_{k>j} dE_k, dE_k = d_cdf_k T_k (k < n; the
  column n is never read).  The kernel folds dE_k = fl(d_cdf_k fl(expf(-E_k))): |d_cdf_k| bT_k plus one rounding; the
  exclusive suffix sum (the inclusive suffix of the lane above plus the carry) adds 5 levels, n_ch - 1 carries and the
  final add, relative to B_j = sum_{k>j} |d_cdf_k| T_k -- without the sample's own term; then two products.
  |d_raw_j - ref| <= delta_j min(sigma_j, e^15) (sum_{k>j} |d_cdf_k| bT_k + (6 + n_ch) u B_j) + 2 u |d_raw_j|.
  With the programmed W0 / w1 and a level-0 table whose features are non-zero, d_enc[:, 0] equals d_raw bit for bit.
  d_b1 is the per-CTA flush of fp32 per-lane sums of d_raw: within (samples per lane + 5 + 8 + CTAs) u sum |d_raw| of
  the float64 sum of the kernel's own d_raw.

* Interlevel loss: the kernel computes the row in float64, so its d_prop_cdf is within u |d64| (the final cast) plus
  float64 rounding of the restatement ``_interlevel`` (test_gpu_prop_level_grad).  Per row, with cs the running sum of
  the blur slopes, h the running heights and X the knots' span: the slopes' sums are off by e_cs = 2 (K + 8) u' max|cs|
  (each partial sum or window is a difference of two cs), the heights by X e_cs + 2 (K + 8) u' max|h|, the cumulative
  area by X times that + 2 (K + 8) u' max|cdf_r|, and each interpolated q by that + 4 u' (|q| + X max w) -- counted for
  both implementations.  The hinge d = max(dq - dP, 0) inherits e_d = e_q(k) + e_q(k + 1), so
  g_k = -2 d / den - d^2 / den^2 (den = dP + 1e-5) moves by e_d (2 / den + 2 (d + e_d) / den^2) + 8 u' |g_k|, and
  d_prop_cdf_k = g_{k-1} - g_k by the two.  The loss is a sum of terms d^2 / den, each within e_d (2 d + e_d) / den,
  cast to fp32 once per CTA and added by fp32 atomics: (CTAs + 1) u sum terms more.  The rows have no zero-width final
  interval: there the reference's heights are NaN, which the kernel's fmax clamps turn into 0 (not pinned here).

Every bound also carries 2^-126 absolute for subnormal results.

Measured on an H100 80GB HBM3 (700 W power limit): the worst element of each check is 0.50 of its bound for the level
CDF, 0.46 for d_raw, 0.04 for d_b1, 0.98 for d_prop_cdf and 0.04 for the loss value, and the file runs in about 25 s.
The cancellation of the backward's fp32 suffix sum, max B_j / |S_j| over samples with S_j != 0, reaches 7.6e6 on the
random d_cdf rows, 3.3e6 on the rows with exact zeros and 3.4e17 on the telescoping rows the interlevel loss produces:
there d_raw is a small difference of large fp32 terms, and only the absolute bound in B_j holds it.  Against the level
kernel that wrote 1 - expf(-E) without the running minimum, only the monotonicity check fails (15 of the 42 forward
cases, a CDF falling by an ulp on up to 77 rows of 8197).  tests/test_prop_bounds_cpu.py shows on the CPU that these
bounds reject plausible slips.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import adapters, hotpath, nerfacc_ref as nf, tcnn_ref
from test_gpu_composite_fp64 import TINY, U, _check, _report, _safe, fwd_bounds, make_rays
from test_gpu_prop_level_grad import _interlevel

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
U53 = 2.0 ** -53
E15 = float(np.float32(3269017.372472111))          # the kernel's fp32 e^15
SIZES = [1, 31, 32, 33, 64, 128, 256]
RAYS = [1, 37, 8192 + 5]
WALL_LANES = (0, 31, 32, 63)


def suffix_excl(v):
    """sum_{k>j} v_k along the last axis."""
    return torch.flip(nf.exclusive_sum(torch.flip(v, [-1])), [-1])


# ------------------------------------------------------------------------------------------------ forward
def check_cdf(tag, cdf, ref, fb):
    """The level's CDF [R, n+1] against composite64's: per sample within bT + u cdf where float64 is finite, NaN
    exactly where it is NaN, non-decreasing, 0 at the first edge and 1 at the last."""
    c = cdf.detach().cpu()
    n = c.shape[-1] - 1
    want = ref["cdf"][:, :n]
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(c[:, :n]), nan), (tag, "NaN pattern", int((torch.isnan(c[:, :n]) ^ nan).sum()))
    _check(f"{tag} cdf", c[:, :n], want, fb["bT"] + U * want.abs(), ~nan)
    assert (c[:, 0] == 0.0).all() and (c[:, n] == 1.0).all(), (tag, "cdf endpoints")
    dec = c[:, 1:] < c[:, :-1]
    assert not dec.any(), (f"{tag}: cdf falls", int(dec.any(-1).sum()), torch.nonzero(dec)[:4].tolist())


BETA = -60.0                      # b1: raw = BETA + enc_0
I_WALL = 8                        # level-0 grid points i >= I_WALL are the wall
X_WALL = (I_WALL - 0.5) / 15.0    # their plane: fmaf(15, x, 0.5) = I_WALL (level 0: scale 15)
WALL_RAW = (16.0, 22.0, 30.0, 40.0)
INF_RAW = 100.0                   # expf(99) = +inf
KIND, NEAR, FAR = "uniform", 0.0, 0.45
RAY_FAMILIES = ("terrain", "wall", "wall", "wall", "inf", "terrain_zero_length", "inf_zero_length")


def _level_net(inst):
    """A bounded proposal DensityField of the instantiation ``inst`` (8 or 4 levels x 1 feature, or 0: 2 levels x 2
    features, the generic kernel) with the programmed MLP."""
    from emernerf_b200.radiance_fields import build_density_field

    levels, feat, maxres, log2 = {8: (8, 1, 512, 15), 4: (4, 1, 96, 12), 0: (2, 2, 32, 12)}[inst]
    torch.manual_seed(inst + 1)
    net = build_density_field(n_input_dims=3, n_levels=levels, max_resolution=maxres, log2_hashmap_size=log2,
                              n_features_per_level=feat, unbounded=False)
    lin = [m for m in net.base_mlp if isinstance(m, torch.nn.Linear)]
    with torch.no_grad():
        lin[0].weight.zero_()
        lin[0].weight[0, 0], lin[0].weight[1, 0] = 1.0, -1.0
        lin[0].bias.zero_()
        lin[1].weight.zero_()
        lin[1].weight[0, 0], lin[1].weight[0, 1] = 1.0, -1.0
        lin[1].bias.fill_(BETA)
    return net, lin


def _level0_points(geom):
    """(ijk [N, 3], entry index [N]) of every point of the dense level 0."""
    assert not geom.hashed[0] and geom.resolutions[0] == 16
    r = torch.arange(16)
    ijk = torch.stack(torch.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3)
    return ijk, tcnn_ref._level_indices(ijk, geom, 0) + geom.offsets[0]


def _paint(net, seed):
    """Level 0, feature 0: columns (y, z) in blocks of 2 x 2 points, block (by, bz) for points 2 b + 1, 2 b + 2; bz 0, 1
    a terrain of N(0, 120) (raw = -60 + enc_0: exact zeros, faint and saturated samples on one ray), bz 2..5 a wall of raw
    WALL_RAW[bz - 2] from I_WALL on behind empty space (exact zeros and raw in [-90, -70]; the point just before the
    wall exactly empty, so the step from 0 to the wall's density happens within 0.2 % of a cell), bz 6 the same with
    raw 100.  The other levels are random and do not reach raw (their W0 columns are 0)."""
    geom = adapters.spec_from_module(net).geom("xyz")
    ijk, idx = _level0_points(geom)
    g = torch.Generator().manual_seed(seed)
    i, j, k = ijk.unbind(-1)
    bz = (k - 1).clamp(0, 13) // 2
    v = torch.randn(len(idx), generator=g) * 120.0
    empty = torch.where(torch.rand(len(idx), generator=g) < 0.5, torch.full_like(v, -1e5),
                        -30.0 + 20.0 * torch.rand(len(idx), generator=g))
    empty[i == I_WALL - 1] = -1e5
    wall_raw = torch.tensor((0.0, 0.0) + WALL_RAW + (INF_RAW,))[bz]
    v = torch.where(bz >= 2, torch.where(i < I_WALL, empty, wall_raw - BETA), v)
    with torch.no_grad():
        tp = net.xyz_encoder.tcnn_encoding.params
        tp.copy_(torch.randn(tp.shape, generator=g) * 0.5)
        tp.view(-1, geom.n_feat)[idx, 0] = v.to(tp.dtype)
    return geom


def level_inputs(n, R, seed):
    """Previous level, jitter and rays of ``RAY_FAMILIES`` (ray r of family r % 7): per ray (prev_s, prev_cdf [R, 4],
    bias [R], origins, dirs [R, 3], family [R], wall lane [R] or -1).  Rays run along +x through the middle of a
    2 x 2 column block; a wall ray starts where the wall plane falls between its samples p - 1 and p (before sample 0
    for p = 0), p cycling over WALL_LANES below n; the s and t edges it needs are importance_sampling's."""
    g = torch.Generator().manual_seed(seed)
    fam = [RAY_FAMILIES[r % len(RAY_FAMILIES)] for r in range(R)]
    zl = torch.tensor(["zero_length" in f for f in fam])
    prev_s = torch.tensor([0.0, 0.25, 0.75, 1.0]).repeat(R, 1)
    prev_cdf = prev_s.clone()
    prev_s[zl] = torch.tensor([0.0, 0.5, 0.5, 1.0])            # 40 % of the mass in a zero-width bin
    prev_cdf[zl] = torch.tensor([0.0, 0.3, 0.7, 1.0])
    bias = torch.rand(R, generator=g)
    iv, _ = nf.importance_sampling(nf.RayIntervals(prev_s), prev_cdf, n, True, jitter=bias)
    t = hotpath._s_to_t(KIND, iv.vals, NEAR, FAR)
    mid = ((t[:, :-1] + t[:, 1:]) / 2.0).double()
    lanes = [p for p in WALL_LANES if p < n]
    origins = torch.zeros(R, 3, dtype=F64)
    wall_lane = torch.full((R,), -1)
    for r, f in enumerate(fam):
        q = r // len(RAY_FAMILIES)
        by = q % 7
        bz = {"terrain": q % 2, "terrain_zero_length": (q + 1) % 2, "wall": 2 + (q + r) % 4}.get(f, 6)
        origins[r, 1], origins[r, 2] = (2 * by + 1) / 15.0, (2 * bz + 1) / 15.0
        if f.startswith("terrain"):
            origins[r, 0] = 0.05 + 0.45 * torch.rand((), generator=g).item()
        elif f == "inf_zero_length":
            origins[r, 0] = 0.4                                   # the zero-length intervals (t = 0.225) in the wall
        else:
            p = lanes[q % len(lanes)]
            wall_lane[r] = p
            at = mid[r, 0] - 0.25 * FAR / n if p == 0 else (mid[r, p - 1] + mid[r, p]) / 2.0
            origins[r, 0] = X_WALL - at
    dirs = torch.tensor([1.0, 0.0, 0.0]).repeat(R, 1)
    return prev_s, prev_cdf, bias, origins.float(), dirs, fam, wall_lane, iv.vals, t


BOX = torch.tensor([0.0, 0.0, 0.0, 1.0, 1.0, 1.0])


def run_level(inst, n, R, seed):
    """One programmed level on the GPU: returns (inputs, (s, t, cdf, sigma) on the CPU, net, lin)."""
    from emernerf_b200 import _ops

    net, lin = _level_net(inst)
    _paint(net, seed)
    net = net.to(DEV)
    ins = level_inputs(n, R, seed + 1)
    prev_s, prev_cdf, bias, o, d = ins[:5]
    s_min, s_max = hotpath.s_bounds(KIND, NEAR, FAR)
    out = _ops.prop_level(prev_s.to(DEV), prev_cdf.to(DEV), n, bias.to(DEV), s_min, s_max, KIND, o.to(DEV), d.to(DEV),
                          BOX.to(DEV), False, net.xyz_encoder.desc, net.xyz_encoder.tcnn_encoding.params,
                          lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias, want_sigma=True)
    torch.cuda.synchronize()
    return ins, [x.cpu() for x in out], net, lin


def _assert_families(n, R, fam, wall_lane, t, sigma, cdf):
    """Each family the module names occurred."""
    delta = (t[:, 1:] - t[:, :-1]).double()
    x = sigma.double() * delta
    zero, faint, sat = sigma == 0, (x > 0) & (x < 1e-6), torch.isfinite(x) & (x > 5.0)
    terrain = torch.tensor([f.startswith("terrain") for f in fam])
    if n >= 32:
        assert (zero & terrain[:, None]).any() and (faint & terrain[:, None]).any()
        assert (zero.any(-1) & faint.any(-1) & sat.any(-1) & terrain).any(), "terrain: zero, faint and saturated"
    for p in (p for p in WALL_LANES if p < n):
        rows = wall_lane == p
        jump = sigma[rows, p] > 1e6
        if p > 0:
            jump &= sigma[rows, p - 1] == 0
        assert jump.any(), f"no ray with a 0 -> >1e6 jump at lane {p}"
    assert torch.isinf(sigma).any(), "no infinite density"
    if n >= 31:
        assert (delta == 0).any(), "no zero-length interval"
        assert torch.isnan(cdf).any(), "no NaN row (inf * 0)"


@pytest.mark.parametrize("R", RAYS)
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("inst", [8, 4])
def test_level_forward_per_sample(inst, n, R):
    _level_forward(inst, n, R)


def test_level_forward_generic_instantiation():
    _level_forward(0, 64, 37)


def _level_forward(inst, n, R):
    from emernerf_b200 import _ops

    seed = 1000 * inst + 7 * n + R
    ins, (s, t, cdf, sigma), net, lin = run_level(inst, n, R, seed)
    prev_s, prev_cdf, bias, o, d, fam, wall_lane, s_want, t_want = ins
    assert torch.equal(s, s_want) and torch.equal(t, t_want), "s / t edges"
    if R >= 37:
        _assert_families(n, R, fam, wall_lane, t, sigma, cdf)
    ref = nf.composite64(t[:, :-1], t[:, 1:], sigma)
    check_cdf(f"level<{inst}> n={n}", cdf, ref, fwd_bounds(ref))

    # the next level, from the rows this one hands on (no NaN): inverse-CDF draws, alone and fused
    rows = ~torch.isnan(cdf).any(-1)
    s1, c1 = s[rows], cdf[rows]
    b2 = torch.rand(int(rows.sum()), generator=torch.Generator().manual_seed(seed + 2))
    iv, _ = nf.importance_sampling(nf.RayIntervals(s1), c1, n, True, jitter=b2)
    t2_want = hotpath._s_to_t(KIND, iv.vals, NEAR, FAR)
    s_min, s_max = hotpath.s_bounds(KIND, NEAR, FAR)
    s2, t2 = _ops.pdf_resample(s1.to(DEV), c1.to(DEV), n, b2.to(DEV), s_min, s_max, KIND)
    s3, t3, _ = _ops.prop_level(s1.to(DEV), c1.to(DEV), n, b2.to(DEV), s_min, s_max, KIND, o[rows].to(DEV),
                                d[rows].to(DEV), BOX.to(DEV), False, net.xyz_encoder.desc,
                                net.xyz_encoder.tcnn_encoding.params, lin[0].weight, lin[0].bias, lin[1].weight,
                                lin[1].bias)
    for tag, a, want in (("pdf_resample s", s2, iv.vals), ("pdf_resample t", t2, t2_want),
                         ("prop_level s", s3, iv.vals), ("prop_level t", t3, t2_want)):
        a = a.cpu()
        assert torch.equal(a, want), (tag, "not bit-exact", int((a != want).sum()))
        assert (a[:, 1:] >= a[:, :-1]).all(), (tag, "falls")


# ----------------------------------------------------------------------------------------------- backward
def level_bwd64(t, sigma, d_cdf):
    """float64 d_raw [R, n] of the level backward from fp32 t edges [R, n+1], sigma [R, n], d_cdf [R, n+1], with its
    bound, S = sum_{k>j} dE_k and B = sum_{k>j} |d_cdf_k| T_k."""
    n = sigma.shape[-1]
    n_ch = (n + 31) // 32
    ref = nf.composite64(t[:, :-1], t[:, 1:], sigma)
    fb = fwd_bounds(ref)
    dc = d_cdf[:, :n].double()
    T = ref["trans"]
    S = suffix_excl(dc * T)
    B = suffix_excl(dc.abs() * T)
    fold = suffix_excl(_safe(dc.abs(), fb["bT"]))
    m = sigma.double().clamp(max=E15)
    d_raw = S * ref["delta"] * m
    bound = ref["delta"] * m * (fold + (6 + n_ch) * U * B) + 2 * U * d_raw.abs() + TINY
    return {"d_raw": d_raw, "bound": bound, "S": S, "B": B}


D_CDF_KINDS = ("random", "zeros", "telescoping", "nan_last")


def make_d_cdf(R, n, seed):
    """d_cdf [R, n+1] fp32, row r of kind D_CDF_KINDS[r % 4]: N(0, 1); N(0, 1) with 30 % exact zeros; the
    telescoping rows g_{k-1} - g_k, |g| ~ 1e5 on 30 % of the samples, that emer_interlevel_loss gives on near-empty
    proposal intervals; N(0, 1) with NaN in column n.  Column n is 1e3 N(0, 1) elsewhere: never read."""
    g = torch.Generator().manual_seed(seed)
    kind = torch.arange(R) % 4
    d = torch.randn(R, n + 1, generator=g)
    d[(kind == 1)[:, None] & (torch.rand(R, n + 1, generator=g) < 0.3)] = 0.0
    gk = torch.randn(R, n, generator=g) * 1e5 * (torch.rand(R, n, generator=g) < 0.3)
    tele = torch.cat([gk[:, :1], gk[:, 1:] - gk[:, :-1], -gk[:, -1:]], -1)      # d_k = g_{k-1} - g_k, g_{-1} = g_n = 0
    d = torch.where((kind == 2)[:, None], -tele, d)
    d[:, n] = 1e3 * torch.randn(R, generator=g)
    d[kind == 3, n] = math.nan
    return d, kind


def backward_inputs(R, n, seed):
    """make_rays' families as a level's t edges [R, n+1] (fp32 prefix sums of its interval lengths, so zero-length
    intervals stay exactly zero) and sigma [R, n]; on every fifth ray sample n // 2 gets sigma = 5e6 > e^15 on an
    interval of ~1e-6, so that the clamped branch of trunc_exp's backward carries gradient from behind it."""
    t0, t1, sigma, _ = make_rays(R, n, seed)
    e = torch.cat([t0[:, :1].double(), t0[:, :1].double() + torch.cumsum((t1 - t0).double(), -1)], -1).float()
    if n >= 2:
        j = n // 2
        rows = (torch.arange(R) % 5 == 1) & (e[:, j + 1] - e[:, j] > 1e-4)
        e[rows, j + 1] = e[rows, j] + 1e-6
        sigma[rows, j] = 5e6
    return e.contiguous(), sigma


@pytest.mark.parametrize("n,R", [(1, 37), (31, 37), (32, 37), (33, 37), (64, 8192 + 5), (128, 37), (256, 8192 + 5)])
@pytest.mark.parametrize("lf", [8, 4])
def test_level_backward_per_sample(lf, n, R):
    from emernerf_b200 import _lib, _ops
    from test_gpu_prop_level_grad import AABB, _rays

    net, lin = _level_net(lf)
    net.set_aabb(AABB)
    geom = adapters.spec_from_module(net).geom("xyz")
    ijk, idx = _level0_points(geom)
    g = torch.Generator().manual_seed(n + R)
    with torch.no_grad():
        tp = net.xyz_encoder.tcnn_encoding.params
        tp.copy_(torch.randn(tp.shape, generator=g))
        tp[idx] = 1.0 + torch.rand(len(idx), generator=g)      # enc_0 in [1, 2]: d_enc[:, 0] = d_raw
    net = net.to(DEV)
    t, sigma = backward_inputs(R, n, seed=5 * n + R)
    d_cdf, kind = make_d_cdf(R, n, seed=n * R)
    o, d = _rays(R, n + 3, DEV)
    xc = torch.empty(R * n, 3, device=DEV)
    d_enc = torch.empty(R * n, lf, device=DEV)
    dw = [torch.zeros(s, device=DEV) for s in ((64, lf), (64,), (64,), (1,))]
    td, sd, dd = t.to(DEV), sigma.to(DEV), d_cdf.to(DEV)
    box, tab = net.aabb.reshape(-1).contiguous(), net.xyz_encoder.tcnn_encoding.params
    w0, b0, w1 = lin[0].weight.detach(), lin[0].bias.detach(), lin[1].weight.detach().reshape(-1).contiguous()
    _lib.call("emer_prop_level_bwd", ctypes.byref(net.xyz_encoder.desc.c), _ops._ptr(td), _ops._ptr(sd),
              _ops._ptr(dd), n, _ops._ptr(o), _ops._ptr(d), _ops._ptr(box), 1, _ops._ptr(tab), _ops._ptr(w0),
              _ops._ptr(b0), _ops._ptr(w1), _ops._ptr(xc), _ops._ptr(d_enc), *[_ops._ptr(x) for x in dw], R,
              _ops._stream())
    torch.cuda.synchronize()
    got = d_enc[:, 0].reshape(R, n).cpu()
    ref = level_bwd64(t, sigma, d_cdf)
    ok = torch.isfinite(ref["d_raw"]) & torch.isfinite(ref["bound"])
    _check(f"level_bwd<{lf}> d_raw", got, ref["d_raw"], ref["bound"], ok)
    assert (ok | ~torch.isfinite(sigma).all(-1, keepdim=True)).all()

    # the cancellation of the fp32 suffix sum: B / |S| where S != 0, per d_cdf kind
    ratio = torch.where(ref["S"] != 0, ref["B"] / ref["S"].abs(), torch.zeros_like(ref["S"]))
    for k, name in enumerate(D_CDF_KINDS):
        _report(f"B/|S| {name}", ratio[(kind == k)].max().item())

    # d_b1: fp32 per-lane sums, the warp butterfly, shared and global atomics
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = min(-(-R // 8), 3 * sms)
    per_lane = -(-n // 32) * -(-R // (ctas * 8))
    dr = got.double()[ok]
    _check(f"level_bwd<{lf}> d_b1", dw[3].cpu(), dr.sum().reshape(1),
           ((per_lane + 5 + 8 + ctas) * U * dr.abs().sum() + TINY).reshape(1))


# ------------------------------------------------------------------------------------------------ interlevel
IL_FAMILIES = ("clustered", "duplicate_edges", "flat", "dip", "grid")


def _increasing32(v):
    """v [R, m] rounded to fp32 and made strictly increasing by whole ulps, column by column."""
    v = v.float()
    for j in range(1, v.shape[1]):
        v[:, j] = torch.maximum(v[:, j], torch.nextafter(v[:, j - 1], torch.tensor(math.inf)))
    return v


def interlevel_rows(R, m, n1, seed, prop=None):
    """Final rows (s, cdf [R, m]) and proposal rows (prop_s, prop_cdf [R, n1]), row r of IL_FAMILIES[r % 5]:
    sampler-like clustered edges (spacings down to 1e-7, histogram heights up to 1e6, opacity < 1) everywhere, and per
    family duplicate proposal edges; flat runs of the proposal CDF (dP = 0 exactly); a 1-ulp dip in it; final edges on
    a grid of 2^-6 (s - r and s + r tie at r = 2^-5).  ``prop``: (prop_s, prop_cdf) rows
    that replace the proposal rows of the first len(prop_s) rays."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *shape: torch.rand(*shape, generator=g, dtype=F64)        # noqa: E731
    fam = torch.arange(R) % len(IL_FAMILIES)
    sp = torch.exp(math.log(1e-7) + rnd(R, m - 1) * (math.log(3e-2) - math.log(1e-7)))
    s = torch.cat([torch.zeros(R, 1, dtype=F64), torch.cumsum(sp, -1)], -1)
    s = 0.02 + 0.96 * s / s[:, -1:]
    s = _increasing32(s)
    s[fam == 4] = torch.arange(m, dtype=torch.float32) / 64.0           # s_j + 2^-5 = s_{j+4} - 2^-5 exactly
    h = torch.exp(rnd(R, m - 1) * math.log(1e6)) * (rnd(R, m - 1) < 0.7)
    w = h * (s[:, 1:] - s[:, :-1]).double()
    cdf = torch.cat([torch.zeros(R, 1, dtype=F64), torch.cumsum(w, -1)], -1)
    cdf = cdf / cdf[:, -1:].clamp_min(1e-30) * (0.5 + 0.5 * rnd(R, 1))
    cdf = torch.cummax(cdf.float(), -1).values
    # proposal: half the edges near the final edges, half uniform
    pick = (rnd(R, n1 // 2) * m).long().clamp(max=m - 1)
    ps = torch.cat([s.double().gather(1, pick) + (rnd(R, n1 // 2) - 0.5) * 1e-4, rnd(R, n1 - n1 // 2 - 2),
                    torch.zeros(R, 1, dtype=F64), torch.ones(R, 1, dtype=F64)], -1).clamp(0, 1)
    ps = torch.sort(ps, -1).values.float()
    dp = rnd(R, n1 - 1) ** 3
    dp[(fam == 2)[:, None] & (rnd(R, n1 - 1) < 0.4)] = 0.0
    pc = torch.cat([torch.zeros(R, 1, dtype=F64), torch.cumsum(dp, -1)], -1)
    pc = (pc / pc[:, -1:]).float()
    pc = torch.cummax(pc, -1).values
    pc[:, -1] = 1.0
    k = (rnd(R) * (n1 - 3)).long() + 1
    dup = fam == 1
    ps[dup, k[dup] + 1] = ps[dup, k[dup]]
    dip = fam == 3
    pc[dip, k[dip] + 1] = torch.nextafter(pc[dip, k[dip]], torch.tensor(-math.inf))
    if prop is not None:
        q = prop[0].shape[0]
        ps[:q], pc[:q] = prop
    return s.contiguous(), cdf.contiguous(), ps.contiguous(), pc.contiguous(), fam


def _blur_magnitudes(s, cdf, r):
    """Per row: the knot span X, max |cs| (running slope sums), max |h| (running heights), max |cdf_r| and max w of
    the blurred step function, in float64 from the restatement's own formulas (hotpath.blur_stepfun)."""
    s_, c_ = s.double(), cdf.double()
    y = (c_[:, 1:] - c_[:, :-1]) / (s_[:, 1:] - s_[:, :-1])
    xr, xr_idx = torch.sort(torch.cat([s_ - r, s_ + r], -1))
    y1 = (torch.cat([y, torch.zeros_like(y[:, :1])], -1) - torch.cat([torch.zeros_like(y[:, :1]), y], -1)) / (2 * r)
    y2 = torch.cat([y1, -y1], -1).take_along_dim(xr_idx[:, :-1], -1)
    cs = torch.cumsum(y2, -1)
    hs = torch.cumsum((xr[:, 1:] - xr[:, :-1]) * cs, -1)
    w = torch.cat([torch.zeros_like(hs[:, :1]), hs.clamp_min(0)], -1)
    area = 0.5 * (w[:, 1:] + w[:, :-1]) * (xr[:, 1:] - xr[:, :-1])
    mx = lambda v: v.abs().nan_to_num(0.0).max(-1, keepdim=True).values          # noqa: E731
    return xr[:, -1:] - xr[:, :1], mx(cs), mx(hs), area.nan_to_num(0.0).sum(-1, keepdim=True), mx(w)


def interlevel64(s, cdf, ps, pc, r):
    """float64 terms [R, n], d_prop_cdf [R, n1] (of the sum of the terms) and their bounds (module docstring); ``r``
    the fp32 pulse width the kernel sees."""
    pc64 = pc.double().requires_grad_(True)
    terms = _interlevel(s, cdf, ps, pc64, r, reduce=False)
    (d64,) = torch.autograd.grad(terms.sum(), pc64)
    terms = terms.detach()
    K = 2 * s.shape[-1]
    c = 2 * (K + 8) * U53
    X, cs, hs, cr, wmax = _blur_magnitudes(s, cdf, r)
    e_cs = c * cs
    e_w = X * e_cs + c * hs
    e_cr = X * e_w + c * cr
    q = cr.expand(-1, ps.shape[-1])                     # |q| <= cdf_r's total
    e_q = 2 * (e_cr + 4 * U53 * (q + X * wmax))
    e_d = e_q[:, 1:] + e_q[:, :-1]
    dp = (pc[:, 1:].double() - pc[:, :-1].double())
    den = dp + 1e-5
    dd = (terms * den).clamp_min(0).sqrt()               # the hinge d
    gk = -2 * dd / den - dd ** 2 / den ** 2
    e_g = e_d * (2 / den.abs() + 2 * (dd + e_d) / den ** 2) + 8 * U53 * gk.abs()
    zero = torch.zeros_like(e_g[:, :1])
    bd = U * d64.abs() + torch.cat([zero, e_g], -1) + torch.cat([e_g, zero], -1) + TINY
    bterm = e_d * (2 * dd + e_d) / den.abs()
    return {"terms": terms, "d": d64, "bound_d": bd, "bound_term": bterm, "g": gk, "hinge": dd, "den": den}


def interlevel_kernel(s, cdf, ps, pc, r):
    """emer_interlevel_loss on the GPU: (fp32 loss sum, d_prop_cdf [R, n1]) as the kernel writes them."""
    from emernerf_b200 import _lib, _ops

    R, m = s.shape
    n1 = ps.shape[1]
    sd, cd, psd, pcd = (x.to(DEV) for x in (s, cdf, ps, pc))
    total = torch.zeros(1, device=DEV)
    grad = torch.empty(R, n1, device=DEV)
    _lib.call("emer_interlevel_loss", _ops._ptr(sd), _ops._ptr(cd), m, _ops._ptr(psd), _ops._ptr(pcd), n1, float(r),
              _ops._ptr(total), _ops._ptr(grad), R, _ops._stream())
    torch.cuda.synchronize()
    return total.cpu(), grad.cpu()


@pytest.mark.parametrize("r", [0.03, 0.003, 2.0 ** -5])
@pytest.mark.parametrize("R", [37, 8192 + 5])
def test_interlevel_per_element(R, r):
    r32 = float(np.float32(r))
    # part of the proposal rows: the fused level's own wall rays (n = 64)
    ins, (s_a, _, cdf_a, _), _, _ = run_level(8, 64, 37, seed=11)
    walls = ins[6] >= 0
    s, cdf, ps, pc, fam = interlevel_rows(R, 65, 65, seed=R + int(1e4 * r), prop=(s_a[walls], cdf_a[walls]))
    if r == 2.0 ** -5:
        knots = torch.cat([s[fam == 4].double() - r32, s[fam == 4].double() + r32], -1)
        srt = torch.sort(knots, -1).values
        assert (srt[:, 1:] == srt[:, :-1]).any(), "no tie of s - r and s + r"
    assert (ps[:, 1:] == ps[:, :-1]).any() and (pc[:, 1:] == pc[:, :-1]).any() and (pc[:, 1:] < pc[:, :-1]).any()
    ref = interlevel64(s, cdf, ps, pc, r32)
    total, got = interlevel_kernel(s, cdf, ps, pc, r32)
    _check(f"interlevel d_prop_cdf r={r}", got, ref["d"], ref["bound_d"])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = min(-(-R // 4), 8 * sms)
    terms = ref["terms"]
    _check(f"interlevel loss r={r}", total, terms.sum().reshape(1),
           (ref["bound_term"].sum() + (ctas + 1) * U * terms.sum() + TINY).reshape(1))

"""Kernel-level parity (through the C ABI) against the CPU oracle: integer work bit-exact, fp32
within the tolerance written at each check."""
import pytest
import torch

from helpers import rel_err
from oracle import hotpath, nerfacc_ref as nf, tcnn_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"

GRIDS = {
    "3d_f4": (3, (4, 8, 64, 10, 4)),          # dense + hashed levels
    "4d_f4": (4, (4, 4, 32, 10, 4)),
    "3d_f1": (3, (4, 16, 96, 12, 1)),
    "4d_f2": (4, (3, 4, 24, 9, 2)),
    "3d_f4_cfg": (3, (10, 16, 8192, 20, 4)),   # configs/default_config.yaml static grid (indices only)
    "4d_f4_cfg": (4, (10, 32, 8192, 18, 4)),
}


def _grid(name):
    from emernerf_b200.grid_desc import GridDesc

    D, args = GRIDS[name]
    cfg = hotpath.hash_encoder_config(*args)
    return D, GridDesc(D, cfg), tcnn_ref.grid_geometry(D, cfg)


def _points(n, D, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, D, generator=g)
    x[: n // 8, :3] = 0.0               # rejected points are encoded at the origin (Q2)
    x[n // 8: n // 4] = torch.rand(n // 4 - n // 8, D, generator=g).round()   # exact corners 0/1
    if D == 4:
        x[-5:, 3] = 1.0                 # t = 1 is a legal timestamp
    return x


@pytest.mark.parametrize("name", list(GRIDS))
def test_grid_corner_indices_bit_exact(name):
    from emernerf_b200 import _ops

    D, desc, geom = _grid(name)
    x = _points(4096, D)
    got = _ops.grid_indices(x.to(DEV), desc).cpu().long()
    for lvl in range(geom.n_levels):
        want, _, _, _ = tcnn_ref.corner_indices_and_weights(x, geom, lvl)
        assert torch.equal(got[:, lvl, :], want), f"level {lvl}"


@pytest.mark.parametrize("name", ["3d_f4", "4d_f4", "3d_f1", "4d_f2"])
def test_grid_forward_backward_vs_oracle(name):
    from emernerf_b200 import _ops

    D, desc, geom = _grid(name)
    g = torch.Generator().manual_seed(1)
    x = _points(3000, D, seed=3)
    params = torch.randn(geom.n_params, generator=g)
    dy = torch.randn(3000, geom.n_output_dims, generator=g)

    xo = x.clone().requires_grad_(True)
    po = params.clone().requires_grad_(True)
    yo = tcnn_ref.grid_forward(xo, po, geom)
    yo.backward(dy)

    xg = x.to(DEV).requires_grad_(True)
    pg = params.to(DEV).requires_grad_(True)
    yg = _ops.grid_encode(xg, pg, desc)
    yg.backward(dy.to(DEV))
    # forward: same fma chain as the oracle -> equal up to the oracle's double-rounding emulation
    assert (yg.cpu() - yo).abs().max().item() <= 1e-6 * yo.abs().max().item()
    assert (yg.cpu() == yo).float().mean().item() > 0.999
    # table gradient: atomics reorder the fp32 sums
    assert rel_err(pg.grad, po.grad) < 2e-5
    # input gradient (dy/dx through the interpolation weights, tcnn semantics)
    assert rel_err(xg.grad, xo.grad) < 2e-5


def test_grid_full_size_properties():
    """BASELINE config size (8192 x 64 points, 10x4 levels, 2^20 table): properties that do not need
    the oracle -- partition of unity, linearity in the table, and the adjoint identity
    <dy, enc_T(x)> == <grad_T, T> that ties backward to forward."""
    from emernerf_b200 import _ops

    _, desc, _ = _grid("3d_f4_cfg")
    n = 8192 * 64
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.rand(n, 3, device=DEV, generator=g)
    ones = torch.ones(desc.n_params, device=DEV)
    y1 = _ops.grid_encode(x, ones, desc)
    assert (y1 - 1).abs().max().item() < 1e-5
    t1 = torch.randn(desc.n_params, device=DEV, generator=g)
    t2 = torch.randn(desc.n_params, device=DEV, generator=g)
    lin = _ops.grid_encode(x, 0.5 * t1 - 2.0 * t2, desc)
    ref = 0.5 * _ops.grid_encode(x, t1, desc) - 2.0 * _ops.grid_encode(x, t2, desc)
    assert (lin - ref).abs().max().item() < 2e-5
    tp = t1.clone().requires_grad_(True)
    y = _ops.grid_encode(x, tp, desc)
    dy = torch.randn(y.shape, device=DEV, generator=g)
    y.backward(dy)
    lhs = (dy.double() * y.detach().double()).sum()
    rhs = (tp.grad.double() * t1.double()).sum()
    assert abs(lhs - rhs).item() <= 1e-4 * abs(lhs).item() + 1e-2


def test_grid_empty_and_ragged_batches():
    from emernerf_b200 import _ops

    D, desc, geom = _grid("3d_f4")
    p = torch.randn(geom.n_params)
    assert _ops.grid_encode(torch.empty(0, 3, device=DEV), p.to(DEV), desc).shape == (0, geom.n_output_dims)
    for n in (1, 31, 257):
        x = torch.rand(n, 3)
        assert rel_err(_ops.grid_encode(x.to(DEV), p.to(DEV), desc), tcnn_ref.grid_forward(x, p, geom)) < 1e-6


def test_contract_forward_backward_vs_oracle():
    from emernerf_b200 import _ops

    g = torch.Generator().manual_seed(0)
    aabb = torch.tensor([-20.0, -40.0, 0.0, 80.0, 40.0, 20.0])
    pos = torch.randn(5000, 3, generator=g) * torch.tensor([200.0, 150.0, 40.0]) + torch.tensor([30.0, 0.0, 10.0])
    pos[:500] = torch.rand(500, 3, generator=g) * torch.tensor([100.0, 80.0, 20.0]) + torch.tensor([-20.0, -40.0, 0.0])
    t = torch.rand(5000, generator=g)
    for unbounded in (True, False):
        po = pos.clone().requires_grad_(True)
        yo = hotpath.contract_points(po, aabb, unbounded)
        w = torch.randn(5000, 3, generator=g)
        (yo * w).sum().backward()
        pg = pos.to(DEV).requires_grad_(True)
        yg = _ops.contract(pg, aabb.to(DEV), None, unbounded)
        (yg * w.to(DEV)).sum().backward()
        assert torch.equal(yg.cpu(), yo.detach()), "contraction is per-op rounded like torch: bit exact"
        assert rel_err(pg.grad, po.grad) < 1e-5
    y4 = _ops.contract(pos.to(DEV), aabb.to(DEV), t.to(DEV), True)
    assert torch.equal(y4[:, 3].cpu(), t) and torch.equal(y4[:, :3].cpu(), hotpath.contract_points(pos, aabb, True))
    raw = _ops.contract_raw(pos.to(DEV), aabb.to(DEV)).cpu()
    assert torch.equal(raw, hotpath.contract(pos, aabb))


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("k,n_out,act", [(40, 64, 1), (64, 128, 0), (113, 64, 1), (177, 64, 1), (64, 3, 2),
                                        (8, 64, 1), (64, 1, 0), (64, 6, 0), (49, 64, 1), (32, 64, 0),
                                        (116, 64, 1), (180, 64, 1), (40, 192, 0)])
def test_linear_forward_backward_vs_fp32_reference(k, n_out, act, impl, monkeypatch):
    """Plain PyTorch fp32 (CPU) reference of the same layer; tolerance 2e-5 relative (fp32 sums of up
    to 180 terms in a different order).  ``tc`` = wgmma 3xTF32 kernels, ``simt`` = FFMA kernels."""
    from emernerf_b200 import _ops

    monkeypatch.setattr(_ops, "LINEAR_IMPL", impl)
    g = torch.Generator().manual_seed(k * 131 + n_out)
    n = 3000 + k
    x = torch.randn(n, k, generator=g)
    w = torch.randn(n_out, k, generator=g) / k ** 0.5
    b = torch.randn(n_out, generator=g)
    dy = torch.randn(n, n_out, generator=g)
    xo, wo, bo = (t.clone().requires_grad_(True) for t in (x, w, b))
    z = torch.nn.functional.linear(xo, wo, bo)
    yo = torch.relu(z) if act == 1 else (torch.sigmoid(z) if act == 2 else z)
    yo.backward(dy)
    xg, wg, bg = (t.to(DEV).requires_grad_(True) for t in (x, w, b))
    yg = _ops.linear(xg, wg, bg, act)
    yg.backward(dy.to(DEV))
    assert rel_err(yg, yo) < 2e-5
    assert rel_err(xg.grad, xo.grad) < 2e-5
    assert rel_err(wg.grad, wo.grad) < 5e-5
    assert rel_err(bg.grad, bo.grad) < 5e-5


@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_linear_strided_input_rows(impl, monkeypatch):
    from emernerf_b200 import _ops

    monkeypatch.setattr(_ops, "LINEAR_IMPL", impl)
    g = torch.Generator().manual_seed(5)
    full = torch.randn(2777, 128, generator=g)
    w = torch.randn(64, 64, generator=g)
    b = torch.randn(64, generator=g)
    fg = full.to(DEV).requires_grad_(True)
    # no activation here: a ReLU mask can legitimately flip for pre-activations within 1e-6 of zero
    y = _ops.linear(fg[:, 64:], w.to(DEV), b.to(DEV), 0)
    fo = full.clone().requires_grad_(True)
    yo = torch.nn.functional.linear(fo[:, 64:], w, b)
    y.sum().backward(); yo.sum().backward()
    assert rel_err(y, yo) < 2e-5 and rel_err(fg.grad, fo.grad) < 2e-5


def test_linear_wgrad_tc_matches_simt(monkeypatch):
    """wgmma weight gradient (dW^T accumulated in registers over many row tiles) vs the FFMA kernel."""
    from emernerf_b200 import _ops

    g = torch.Generator(device=DEV).manual_seed(3)
    for k, n_out, act in ((177, 64, 1), (64, 128, 0), (40, 64, 1), (64, 3, 2), (256, 128, 0)):
        n = 64 * 1500 + 21
        x = torch.randn(n, k, device=DEV, generator=g)
        w = (torch.randn(n_out, k, device=DEV, generator=g) / k ** 0.5)
        b = torch.randn(n_out, device=DEV, generator=g)
        dy = torch.randn(n, n_out, device=DEV, generator=g)
        grads = {}
        for impl in ("tc", "simt"):
            monkeypatch.setattr(_ops, "LINEAR_WGRAD_IMPL", impl)
            wp, bp = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
            _ops.linear(x, wp, bp, act).backward(dy)
            grads[impl] = (wp.grad, bp.grad)
        assert rel_err(grads["tc"][0], grads["simt"][0]) < 2e-5, (k, n_out)
        assert rel_err(grads["tc"][1], grads["simt"][1]) < 2e-5, (k, n_out)


def test_linear_tc_many_tiles_and_ragged_tail():
    """More tiles than CTAs (persistent loop over several tiles per CTA) and a ragged last tile."""
    from emernerf_b200 import _ops

    g = torch.Generator(device=DEV).manual_seed(11)
    n = 128 * 700 + 37
    x = torch.randn(n, 64, device=DEV, generator=g)
    w = torch.randn(64, 64, device=DEV, generator=g) / 8
    b = torch.randn(64, device=DEV, generator=g)
    y = _ops.linear(x, w, b, 1)
    ref = torch.relu(x.double() @ w.double().t() + b.double()).float()
    assert rel_err(y, ref) < 5e-6


@pytest.mark.parametrize("m1,n", [(2, 128), (129, 64), (65, 64), (33, 16), (17, 7)])
@pytest.mark.parametrize("stratified", [False, True])
def test_pdf_resample_bit_exact(m1, n, stratified):
    """Identical CDFs in -> bit-identical bins, s edges and t edges out (BASELINE: 'bit-exact sample
    indices and ray offsets')."""
    from emernerf_b200 import _ops

    g = torch.Generator().manual_seed(m1 * 7 + n)
    R = 513
    if m1 == 2:
        vals = torch.tensor([[0.0, 1.0]]).repeat(R, 1)
        cdfs = vals.clone()
    else:
        vals = torch.sort(torch.rand(R, m1, generator=g), -1).values
        w = torch.rand(R, m1 - 1, generator=g) ** 4
        w[:, ::5] = 0.0                       # flat CDF stretches (du < 1e-10 branch)
        cdfs = torch.cat([torch.zeros(R, 1), torch.cumsum(w / w.sum(-1, keepdim=True), -1)], -1)
        cdfs[:, -1] = 1.0
    jit = torch.rand(R, 1, generator=g) if stratified else None
    s_min, s_max = hotpath.s_bounds("uniform_lindisp", 0.1, 1000.0)
    bias = jit if stratified else torch.full((R, 1), 0.5)
    _, p0, p1 = nf.importance_sampling_bins(cdfs, n, bias)
    iv, _ = nf.importance_sampling(nf.RayIntervals(vals), cdfs, n, stratified, jitter=jit)
    t_want = hotpath._s_to_t("uniform_lindisp", iv.vals, 0.1, 1000.0)
    s_got, t_got, bins = _ops.pdf_resample(vals.to(DEV), cdfs.to(DEV), n, None if jit is None else jit.to(DEV),
                                           s_min, s_max, "uniform_lindisp", want_bins=True)
    bins = bins.cpu().long()
    assert torch.equal((bins - 1).clamp(0, m1 - 1), p0) and torch.equal(bins.clamp(0, m1 - 1), p1)
    assert torch.equal(s_got.cpu(), iv.vals)
    assert torch.equal(t_got.cpu(), t_want)
    assert (s_got[:, 1:] >= s_got[:, :-1]).all()
    # the fused proposal level draws the same edges from the same CDF rows (whatever its grid and MLP hold)
    _, desc, geom = _grid("3d_f1")
    zeros = lambda *shape: torch.zeros(*shape, device=DEV)
    box = torch.tensor([-1.0, -1.0, -1.0, 1.0, 1.0, 1.0], device=DEV)
    s_pl, t_pl, _ = _ops.prop_level(vals.to(DEV), cdfs.to(DEV), n, None if jit is None else jit.to(DEV), s_min, s_max,
                                    "uniform_lindisp", zeros(R, 3), zeros(R, 3), box, True, desc,
                                    zeros(geom.n_params), zeros(64, 4), zeros(64), zeros(1, 64), zeros(1))
    assert torch.equal(s_pl, s_got) and torch.equal(t_pl, t_got)


@pytest.mark.parametrize("kind", ["uniform", "lindisp", "sqrt", "uniform_lindisp_0"])
def test_pdf_resample_other_warps(kind):
    from emernerf_b200 import _ops

    R, n = 64, 32
    vals = torch.tensor([[0.0, 1.0]]).repeat(R, 1)
    s_min, s_max = hotpath.s_bounds(kind, 0.5, 100.0)
    iv, _ = nf.importance_sampling(nf.RayIntervals(vals), vals.clone(), n, False)
    want = hotpath._s_to_t(kind, iv.vals, 0.5, 100.0)
    _, t = _ops.pdf_resample(vals.to(DEV), vals.to(DEV), n, None, s_min, s_max, kind)
    assert torch.equal(t.cpu(), want)


@pytest.mark.parametrize("S", [64, 128, 16, 45, 1])
def test_composite_forward_backward_vs_oracle(S):
    from emernerf_b200 import _ops

    g = torch.Generator().manual_seed(S)
    R = 300
    edges = torch.sort(torch.rand(R, S + 1, generator=g) * 50, -1).values
    t0, t1 = edges[:, :-1].contiguous(), edges[:, 1:].contiguous()
    sigma = torch.rand(R, S, generator=g) ** 3 * 2
    sigma[:10] = 0.0                                          # empty rays: opacity clamps at 1e-6
    sigma[10:20] *= 50                                        # saturating rays
    so = sigma.clone().requires_grad_(True)
    trans, alphas = nf.render_transmittance_from_density(t0, t1, so)
    w = trans * alphas
    op = nf.accumulate_along_rays(w, None).clamp(1e-6, 1.0)
    mid = (t0 + t1)[..., None] / 2.0
    dep = nf.accumulate_along_rays(w, mid) / op
    cw = torch.cumsum(w, -1)
    mi = torch.searchsorted(cw, torch.full((R, 1), 0.5), side="left").clamp(0, S - 1)
    med = torch.gather(mid[..., 0], -1, mi)
    gw, gt = torch.randn(R, S, generator=g), torch.randn(R, S, generator=g)
    go, gd = torch.randn(R, 1, generator=g), torch.randn(R, 1, generator=g) * 0.1
    cdf_o = 1.0 - torch.cat([trans, torch.zeros_like(trans[..., :1])], -1)
    gc = torch.randn(R, S + 1, generator=g)
    ((w * gw).sum() + (trans * gt).sum() + (op * go).sum() + (dep * gd).sum() + (cdf_o * gc).sum()).backward()

    sg = sigma.to(DEV).requires_grad_(True)
    W, T, O, D, M, C = _ops.composite(t0.to(DEV), t1.to(DEV), sg, want_cdf=True)
    ((W * gw.to(DEV)).sum() + (T * gt.to(DEV)).sum() + (O * go.to(DEV)).sum() + (D * gd.to(DEV)).sum()
     + (C * gc.to(DEV)).sum()).backward()
    tol = 1e-5       # expf differs by ulps between host and device; scan order differs from cumsum
    assert rel_err(W, w) < tol and rel_err(T, trans) < tol and rel_err(O, op) < tol and rel_err(D, dep) < tol
    assert rel_err(C, cdf_o) < tol
    agree = (M.cpu() == med).float().mean().item()
    assert agree > 0.98, agree                                # median index flips only at cw ~= 0.5 ties
    assert rel_err(sg.grad, so.grad) < 5e-5
    # telescoping identity: sum of weights == 1 - T_end*(1 - alpha_end)
    assert torch.allclose(W.sum(-1), 1 - T[:, -1] * torch.exp(-(sg.detach()[:, -1] * (t1 - t0).to(DEV)[:, -1])), atol=1e-5)


@pytest.mark.parametrize("C", [1, 3, 6, 64])
def test_accumulate_forward_backward(C):
    from emernerf_b200 import _ops

    g = torch.Generator().manual_seed(C)
    R, S = 257, 64
    w = torch.rand(R, S, generator=g)
    v = torch.randn(R, S, C, generator=g)
    go = torch.randn(R, C, generator=g)
    wo, vo = w.clone().requires_grad_(True), v.clone().requires_grad_(True)
    nf.accumulate_along_rays(wo, vo).backward(go)
    wg, vg = w.to(DEV).requires_grad_(True), v.to(DEV).requires_grad_(True)
    out = _ops.accumulate(wg, vg)
    out.backward(go.to(DEV))
    assert rel_err(out, nf.accumulate_along_rays(w, v)) < 1e-5
    assert rel_err(wg.grad, wo.grad) < 1e-5 and rel_err(vg.grad, vo.grad) < 1e-6


def test_trunc_exp():
    from emernerf_b200 import _ops

    x = torch.linspace(-20, 25, 1001)
    xo = x.clone().requires_grad_(True)
    hotpath.density_activation(xo).sum().backward()
    xg = x.to(DEV).requires_grad_(True)
    y = _ops.density_activation(xg)
    y.sum().backward()
    assert rel_err(y, hotpath.density_activation(x)) < 1e-6
    assert torch.allclose(xg.grad.cpu(), xo.grad, rtol=2e-6)
    assert xg.grad.max().item() <= float(torch.exp(torch.tensor(15.0))) * (1 + 1e-6)     # clamped backward


@pytest.mark.parametrize("stratified", [False, True])
def test_fused_proposal_level_vs_oracle(stratified):
    """emer_prop_level (resample + march + contraction + grid + MLP + scan in one launch): s/t edges are
    bit-exact against the oracle's importance_sampling, the CDF within 2e-5 (FFMA sums / expf ulps)."""
    import types
    import cases
    from helpers import Golden
    from emernerf_b200 import _ops
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder
    from oracle import adapters

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField, build_density_field=build_density_field)
    _, props = cases.build_models(ns, "static")
    g = Golden("static")
    net = props[1]
    net.load_state_dict(g.tensors("sd/prop1"))
    batch = g.tensors("in/pixel")
    R, n = batch["origins"].shape[0], 32
    gen = torch.Generator().manual_seed(9)
    prev_s = torch.tensor([[0.0, 1.0]]).repeat(R, 1)
    prev_cdf = prev_s.clone()
    jit = torch.rand(R, 1, generator=gen) if stratified else None
    s_min, s_max = hotpath.s_bounds("uniform_lindisp", 0.1, 1000.0)
    iv, _ = nf.importance_sampling(nf.RayIntervals(prev_s), prev_cdf, n, stratified, jitter=jit)
    t = hotpath._s_to_t("uniform_lindisp", iv.vals, 0.1, 1000.0)
    pos = batch["origins"][:, None, :] + batch["viewdirs"][:, None, :] * (t[:, :-1] + t[:, 1:])[..., None] / 2.0
    sd = adapters.cpu_state_dict(net)
    sig = hotpath.density_field_forward(sd, adapters.spec_from_module(net), pos)["density"].squeeze(-1)
    trans, _ = nf.render_transmittance_from_density(t[:, :-1], t[:, 1:], sig)
    cdf_want = 1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], -1)

    net = net.to(DEV)
    lin = [m for m in net.base_mlp if isinstance(m, torch.nn.Linear)]
    s_got, t_got, cdf_got = _ops.prop_level(
        prev_s.to(DEV), prev_cdf.to(DEV), n, None if jit is None else jit.to(DEV), s_min, s_max, "uniform_lindisp",
        batch["origins"].to(DEV), batch["viewdirs"].to(DEV), net.aabb, True, net.xyz_encoder.desc,
        net.xyz_encoder.tcnn_encoding.params, lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias)
    assert torch.equal(s_got.cpu(), iv.vals) and torch.equal(t_got.cpu(), t)
    assert rel_err(cdf_got, cdf_want) < 2e-5
    assert torch.equal(cdf_got[:, -1].cpu(), torch.ones(R))

    # the reference's pipeline hands over NON-contiguous origins (broadcast of c2w[:, :3, -1], pixel_source.py:71);
    # converted copies must outlive the launch (they used to be temporaries whose blocks were reused): slices of an
    # [R, 6] tensor and fp64 rays give the same result as contiguous fp32 ones
    od = torch.cat([batch["origins"], batch["viewdirs"]], -1).to(DEV)
    s2, t2, cdf2 = _ops.prop_level(
        prev_s.to(DEV), prev_cdf.to(DEV), n, None if jit is None else jit.to(DEV), s_min, s_max, "uniform_lindisp",
        od[:, :3], od[:, 3:].double(), net.aabb, True, net.xyz_encoder.desc,
        net.xyz_encoder.tcnn_encoding.params, lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias)
    torch.cuda.synchronize()
    assert torch.equal(s2, s_got) and torch.equal(t2, t_got) and torch.equal(cdf2, cdf_got)


@pytest.mark.parametrize("n_levels,n,R", [(4, 32, 64), (8, 128, 96), (8, 64, 33), (8, 40, 2100)])
def test_fused_proposal_level_backward_vs_oracle(n_levels, n, R):
    """emer_prop_level_bwd (+ emer_grid_bwd for the scatter): gradient of a proposal level's CDF row w.r.t. the hash
    table and the 8->64->1 MLP, against autograd through the oracle's DensityField + transmittance on CPU
    (third_party/nerfacc_prop_net.py:161-170 -> render_utils.py:314-324 -> radiance_field.py:825-841 of the reference).
    The forward of the training form is the no-grad kernel itself (bit-identical samples and CDF).  Every warp of the
    persistent backward handles at most one ray at these sizes (2100 rays need 263 CTAs, fewer than 3 per SM);
    test_gpu_prop_level_grad.py holds the rays-per-warp loop and the benchmark's 8192 rays to fp64."""
    from emernerf_b200 import _ops
    from emernerf_b200.radiance_fields import build_density_field
    from oracle import adapters

    torch.manual_seed(3)
    net = build_density_field(n_input_dims=3, n_levels=n_levels, max_resolution=96 if n_levels == 4 else 512,
                              log2_hashmap_size=12 if n_levels == 4 else 15, n_features_per_level=1, unbounded=True)
    net.set_aabb([-20.0, -20.0, -5.0, 20.0, 20.0, 10.0])
    gen = torch.Generator().manual_seed(5)
    with torch.no_grad():
        net.xyz_encoder.tcnn_encoding.params.copy_(torch.randn(net.xyz_encoder.tcnn_encoding.params.shape, generator=gen) * 0.5)
    origins = torch.randn(R, 3, generator=gen) * 2.0
    dirs = torch.randn(R, 3, generator=gen)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    prev_s = torch.tensor([[0.0, 1.0]]).repeat(R, 1)
    prev_cdf = prev_s.clone()
    jit = torch.rand(R, 1, generator=gen)
    up = torch.randn(R, n + 1, generator=gen)
    s_min, s_max = hotpath.s_bounds("uniform_lindisp", 0.1, 1000.0)

    # oracle, CPU autograd
    iv, _ = nf.importance_sampling(nf.RayIntervals(prev_s), prev_cdf, n, True, jitter=jit)
    t = hotpath._s_to_t("uniform_lindisp", iv.vals, 0.1, 1000.0)
    pos = origins[:, None, :] + dirs[:, None, :] * (t[:, :-1] + t[:, 1:])[..., None] / 2.0
    sd = adapters.cpu_state_dict(net, requires_grad=True)
    sig = hotpath.density_field_forward(sd, adapters.spec_from_module(net), pos)["density"].squeeze(-1)
    trans, _ = nf.render_transmittance_from_density(t[:, :-1], t[:, 1:], sig)
    cdf_want = 1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], -1)
    names = [k for k, _ in net.named_parameters()]
    want = dict(zip(names, torch.autograd.grad((cdf_want * up).sum(), [sd[k] for k in names])))

    net = net.to(DEV)
    lin = [m for m in net.base_mlp if isinstance(m, torch.nn.Linear)]
    args = (prev_s.to(DEV), prev_cdf.to(DEV), n, jit.to(DEV), s_min, s_max, "uniform_lindisp", origins.to(DEV),
            dirs.to(DEV), net.aabb, True, net.xyz_encoder.desc, net.xyz_encoder.tcnn_encoding.params, lin[0].weight,
            lin[0].bias, lin[1].weight, lin[1].bias)
    s0, t0, cdf0 = _ops.prop_level(*args)
    s1, t1, cdf1 = _ops.prop_level_train(*args)
    assert torch.equal(s0, s1) and torch.equal(t0, t1) and torch.equal(cdf0, cdf1)
    assert cdf1.requires_grad and not s1.requires_grad and not t1.requires_grad
    assert rel_err(cdf1, cdf_want) < 2e-5
    (cdf1 * up.to(DEV)).sum().backward()
    got = dict(net.named_parameters())
    for k in names:
        assert got[k].grad is not None, k
        assert rel_err(got[k].grad, want[k]) < 2e-4, (k, rel_err(got[k].grad, want[k]))


@pytest.mark.parametrize("with_emb,extra,front", [(True, 0, 0), (True, 64, 0), (False, 0, 0), (True, 0, 64),
                                                  (False, 64, 32)])
def test_field_tail_forward_backward_vs_torch(with_emb, extra, front):
    """Fused field tail vs the reference's op chain in plain PyTorch (CPU): density, [geo | dir | emb]
    assembly, and the gradients w.r.t. the features and the embedding table."""
    from emernerf_b200 import _ops
    from oracle import hotpath

    g = torch.Generator().manual_seed(2)
    R, S, G, E = 37, 16, 64, 16
    feats = torch.randn(R, S, G + extra, generator=g)
    dirs = torch.randn(R, 3, generator=g)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    idx = torch.randint(0, 11, (R,), generator=g)
    emb = torch.randn(11, E, generator=g)
    g_sig = torch.randn(R, S, generator=g)
    width = G + 33 + (E if with_emb else 0)
    g_in = torch.randn(R, S, width, generator=g)

    fo, eo = feats.clone().requires_grad_(True), emb.clone().requires_grad_(True)
    sig_o = hotpath.density_activation(fo[..., 0])
    h = hotpath.sinusoidal((dirs + 1.0) / 2.0)[:, None, :].expand(R, S, 33)
    parts = [fo[..., :G], h] + ([torch.nn.functional.embedding(idx, eo)[:, None, :].expand(R, S, E)] if with_emb else [])
    in_o = torch.cat(parts, -1)
    ((sig_o * g_sig).sum() + (in_o * g_in).sum()).backward()

    fg, eg = feats.to(DEV).requires_grad_(True), emb.to(DEV).requires_grad_(True)
    res = _ops.field_tail(fg, dirs.to(DEV), idx.to(DEV) if with_emb else None, eg if with_emb else None, G,
                          front=front)
    sig, rgb_in = res[0], res[1]
    assert rgb_in.shape == (R, S, width)
    if front:
        # rows sit behind ``front`` spare columns of the concat buffer handed to the colour head
        catbuf = res[2]
        assert catbuf.shape == (R * S, (front + width + 3) // 4 * 4) and not catbuf.requires_grad
        assert rgb_in.data_ptr() == catbuf.data_ptr() + 4 * front
        assert torch.equal(catbuf[:, front:front + width], rgb_in.reshape(R * S, width))
        assert (catbuf[:, front + width:] == 0).all()
    ((sig * g_sig.to(DEV)).sum() + (rgb_in * g_in.to(DEV)).sum()).backward()
    assert rel_err(sig, sig_o) < 2e-6
    assert rel_err(rgb_in, in_o) < 2e-6          # sinf on device vs host: ulps
    assert torch.equal(rgb_in[..., :G].cpu(), feats[..., :G])
    assert rel_err(fg.grad, fo.grad) < 1e-5
    if with_emb:
        assert rel_err(eg.grad, eo.grad) < 1e-5


@pytest.mark.parametrize("impl", ["stack", "add"])
@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("n", [300, 128 * 70 + 19])
def test_colour_head_chain_skip_variants(impl, shared, n, monkeypatch):
    """The colour head (113 -> 64 -> [64 | 113] -> 64 -> 3, sigmoid; radiance_fields/mlp.py:38-46) through the
    chain in its four bookkeeping variants -- stacked / two-product skip gradient, shared / copied
    concatenation buffer -- against fp64 autograd.  n = 300 runs the CUDA-core layers, the larger n the
    tensor-core ones (3xTF32: ~1e-6).  Rows with a ReLU input within 1e-5 of zero get no upstream gradient:
    there the mask is decided by fp32 rounding, which differs with any summation order (the data has an
    input of 3e-7 against ~1e-6 of rounding in its row)."""
    from emernerf_b200 import _ops

    monkeypatch.setattr(_ops, "SKIP_BWD_IMPL", impl)
    g = torch.Generator().manual_seed(5)
    k0, h = 113, 64
    dims = [(h, k0), (h, h + k0), (3, h)]
    ws = [(torch.randn(o, k, generator=g) / k ** 0.5) for o, k in dims]
    bs = [torch.randn(o, generator=g) * 0.1 for o, _ in dims]
    x = torch.randn(n, k0, generator=g)
    up = torch.randn(n, 3, generator=g)

    wd = [w.double().requires_grad_() for w in ws]
    bd = [b.double().requires_grad_() for b in bs]
    xd = x.double().requires_grad_()
    z1 = xd @ wd[0].t() + bd[0]
    h1 = torch.relu(z1)
    z2 = torch.cat([h1, xd], -1) @ wd[1].t() + bd[1]
    h2 = torch.relu(z2)
    yd = torch.sigmoid(h2 @ wd[2].t() + bd[2])
    ill = (z1.detach().abs() < 1e-5).any(-1) | (z2.detach().abs() < 1e-5).any(-1)
    assert int(ill.sum()) <= 16
    up = up * (~ill).float()[:, None]
    (yd * up.double()).sum().backward()

    wg = [w.to(DEV).requires_grad_() for w in ws]
    bg = [b.to(DEV).requires_grad_() for b in bs]
    catbuf = None
    if shared:
        catbuf = torch.zeros(n, (h + k0 + 3) // 4 * 4, device=DEV)
        catbuf[:, h:h + k0] = x.to(DEV)
        xg = catbuf[:, h:h + k0].detach().requires_grad_()      # same memory, a leaf for dX
        assert xg.data_ptr() == catbuf.data_ptr() + 4 * h
    else:
        xg = x.to(DEV).requires_grad_()
    y = _ops.mlp_chain(xg, wg, bg, _ops.ACT_SIGMOID, 1, catbuf=catbuf)
    (y * up.to(DEV)).sum().backward()
    if shared:
        assert rel_err(catbuf[:, :h], h1.detach()) < 5e-6       # layer 0 wrote into the shared buffer
    assert rel_err(y, yd.detach()) < 5e-6
    assert rel_err(xg.grad, xd.grad) < 2e-5
    for a, b in zip(wg + bg, wd + bd):
        assert rel_err(a.grad, b.grad) < 2e-5


# ----------------------------------------------------------------------------- fused field chain (wgmma, register-resident)
def _chain_reference(enc, rb, S, wb0, bb0, wb1, bb1, w0, w1, w2, b2, c, masks=None):
    """fp64 restatement of the chain.  ``masks`` = the ReLU masks of the kernel's own (saved) activations: with 10^6+
    pre-activations a handful sit within rounding distance of zero, where the fp32 kernel and fp64 disagree about
    relu'(x) -- a different (equally valid) subgradient, O(1) different in that row; the gradient check uses the
    kernel's masks on both sides."""
    d = lambda t: t.double()
    act = (lambda x, i: torch.relu(x)) if masks is None else (lambda x, i: x * masks[i])
    hb = act(d(enc) @ d(wb0).T + d(bb0), 0)
    feats = hb @ d(wb1).T + d(bb1)
    geo = feats[:, :64]
    r = d(rb)[torch.arange(enc.shape[0], device=enc.device) // S]
    h0 = act(geo @ d(w0)[:, c:].T + r[:, :64], 1)
    h1 = act(h0 @ d(w1)[:, :64].T + geo @ d(w1)[:, 64 + c:].T + r[:, 64:], 2)
    rgb = torch.sigmoid(h1 @ d(w2).T + d(b2))
    return _trunc_exp64(feats[:, 0] - 1), rgb, geo, feats[:, 64:], hb, h0, h1


def _trunc_exp64(x):
    """trunc_exp (nerf_utils.py:59-75, as oracle.hotpath.density_activation) in fp64: exp(x) forward, the gradient
    g * exp(min(x, 15))."""
    xd = x.detach()
    return torch.exp(xd) + (x - xd) * torch.exp(xd.clamp(max=15.0))


# (k_enc, n_feat, n, S, c, outputs, enc, clamp).  outputs: which of sigma / rgb / geo / sem enter the loss.  enc: "plain",
# "strided" (a 32-byte-aligned column view of a wider buffer: read in place), "misaligned" (copied first), "nograd",
# "accum" (into an existing .grad).  clamp: bb1[0] += 15.5, so about a fifth of the rows have a density pre-activation
# above 15, where trunc_exp's backward clamps.
_ALL = ("sigma", "rgb", "geo", "sem")
_CHAIN_OLD = [(40, 64, 128 * 6 + 37, 64, 49), (40, 128, 4096, 48, 49), (32, 64, 333, 16, 33), (64, 64, 128 * 300, 64, 49)]
_CHAIN_CASES = [(*t, _ALL, "plain", False) for t in _CHAIN_OLD]
_CHAIN_CASES += [(32, 64, 4096, 32, 33, _ALL, "plain", True), (32, 128, 4096, 64, 49, _ALL, "plain", True),
                 (40, 64, 8192, 64, 49, _ALL, "plain", True), (40, 128, 8192, 64, 49, _ALL, "plain", True),
                 (64, 64, 4096, 128, 33, _ALL, "plain", True), (64, 128, 4096, 32, 49, _ALL, "plain", True),
                 (40, 64, 64 * 100 + 37, 64, 49, _ALL, "plain", True)]              # ragged last ray, fused
_CHAIN_CASES += [(40, 128, 4096, 64, 49, o, "plain", True)
                 for o in (("rgb",), ("sigma",), ("geo",), ("sem",), ("sigma", "geo", "sem"))]
_CHAIN_CASES += [(40, 64, 4096, 64, 49, _ALL, e, False) for e in ("strided", "misaligned", "nograd", "accum")]
_CHAIN_PARAMS = []
for _case in _CHAIN_CASES:
    for _bwd in ("fused", "layers"):
        _k, _f, _n, _S, _c, _o, _e, _cl = _case
        _id = f"{_k}-{_f}-{_n}-{_S}-{_c}"
        if not (_case[:5] in _CHAIN_OLD and _bwd == "fused"):
            _id += f"-{_bwd}-{'+'.join(_o)}-{_e}" + ("-clamp" if _cl else "")
        _CHAIN_PARAMS.append(pytest.param(*_case, _bwd, id=_id))


@pytest.mark.parametrize("k_enc,n_feat,n,S,c,outputs,enc_kind,clamp,chain_bwd", _CHAIN_PARAMS)
def test_field_chain_forward_backward_vs_fp64(k_enc, n_feat, n, S, c, outputs, enc_kind, clamp, chain_bwd, monkeypatch):
    """emer_field_fwd (csrc/field_fused.cu): outputs within 2e-5 of an fp64 restatement of the chain (3xTF32),
    ragged last tile / last ray, both warpgroups and many tiles per CTA; gradients of every input through the op's
    backward within 5e-5 of fp64 autograd, from emer_field_bwd (``chain_bwd`` = fused, where S % 32 == 0 and
    n >= TC_MIN_ROWS) or the layer walk, and the two data paths within 1e-5 of each other (measured on an H100 80GB
    HBM3 at 400 W: at most 9.3e-6 and 1.7e-6; one dropped product of a 3xTF32 stage gives ~5e-4).  Outputs left out
    of the loss reach the backward as None: the weights they alone depend on get None, like fp64 autograd, and the
    semantic rows of wb1 / bb1 stay exactly zero."""
    from emernerf_b200 import _lib, _ops

    monkeypatch.setattr(_ops, "CHAIN_BWD", chain_bwd)
    gen = torch.Generator().manual_seed(k_enc + n)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=gen) * scale).to(DEV)
    R = (n + S - 1) // S
    if enc_kind == "strided":
        src = rnd(n, k_enc + 24, scale=0.5).requires_grad_(True)        # row stride k_enc + 24, first column 32 B in
        enc = src[:, 8:8 + k_enc]
    elif enc_kind == "misaligned":
        src = rnd(n, k_enc + 8, scale=0.5).requires_grad_(True)
        enc = src[:, 1:1 + k_enc]
    else:
        src = enc = rnd(n, k_enc, scale=0.5).requires_grad_(enc_kind != "nograd")
    rb = rnd(R, 128, scale=0.3).requires_grad_(True)
    ws = [rnd(64, k_enc, scale=0.2), rnd(64, scale=0.1), rnd(n_feat, 64, scale=0.15), rnd(n_feat, scale=0.1),
          rnd(64, 64 + c, scale=0.12), rnd(64, 128 + c, scale=0.1), rnd(3, 64, scale=0.2), rnd(3, scale=0.1)]
    if clamp:
        ws[3][0] += 15.5
    ws = [w.requires_grad_(True) for w in ws]
    sigma, rgb, geo, sem = _ops.field_chain(enc, rb, S, ws[:4], ws[4:], want_geo=True)
    want = _chain_reference(enc.detach(), rb.detach(), S, *[w.detach() for w in ws], c)
    assert rel_err(sigma, want[0]) < 2e-5 and rel_err(rgb, want[1]) < 2e-5 and rel_err(geo, want[2]) < 2e-5
    if n_feat == 128:
        assert rel_err(sem, want[3]) < 2e-5
    else:
        assert sem is None
    if enc_kind in ("strided", "misaligned"):                   # read in place, or copied to aligned rows first
        assert (sigma.grad_fn.saved_tensors[0].data_ptr() == enc.data_ptr()) == (enc_kind == "strided")
    saved = [t.clone() for t in sigma.grad_fn.saved_tensors[:4]]        # enc, hb, [h0 | geo], h1 (freed by the backward pass)
    # gradients: a scalar over the chosen outputs
    g_s, g_c, g_g = rnd(n), rnd(n, 3), rnd(n, 64, scale=0.1)
    if clamp:
        assert 0.01 < float((want[0] > 3269017.25).double().mean()) < 0.99
        g_s = g_s / sigma.detach().clamp(1.0, 3269017.25)        # d_sigma * min(sigma, e^15) is O(1) in every row
    used = [o for o in outputs if o != "sem" or n_feat == 128]
    terms = dict(sigma=lambda o: (o[0] * g_s).sum(), rgb=lambda o: (o[1] * g_c).sum(), geo=lambda o: (o[2] * g_g).sum(),
                 sem=lambda o: (o[3] * g_g).sum())
    loss_of = lambda o: sum(terms[k](o) for k in used)
    leaves = ([src] if enc_kind != "nograd" else []) + [rb] + ws
    names = (["enc"] if enc_kind != "nograd" else []) + ["ray_bias", "wb0", "bb0", "wb1", "bb1", "w0", "w1", "w2", "b2"]
    loss = loss_of((sigma, rgb, geo, sem))

    def backward(path, retain):
        monkeypatch.setattr(_ops, "CHAIN_BWD", path)
        rec = []
        _lib.set_profile(lambda name, args: True, rec)
        try:
            if enc_kind == "accum":
                g0 = rnd(n, k_enc)
                src.grad = g0.clone()
                loss.backward(inputs=leaves, retain_graph=retain)
                res = [src.grad - g0] + [t.grad for t in leaves[1:]]
                for t in leaves:
                    t.grad = None
            else:
                res = list(torch.autograd.grad(loss, leaves, retain_graph=retain, allow_unused=True))
        finally:
            _lib.set_profile(None, None)
        launched = {r[0] for r in rec}
        assert ("emer_field_bwd" in launched) == (path == "fused" and S % 32 == 0 and n >= _ops.TC_MIN_ROWS), launched
        assert "emer_field_wgrad" in launched, launched
        return res

    other = backward("layers" if chain_bwd == "fused" else "fused", True)
    got = backward(chain_bwd, False)
    src64 = src.detach().double().requires_grad_(True)
    enc64 = src64 if src is enc else src64[:, 8:8 + k_enc] if enc_kind == "strided" else src64[:, 1:1 + k_enc]
    rb64 = rb.detach().double().requires_grad_(True)
    ws64 = [w.detach().double().requires_grad_(True) for w in ws]
    masks = [(saved[1] > 0).double(), (saved[2][:, :64] > 0).double(), (saved[3] > 0).double()]
    for got_act, want_act in ((saved[1], want[4]), (saved[2][:, :64], want[5]), (saved[3], want[6])):
        assert rel_err(got_act, want_act) < 2e-5               # what the backward pass reads
    r = _chain_reference(enc64, rb64, S, *ws64, c, masks=masks)
    leaves64 = ([src64] if enc_kind != "nograd" else []) + [rb64] + ws64
    want_g = torch.autograd.grad(loss_of(r), leaves64, allow_unused=True)
    errs = {}
    for name, a, o, b in zip(names, got, other, want_g):
        assert (a is None) == (b is None) and (o is None) == (b is None), (name, a is None, o is None, b is None)
        if b is not None:
            errs[name] = (rel_err(a, b), rel_err(a, o))
    print(" ".join(f"{k} {e:.1e}/{p:.1e}" for k, (e, p) in errs.items()))
    for name, (e, p) in errs.items():
        assert e < 5e-5 and p < 1e-5, (name, e, p)
    g = dict(zip(names, got))
    if "rgb" in used:
        # per-ray columns of the head weights belong to the ray-bias product, not to this op
        assert float(g["w0"][:, :c].abs().max()) == 0.0 and float(g["w1"][:, 64:64 + c].abs().max()) == 0.0
    if n_feat == 128 and "sem" not in used:
        assert float(g["wb1"][64:].abs().max()) == 0.0 and float(g["bb1"][64:].abs().max()) == 0.0
    if enc_kind in ("strided", "misaligned"):                     # the columns around the view get no gradient
        off = 8 if enc_kind == "strided" else 1
        rest = torch.cat([g["enc"][:, :off], g["enc"][:, off + k_enc:]], 1)
        assert float(rest.abs().max()) == 0.0


def test_field_chain_inference_writes_no_saves():
    """Under no_grad the op allocates neither the hidden activations nor [h0 | geo] (inference traffic only) and gives
    the same outputs as the training call, with and without the semantic half."""
    from emernerf_b200 import _ops

    gen = torch.Generator().manual_seed(3)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=gen) * scale).to(DEV)
    n, S = 128 * 40, 64
    for n_feat in (64, 128):
        enc, rb = rnd(n, 40, scale=0.5), rnd(n // S, 128, scale=0.3)
        ws = [rnd(64, 40, scale=0.2), rnd(64), rnd(n_feat, 64, scale=0.15), rnd(n_feat), rnd(64, 113, scale=0.12),
              rnd(64, 177, scale=0.1), rnd(3, 64, scale=0.2), rnd(3)]
        with torch.no_grad():
            s0, c0, g0, e0 = _ops.field_chain(enc, rb, S, ws[:4], ws[4:])
        assert g0 is None
        s1, c1, _, e1 = _ops.field_chain(enc.clone().requires_grad_(True), rb, S, ws[:4], ws[4:])
        assert torch.equal(s0, s1) and torch.equal(c0, c1)
        assert (e0 is None and e1 is None) if n_feat == 64 else torch.equal(e0, e1)


# ----------------------------------------------------------------------------- optimizer
def test_fused_adam_matches_torch_adam_on_device():
    """emer_adam_step (csrc/optim.cu) through emernerf_b200.optim.FusedAdam: same gradients in, torch.optim.Adam's
    parameters out (<= 1e-6 after 5 steps: the two differ only in FMA contraction and the fp64 bias corrections),
    gradients zeroed by the step, untouched parameters skipped, ragged block sizes."""
    from emernerf_b200 import _ops
    from emernerf_b200.optim import FusedAdam

    _ops.clear_grad_sinks()
    adam = dict(lr=0.01, eps=1e-15, weight_decay=1e-5, betas=(0.9, 0.99))
    torch.manual_seed(2)
    shapes = ((1 << 21,), (64, 40), (64,), (3, 64), (1000003,), (7,))
    pa = [torch.nn.Parameter(torch.randn(s, device=DEV)) for s in shapes]
    pb = [torch.nn.Parameter(p.detach().clone()) for p in pa]
    idle = torch.nn.Parameter(torch.randn(100, device=DEV))
    idle0 = idle.detach().clone()
    a, b = torch.optim.Adam(pa, **adam), FusedAdam(pb + [idle], **adam)
    for step in range(5):
        for x, y in zip(pa, pb):
            gr = torch.randn_like(x) * (10.0 ** (step - 2))
            x.grad = gr.clone()
            y.grad.add_(gr)
            b._mark(y)
        a.step(); b.step()
        assert all(float(g.abs().max()) == 0.0 for g in b.flat_grads())
    for x, y in zip(pa, pb):
        assert rel_err(y, x) < 1e-6, rel_err(y, x)
    assert torch.equal(idle.detach(), idle0)              # never touched: no update, no weight decay
    _ops.clear_grad_sinks()


# ----------------------------------------------------------------------------- ray generation
def _get_rays_reference(x, y, c2w, intrinsic):
    """datasets/base/pixel_source.py:39-76, restated."""
    cam = torch.nn.functional.pad(torch.stack([(x - intrinsic[:, 0, 2] + 0.5) / intrinsic[:, 0, 0],
                                               (y - intrinsic[:, 1, 2] + 0.5) / intrinsic[:, 1, 1]], dim=-1), (0, 1), value=1.0)
    directions = (cam[:, None, :] * c2w[:, :3, :3]).sum(dim=-1)
    origins = torch.broadcast_to(c2w[:, :3, -1], directions.shape)
    norm = torch.linalg.norm(directions, dim=-1, keepdims=True)
    return origins, directions / (norm + 1e-8), norm


def test_gen_rays_matches_the_reference_formula():
    from emernerf_b200 import raygen, synthetic

    g = torch.Generator().manual_seed(5)
    M, R, Hh, Ww = 600, 8192 + 13, 640, 960
    c2w = torch.eye(4).repeat(M, 1, 1)
    yaw = torch.rand(M, generator=g) * 6.28
    c2w[:, 0, 0], c2w[:, 0, 1], c2w[:, 1, 0], c2w[:, 1, 1] = torch.cos(yaw), -torch.sin(yaw), torch.sin(yaw), torch.cos(yaw)
    c2w[:, :3, 3] = torch.randn(M, 3, generator=g) * 30
    K = torch.tensor([[1030.0, 0, 480.0], [0, 1030.0, 320.0], [0, 0, 1.0]]).repeat(M, 1, 1) * (1 + 0.01 * torch.rand(M, 1, 1, generator=g))
    ts = torch.linspace(0, 1, M)
    idx = torch.randint(0, M, (R,), generator=g)
    y, x = torch.randint(0, Hh, (R,), generator=g), torch.randint(0, Ww, (R,), generator=g)
    out = raygen.train_rays(idx.to(DEV), y.to(DEV), x.to(DEV), c2w.to(DEV), K.to(DEV), Hh, Ww, ts.to(DEV))
    o, d, n = _get_rays_reference(x.float(), y.float(), c2w[idx], K[idx])
    assert torch.equal(out["origins"].cpu(), o)
    assert rel_err(out["viewdirs"], d) < 1e-6 and rel_err(out["direction_norms"], n) < 1e-6
    assert torch.equal(out["pixel_coords"].cpu(), torch.stack([y / Hh, x / Ww], -1))
    assert torch.equal(out["normed_timestamps"].cpu(), ts[idx]) and torch.equal(out["img_idx"].cpu(), idx)
    # the reference's own call shape: per-ray gathered matrices
    o2, d2, n2 = raygen.get_rays(x.float().to(DEV), y.float().to(DEV), c2w[idx].to(DEV), K[idx].to(DEV))
    assert torch.equal(o2, out["origins"]) and torch.equal(d2, out["viewdirs"]) and torch.equal(n2, out["direction_norms"])
    # unit directions
    assert float((out["viewdirs"].norm(dim=-1) - 1).abs().max()) < 1e-6


@pytest.mark.parametrize("k,n,ldx,lddz", [(64, 64 * 1500 + 21, 64, 64), (40, 128 * 700 + 5, 40, 64), (128, 64 * 900 + 63, 128, 64),
                                          (64, 37, 128, 128), (100, 64 * 400, 104, 64), (64, 524288, 128, 128)])
def test_tc_weight_gradient_row_major_operands(k, n, ldx, lddz):
    """emer_linear_tc_bwd_weight (csrc/wgrad_mn.cu: operands read as they lie in memory, row-major X and dZ)
    against fp64: dW and db within 2e-5 of the sum over all rows; ragged last tile, strided
    rows, k not a multiple of 32, accumulation into a non-zero buffer."""
    import ctypes

    from emernerf_b200 import _lib, _ops

    g = torch.Generator(device=DEV).manual_seed(k + n)
    xb = torch.randn(n, ldx, device=DEV, generator=g)
    zb = torch.randn(n, lddz, device=DEV, generator=g)
    x, dz = xb[:, :k], zb[:, :64]
    dw0, db0 = torch.randn(64, k, device=DEV, generator=g), torch.randn(64, device=DEV, generator=g)
    dw, db = dw0.clone(), db0.clone()
    _ops._need_cuda(x)
    _lib.call("emer_linear_tc_bwd_weight", _ops._ptr(x), ldx, _ops._ptr(dz), lddz, _ops._ptr(dw), _ops._ptr(db), n, k, 64,
              _ops._stream())
    want_w = dw0.double() + dz.double().T @ x.double()
    want_b = db0.double() + dz.double().sum(0)
    tol = 2e-5 if n < 200000 else 5e-5               # fp32 accumulation over thousands of row tiles in registers + one partial sum per CTA
    assert rel_err(dw, want_w) < tol, rel_err(dw, want_w)
    assert rel_err(db, want_b) < tol, rel_err(db, want_b)


@pytest.mark.parametrize("k,n_out,n,ldx,lddz", [(64, 3, 40000 + 13, 64, 3), (64, 3, 524288, 64, 4), (64, 1, 9000, 128, 4),
                                                (40, 4, 777, 40, 4), (256, 2, 5000, 256, 2), (37, 3, 4000, 37, 3),
                                                (64, 6, 3000, 64, 8), (64, 3, 5, 64, 3)])
@pytest.mark.parametrize("bias", [True, False])
def test_narrow_weight_gradient(k, n_out, n, ldx, lddz, bias):
    """emer_linear_narrow_bwd_weight (heads with n_out <= 8: sigma, rgb, sky, shadow): dW [n_out, k] and db accumulate
    dZ^T X / column sums of dZ over all rows, against fp64.  Covers the 16-byte-vector kernel (k % 4 == 0, n_out <= 4;
    dZ rows padded to 4 floats or not) and the scalar one (odd k, n_out > 4), strided rows and a ragged row count."""
    from emernerf_b200 import _lib, _ops

    g = torch.Generator(device=DEV).manual_seed(k * 7 + n_out)
    xb = torch.randn(n, ldx, device=DEV, generator=g)
    zb = torch.randn(n, lddz, device=DEV, generator=g)
    x, dz = xb[:, :k], zb[:, :n_out]
    dw0, db0 = torch.randn(n_out, k, device=DEV, generator=g), torch.randn(n_out, device=DEV, generator=g)
    dw, db = dw0.clone(), db0.clone()
    _ops._need_cuda(x)
    _lib.call("emer_linear_narrow_bwd_weight", _ops._ptr(xb), ldx, _ops._ptr(zb), lddz, _ops._ptr(dw),
              _ops._ptr(db) if bias else None, n, k, n_out, _ops._stream())
    want_w = dw0.double() + dz.double().T @ x.double()
    assert rel_err(dw, want_w) < 2e-5, rel_err(dw, want_w)
    if bias:
        assert rel_err(db, db0.double() + dz.double().sum(0)) < 2e-5
    else:
        assert torch.equal(db, db0)


@pytest.mark.parametrize("S,n,R,r", [(64, 128, 300, 0.03), (64, 64, 300, 0.003), (16, 7, 50, 0.03), (128, 256, 40, 0.003),
                                     (1, 1, 9, 0.03), (64, 128, 5000, 0.03)])
def test_interlevel_loss_value_and_gradient_vs_oracle(S, n, R, r):
    """emer_interlevel_loss: one proposal level's anti-aliased interlevel term (blur of the final histogram by merging
    s - r / s + r, piecewise-quadratic cdf, interpolation at the level's edges, hinge) and its gradient w.r.t. the
    level's CDF, against the oracle's restatement of the reference (sort + dense bracketing masks,
    third_party/nerfacc_prop_net.py:22-60,182-240) with autograd, evaluated in fp64.  Edge lists as the sampler
    produces them: sorted, in [0, 1], spacings within a factor 50 of each other (so blurred knots of neighbouring edges
    interleave), a quarter of the rays on the uniform first level.  (With spacings down to 1e-7 the histogram heights
    reach 1e6 and the fp32 reference itself is 2 % off its fp64 evaluation -- the double cumulative sum cancels.)"""
    from emernerf_b200 import _ops

    g = torch.Generator().manual_seed(S * 1000 + n)

    def edges(k):
        inc = torch.rand(R, k, generator=g) ** 2 + 0.02
        e = torch.cat([torch.zeros(R, 1), torch.cumsum(inc, -1)], -1)
        e = e / e[:, -1:]
        e[: R // 4] = torch.linspace(0, 1, k + 1)[None]
        e[:, -1] = 1.0
        return e

    def cdf_rows(k):
        w = torch.rand(R, k, generator=g) ** 4 + 1e-6
        w[R // 2:, : k // 2] *= 1e-4                                      # mass far away: flat beginnings
        c = torch.cat([torch.zeros(R, 1), torch.cumsum(w, -1)], -1)
        return c / c[:, -1:] * torch.rand(R, 1, generator=g)              # opacity < 1
    s, cdf, ps, pc = edges(S), cdf_rows(S), edges(n), cdf_rows(n)

    s64, cdf64, ps64 = s.double(), cdf.double(), ps.double()
    pc_o = pc.double().requires_grad_()
    w_n = (cdf64[:, 1:] - cdf64[:, :-1]) / (s64[:, 1:] - s64[:, :-1])
    c, w = hotpath.blur_stepfun(s64, w_n, r)
    area = 0.5 * (w[:, 1:] + w[:, :-1]) * (c[:, 1:] - c[:, :-1])
    cd = torch.cat([torch.zeros_like(area[:, :1]), torch.cumsum(area, -1)], -1)
    wp = pc_o[:, 1:] - pc_o[:, :-1]
    w_s = torch.diff(hotpath.sorted_interp_quad(ps64, c, w, cd), dim=-1)
    want = ((w_s - wp).clamp_min(0) ** 2 / (wp + 1e-5)).mean()
    (want_g,) = torch.autograd.grad(want * 3.0, pc_o)

    pc_g = pc.to(DEV).requires_grad_()
    got = _ops.interlevel_loss(s.to(DEV), cdf.to(DEV), ps.to(DEV), pc_g, r)
    (got * 3.0).backward()
    assert got.dim() == 0
    assert abs(got.item() - want.item()) <= 1e-4 * abs(want.item()), (got.item(), want.item())
    assert rel_err(pc_g.grad, want_g) < 2e-4, rel_err(pc_g.grad, want_g)
    # no gradient wanted: the value alone
    alone = _ops.interlevel_loss(s.to(DEV), cdf.to(DEV), ps.to(DEV), pc.to(DEV), r)
    assert abs(alone.item() - want.item()) <= 1e-4 * abs(want.item())

"""The hash grid's input gradient (grid_bwd_dx_kernel) and ``grid_encode_rows`` against float64.

The flow variants learn their scene flow through this gradient: the loss reaches the dynamic features at the
flow-warped points and goes on through the grid's input gradient, the flow warp and the flow field.  Tested here at the
grids that take it in training -- the dynamic grid (4-D, 10 levels x 4 features, base 32, max 8192, 2^18 entries per
level) and the flow grid (base 16, max 4096), both read from the model builder -- and at the proposal-sized 3-D grids
and the small grids of every (D, F) the library instantiates.

Error bounds.  dx_d of a row is an fp32 evaluation of sum_l scale_l sum_{c: bit d clear} prod_{e != d} w_e
(s_{c|d} - s_c), s_c = <dy_l, table[idx_c]>.  To first order in u = 2^-24 its error is at most gamma u mag_d, where
mag_d is the same sum over |dy_l| . |table[idx]| of both corners (``tcnn_ref.grid_input_grad64``) and
gamma = F (the dot product's fmas) + 1 (the difference) + 2 (D - 1) (the weight product and the roundings of 1 - w)
+ 2^(D-1) (a level's fmas) + L (the sum over levels).  gamma is at most 29 for every grid here (D = 4, F = 4, L = 10),
so every row and component is held to C_DX = 32 u mag.  The reference's cells, fractions and corner indices are the
kernel's bit for bit, and its own rounding (about 2^-53 mag) is negligible.  A table entry that receives K
contributions is an fp32 sum of K rounded products in the order the atomics land: at most K u sum |w dy| to first
order, held to C_TAB (K + 1) u (sum |w dy| + |g0|), g0 a gradient already in the buffer.

Measured on an H100 80GB HBM3 (700 W power limit): the worst input-gradient row is 4.6 u mag (of 32), the worst
table entry 0.91 of its bound (a pre-filled optimizer buffer), and the file runs in about 35 s.
"""
import functools

import pytest
import torch

from helpers import rel_err
from oracle import hotpath, tcnn_ref
from test_gpu_flow_branch import AABB, _contract64, _warp_inputs
from test_gpu_layer_instantiations import GRID_CASES

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
C_DX = 32
C_TAB = 1
N_BIG = (1 << 20) + 17
TD = 0.1                                      # the warp's time step: large enough that the time clamp bites often

SMALL = {f"small_{D}d_f{F}": (D, args) for (D, F), args in GRID_CASES.items()}
PROP = {"prop_512": (3, (8, 16, 512, 20, 1)), "prop_2048": (3, (8, 16, 2048, 20, 1))}     # configs.py propnet


@functools.lru_cache(maxsize=None)
def _model_grids():
    """The encoding configs of the flow variants' dynamic and flow grids, as the model builder makes them."""
    from emernerf_b200 import configs
    from emernerf_b200.radiance_fields import build_radiance_field_from_cfg

    field = build_radiance_field_from_cfg(configs.make_cfg("flow").nerf.model, verbose=False)
    return {"dynamic": field.dynamic_xyz_encoder.encoding_config, "flow": field.flow_xyz_encoder.encoding_config}


def _grid(name):
    from emernerf_b200.grid_desc import GridDesc

    if name in ("dynamic", "flow"):
        D, cfg = 4, _model_grids()[name]
    else:
        D, args = {**SMALL, **PROP}[name]
        cfg = hotpath.hash_encoder_config(*args)
    return D, GridDesc(D, cfg), tcnn_ref.grid_geometry(D, cfg)


def _report(check, worst, bound, re=None):
    """One line per check for the test log: the worst observed error in units of its bound's scale."""
    print(f"\n[{check}] worst {worst:.3g} (bound {bound})" + ("" if re is None else f", rel err {re:.3g}"))


# ----------------------------------------------------------------------------------------------- inputs
def _face_rows(D, geom, m, g):
    """m rows with coordinates on a cell face of a random level: fmaf(scale, x, 0.5) integral, so w = 0 there and the
    derivative is the one-sided one of the kernel's cell.  One dimension per row in the first half, all of them in
    the second; x is the first of the fp32 values around (k - 0.5) / scale whose fma lands on the integer."""
    x = torch.rand(m, D, generator=g)
    every = (torch.arange(m) >= m // 2)[:, None] | torch.nn.functional.one_hot(
        torch.randint(0, D, (m,), generator=g), D).bool()
    sc = torch.tensor(geom.scales, dtype=torch.float32)[torch.randint(0, geom.n_levels, (m, D), generator=g)]
    k = (torch.rand(m, D, generator=g) * sc.floor()).floor() + 1                      # 1 .. floor(scale)
    up = dn = ((k.double() - 0.5) / sc.double()).float()
    cands = [up]
    for _ in range(3):
        up, dn = torch.nextafter(up, torch.full_like(up, 2.0)), torch.nextafter(dn, torch.full_like(dn, -1.0))
        cands += [up, dn]
    cands = torch.stack(cands, -1)                                                     # [m, D, 7]
    pos = tcnn_ref._fma32(sc[..., None].expand_as(cands), cands, torch.full_like(cands, 0.5))
    hit = pos == pos.floor()
    pick = cands.gather(-1, hit.float().argmax(-1, keepdim=True))[..., 0]
    on_face = every & hit.any(-1)
    x = torch.where(on_face, pick, x)
    assert on_face.any(-1).float().mean() > 0.9
    return x


def _points(D, geom, n, seed):
    """n rows: rows on cell faces, at x = 1 (single coordinates and whole rows), uniform rows and rows with xyz = 0 (a
    point the in-cube selector rejected), then the flow warp's output for _warp_inputs (both warps; t exactly 0 and 1
    where the time clamp bites; points on the contraction's faces).  3-D grids take the xyz columns."""
    from emernerf_b200 import _ops

    g = torch.Generator().manual_seed(seed)
    face = _face_rows(D, geom, 8192, g)
    ones = torch.rand(1024, D, generator=g)
    ones[torch.rand(1024, D, generator=g) < 0.5] = 1.0
    ones[:64] = 1.0
    origin = torch.rand(1024, D, generator=g)
    origin[:, :3] = 0.0
    special = torch.cat([face, ones, torch.rand(4096, D, generator=g), origin])
    nw = (n - special.shape[0] + 1) // 2
    pos, flow, noise, t = (v.to(DEV) for v in _warp_inputs(nw, seed))
    warped = _ops.flow_warp(pos, flow, noise, t, torch.tensor(AABB, device=DEV), TD, True)
    x = torch.cat([special.to(DEV), warped[:, :D]])[:n].contiguous()
    if D == 4:
        assert (x[:, 3] == 0).any() and (x[:, 3] == 1).any()
    assert ((x[:, :3] == 0).all(-1)).sum() >= 1024
    return x


def _dy(n, geom, seed):
    """Upstream gradient with whole levels zero (the kernel skips such a level), single zero components within a level
    and rows with no gradient at all (their dx is exactly zero)."""
    g = torch.Generator().manual_seed(seed)
    L, F = geom.n_levels, geom.n_feat
    dy = torch.randn(n, L, F, generator=g)
    r = torch.arange(n)
    dy[r % 3 == 0, (r[r % 3 == 0] // 3) % L] = 0.0
    dy[r % 7 == 4, : L // 2] = 0.0
    s = r[r % 5 == 1]
    dy[s, torch.randint(0, L, s.shape, generator=g), torch.randint(0, F, s.shape, generator=g)] = 0.0
    dy[r % 11 == 2] = 0.0
    return dy.view(n, L * F).to(DEV)


def _check_dx(check, got, want, mag):
    """Every row and component within C_DX u mag, and 1e-5 of the max-abs overall; returns the worst ratio."""
    err = (got.double() - want).abs()
    bad = err > C_DX * U * mag
    if bad.any():
        i = int(bad.any(-1).nonzero()[0])
        pytest.fail(f"{check}: {int(bad.any(-1).sum())} rows beyond {C_DX} u mag; row {i}: got {got[i].tolist()} "
                    f"want {want[i].tolist()} mag {mag[i].tolist()}")
    re = rel_err(got, want)
    assert re <= 1e-5, (check, re)
    live = mag > 0
    return (err[live] / (U * mag[live])).max().item() if live.any() else 0.0, re


def _check_table(check, got, want, mag, count, g0=None):
    """Every entry within C_TAB (K + 1) u (sum |w dy| + |g0|) of its K contributions and the gradient g0 already in the
    buffer, entries no corner reaches untouched, and 2e-5 of the max-abs overall; returns the worst ratio."""
    got = got.double()
    base = torch.zeros_like(want) if g0 is None else g0.double()
    err = (got - base - want).abs()
    scale = (count + 1) * U * (mag + base.abs())
    bad = err > C_TAB * scale
    assert not bad.any(), (check, int(bad.sum()), (err / scale.clamp_min(1e-300)).max().item())
    assert torch.equal(got[count == 0], base[count == 0]), check
    re = rel_err(got, base + want)
    assert re <= 2e-5, (check, re)
    live = count > 0
    return (err[live] / scale[live].clamp_min(1e-300)).max().item(), re


# ----------------------------------------------------------------------------------------------- 1. input gradient
@pytest.mark.parametrize("name", ["dynamic", "flow"] + list(PROP) + list(SMALL))
def test_grid_input_grad_vs_fp64(name):
    """emer_grid_bwd with dx only (x requires grad, the table does not) in every (D, F) instantiation, at 2^20 + 17 rows
    and at ragged prefixes of them."""
    from emernerf_b200 import _ops

    D, desc, geom = _grid(name)
    seed = sum(map(ord, name))
    x = _points(D, geom, N_BIG, seed)
    params = (torch.randn(geom.n_params, generator=torch.Generator().manual_seed(seed)) * 0.3).to(DEV)
    dy = _dy(N_BIG, geom, seed + 1)
    want, mag = tcnn_ref.grid_input_grad64(x, params, dy, geom)
    assert (mag == 0).all(-1).sum() >= N_BIG // 11
    worst = 0.0
    for m in (1, 31, 257, N_BIG):
        xg = x[:m].clone().requires_grad_(True)
        _ops.grid_encode(xg, params, desc).backward(dy[:m])
        assert xg.grad.shape == (m, D)
        w, re = _check_dx(f"{name} n={m}", xg.grad, want[:m], mag[:m])
        worst = max(worst, w)
    _report(f"dx {name}", worst, C_DX, re)


# ----------------------------------------------------------------------------------------------- 2. grid_encode_rows
def _rows_inputs(D, n, seed):
    """x_fixed: n ray-major rows (64 samples per ray, in ray order as the renderer feeds them) = [contract(pos) | t];
    x_var: their forward and backward flow warps.  A quarter of the rows have flow = 0 (the warped row has the current
    row's xyz cells) and an eighth noise = 0 as well (the warped row IS the current row)."""
    from emernerf_b200 import _ops

    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(AABB[:3]), torch.tensor(AABB[3:])
    rays = (n + 63) // 64
    o = lo + (hi - lo) * (torch.rand(rays, 1, 3, generator=g) * 2 - 0.5)
    d = torch.nn.functional.normalize(torch.randn(rays, 1, 3, generator=g), dim=-1)
    s = torch.sort(torch.rand(rays, 64, 1, generator=g), dim=1).values * torch.rand(rays, 1, 1, generator=g) * 60
    pos = (o + d * s).reshape(-1, 3)[:n].contiguous()
    t = torch.rand(rays, 1, generator=g).expand(rays, 64).reshape(-1)[:n].contiguous()
    flow = torch.randn(n, 6, generator=g) * 2
    noise = torch.rand(n, generator=g)
    r = torch.arange(n)
    flow[r % 4 == 0] = 0.0
    noise[r % 8 == 0] = 0.0
    aabb = torch.tensor(AABB, device=DEV)
    pos, t = pos.to(DEV), t.to(DEV)
    cur = _ops.contract(pos, aabb, t, True)
    warped = _ops.flow_warp(pos, flow.to(DEV), noise.to(DEV), t, aabb, TD, True)
    same = (warped[:n] == cur).all(-1)
    assert same.sum() >= n // 8 and (warped[:n, :3] == cur[:, :3]).all(-1).sum() >= n // 4
    return cur[:, :D].contiguous(), warped[:, :D].contiguous()


ROWS_CASES = {
    # name: (N0, N1, flags)
    "branch": (64 * 129, 2 * 64 * 129, ()),         # the fused flow branch: N current rows, 2N warped rows
    "n0_zero": (0, 64 * 97 + 5, ()),
    "n1_zero": (64 * 97 + 5, 0, ()),
    "odd_n0": (64 * 97 + 3, 2 * 64 * 97 + 3, ()),
    "dy_strided": (64 * 65 + 1, 2 * 64 * 65 + 1, ("strided",)),
    "no_table_grad": (64 * 65, 2 * 64 * 65, ("frozen",)),
    "sink": (64 * 65 + 7, 2 * 64 * 65 + 7, ("sink",)),
}


@pytest.mark.parametrize("case", list(ROWS_CASES))
@pytest.mark.parametrize("name", ["dynamic", "small_4d_f2", "small_3d_f4"])
def test_grid_encode_rows_vs_fp64(name, case):
    """grid_encode_rows(x_fixed, x_var): the forward is grid_encode of the stacked rows bit for bit; the table gradient
    is the scatter of ALL N0 + N1 rows, the input gradient is x_var's alone ([N1, D]) and x_fixed takes none even when
    it requires grad.  small_4d_f2 (24-byte rows of dy) and small_3d_f4 (12-byte rows of x) put the x_var half off a
    16-byte boundary when N0 is odd."""
    from emernerf_b200 import _ops
    from emernerf_b200.optim import FusedAdam

    n0, n1, flags = ROWS_CASES[case]
    D, desc, geom = _grid(name)
    seed = sum(map(ord, name + case))
    cur, warped = _rows_inputs(D, max(n0, (n1 + 1) // 2), seed)
    xf = cur[:n0].clone().requires_grad_(True)
    xv = warped[:n1].clone().requires_grad_(True)
    g = torch.Generator().manual_seed(seed)
    p0 = (torch.randn(geom.n_params, generator=g) * 0.3).to(DEV)
    g0 = None
    if "frozen" in flags:
        p = p0
    elif "sink" in flags:
        p = torch.nn.Parameter(p0.clone())
        FusedAdam([p], lr=1e-3)
        sink = p.grad
        g0 = torch.randn(geom.n_params, generator=g).to(DEV)
        sink.copy_(g0)
    else:
        p = p0.clone().requires_grad_(True)
    y = _ops.grid_encode_rows(xf, xv, p, desc)
    x_all = torch.cat([cur[:n0], warped[:n1]])
    assert torch.equal(y, _ops.grid_encode(x_all, p0, desc))

    dy = _dy(n0 + n1, geom, seed)
    if "strided" in flags:
        wide = torch.randn(n0 + n1, geom.n_output_dims + 8, generator=g).to(DEV)
        wide[:, 3:3 + geom.n_output_dims] = dy
        dy = wide[:, 3:3 + geom.n_output_dims]
        assert not dy.is_contiguous()
    y.backward(dy)

    assert xf.grad is None
    assert xv.grad is not None and xv.grad.shape == (n1, D)
    if n1:
        want, mag = tcnn_ref.grid_input_grad64(warped[:n1], p0, dy[n0:], geom)
        worst, re = _check_dx(f"rows {name} {case} dx", xv.grad, want, mag)
        _report(f"rows dx {name} {case}", worst, C_DX, re)
    if "frozen" in flags:
        return
    if "sink" in flags:
        assert p.grad.data_ptr() == sink.data_ptr()
    want, mag, count = tcnn_ref.grid_table_grad64(x_all, dy, geom)
    worst, re = _check_table(f"rows {name} {case} table", p.grad, want, mag, count, g0)
    _report(f"rows table {name} {case}", worst, C_TAB, re)


# ----------------------------------------------------------------------------------------------- 3. warp -> encodings
def test_warp_to_encoding_segment_vs_fp64():
    """The flow branch's segment between the flow field's output and the chain's input, at training size (8192 rays x 64
    samples) with the two model grids: a leaf flow [N, 6] through flow_warp (training noise), the warped rows through
    grid_encode_rows on the dynamic table (current rows [contract(pos) | t]) and grid_encode on the flow table, each
    projected by a fixed random matrix and weighted by a random upstream gradient.  The gradients of the flow, of the
    dynamic table and of the flow table against float64: the grid at the fp32 warped points the kernel produced, the
    contraction's Jacobian at the fp32 point flow_warp forms first (as test_flow_warp_matches_fp64), the rows where
    fp32 and fp64 disagree on the arg-max coordinate or the in-cube selector counted rather than compared."""
    from emernerf_b200 import _ops

    n = 8192 * 64
    _, desc_d, geom_d = _grid("dynamic")
    _, desc_f, geom_f = _grid("flow")
    pos, flow, noise, t = _warp_inputs(n, seed=5)
    g = torch.Generator().manual_seed(6)
    p_d = (torch.randn(geom_d.n_params, generator=g) * 0.3).to(DEV).requires_grad_(True)
    p_f = (torch.randn(geom_f.n_params, generator=g) * 0.3).to(DEV).requires_grad_(True)
    m_d, m_f = (torch.randn(40, 16, generator=g) / 40 ** 0.5 for _ in range(2))
    w_d, w_f = torch.randn(3 * n, 16, generator=g), torch.randn(2 * n, 16, generator=g)
    aabb = torch.tensor(AABB)

    fl = flow.to(DEV).requires_grad_(True)
    pos_g, t_g, aabb_g = pos.to(DEV), t.to(DEV), aabb.to(DEV)
    coords = _ops.flow_warp(pos_g, fl, noise.to(DEV), t_g, aabb_g, TD, True)
    cur = _ops.contract(pos_g, aabb_g, t_g, True)
    enc_d = _ops.grid_encode_rows(cur, coords, p_d, desc_d)
    enc_f = _ops.grid_encode(coords, p_f, desc_f)
    dys = {}
    enc_d.register_hook(lambda gr: dys.__setitem__("d", gr))
    enc_f.register_hook(lambda gr: dys.__setitem__("f", gr))
    loss = ((enc_d @ m_d.to(DEV)) * w_d.to(DEV)).sum() + ((enc_f @ m_f.to(DEV)) * w_f.to(DEV)).sum()
    loss.backward()

    # the upstream gradients the grids received are the projections' (fp32 matmul): the grids' references take them
    assert rel_err(dys["d"], w_d.double() @ m_d.double().T) < 1e-5
    assert rel_err(dys["f"], w_f.double() @ m_f.double().T) < 1e-5
    x32 = coords.detach()
    dx_d, _ = tcnn_ref.grid_input_grad64(x32, p_d, dys["d"][n:], geom_d)
    dx_f, _ = tcnn_ref.grid_input_grad64(x32, p_f, dys["f"], geom_f)
    d_coords = (dx_d + dx_f).cpu()
    tab_d, mag_d, cnt_d = tcnn_ref.grid_table_grad64(torch.cat([cur, x32]), dys["d"], geom_d)
    tab_f, mag_f, cnt_f = tcnn_ref.grid_table_grad64(x32, dys["f"], geom_f)
    w1, re1 = _check_table("segment dynamic table", p_d.grad, tab_d, mag_d, cnt_d)
    w2, re2 = _check_table("segment flow table", p_f.grad, tab_f, mag_f, cnt_f)
    _report("segment dynamic table", w1, C_TAB, re1)
    _report("segment flow table", w2, C_TAB, re2)

    # the warp in float64 at the fp32 point x32 = pos + flow * noise, as test_flow_warp_matches_fp64
    nz = noise[:, None]
    a64 = aabb.double()
    rows, grads, ties = [], [], []
    for d in range(2):
        xw = pos + flow[:, 3 * d: 3 * d + 3] * nz
        top = ((xw.double() - a64[:3]) / (a64[3:] - a64[:3]) * 2 - 1).abs().topk(2, dim=-1).values
        ties.append((top[:, 0] >= 1) & (top[:, 0] - top[:, 1] <= 4e-7 * top[:, 0]))
        f64 = flow[:, 3 * d: 3 * d + 3].double().requires_grad_(True)
        y = _contract64(xw.double() + (f64 - f64.detach()) * nz.double(), a64)
        rows.append(y.detach())
        (gf,) = torch.autograd.grad(y, f64, d_coords[d * n:(d + 1) * n, :3])
        grads.append(gf)
    got_xyz = x32[:, :3].cpu().double()
    want_xyz = torch.cat(rows)
    same = (got_xyz != 0).any(-1) == (want_xyz != 0).any(-1)
    assert (~same).sum() <= 16, int((~same).sum())
    assert rel_err(got_xyz[same], want_xyz[same]) < 1e-6
    d_want = torch.cat(grads, 1)
    centre = ~torch.isfinite(d_want).all(-1)           # torch.where's backward at the cube's centre, see the warp test
    tie = ties[0] | ties[1]
    assert tie.sum() <= 16 and centre.sum() <= n // 32, (int(tie.sum()), int(centre.sum()))
    ok = same[:n] & same[n:] & ~centre & ~tie
    re = rel_err(fl.grad.cpu().double()[ok], d_want[ok])
    _report("segment d_flow", re, 1e-5)
    assert re <= 1e-5, re
    assert torch.isfinite(fl.grad).all()

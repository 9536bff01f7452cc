"""CPU emulator of the C ABI (include/emer_b200.h) -- TEST INFRASTRUCTURE ONLY.

Every entry point of ``libemer_b200.so`` restated on host memory, through the same raw pointers, row
strides and sizes the product hands to the library, with the arithmetic of ``oracle/`` (which is pinned
against the reference's own Python, tests/golden/make_golden.py).  ``install(monkeypatch)`` swaps it in
for ``emernerf_b200._lib.call``, so that the whole host side of the product -- the drop-in modules, the
autograd wrappers of ``_ops.py``, their buffer / stride / padding bookkeeping and the ctypes argument
lists -- runs on CPU tensors in the ``-m "not gpu"`` suite and is compared with the same golden vectors
as the GPU path.  Nothing under ``emernerf_b200/`` imports this module; without it every op raises on CPU
tensors (tests/test_abi_and_host.py::test_ops_refuse_cpu_tensors).
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from oracle import hotpath, nerfacc_ref as nf, tcnn_ref

CALLS = []          # names of the entry points hit since the last reset (tests assert on coverage)


def _addr(p):
    if p is None:
        return 0
    if isinstance(p, int):
        return p
    return p.value or 0


def _require(cond, msg: str) -> None:
    """The library's EMER_REQUIRE checks, mirrored: a call the .so would refuse must fail here too."""
    if not cond:
        raise RuntimeError(f"cabi_emulator (as the library would): {msg}")


def _aligned16(*ptrs) -> bool:
    return all(_addr(p) % 16 == 0 for p in ptrs)


def _aligned32(*ptrs) -> bool:
    return all(_addr(p) % 32 == 0 for p in ptrs)


def _view(ptr, rows: int, cols: int, ld=None, ctype=ctypes.c_float, dtype=np.float32):
    """[rows, cols] tensor aliasing the caller's memory at ``ptr`` with row stride ``ld`` (elements)."""
    addr = _addr(ptr)
    if not addr:
        return None
    ld = cols if ld is None else int(ld)
    if rows == 0 or cols == 0:
        return torch.from_numpy(np.zeros((rows, cols), dtype))
    count = (rows - 1) * ld + cols
    arr = np.ctypeslib.as_array((ctype * count).from_address(addr))
    return torch.from_numpy(arr).as_strided((rows, cols), (ld, 1))


def _vec(ptr, n: int, **kw):
    v = _view(ptr, 1, n, **kw)
    return None if v is None else v[0]


def _geom(desc_ref) -> tcnn_ref.GridGeometry:
    g = desc_ref._obj
    L = g.n_levels
    return tcnn_ref.GridGeometry(g.n_dims, L, g.n_feat, [float(g.scale[i]) for i in range(L)],
                                 [int(g.resolution[i]) for i in range(L)], [int(g.offset[i]) for i in range(L + 1)],
                                 [bool(g.hashed[i]) for i in range(L)])


def _act(v, act):
    if act == 1:
        return torch.relu(v)
    if act == 2:
        return torch.sigmoid(v)
    return v


def _act_grad(g, y, act):
    if act == 1:
        return g * (y > 0)
    if act == 2:
        return g * (y * (1.0 - y))
    return g


# ----------------------------------------------------------------------------- hash grid
def _check_grid(geom):
    _require(geom.n_dims in (3, 4) and 1 <= geom.n_levels <= 16 and geom.n_feat in (1, 2, 4), "grid: bad descriptor")
    for l in range(geom.n_levels):
        size = geom.offsets[l + 1] - geom.offsets[l]
        _require(size > 0 and (not geom.hashed[l] or size & (size - 1) == 0), f"grid: level {l} size {size}")


def emer_grid_fwd(desc, x, table, y, n, stream):
    geom = _geom(desc)
    _check_grid(geom)
    _require(_aligned16(x, table, y), "emer_grid_fwd: pointers must be 16-byte aligned")
    xs = _view(x, n, geom.n_dims)
    tb = _vec(table, geom.n_params)
    with torch.no_grad():
        _view(y, n, geom.n_output_dims).copy_(tcnn_ref.grid_forward(xs, tb, geom))


def emer_grid_bwd(desc, x, table, dy, dtable, dx, n, stream):
    geom = _geom(desc)
    _check_grid(geom)
    _require(_aligned16(x, table, dy, dtable, dx), "emer_grid_bwd: pointers must be 16-byte aligned")
    xs = _view(x, n, geom.n_dims).clone().requires_grad_(bool(_addr(dx)))
    tb = _vec(table, geom.n_params).clone().requires_grad_(bool(_addr(dtable)))
    g = _view(dy, n, geom.n_output_dims)
    wanted = [t for t in (tb, xs) if t.requires_grad]
    if not wanted or n == 0:
        return
    with torch.enable_grad():
        grads = list(torch.autograd.grad(tcnn_ref.grid_forward(xs, tb, geom), wanted, g))
    if tb.requires_grad:
        _vec(dtable, geom.n_params).add_(grads.pop(0))          # accumulated: the caller zeroes
    if xs.requires_grad:
        _view(dx, n, geom.n_dims).copy_(grads.pop(0))


# ----------------------------------------------------------------------------- contraction, activation
def _contract(pos, aabb, unbounded, apply_selector):
    if apply_selector:
        return hotpath.contract_points(pos, aabb, bool(unbounded))
    if unbounded:
        return hotpath.contract(pos, aabb)
    lo, hi = torch.split(aabb, 3, dim=-1)
    return (pos - lo) / (hi - lo)


def emer_contract_fwd(pos, aabb6, time, out, out_dim, unbounded, apply_selector, n, stream):
    _require(out_dim in (3, 4) and (out_dim == 3 or _aligned16(out)), "emer_contract_fwd: out_dim / alignment")
    _require(out_dim == 3 or _addr(time), "emer_contract_fwd: out_dim 4 needs the time column")
    o = _view(out, n, out_dim)
    with torch.no_grad():
        o[:, :3] = _contract(_view(pos, n, 3), _vec(aabb6, 6), unbounded, apply_selector)
        if out_dim == 4:
            o[:, 3] = _vec(time, n)


def emer_contract_bwd(pos, aabb6, dout, dpos, dtime, out_dim, unbounded, apply_selector, n, stream):
    g = _view(dout, n, out_dim)
    p = _view(pos, n, 3).clone().requires_grad_(True)
    with torch.enable_grad():
        (gp,) = torch.autograd.grad(_contract(p, _vec(aabb6, 6), unbounded, apply_selector), p, g[:, :3].contiguous())
    _view(dpos, n, 3).copy_(gp)
    if _addr(dtime):
        _vec(dtime, n).copy_(g[:, 3])


def emer_trunc_exp_fwd(x, ldx, y, n, stream):
    with torch.no_grad():
        _vec(y, n).copy_(torch.exp(_view(x, n, 1, ldx)[:, 0] - 1.0))


def emer_trunc_exp_bwd(x, ldx, dy, dx, n, stream):
    with torch.no_grad():
        _vec(dx, n).copy_(_vec(dy, n) * torch.exp(torch.clamp(_view(x, n, 1, ldx)[:, 0] - 1.0, max=15.0)))


# ----------------------------------------------------------------------------- dense layers
def emer_linear_fwd(x, ldx, w, b, y, ldy, n, k, n_out, act, stream):
    _require(k > 0 and n_out > 0 and ldx >= k and ldy >= n_out, f"emer_linear_fwd: bad shape k={k} n_out={n_out}")
    with torch.no_grad():
        v = _view(x, n, k, ldx) @ _view(w, n_out, k).t()
        if _addr(b):
            v = v + _vec(b, n_out)
        _view(y, n, n_out, ldy).copy_(_act(v, act))


def _r(v, m):
    return (v + m - 1) // m * m


def _check_tc(kred, ncols, what):
    """linear_tc.cu launch<>: the padded output width is at most 256; the resident weight panels fit shared memory."""
    n_pad, kred_pad = _r(ncols, 16), _r(kred, 32)
    _require(n_pad <= 256, f"{what}: output width {ncols} exceeds one MMA (256)")
    smem = 2 * (kred_pad // 4) * n_pad * 16 + n_pad * 4
    _require(smem <= 227 * 1024, f"{what}: layer needs {smem} B of shared memory")


def _check_narrow(k, n_out, what):
    _require(1 <= n_out <= 8 and 1 <= k <= 256, f"{what}: k={k} n_out={n_out}")


def emer_linear_tc_fwd(x, ldx, w, b, y, ldy, n, k, n_out, act, stream):
    _check_tc(k, n_out, "emer_linear_tc_fwd")
    emer_linear_fwd(x, ldx, w, b, y, ldy, n, k, n_out, act, stream)


def emer_linear_narrow_fwd(x, ldx, w, b, y, ldy, n, k, n_out, act, stream):
    _check_narrow(k, n_out, "emer_linear_narrow_fwd")
    emer_linear_fwd(x, ldx, w, b, y, ldy, n, k, n_out, act, stream)


def _bwd_data(dz, w, dx, relu_src, relu_cols, accumulate):
    with torch.no_grad():
        g = dz @ w
        if relu_src is not None and relu_cols > 0:
            g[:, :relu_cols] = g[:, :relu_cols] * (relu_src[:, :relu_cols] > 0)
        if accumulate:
            dx.add_(g)
        else:
            dx.copy_(g)


def emer_linear_bwd_data(dy, lddy, y, ldy, act, w, dx, lddx, n, k, n_out, accumulate, stream):
    dz = _act_grad(_view(dy, n, n_out, lddy), _view(y, n, n_out, ldy) if act else None, act)
    _bwd_data(dz, _view(w, n_out, k), _view(dx, n, k, lddx), None, 0, accumulate)


def emer_linear_tc_bwd_data(dy, lddy, y, ldy, act, w, dx, lddx, relu_src, ld_relu, relu_cols, n, k, n_out, accumulate,
                            stream):
    _check_tc(n_out, k, "emer_linear_tc_bwd_data")
    dz = _act_grad(_view(dy, n, n_out, lddy), _view(y, n, n_out, ldy) if act else None, act)
    mask = _view(relu_src, n, relu_cols, ld_relu) if _addr(relu_src) and relu_cols > 0 else None
    _bwd_data(dz, _view(w, n_out, k), _view(dx, n, k, lddx), mask, relu_cols, accumulate)


def emer_linear_narrow_bwd_data(dz, lddz, w, dx, lddx, relu_src, ld_relu, relu_cols, n, k, n_out, stream):
    _check_narrow(k, n_out, "emer_linear_narrow_bwd_data")
    mask = _view(relu_src, n, relu_cols, ld_relu) if _addr(relu_src) and relu_cols > 0 else None
    _bwd_data(_view(dz, n, n_out, lddz), _view(w, n_out, k), _view(dx, n, k, lddx), mask, relu_cols, 0)


def _bwd_weight(x, dz, dw, db):
    with torch.no_grad():
        dw.add_(dz.t() @ x)                                  # accumulated: the caller zeroes
        if db is not None:
            db.add_(dz.sum(0))


def emer_linear_bwd_weight(x, ldx, dy, lddy, y, ldy, act, dw, db, n, k, n_out, stream):
    dz = _act_grad(_view(dy, n, n_out, lddy), _view(y, n, n_out, ldy) if act else None, act)
    _bwd_weight(_view(x, n, k, ldx), dz, _view(dw, n_out, k), _vec(db, n_out))


def _check_tc_wgrad(x, ldx, dz, lddz, k, n_out):
    """emer_linear_tc_bwd_weight's EMER_REQUIREs (csrc/wgrad_mn.cu), restated independently of _ops."""
    _require(n_out <= 128 and k <= 256, f"emer_linear_tc_bwd_weight: widths k={k} n_out={n_out} out of range")
    _require(ldx % 4 == 0 and lddz % 4 == 0 and _aligned16(x, dz), "emer_linear_tc_bwd_weight: rows must be 16-byte aligned")
    _require(_r(k, 4) <= ldx, "emer_linear_tc_bwd_weight: row stride shorter than the padded width")
    _require(_r(n_out, 4) <= lddz, "emer_linear_tc_bwd_weight: dZ rows too short")


def emer_linear_tc_bwd_weight(x, ldx, dz, lddz, dw, db, n, k, n_out, stream):
    if n == 0:
        return
    _check_tc_wgrad(x, ldx, dz, lddz, k, n_out)
    _bwd_weight(_view(x, n, k, ldx), _view(dz, n, n_out, lddz), _view(dw, n_out, k), _vec(db, n_out))


def emer_linear_narrow_bwd_weight(x, ldx, dz, lddz, dw, db, n, k, n_out, stream):
    _check_narrow(k, n_out, "emer_linear_narrow_bwd_weight")
    _bwd_weight(_view(x, n, k, ldx), _view(dz, n, n_out, lddz), _view(dw, n_out, k), _vec(db, n_out))


# ----------------------------------------------------------------------------- sampling
_S_TO_T = {
    0: lambda v: v,
    1: lambda v: 1 / v,
    2: lambda v: v ** 2,
    3: lambda v: torch.exp(v),
    4: lambda v: torch.where(v < 0.5, v * 400, 200 / (2 - 2 * v)),
    5: lambda v: torch.where(v < 0.5, 2 * v, 1 / (2 - 2 * v)),
}


def _resample(vals, cdfs, n, bias, s_min, s_max, kind):
    R = vals.shape[0]
    jitter = None if bias is None else bias.reshape(R, 1)
    iv, _ = nf.importance_sampling(nf.RayIntervals(vals), cdfs, n, jitter is not None, jitter=jitter)
    s = iv.vals
    smin, smax = torch.tensor(s_min, dtype=torch.float32), torch.tensor(s_max, dtype=torch.float32)
    return s, _S_TO_T[kind](s * smax + (1 - s) * smin)


def emer_pdf_resample(vals, cdfs, m1, n, bias, s_min, s_max, kind, out_s, out_t, out_bins, n_rays, stream):
    _require(m1 >= 2 and n >= 1 and kind in _S_TO_T, "emer_pdf_resample: need m1 >= 2 edges, n >= 1 intervals, a known warp")
    v, c = _view(vals, n_rays, m1), _view(cdfs, n_rays, m1)
    b = _vec(bias, n_rays)
    with torch.no_grad():
        s, t = _resample(v, c, n, b, s_min, s_max, kind)
        _view(out_s, n_rays, n + 1).copy_(s)
        _view(out_t, n_rays, n + 1).copy_(t)
        if _addr(out_bins):
            bb = torch.full((n_rays, 1), 0.5) if b is None else b.reshape(n_rays, 1)
            u = c[:, :1] + (torch.arange(n + 1, dtype=torch.float32)[None] + (bb - 0.5)) * ((c[:, -1:] - c[:, :1]) / n)
            p = torch.searchsorted(c.contiguous(), u.contiguous(), right=True)
            _view(out_bins, n_rays, n + 1, ctype=ctypes.c_int32, dtype=np.int32).copy_(p.to(torch.int32))


def emer_prop_level(desc, prev_s, prev_cdf, m1, n, bias, s_min, s_max, kind, origins, dirs, aabb6, unbounded, table,
                    w0, b0, w1, b1, out_s, out_t, out_cdf, out_sigma, n_rays, stream):
    geom = _geom(desc)
    lf = geom.n_output_dims
    _check_grid(geom)
    _require(geom.n_dims == 3 and lf <= 16 and geom.n_feat <= 4, "emer_prop_level: 3-D grids with at most 16 features")
    _require(m1 >= 2 and n >= 1 and n + 1 <= 257, f"emer_prop_level: n={n} out of range")
    with torch.no_grad():
        s, t = _resample(_view(prev_s, n_rays, m1), _view(prev_cdf, n_rays, m1), n, _vec(bias, n_rays), s_min, s_max,
                         kind)
        t0, t1 = t[:, :-1], t[:, 1:]
        pos = _view(origins, n_rays, 3)[:, None, :] + _view(dirs, n_rays, 3)[:, None, :] * (t0 + t1)[..., None] / 2.0
        x = hotpath.contract_points(pos.reshape(-1, 3), _vec(aabb6, 6), bool(unbounded))
        h = torch.relu(tcnn_ref.grid_forward(x, _vec(table, geom.n_params), geom) @ _view(w0, 64, lf).t() + _vec(b0, 64))
        raw = h @ _view(w1, 1, 64).t() + _vec(b1, 1)
        sigma = torch.exp(raw[:, 0] - 1.0).reshape(n_rays, n)
        trans, _ = nf.render_transmittance_from_density(t0, t1, sigma)
        _view(out_s, n_rays, n + 1).copy_(s)
        _view(out_t, n_rays, n + 1).copy_(t)
        _view(out_cdf, n_rays, n + 1).copy_(1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], -1))
        if _addr(out_sigma):
            _view(out_sigma, n_rays, n).copy_(sigma)


def emer_prop_level_bwd(desc, t_edges, sigma, d_cdf, n, origins, dirs, aabb6, unbounded, table, w0, b0, w1, xc, d_enc,
                        d_w0, d_b0, d_w1, d_b1, n_rays, stream):
    """Autograd through the restated forward of the level (from the grid features on; the scatter is emer_grid_bwd)."""
    geom = _geom(desc)
    lf = geom.n_output_dims
    _check_grid(geom)
    _require(geom.n_dims == 3 and geom.n_feat == 1 and lf in (4, 8), "emer_prop_level_bwd: 3-D grids of 4 or 8 levels x 1 feature")
    _require(n >= 1 and n + 1 <= 257, f"emer_prop_level_bwd: n={n} out of range")
    _require(_aligned16(d_enc), "emer_prop_level_bwd: d_enc must be 16-byte aligned")
    t = _view(t_edges, n_rays, n + 1)
    t0, t1 = t[:, :-1], t[:, 1:]
    with torch.no_grad():
        pos = _view(origins, n_rays, 3)[:, None, :] + _view(dirs, n_rays, 3)[:, None, :] * (t0 + t1)[..., None] / 2.0
        x = hotpath.contract_points(pos.reshape(-1, 3), _vec(aabb6, 6), bool(unbounded))
        enc0 = tcnn_ref.grid_forward(x, _vec(table, geom.n_params), geom)
    enc = enc0.clone().requires_grad_()
    W0 = _view(w0, 64, lf).clone().requires_grad_()
    B0 = _vec(b0, 64).clone().requires_grad_()
    W1 = _view(w1, 1, 64).clone().requires_grad_()
    # Like the kernel, work from the SAVED densities: sigma = exp(raw - 1) has d sigma / d raw = exp(min(raw - 1, 15))
    # = min(sigma, e^15) (nerf_utils.py:59-75), so b1's value is not needed -- only that raw depends on it.
    B1 = torch.zeros(1, requires_grad=True)
    with torch.enable_grad():
        raw = (torch.relu(enc @ W0.t() + B0) @ W1.t() + B1)[:, 0].reshape(n_rays, n)
        sg = _view(sigma, n_rays, n)
        sig = sg + torch.clamp(sg, max=float(np.exp(np.float32(15.0)))) * (raw - raw.detach())
        trans, _ = nf.render_transmittance_from_density(t0, t1, sig)
        cdf = 1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], -1)
        g_enc, g_w0, g_b0, g_w1, g_b1 = torch.autograd.grad(cdf, (enc, W0, B0, W1, B1), _view(d_cdf, n_rays, n + 1))
    with torch.no_grad():
        _view(xc, n_rays * n, 3).copy_(x)
        _view(d_enc, n_rays * n, lf).copy_(g_enc)
        _view(d_w0, 64, lf).add_(g_w0)
        _vec(d_b0, 64).add_(g_b0)
        _vec(d_w1, 64).add_(g_w1.reshape(-1))
        _vec(d_b1, 1).add_(g_b1)


def emer_interlevel_loss(s, cdf, m, prop_s, prop_cdf, n1, pulse_width, loss_sum, d_prop_cdf, n_rays, stream):
    """One level's term of oracle.hotpath.proposal_loss (sum instead of mean) and autograd's gradient of it."""
    _require(2 <= m <= 129 and 2 <= n1 <= 257, f"emer_interlevel_loss: {m} final edges / {n1} proposal edges out of range")
    _require(pulse_width > 0, "emer_interlevel_loss: pulse width must be positive")
    S, C, PS = _view(s, n_rays, m), _view(cdf, n_rays, m), _view(prop_s, n_rays, n1)
    PC = _view(prop_cdf, n_rays, n1).clone().requires_grad_()
    with torch.enable_grad():
        w_n = (C[:, 1:] - C[:, :-1]) / (S[:, 1:] - S[:, :-1])
        c, w = hotpath.blur_stepfun(S, w_n, pulse_width)
        area = 0.5 * (w[:, 1:] + w[:, :-1]) * (c[:, 1:] - c[:, :-1])
        cd = torch.cat([torch.zeros_like(area[:, :1]), torch.cumsum(area, -1)], -1)
        wp = PC[:, 1:] - PC[:, :-1]
        w_s = torch.diff(hotpath.sorted_interp_quad(PS, c, w, cd), dim=-1)
        total = ((w_s - wp).clamp_min(0) ** 2 / (wp + 1e-5)).sum()
        (g,) = torch.autograd.grad(total, PC)
    with torch.no_grad():
        _vec(loss_sum, 1).add_(total.detach())
        if _addr(d_prop_cdf):
            _view(d_prop_cdf, n_rays, n1).copy_(g)


# ----------------------------------------------------------------------------- field tail
FT_DIR = 33


def emer_field_tail_fwd(feats, ld_feats, g_dim, dirs, idx, emb, e_dim, out, ld_out, sigma, n_rays, n_samples, stream):
    n = n_rays * n_samples
    width = g_dim + FT_DIR + e_dim
    w4 = (width + 3) // 4 * 4
    _require(e_dim == 0 or (_addr(idx) and _addr(emb)), "emer_field_tail_fwd: embedding needs indices and a table")
    _require(ld_out % 4 == 0 and ld_out >= w4 and _aligned16(out),
             "emer_field_tail_fwd: output rows must be 16-byte aligned and wide enough")
    _require(g_dim % 4 == 0 and w4 - g_dim <= 72, f"emer_field_tail_fwd: geometry width {g_dim} must be a multiple of 4 "
             "and the tail at most 72 floats")
    f = _view(feats, n, g_dim, ld_feats)
    o = _view(out, n, w4, ld_out)
    with torch.no_grad():
        o[:, :g_dim] = f
        enc = hotpath.sinusoidal((_view(dirs, n_rays, 3) + 1.0) / 2.0)
        o[:, g_dim:g_dim + FT_DIR] = enc.repeat_interleave(n_samples, 0)
        if e_dim:
            ix = _vec(idx, n_rays, ctype=ctypes.c_int64, dtype=np.int64)
            table = _view(emb, int(ix.max()) + 1, e_dim)
            o[:, g_dim + FT_DIR:width] = table[ix].repeat_interleave(n_samples, 0)
        o[:, width:] = 0.0
        if _addr(sigma):
            _vec(sigma, n).copy_(torch.exp(f[:, 0] - 1.0))


def emer_field_tail_bwd(feats, ld_feats, d_out, ld_out, g_dim, d_sigma, idx, d_emb, e_dim, n_rays, n_samples, stream):
    n = n_rays * n_samples
    _require(e_dim <= 32, f"emer_field_tail_bwd: embedding width {e_dim} > 32")
    g = _view(d_out, n, g_dim + FT_DIR + e_dim, ld_out)
    with torch.no_grad():
        if _addr(d_sigma):
            f0 = _view(feats, n, 1, ld_feats)[:, 0]
            g[:, 0] += _vec(d_sigma, n) * torch.exp(torch.clamp(f0 - 1.0, max=15.0))
        if _addr(d_emb):
            ix = _vec(idx, n_rays, ctype=ctypes.c_int64, dtype=np.int64)
            per_ray = g[:, g_dim + FT_DIR:].reshape(n_rays, n_samples, e_dim).sum(1)
            _view(d_emb, int(ix.max()) + 1, e_dim).index_add_(0, ix, per_ray)      # accumulated: the caller zeroes


# ----------------------------------------------------------------------------- volume rendering
def _composite(t0, t1, sigma):
    w, trans, _ = nf.render_weight_from_density(t0, t1, sigma)
    opacity = nf.accumulate_along_rays(w, None).clamp(1e-6, 1.0)
    steps = (t0 + t1)[..., None] / 2.0
    depth = nf.accumulate_along_rays(w, steps) / opacity
    return w, trans, opacity, depth, steps


def emer_composite_fwd(t0, t1, sigma, weights, trans, opacity, depth, median, cdf, n_rays, n_samples, stream):
    _require(n_samples >= 1, "emer_composite_fwd: n_samples must be >= 1")
    a, b, s = (_view(p, n_rays, n_samples) for p in (t0, t1, sigma))
    with torch.no_grad():
        w, tr, op, dep, steps = _composite(a, b, s)
        _view(weights, n_rays, n_samples).copy_(w)
        _view(trans, n_rays, n_samples).copy_(tr)
        _view(opacity, n_rays, 1).copy_(op)
        _view(depth, n_rays, 1).copy_(dep)
        cw = torch.cumsum(w, dim=-1)
        mi = torch.clamp(torch.searchsorted(cw, torch.full((n_rays, 1), 0.5), side="left"), 0, n_samples - 1)
        _view(median, n_rays, 1).copy_(torch.gather(steps[..., 0], -1, mi))
        if _addr(cdf):
            _view(cdf, n_rays, n_samples + 1).copy_(1.0 - torch.cat([tr, torch.zeros_like(tr[:, :1])], -1))


def emer_composite_bwd(t0, t1, sigma, weights, trans, g_w, g_t, g_o, g_d, dsigma, n_rays, n_samples, stream):
    a, b = _view(t0, n_rays, n_samples), _view(t1, n_rays, n_samples)
    s = _view(sigma, n_rays, n_samples).clone().requires_grad_(True)
    with torch.enable_grad():
        w, tr, op, dep, _ = _composite(a, b, s)
        outs, grads = [], []
        for o, g, cols in ((w, g_w, n_samples), (tr, g_t, n_samples), (op, g_o, 1), (dep, g_d, 1)):
            if _addr(g):
                outs.append(o)
                grads.append(_view(g, n_rays, cols))
        (gs,) = torch.autograd.grad(outs, s, grads)
    _view(dsigma, n_rays, n_samples).copy_(gs)


ACC_MAX_CHANNELS = 32 * 8          # composite.cu: ACC_MAX_PER_LANE = 8


def emer_accumulate_fwd(w, v, out, n_rays, n_samples, c, stream):
    _require(1 <= c <= ACC_MAX_CHANNELS, f"emer_accumulate_fwd: channels {c} out of range")
    with torch.no_grad():
        ww = _view(w, n_rays, n_samples)
        vv = _view(v, n_rays * n_samples, c).reshape(n_rays, n_samples, c)
        _view(out, n_rays, c).copy_((ww[..., None] * vv).sum(1))


def emer_accumulate_bwd(w, v, g, dw, dv, n_rays, n_samples, c, stream):
    with torch.no_grad():
        ww = _view(w, n_rays, n_samples)
        vv = _view(v, n_rays * n_samples, c).reshape(n_rays, n_samples, c)
        gg = _view(g, n_rays, c)
        if _addr(dw):
            _view(dw, n_rays, n_samples).copy_((gg[:, None, :] * vv).sum(-1))
        if _addr(dv):
            _view(dv, n_rays * n_samples, c).copy_((ww[..., None] * gg[:, None, :]).reshape(-1, c))


# ----------------------------------------------------------------------------- fused field chain
def emer_field_fwd(enc, ld_enc, k_enc, wb0, bb0, wb1, bb1, n_feat, w0g, ld_w0, w1h, w1g, ld_w1, w2, b2, ray_bias,
                   samples, sigma, rgb, save_hb, save_hg, save_h1, save_sem, n, stream):
    _require(k_enc in (32, 40, 64), f"emer_field_fwd: k_enc={k_enc} (L*F of the grid) must be 32, 40 or 64")
    _require(n_feat in (64, 128), f"emer_field_fwd: n_feat={n_feat} must be 64 or 128")
    _require(samples > 0, "emer_field_fwd: samples per ray must be positive")
    _require(ld_enc % 8 == 0 and _aligned32(enc, save_hb, save_hg, save_h1, save_sem) and _aligned16(ray_bias),
             "emer_field_fwd: rows must be 32-byte aligned")
    _require(n_feat == 64 or _addr(save_sem), "emer_field_fwd: the semantic half needs its output buffer")
    if n == 0:
        return
    n_rays = (n + samples - 1) // samples
    with torch.no_grad():
        x = _view(enc, n, k_enc, ld_enc)
        hb = torch.relu(x @ _view(wb0, 64, k_enc).T + _vec(bb0, 64))
        feats = hb @ _view(wb1, n_feat, 64).T + _vec(bb1, n_feat)
        geo = feats[:, :64]
        rb = _view(ray_bias, n_rays, 128)[torch.arange(n) // samples]
        h0 = torch.relu(geo @ _view(w0g, 64, 64, ld_w0).T + rb[:, :64])
        h1 = torch.relu(h0 @ _view(w1h, 64, 64, ld_w1).T + geo @ _view(w1g, 64, 64, ld_w1).T + rb[:, 64:])
        _vec(sigma, n).copy_(torch.exp(feats[:, 0] - 1.0))
        _view(rgb, n, 3).copy_(torch.sigmoid(h1 @ _view(w2, 3, 64).T + _vec(b2, 3)))
        if _addr(save_hb):
            _view(save_hb, n, 64).copy_(hb)
        if _addr(save_hg):
            _view(save_hg, n, 128).copy_(torch.cat([h0, geo], -1))
        if _addr(save_h1):
            _view(save_h1, n, 64).copy_(h1)
        if n_feat == 128:
            _view(save_sem, n, 64).copy_(feats[:, 64:])


def emer_field_bwd(d_rgb, rgb, d_sigma, sigma, d_geo, d_sem, hb, hg, h1, wb0, k_enc, wb1, n_feat, w0g, ld_w0, w1h, w1g,
                   ld_w1, w2, dz2, dz1, d1, dzb, d_enc, ld_denc, d_ray_bias, samples, n, stream):
    _require(all(_addr(p) for p in (rgb, sigma, hb, hg, h1, wb0, wb1, w0g, w1h, w1g, w2, dz1, d1, dzb)),
             "emer_field_bwd: NULL pointer")
    _require(k_enc in (32, 40, 64) and n_feat in (64, 128) and samples > 0, "emer_field_bwd: bad shape")
    _require(not _addr(d_enc) or (ld_denc % 8 == 0 and ld_denc >= k_enc), "emer_field_bwd: d_enc rows must be 32-byte aligned")
    _require(_aligned32(hb, hg, h1, dz1, d1, dzb, d_enc, d_geo, d_sem), "emer_field_bwd: row buffers must be 32-byte aligned")
    _require(not _addr(d_ray_bias) or samples % 32 == 0, "emer_field_bwd: per-ray sums need samples % 32 == 0")
    if n == 0:
        return
    with torch.no_grad():
        z2 = torch.zeros(n, 3)
        if _addr(d_rgb):
            y = _view(rgb, n, 3)
            z2 = _view(d_rgb, n, 3) * (y * (1.0 - y))
            if _addr(dz2):                  # (without d_rgb the library leaves dz2 as it is)
                _view(dz2, n, 3).copy_(z2)
        z1 = (z2 @ _view(w2, 3, 64)) * (_view(h1, n, 64) > 0)
        _view(dz1, n, 64).copy_(z1)
        h0 = _view(hg, n, 64, 128)
        z0 = (z1 @ _view(w1h, 64, 64, ld_w1)) * (h0 > 0)
        dF = z1 @ _view(w1g, 64, 64, ld_w1) + z0 @ _view(w0g, 64, 64, ld_w0)
        if _addr(d_geo):
            dF = dF + _view(d_geo, n, 64)
        if _addr(d_sigma):
            dF[:, 0] += _vec(d_sigma, n) * torch.clamp(_vec(sigma, n), max=3269017.25)
        out = _view(d1, n, 128)
        out[:, :64] = z0
        out[:, 64:] = dF
        wb1_ = _view(wb1, n_feat, 64)
        dhb = dF @ wb1_[:64]
        if n_feat == 128 and _addr(d_sem):
            dhb = dhb + _view(d_sem, n, 64) @ wb1_[64:]
        zb = dhb * (_view(hb, n, 64) > 0)
        _view(dzb, n, 64).copy_(zb)
        if _addr(d_enc):
            _view(d_enc, n, k_enc, ld_denc).copy_(zb @ _view(wb0, 64, k_enc))
        if _addr(d_ray_bias):
            n_rays = (n + samples - 1) // samples
            acc = _view(d_ray_bias, n_rays, 128)
            ray = torch.arange(n) // samples
            acc[:, :64].index_add_(0, ray, z0)
            acc[:, 64:].index_add_(0, ray, z1)


def emer_field_wgrad(enc, ld_enc, k_enc, hb, hg, h1, dz2, dz1, d1, dzb, d_sem, n_feat, dwb0, dbb0, dwb1, dbb1, dw0g, ld_w0,
                     dw1h, dw1g, ld_w1, dw2, db2, n, stream):
    if n == 0:
        return
    _require(all(_addr(p) for p in (enc, hb, d1, dzb, dwb0, dbb0, dwb1, dbb1)), "emer_field_wgrad: NULL pointer")
    _require(not _addr(dz2) or all(_addr(p) for p in (hg, h1, dz1, dw0g, dw1h, dw1g, dw2, db2)),
             "emer_field_wgrad: NULL pointer among the colour head's buffers")
    _require(k_enc in (32, 40, 64) and n_feat in (64, 128), "emer_field_wgrad: bad shape")
    _require(not _addr(d_sem) or n_feat == 128, "emer_field_wgrad: d_sem needs n_feat = 128")
    _require(ld_enc % 4 == 0 and ld_enc >= k_enc, "emer_field_wgrad: ld_enc")
    _require(not _addr(dz2) or (ld_w0 >= 64 and ld_w1 >= 64), "emer_field_wgrad: ld_w0 / ld_w1 shorter than a block")
    _require(_aligned16(enc, hb, hg, h1, dz2, dz1, d1, dzb, d_sem), "emer_field_wgrad: row buffers must be 16-byte aligned")
    D1, hb_ = _view(d1, n, 128), _view(hb, n, 64)
    _bwd_weight(_view(enc, n, k_enc, ld_enc), _view(dzb, n, 64), _view(dwb0, 64, k_enc), _vec(dbb0, 64))
    _bwd_weight(hb_, D1[:, 64:], _view(dwb1, 64, 64), _vec(dbb1, 64))
    if _addr(d_sem):
        _bwd_weight(hb_, _view(d_sem, n, 64), _view(_addr(dwb1) + 64 * 64 * 4, 64, 64), _vec(_addr(dbb1) + 64 * 4, 64))
    if _addr(dz2):
        h0, geo, z1 = _view(hg, n, 64, 128), _view(_addr(hg) + 64 * 4, n, 64, 128), _view(dz1, n, 64)
        _bwd_weight(geo, D1[:, :64], _view(dw0g, 64, 64, ld_w0), None)
        _bwd_weight(h0, z1, _view(dw1h, 64, 64, ld_w1), None)
        _bwd_weight(geo, z1, _view(dw1g, 64, 64, ld_w1), None)
        _bwd_weight(_view(h1, n, 64), _view(dz2, n, 3), _view(dw2, 3, 64), _vec(db2, 3))


# ----------------------------------------------------------------------------- ray generation
def emer_gen_rays(img_idx, x, y, c2w, intrinsics, per_ray_mats, timestamps, height, width, origins, viewdirs, norms,
                  pixel_coords, out_times, n, stream):
    if n == 0:
        return
    _require(not _addr(pixel_coords) or (height > 0 and width > 0), "emer_gen_rays: pixel coordinates need the image size")
    xs, ys = _vec(x, n), _vec(y, n)
    if _addr(img_idx):
        idx = _vec(img_idx, n, ctype=ctypes.c_int64, dtype=np.int64)
        n_m = int(idx.max()) + 1
    else:
        idx = torch.arange(n) if per_ray_mats else torch.zeros(n, dtype=torch.int64)
        n_m = n if per_ray_mats else 1
    C = _view(c2w, n_m, 16)[idx].view(n, 4, 4)
    K = _view(intrinsics, n_m, 9)[idx].view(n, 3, 3)
    cam = torch.stack([(xs - K[:, 0, 2] + 0.5) / K[:, 0, 0], (ys - K[:, 1, 2] + 0.5) / K[:, 1, 1], torch.ones(n)], -1)
    d = (cam[:, None, :] * C[:, :3, :3]).sum(-1)
    nrm = torch.linalg.norm(d, dim=-1, keepdims=True)
    _view(origins, n, 3).copy_(C[:, :3, 3])
    _view(viewdirs, n, 3).copy_(d / (nrm + 1e-8))
    if _addr(norms):
        _view(norms, n, 1).copy_(nrm)
    if _addr(pixel_coords):
        _view(pixel_coords, n, 2).copy_(torch.stack([ys / height, xs / width], -1))
    if _addr(out_times) and _addr(timestamps):
        _vec(out_times, n).copy_(_vec(timestamps, n_m)[idx])


# ----------------------------------------------------------------------------- optimizer
def emer_adam_step(blocks, prefix, n_blocks, total, hyper, beta1, beta2, eps, weight_decay, zero_grad, stream):
    if n_blocks == 0 or total == 0:
        return
    rows = _view(blocks, n_blocks, 5, ctype=ctypes.c_int64, dtype=np.int64)
    step, lr = [float(v) for v in _vec(hyper, 2)]
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    with torch.no_grad():
        for r in rows.tolist():
            n = r[4]
            p, g, m, v = (_vec(a, n) for a in r[:4])
            _require(all(a % 16 == 0 for a in r[:4]), "emer_adam_step: blocks must be 16-byte aligned")
            gg = g + weight_decay * p if weight_decay != 0 else g.clone()
            m.add_((1.0 - beta1) * (gg - m))
            v.mul_(beta2).add_((1.0 - beta2) * gg * gg)
            p.sub_(np.float32(lr / bc1) * (m / (v.sqrt() * np.float32(1.0 / np.sqrt(bc2)) + eps)))
            if zero_grad:
                g.zero_()


# ----------------------------------------------------------------------------- dispatch
def call(name: str, *args) -> None:
    """Stand-in for ``emernerf_b200._lib.call``: same names, same positional arguments."""
    fn = globals().get(name)
    if fn is None or not name.startswith("emer_"):
        raise NotImplementedError(f"cabi_emulator: {name}")
    CALLS.append(name)
    plain = [a.value if isinstance(a, (ctypes.c_int, ctypes.c_int64, ctypes.c_float)) else a for a in args]
    fn(*plain)


def install(monkeypatch) -> None:
    """Route the product's C-ABI calls to this emulator and let its fused-path selectors accept CPU tensors."""
    from emernerf_b200 import _lib, _ops

    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(_ops, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(_ops, "_stream", lambda: None)
    monkeypatch.setattr(_ops, "on_device", lambda t: True)
    monkeypatch.setattr(_ops, "TC_MIN_ROWS", 64)       # send the larger layers through the tensor-core entry points
    monkeypatch.setattr(_ops, "WGRAD_STREAM", False)   # host memory has no side stream
    del CALLS[:]

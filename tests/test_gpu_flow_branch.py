"""EMER_FLOW_BRANCH=fused: the flow variants' temporal aggregation on the three-query field chain.

- the flow warp (emer_flow_warp_fwd / _bwd) against fp64 restatements of the reference lines, at 2^20 + 17 points with
  points placed on every branch of the contraction, on the aabb faces and where the time clamp bites;
- the three-query chain (emer_flow_field_fwd / _bwd + emer_field_wgrad) against an fp64 restatement, buffer by buffer;
- the whole field with the switch on against the switch off, and the reference-derived goldens under the switch.
"""
import pytest
import torch

import test_gpu_fullsize as tfs
import test_gpu_golden as tgg
from helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
AABB = [-20.0, -40.0, 0.0, 80.0, 40.0, 20.0]


# ----------------------------------------------------------------------------------------------- flow warp
def _contract64(x, aabb):
    """radiance_field.py:278-300 / nerf_utils.py:13-28 with the in-cube selector, in the dtype of x."""
    lo, hi = aabb[:3], aabb[3:]
    xn = (x - lo) / (hi - lo) * 2 - 1
    mag = xn.abs().max(dim=-1, keepdim=True).values
    y = torch.where(mag < 1, xn, (2 - 1 / mag) * (xn / mag)) / 4 + 0.5
    sel = ((y > 0) & (y < 1)).all(dim=-1, keepdim=True)
    return y * sel


def _warp_inputs(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(AABB[:3]), torch.tensor(AABB[3:])
    pos = lo + (hi - lo) * (torch.rand(n, 3, generator=g) * 3 - 1)           # |xn| up to 5: both contraction branches
    flow = torch.randn(n, 6, generator=g) * 5
    noise = torch.rand(n, generator=g)
    t = torch.rand(n, generator=g)
    k = n // 8
    flow[:k] = 0.0                                                            # warped point == pos for these
    # ||xn||_inf == 1 exactly (the cube's faces) and the aabb faces themselves
    pos[: k // 4, 0] = hi[0]
    pos[k // 4: k // 2, 1] = lo[1]
    pos[k // 2: 3 * k // 4] = (lo + hi) / 2
    # the time clamp: t +- dt * noise landing on 0 and 1, and beyond
    t[k: k + 1000], noise[k: k + 1000] = 0.9, 1.0
    t[k + 1000: k + 2000], noise[k + 1000: k + 2000] = 0.1, 1.0
    t[k + 2000: k + 3000] = 0.0
    t[k + 3000: k + 4000] = 1.0
    return pos, flow, noise, t


def test_flow_warp_matches_fp64():
    from emernerf_b200 import _ops

    n = (1 << 20) + 17
    td = 0.1
    pos, flow, noise, t = _warp_inputs(n)
    aabb = torch.tensor(AABB)
    fl = flow.to(DEV).requires_grad_(True)
    coords = _ops.flow_warp(pos.to(DEV), fl, noise.to(DEV), t.to(DEV), aabb.to(DEV), td, True)
    assert coords.shape == (2 * n, 4)
    g = torch.randn(2 * n, 4, generator=torch.Generator().manual_seed(1))
    (d_flow,) = torch.autograd.grad(coords, fl, g.to(DEV))

    # fp64 reference of the same lines, evaluated at the fp32 warped point the reference forms first
    nz = noise[:, None]
    a64 = aabb.double()
    rows, grads, ties = [], [], []
    for d, sign in ((0, 1.0), (1, -1.0)):
        x32 = pos + flow[:, 3 * d: 3 * d + 3] * nz
        # the inf-norm's subgradient goes to the arg-max coordinate: where the two largest |xn| are equal to within fp32
        # rounding, fp32 and fp64 may pick different coordinates and the Jacobian is discontinuous there.  Such rows
        # are counted, not compared
        top = ((x32.double() - a64[:3]) / (a64[3:] - a64[:3]) * 2 - 1).abs().topk(2, dim=-1).values
        ties.append((top[:, 0] >= 1) & (top[:, 0] - top[:, 1] <= 4e-7 * top[:, 0]))
        f64 = flow[:, 3 * d: 3 * d + 3].double().requires_grad_(True)
        x64 = x32.double() + (f64 - f64.detach()) * nz.double()             # value of x32, gradient d x / d flow = noise
        y = _contract64(x64, a64)
        w_t = torch.clamp(t.double() + sign * td * noise.double(), 0, 1)
        rows.append(torch.cat([y.detach(), w_t[:, None]], -1))
        (gf,) = torch.autograd.grad(y, f64, g[d * n:(d + 1) * n, :3].double())
        grads.append(gf)
    want = torch.cat(rows)
    got = coords.detach().cpu().double()
    # the in-cube selector may flip where fp32 and fp64 disagree on a face: such rows are counted, not compared
    same = ((got[:, :3] != 0).any(-1) == (want[:, :3] != 0).any(-1))
    assert (~same).sum() <= 16, int((~same).sum())
    assert rel_err(got[same, :3], want[same, :3]) < 1e-6
    assert rel_err(got[:, 3], want[:, 3]) < 1e-6
    assert torch.equal(got[:, 3].clamp(0, 1), got[:, 3])
    d_want = torch.cat(grads, 1)
    # torch.where's backward is NaN at the cube's centre (the unused branch divides by |xn| = 0): those rows are
    # checked on their own, the kernel's contraction is the identity there
    centre = ~torch.isfinite(d_want).all(-1)
    assert centre.sum() <= n // 32
    tie = ties[0] | ties[1]
    assert tie.sum() <= 16, int(tie.sum())
    ok = same[:n] & same[n:] & ~centre & ~tie
    assert rel_err(d_flow.cpu().double()[ok], d_want[ok]) < 1e-6
    assert torch.isfinite(d_flow).all()


# ----------------------------------------------------------------------------------------------- three-query chain
def _chain64(enc, base, head, ray_bias, samples, density_only):
    wb0, bb0, wb1, bb1 = base
    w0, w1, w2, b2 = head
    n = enc.shape[0] // 3
    F = []
    for q in range(3):
        hb = torch.relu(enc[q * n:(q + 1) * n] @ wb0.T + bb0)
        F.append(hb @ wb1.T + bb1)
    feats = (F[0] + 0.5 * F[1] + 0.5 * F[2]) / 2.0
    sigma = torch.exp(feats[:, 0] - 1.0)
    geo = feats[:, :64]
    sem = feats[:, 64:] if feats.shape[1] > 64 else None
    if density_only:
        return sigma, None, geo, sem
    c = w0.shape[1] - 64
    rb = ray_bias[torch.arange(n, device=enc.device) // samples]
    h0 = torch.relu(geo @ w0[:, c:].T + rb[:, :64])
    h1 = torch.relu(h0 @ w1[:, :64].T + geo @ w1[:, 64 + c:].T + rb[:, 64:])
    return sigma, torch.sigmoid(h1 @ w2.T + b2), geo, sem


@pytest.mark.parametrize("n_feat", [64, 128])
@pytest.mark.parametrize("k_enc", [40, 64])
@pytest.mark.parametrize("mode", ["train", "train_geo_sem", "density", "infer"])
def test_flow_field_chain_matches_fp64(n_feat, k_enc, mode):
    from emernerf_b200 import _ops

    g = torch.Generator().manual_seed(k_enc + n_feat)
    samples, n_rays = 64, 97
    n = samples * n_rays - 13                              # not a multiple of the 64-row tile; a ragged last ray
    r = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc)
    enc = r(3 * n, k_enc, sc=0.5)
    base = [r(64, k_enc, sc=k_enc ** -0.5), r(64, sc=0.1), r(n_feat, 64, sc=0.125), r(n_feat, sc=0.1)]
    head = [r(64, 113, sc=0.1), r(64, 177, sc=0.1), r(3, 64, sc=0.125), r(3, sc=0.1)]
    n_r = (n + samples - 1) // samples
    rb = r(n_r, 128, sc=0.1)
    density_only = mode == "density"
    train = mode != "infer"
    t32 = [x.to(DEV).requires_grad_(train) for x in [enc, rb] + base + head]
    t64 = [x.double().to(DEV).requires_grad_(train) for x in [enc, rb] + base + head]
    with torch.set_grad_enabled(train):
        got = _ops.flow_field_chain(t32[0], None if density_only else t32[1], samples, t32[2:6], t32[6:10])
        want = _chain64(t64[0], t64[2:6], t64[6:10], t64[1], samples, density_only)
    for name, a, b in zip(("sigma", "rgb", "geo", "sem"), got, want):
        assert (a is None) == (b is None), name
        if a is not None:
            assert rel_err(a.detach().double(), b.detach()) < 1e-5, (name, rel_err(a.detach().double(), b.detach()))
    if not train:
        return
    gs = [torch.randn(x.shape, generator=g).to(DEV) if x is not None else None for x in want]
    if mode == "train":                                   # no shadow / dino gradient
        gs[2] = None
        gs[3] = None
    pairs = [(a, gg) for a, gg in zip(got, gs) if a is not None and gg is not None]
    pairs64 = [(b, gg.double()) for b, gg in zip(want, gs) if b is not None and gg is not None]
    g32 = torch.autograd.grad([a for a, _ in pairs], t32, [gg for _, gg in pairs], allow_unused=True)
    g64 = torch.autograd.grad([b for b, _ in pairs64], t64, [gg for _, gg in pairs64], allow_unused=True)
    names = ["d_enc", "d_ray_bias", "wb0", "bb0", "wb1", "bb1", "w0", "w1", "w2", "b2"]
    for name, a, b in zip(names, g32, g64):
        if b is None or not b.abs().sum():
            continue
        assert a is not None, name
        if name == "d_enc":
            for q in range(3):                            # the three row sets
                assert rel_err(a[q * n:(q + 1) * n].double(), b[q * n:(q + 1) * n]) < 1e-4, (name, q)
        else:
            assert rel_err(a.double(), b) < 1e-4, (name, rel_err(a.double(), b))


# ----------------------------------------------------------------------------------------------- whole field
FUSED = {"emer_flow_warp_fwd", "emer_flow_field_fwd"}
FUSED_BWD = {"emer_flow_warp_bwd", "emer_flow_field_bwd"}


@pytest.fixture
def calls(monkeypatch):
    """Names of the library entry points called, in order (so a test can tell which path ran)."""
    from emernerf_b200 import _lib

    names, real = [], _lib.call

    def record(name, *args):
        names.append(name)
        return real(name, *args)

    monkeypatch.setattr(_lib, "call", record)
    return names


def _grads(field):
    return {k: v.grad.detach().clone() for k, v in field.named_parameters() if v.grad is not None}


@pytest.mark.parametrize("variant", ["flow", "flow_feat"])
@pytest.mark.parametrize("mode", ["train", "lidar", "eval"])
def test_switch_on_matches_switch_off(variant, mode, monkeypatch, calls):
    from emernerf_b200 import _ops

    g, field, props, est = tfs._build(variant)
    res = {}
    for sw in ("layers", "fused"):
        monkeypatch.setattr(_ops, "FLOW_BRANCH", sw)
        del calls[:]
        out = tfs._render(g, field, props, est, mode)
        if mode != "eval":
            loss = sum((v.float() ** 2).mean() for k, v in out.items() if torch.is_tensor(v) and v.requires_grad)
            loss.backward()
        res[sw] = (out, _grads(field) if mode != "eval" else {})
        want = (FUSED | FUSED_BWD) if mode != "eval" else FUSED
        if sw == "fused":
            assert want <= set(calls), sorted(want - set(calls))
        else:
            assert not (FUSED | FUSED_BWD) & set(calls)
    (a, ga), (b, gb) = res["layers"], res["fused"]
    tol = tfs._tols(mode)
    for k, v in a.items():
        if torch.is_tensor(v):
            assert rel_err(b[k].float(), v.float()) < tol.get(k, tol["*"]), (k, rel_err(b[k].float(), v.float()))
    assert ga.keys() == gb.keys()
    for k in ga:
        assert rel_err(gb[k], ga[k]) < 5e-3, (k, rel_err(gb[k], ga[k]))


@pytest.mark.parametrize("variant", ["flow", "flow_feat"])
def test_switch_keeps_keys_and_generator_state(variant, monkeypatch):
    """Without a noise override the fused path draws the warp's noise with the same call in the same place."""
    from emernerf_b200 import _ops
    from emernerf_b200.radiance_fields.render_utils import render_rays
    from golden import full_cases as fc

    g, field, props, est = tfs._build(variant)
    batch = g.tensors("in/pixel", DEV)
    field.train(True); est.train(True)
    field._noise_override = None
    est._jitter_override = None
    outs, states = {}, {}
    for sw in ("layers", "fused"):
        monkeypatch.setattr(_ops, "FLOW_BRANCH", sw)
        torch.manual_seed(7)
        est.prop_cache.clear()
        out = render_rays(field, est, props, batch, fc.render_cfg(), proposal_requires_grad=False)
        outs[sw], states[sw] = out, torch.cuda.get_rng_state()
    assert torch.equal(states["layers"], states["fused"])
    ea, eb = outs["layers"]["extras"], outs["fused"]["extras"]
    assert list(ea) == list(eb)
    for k in ea:
        if torch.is_tensor(ea[k]):
            assert ea[k].shape == eb[k].shape, k


@pytest.mark.parametrize("variant", ["flow", "flow_feat"])
@pytest.mark.parametrize("mode", ["eval", "lidar", "train"])
def test_full_size_goldens_under_the_switch(variant, mode, monkeypatch, calls):
    from emernerf_b200 import _ops

    monkeypatch.setattr(_ops, "FLOW_BRANCH", "fused")
    tfs.test_full_size_render_matches_reference(variant, mode)
    assert FUSED <= set(calls)


@pytest.mark.parametrize("variant", ["flow", "flow_feat"])
def test_full_size_gradients_under_the_switch(variant, monkeypatch, calls):
    from emernerf_b200 import _ops

    monkeypatch.setattr(_ops, "FLOW_BRANCH", "fused")
    tfs.test_full_size_gradients_and_proposal_loss(variant)
    assert (FUSED | FUSED_BWD) <= set(calls)


@pytest.mark.parametrize("case", ["flow", "flow_feat"])
@pytest.mark.parametrize("mode", ["eval", "lidar", "train"])
def test_small_goldens_under_the_switch_take_the_per_layer_path(case, mode, monkeypatch, calls):
    """The miniature cases' dynamic grid has L*F = 16, a shape the chain does not cover: with the switch on they run the
    per-layer path and still match their goldens."""
    from emernerf_b200 import _ops

    monkeypatch.setattr(_ops, "FLOW_BRANCH", "fused")
    tgg.test_render_rays_matches_reference_outputs(case, mode)
    assert not (FUSED | FUSED_BWD) & set(calls)


# ----------------------------------------------------------------------------------------------- saves, buffer by buffer
@pytest.mark.parametrize("n_feat", [64, 128])
@pytest.mark.parametrize("k_enc", [40, 64])
def test_flow_field_saves_and_data_gradients_match_fp64(n_feat, k_enc):
    """Every buffer emer_flow_field_fwd / _bwd write, against the fp64 autograd of the same lines: hb for the three
    row sets, [h0 | geo], h1, the blended semantic half; dz2, dz1, [dz0 | dF_q] (dF_q = d loss / d F_q), dzb, d_sem_q,
    d_enc and the per-ray sums."""
    from emernerf_b200 import _lib, _ops

    g = torch.Generator().manual_seed(3 * k_enc + n_feat)
    samples, n_rays = 64, 53
    n = samples * n_rays
    r = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc).double().to(DEV)
    enc = r(3 * n, k_enc, sc=0.5)
    wb0, bb0, wb1, bb1 = r(64, k_enc, sc=k_enc ** -0.5), r(64, sc=0.1), r(n_feat, 64, sc=0.125), r(n_feat, sc=0.1)
    w0, w1, w2, b2 = r(64, 113, sc=0.1), r(64, 177, sc=0.1), r(3, 64, sc=0.125), r(3, sc=0.1)
    rb = r(n_rays, 128, sc=0.1)
    d_rgb, d_sigma, d_geo = r(n, 3), r(n), r(n, 64)
    d_sem = r(n, 64) if n_feat == 128 else None

    # fp64 reference with every intermediate kept
    pre_b = [(enc[q * n:(q + 1) * n] @ wb0.T + bb0).requires_grad_(True) for q in range(3)]
    hb = [torch.relu(p) for p in pre_b]
    F = [(h @ wb1.T + bb1).requires_grad_(True) for h in hb]
    feats = (F[0] + 0.5 * F[1] + 0.5 * F[2]) / 2.0
    geo = feats[:, :64]
    ray = torch.arange(n, device=DEV) // samples
    a0 = (geo @ w0[:, 49:].T + rb[ray, :64]).requires_grad_(True)
    h0 = torch.relu(a0)
    a1 = (h0 @ w1[:, :64].T + geo @ w1[:, 113:].T + rb[ray, 64:]).requires_grad_(True)
    h1 = torch.relu(a1)
    z = (h1 @ w2.T + b2).requires_grad_(True)
    rgb, sigma = torch.sigmoid(z), torch.exp(feats[:, 0] - 1.0)
    loss = (rgb * d_rgb).sum() + (sigma * d_sigma).sum() + (geo * d_geo).sum()
    if d_sem is not None:
        loss = loss + (feats[:, 64:] * d_sem).sum()
    gz, ga1, ga0, *gF = torch.autograd.grad(loss, [z, a1, a0] + F, retain_graph=True)
    gpre = torch.autograd.grad(loss, pre_b)

    f32 = lambda t: None if t is None else t.float().contiguous()
    e32, wb0f, bb0f, wb1f, bb1f, w0f, w1f, w2f, b2f, rbf = (f32(t) for t in (enc, wb0, bb0, wb1, bb1, w0, w1, w2, b2, rb))
    e = lambda *s: torch.empty(*s, dtype=torch.float32, device=DEV)
    sig, rgb_o, hb_o, hg_o, h1_o = e(n), e(n, 3), e(3 * n, 64), e(n, 128), e(n, 64)
    sem_o = e(n, 64) if n_feat == 128 else None
    P = _ops._ptr
    _ops._need_cuda(e32)
    _lib.call("emer_flow_field_fwd", P(e32), k_enc, k_enc, P(wb0f), P(bb0f), P(wb1f), P(bb1f), n_feat, P(w0f[:, 49:]), 113,
              P(w1f[:, :64]), P(w1f[:, 113:]), 177, P(w2f), P(b2f), P(rbf), samples, P(sig), P(rgb_o), P(hb_o), P(hg_o),
              P(h1_o), P(sem_o), n, _ops._stream())
    chk = lambda name, a, b, tol=1e-5: (lambda err: None if err < tol else pytest.fail(f"{name}: {err}"))(
        rel_err(a.double(), b.detach()))
    for q in range(3):
        chk(f"hb[{q}]", hb_o[q * n:(q + 1) * n], hb[q])
    chk("h0", hg_o[:, :64], h0)
    chk("geo", hg_o[:, 64:], geo)
    chk("h1", h1_o, h1)
    chk("sigma", sig, sigma)
    chk("rgb", rgb_o, rgb)
    if sem_o is not None:
        chk("sem", sem_o, feats[:, 64:])

    w1hg = torch.cat([w1f[:, :64], w1f[:, 113:]], dim=1)
    w0g = w0f[:, 49:].contiguous()
    dz2, dz1, D1, dzb, d_enc = e(n, 3), e(n, 64), e(3 * n, 128), e(3 * n, 64), e(3 * n, k_enc)
    d_sem_q = e(3 * n, 64) if d_sem is not None else None
    d_rb = torch.zeros(n_rays, 128, device=DEV)
    d_rgb32, d_sigma32, d_geo32, d_sem32 = (f32(t) for t in (d_rgb, d_sigma, d_geo, d_sem))     # (kept alive)
    _lib.call("emer_flow_field_bwd", P(d_rgb32), P(rgb_o), P(d_sigma32), P(sig), P(d_geo32), P(d_sem32),
              P(hb_o), P(hg_o), P(h1_o), P(wb0f), k_enc, P(wb1f), n_feat, P(w0g), 64, P(w1hg), P(w1hg[:, 64:]), 128,
              P(w2f), P(dz2), P(dz1), P(D1), P(dzb), P(d_enc), k_enc, P(d_rb), P(d_sem_q), samples, n, _ops._stream())
    chk("dz2", dz2, gz)
    chk("dz1", dz1, ga1, 1e-4)
    chk("dz0", D1[:n, :64], ga0, 1e-4)
    for q in range(3):
        chk(f"dF[{q}]", D1[q * n:(q + 1) * n, 64:], gF[q][:, :64], 1e-4)
        chk(f"dzb[{q}]", dzb[q * n:(q + 1) * n], gpre[q], 1e-4)
        chk(f"d_enc[{q}]", d_enc[q * n:(q + 1) * n], gpre[q] @ wb0, 1e-4)
        if d_sem_q is not None:
            chk(f"d_sem_q[{q}]", d_sem_q[q * n:(q + 1) * n], gF[q][:, 64:])
    chk("d_ray_bias", d_rb, torch.cat([torch.zeros(n_rays, 64, device=DEV, dtype=torch.float64).index_add_(0, ray, ga0),
                                       torch.zeros(n_rays, 64, device=DEV, dtype=torch.float64).index_add_(0, ray, ga1)], 1),
        1e-4)


# ----------------------------------------------------------------------------------------------- a training step
def _field_step_inputs(g):
    batch = g.tensors("in/pixel", DEV)
    S = 64
    tv = torch.linspace(2.0, 60.0, S, device=DEV).expand(batch["origins"].shape[0], S)
    d = batch["viewdirs"][:, None, :].expand(-1, S, -1)
    sub = {k: v.unsqueeze(-1).expand(*v.shape, S) for k, v in batch.items()
           if k not in ("viewdirs", "origins", "pixel_coords")}
    sub["pixel_coords"] = batch["pixel_coords"]
    return batch["origins"][:, None, :] + d * tv[..., None], d, sub


@pytest.mark.parametrize("variant", ["flow", "flow_feat"])
def test_fused_training_step_is_sync_free_and_replays_in_a_graph(variant, monkeypatch, calls):
    """Field forward + backward of a training step under the switch: no host sync (set_sync_debug_mode("error")), and
    captured into a CUDA graph its replay computes what the eager step computes."""
    from emernerf_b200 import _ops

    monkeypatch.setattr(_ops, "FLOW_BRANCH", "fused")
    g, field, props, est = tfs._build(variant)
    pos, d, sub = _field_step_inputs(g)
    field.train(True)
    field._noise_override = torch.rand(*pos.shape[:2], 1, generator=torch.Generator().manual_seed(2)).to(DEV)
    params = [p for p in field.parameters() if p.requires_grad]

    def step():
        out = field(pos, d, sub)
        loss = sum((v.float() ** 2).mean() for k, v in out.items() if torch.is_tensor(v) and v.requires_grad)
        grads = torch.autograd.grad(loss, params, allow_unused=True)
        return out["dynamic_density"], [gr for gr in grads if gr is not None]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            want_density, want_grads = step()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            step()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.current_stream().wait_stream(side)
    assert FUSED | FUSED_BWD <= set(calls)

    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got_density, got_grads = step()
    graph.replay()
    torch.cuda.synchronize()
    assert rel_err(got_density, want_density) < 1e-6
    for a, b in zip(got_grads, want_grads):
        assert rel_err(a, b) < 1e-4

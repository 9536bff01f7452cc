"""Known-answer tests for the nerfacc restatement (the only published vectors available
offline: the ``importance_sampling`` docstring example of nerfacc@8340e19)."""
import torch

from oracle import nerfacc_ref as nf


def test_importance_sampling_docstring_example():
    # nerfacc/pdf.py docstring: ray 0 vals [0,1] cdfs [0,.5]; ray 1 vals [0,1,2] cdfs [0,.5,1]; n=2
    iv, sm = nf.importance_sampling(nf.RayIntervals(torch.tensor([[0.0, 1.0]])), torch.tensor([[0.0, 0.5]]), 2)
    assert torch.equal(iv.vals, torch.tensor([[0.0, 0.5, 1.0]]))
    assert torch.equal(sm.vals, torch.tensor([[0.25, 0.75]]))
    iv, sm = nf.importance_sampling(nf.RayIntervals(torch.tensor([[0.0, 1.0, 2.0]])),
                                    torch.tensor([[0.0, 0.5, 1.0]]), 2)
    assert torch.equal(iv.vals, torch.tensor([[0.0, 1.0, 2.0]]))
    assert torch.equal(sm.vals, torch.tensor([[0.5, 1.5]]))


def test_importance_sampling_edges_sorted_and_bounded():
    g = torch.Generator().manual_seed(0)
    R, m, n = 64, 33, 17
    vals = torch.sort(torch.rand(R, m, generator=g), -1).values
    w = torch.rand(R, m - 1, generator=g)
    cdfs = torch.cat([torch.zeros(R, 1), torch.cumsum(w / w.sum(-1, keepdim=True), -1)], -1)
    cdfs[:, -1] = 1.0
    for strat in (False, True):
        iv, _ = nf.importance_sampling(nf.RayIntervals(vals), cdfs, n, strat, jitter=torch.rand(R, 1, generator=g))
        e = iv.vals
        assert e.shape == (R, n + 1)
        assert (e[:, 1:] >= e[:, :-1]).all()
        assert (e >= vals[:, :1]).all() and (e <= vals[:, -1:]).all()


def test_volrend_identities():
    g = torch.Generator().manual_seed(1)
    t = torch.sort(torch.rand(8, 17, generator=g), -1).values
    sig = torch.rand(8, 16, generator=g) * 5
    w, tr, al = nf.render_weight_from_density(t[:, :-1], t[:, 1:], sig)
    # telescoping: sum of weights = 1 - T_end
    t_end = tr[:, -1] * (1 - al[:, -1])
    assert torch.allclose(w.sum(-1), 1 - t_end, atol=1e-6)
    assert torch.equal(tr[:, 0], torch.ones(8))
    assert torch.allclose(nf.accumulate_along_rays(w, None)[:, 0], w.sum(-1))


def test_composite64_matches_autograd_through_the_restatement():
    """composite64 against float64 autograd through render_transmittance_from_density / accumulate_along_rays on empty
    (clamped at 1e-6), faint, partial and saturated rays; the clamp at 1, which only an fp32 sum reaches, taken from the
    kernel's weights; and its kernel-order fp32 ray sum against a plain loop over lanes."""
    g = torch.Generator().manual_seed(3)
    R, S = 12, 45
    edges = torch.sort(torch.rand(R, S + 1, generator=g) * 10, -1).values
    t0, t1 = edges[:, :-1].contiguous(), edges[:, 1:].contiguous()
    sigma = torch.rand(R, S, generator=g) * 2
    sigma[:3] = 0.0
    sigma[3:6] *= 1e-5
    sigma[6:9] *= 100
    gw, gt, gc = (torch.randn(R, n, generator=g) for n in (S, S, S + 1))
    go, gd = torch.randn(R, 1, generator=g), torch.randn(R, 1, generator=g)
    got = nf.composite64(t0, t1, sigma, None, gw, gt, go, gd, gc)

    f64 = torch.float64
    delta = (t1 - t0).to(f64)
    mid = ((t0 + t1) / 2.0).to(f64)
    so = sigma.to(f64).requires_grad_(True)
    trans, alphas = nf.render_transmittance_from_density(t0.to(f64), (t0.to(f64) + delta), so)
    w = trans * alphas
    op = nf.accumulate_along_rays(w, None).clamp(1e-6, 1.0)
    dep = nf.accumulate_along_rays(w, mid[..., None]) / op
    cdf = 1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], -1)
    loss = (w * gw).sum() + (trans * gt).sum() + (op * go).sum() + (dep * gd).sum() + (cdf * gc).sum()
    (ds,) = torch.autograd.grad(loss, so, retain_graph=True)
    (G,) = torch.autograd.grad(loss, w)
    for k, want in (("weights", w), ("trans", trans), ("opacity", op), ("depth", dep), ("cdf", cdf), ("dsigma", ds),
                    ("G", G)):
        assert torch.allclose(got[k], want.detach(), rtol=1e-12, atol=1e-300), k
    assert got["in_range"][:3].logical_not().all() and got["in_range"][3:].all()
    cw = torch.cumsum(w.detach(), -1)
    idx = torch.searchsorted(cw, torch.full((R, 1), 0.5), side="left").clamp(0, S - 1)
    assert torch.equal(got["median_idx"], idx[:, 0])
    e = torch.cat([torch.zeros(R, 1, dtype=f64), torch.cumsum(so.detach() * delta, -1)[:, :-1]], -1)
    assert torch.allclose(got["E"], e, rtol=1e-12)
    q = G.abs() * w.detach() + (gt.to(f64) - gc[:, :S].to(f64)).abs() * trans.detach()
    b = torch.stack([q[:, i + 1:].sum(-1) for i in range(S)], -1)
    assert torch.allclose(got["B"], b, rtol=1e-12)
    assert torch.allclose(got["A"], G.abs() * trans.detach() * torch.exp(-(so.detach() * delta)), rtol=1e-12)

    # fp32 weights whose kernel-order sum passes 1 take the upper clamp: opacity 1, no gradient through it
    w32 = w.detach().float()
    w32[6:9] *= 1.01
    hi = nf.composite64(t0, t1, sigma, w32, gw, gt, go, gd, gc)
    assert hi["in_range"][:3].logical_not().all() and hi["in_range"][3:6].all()
    assert hi["in_range"][6:9].logical_not().all()
    assert torch.equal(hi["opacity"][6:9], torch.ones(3, 1, dtype=f64))
    assert torch.allclose(hi["G"][6:9], gw[6:9].to(f64) + gd[6:9].to(f64) * mid[6:9], rtol=1e-12)
    assert torch.allclose(hi["G"][:6], G[:6], rtol=1e-12)

    w32 = torch.rand(R, 70, generator=g)
    lanes = [torch.zeros(R) for _ in range(32)]
    for s in range(70):
        lanes[s % 32] = lanes[s % 32] + w32[:, s]
    for o in (16, 8, 4, 2, 1):
        lanes = [lanes[i] + lanes[i ^ o] for i in range(32)]
    assert torch.equal(nf.warp_sum32(w32), lanes[0])

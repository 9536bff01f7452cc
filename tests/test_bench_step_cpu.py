"""bench.py's two arms compute the same workload: one training step of the GPU arm (``Trainer._step_body`` --
render_rays + proposal update + pixel losses + backward + Adam, here on CPU with the C ABI answered by
tests/cabi_emulator.py) against the step the reference arm times (``cpu_baseline``: oracle render_rays +
the same losses + backward), on the same full-size default configuration, tables, batch and random draws."""
import importlib.util
import os
import types

import pytest
import torch

import cabi_emulator
from helpers import rel_err
from oracle import adapters, hotpath

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bench():
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("variant", ["static"])        # (flow_feat: same code path, 90 s on CPU -- run by hand)
def test_training_step_of_both_arms_is_the_same_computation(monkeypatch, variant):
    from emernerf_b200 import configs, synthetic

    bench = _bench()
    cabi_emulator.install(monkeypatch)
    n_rays, samples = 24, 64
    cfg = configs.make_cfg(variant, num_samples=samples)
    field, props, est, opt = configs.build_hot_path(cfg, "cpu", table_std=0.3)
    feats = variant == "flow_feat"
    batch = synthetic.pixel_batch(n_rays, cfg.data.num_timesteps, 3, seed=5, features=feats)

    # ---- reference arm's step (what cpu_baseline times), on copies of the same parameters
    fsd = adapters.cpu_state_dict(field, requires_grad=True)
    psd = [adapters.cpu_state_dict(p, requires_grad=True) for p in props]
    torch.manual_seed(123)
    out_o, cache = hotpath.render_rays(fsd, adapters.spec_from_module(field), psd,
                                       [adapters.spec_from_module(p) for p in props], batch, num_samples=samples,
                                       prop_samples=cfg.nerf.propnet.num_samples_per_prop, near_plane=0.1,
                                       far_plane=1000.0, training=True, proposal_requires_grad=True)
    loss_o = bench.pixel_losses(out_o, batch)
    ploss_o = hotpath.proposal_loss(cache, out_o["extras"]["trans"], tuple(cfg.nerf.propnet.anti_aliasing_pulse_width),
                                    1024.0)
    names = [k for k, v in fsd.items() if v.requires_grad]
    grads_o = dict(zip(names, torch.autograd.grad(loss_o * 1024.0, [fsd[k] for k in names], allow_unused=True)))

    # ---- GPU arm's step body, unmodified
    tr = bench.Trainer.__new__(bench.Trainer)
    tr.args = types.SimpleNamespace(variant=variant, rays=n_rays, samples=samples)
    tr.rank, tr.world, tr.device, tr.cfg = 0, 1, "cpu", cfg
    tr.dp = None                      # torch.optim.Adam arm: the gradients stay inspectable after the step
    tr.field, tr.props, tr.est, tr.opt = field, props, est, opt
    tr.params = list(field.parameters())
    tr.prop_params = [p for m in props for p in m.parameters()]
    field.train(); est.train()
    [p.train() for p in props]
    before = {k: v.detach().clone() for k, v in field.named_parameters()}
    prop_before = [p.detach().clone() for p in tr.prop_params]
    torch.manual_seed(123)
    loss = tr._step_body(batch, True)                      # a proposal-update step

    assert abs(loss.item() - loss_o.item()) <= 2e-6 * max(1.0, abs(loss_o.item()))
    # same gradients reached the optimizer ...
    checked = 0
    for k, v in field.named_parameters():
        g = grads_o.get(k)
        if g is None:
            continue
        assert v.grad is not None, k
        assert rel_err(v.grad, g) < 2e-5, k
        checked += 1
    assert checked >= 10
    # ... Adam moved the parameters, and the proposal update moved the LAST proposal network only (Q21)
    moved = [k for k, v in field.named_parameters() if not torch.equal(v.detach(), before[k])]
    assert len(moved) >= checked
    n0 = len(list(props[0].parameters()))
    assert all(torch.equal(p.detach(), b) for p, b in zip(tr.prop_params[:n0], prop_before[:n0]))
    assert any(not torch.equal(p.detach(), b) for p, b in zip(tr.prop_params[n0:], prop_before[n0:]))
    assert ploss_o.item() > 0 and len(est.prop_cache) == 0   # the cache was consumed by the update

    # a step without proposal gradients goes through the fused proposal level
    del cabi_emulator.CALLS[:]
    tr._step_body(batch, False)
    assert "emer_prop_level" in cabi_emulator.CALLS


def test_lidar_half_of_the_iteration_runs_and_matches_the_reference_losses(monkeypatch):
    """bench.py's lidar pass (density-only render, range + line-of-sight losses, backward, second Adam step) on CPU
    through the emulator; its loss restated with the reference's own formulas (boolean indexing, loss/base.py:188-269,
    430-464) gives the same number."""
    from emernerf_b200 import configs, synthetic

    bench = _bench()
    cabi_emulator.install(monkeypatch)
    cfg = configs.make_cfg("dynamic", num_samples=64)
    field, props, est, opt = configs.build_hot_path(cfg, "cpu", table_std=0.3)
    tr = bench.Trainer.__new__(bench.Trainer)
    tr.rank, tr.world, tr.device, tr.cfg, tr.dp = 0, 1, "cpu", cfg, None
    tr.field, tr.props, tr.est, tr.opt = field, props, est, opt
    tr.params = list(field.parameters())
    tr.prop_params = [p for m in props for p in m.parameters()]
    field.train(); est.train()
    [p.train() for p in props]
    lb = synthetic.lidar_batch(24, cfg.data.num_timesteps, seed=3)
    before = field.xyz_encoder.tcnn_encoding.params.detach().clone()
    torch.manual_seed(7)
    loss = tr._lidar_body(lb, False)
    assert torch.isfinite(loss) and not torch.equal(field.xyz_encoder.tcnn_encoding.params.detach(), before)

    from emernerf_b200.radiance_fields.render_utils import render_rays
    torch.manual_seed(7)
    field.eval(); est.eval()
    with torch.no_grad():
        out = render_rays(field, est, props, lb, cfg, prefix="lidar_")
    gt = lb["lidar_ranges"].squeeze()
    pred = out["depth"].squeeze()
    valid = (gt > 0.01) & (gt < 80)
    want = torch.nn.functional.mse_loss(torch.clamp(pred[valid] / 80, 0, 1), torch.clamp(gt[valid] / 80, 0, 1))
    w, t = out["extras"]["weights"], out["extras"]["t_vals"]
    g = gt.unsqueeze(-1)
    eps = 2.0
    dirac = (1 / (2 * torch.pi * (eps / 3) ** 2) ** 0.5) * torch.exp(-((t - g) ** 2) / (2 * (eps / 3) ** 2))
    sight = ((w.square() * (t < g - eps)).sum(-1, keepdim=True).mean()
             + ((w - dirac).square() * ((t > g - eps) & (t < g + eps))).sum(-1, keepdim=True).mean()) * (gt > 0)
    want = want + 0.1 * sight.mean() + 0.01 * out["extras"]["dynamic_density"].mean()
    got = bench.lidar_losses(out, lb)
    assert abs(got.item() - want.item()) <= 1e-6 * max(1.0, abs(want.item()))

"""``train.CapturedIteration``'s host side and the live line-of-sight loss on CPU.

* ``CapturedIteration.__call__`` over every step of the default 25 000-iteration run, its graphs stubbed out: each
  pass's key, the learning rates both optimizers hold when it starts, the staged line-of-sight constants and the CPU
  generator's draws, against a restatement of train_emernerf.py:612-855's host side with builders.py's schedulers.
* The refusals: check_nan, the reference's loss classes, an optimizer other than FusedAdam, more than one rank, a
  source without the device sampler.
* The live entry points through the emulator: value and gradient equal to the float entries' for the same epsilon and
  decay weight, and ``line_of_sight_consts`` rounds what the float call rounds.
"""
import ctypes
import types

import numpy as np
import pytest
import torch

import cabi_emulator
import live_loss_emulator

NS = types.SimpleNamespace


def default_cfg(num_iters=25000):
    los = NS(enable=True, start_iter=2000, decay_steps=2000, decay_rate=0.5, start_epsilon=6.0, end_epsilon=2.5)
    return NS(supervision=NS(depth=NS(enable=True, line_of_sight=los)), optim=NS(num_iters=num_iters),
              data=NS(pixel_source=NS(load_rgb=True), lidar_source=NS(load_lidar=True)))


def builders_scheduler(opt, num_iters):
    """builders.py:67-89 and 129-142."""
    milestones = [num_iters // 2, num_iters * 3 // 4, num_iters * 9 // 10]
    if num_iters >= 10000:
        milestones.insert(0, num_iters // 4)
    return torch.optim.lr_scheduler.ChainedScheduler([
        torch.optim.lr_scheduler.LinearLR(opt, start_factor=0.01, total_iters=num_iters // 10),
        torch.optim.lr_scheduler.MultiStepLR(opt, milestones=milestones, gamma=0.33)])


def host_fused_adam(lr=0.01):
    """A FusedAdam with param_groups and nothing on a device: what the schedulers and the refusals look at."""
    from emernerf_b200.optim import FusedAdam

    opt = FusedAdam.__new__(FusedAdam)
    torch.optim.Optimizer.__init__(opt, [torch.nn.Parameter(torch.zeros(1))], dict(lr=lr))
    return opt


class Split:
    def __init__(self, source, split_indices):
        self.datasource, self.split_indices = source, split_indices

    def __len__(self):
        return 1000000


def reference_passes(cfg):
    """train_emernerf.py:612-855's host side with builders.py's schedulers: per pass, (key branch, main lr, proposal
    lr, epsilon and decay weight or None), and the CPU generator's state at the end."""
    from emernerf_b200.third_party.nerfacc_prop_net import get_proposal_requires_grad_fn

    los = cfg.supervision.depth.line_of_sight
    opt, prop_opt = (torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.01) for _ in range(2))
    sched, prop_sched = builders_scheduler(opt, cfg.optim.num_iters), builders_scheduler(prop_opt, cfg.optim.num_iters)
    req = get_proposal_requires_grad_fn()
    epsilon_final, epsilon_start = los.end_epsilon, los.start_epsilon
    decay, passes = 1.0, []
    torch.manual_seed(0)
    for step in np.arange(0, cfg.optim.num_iters + 1):          # the reference iterates numpy integers
        if step > los.start_iter and (step - los.start_iter) % los.decay_steps == 0:
            decay *= los.decay_rate
        for kind in ("pixel", "lidar"):
            prg = req(int(step))
            torch.randint(0, 1000000, (1,)).item()
            sight = None
            if kind == "lidar" and step > los.start_iter:
                m = (epsilon_final - epsilon_start) / (cfg.optim.num_iters - los.start_iter)
                b = epsilon_start - m * los.start_iter
                eps = epsilon_start if step < los.start_iter else epsilon_final if step > cfg.optim.num_iters else m * step + b
                sight = (eps, decay)
            branch = (prg, False) if kind == "pixel" else (prg, sight is not None)
            passes.append((kind, branch, opt.param_groups[0]["lr"], prop_opt.param_groups[0]["lr"], sight))
            prop_sched.step()                   # update_every_n_steps, either branch
            sched.step()
    return passes, torch.get_rng_state()


def test_keys_learning_rates_and_line_of_sight_of_every_pass_over_the_default_run(monkeypatch):
    """CapturedIteration.__call__ over the 25 001 steps of the default schedule, with its graphs stubbed out: the key of
    every pass, the learning rates of both optimizers when the pass starts (what sync_lr writes), the staged epsilon and
    decay weight, and the CPU generator's draws, against the restatement above."""
    import warnings

    from emernerf_b200 import loss, raygen
    from emernerf_b200.third_party.nerfacc_prop_net import get_proposal_requires_grad_fn
    from emernerf_b200.train import CapturedIteration

    cfg = default_cfg()
    want, want_rng = reference_passes(cfg)
    got, staged = [], []

    def run(self, key, body, held):
        sight = staged.pop() if key[0] == "lidar" and key[1][1] else None
        got.append((key[0], key[1], self.optimizer.param_groups[0]["lr"], self.est.optimizer.param_groups[0]["lr"],
                    sight))
        return []

    monkeypatch.setattr(CapturedIteration, "_device_state", lambda self, dev: None)
    monkeypatch.setattr(CapturedIteration, "_run", run)
    monkeypatch.setattr(CapturedIteration, "_stage_sight", lambda self, vals: staged.append(vals))
    monkeypatch.setattr(CapturedIteration, "_read_ring", lambda self: self._pending.clear() or [])
    pix = NS(buffer_ratio=0.25, pixel_error_buffered=False, pixel_error_maps=None)
    pix.get_train_rays = raygen.PixelRaySampler(pix).get_train_rays
    lid = NS()
    lid.get_train_rays = raygen.LidarRaySampler(lid).get_train_rays
    dataset = NS(train_pixel_set=Split(pix, [0, 2, 3]), train_lidar_set=Split(lid, [1, 4]))
    opt, prop_opt = host_fused_adam(), host_fused_adam()
    est = torch.nn.Module()
    est.optimizer, est.scheduler = prop_opt, builders_scheduler(prop_opt, cfg.optim.num_iters)
    losses = {"rgb": loss.RealValueLoss(), "depth": loss.DepthLoss(), "line_of_sight": loss.LineOfSightLoss()}

    it = CapturedIteration(cfg, dataset, torch.nn.Linear(1, 1), est, [], opt,
                           builders_scheduler(opt, cfg.optim.num_iters), losses, get_proposal_requires_grad_fn())
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                   # the stubbed passes never call optimizer.step()
        for step in np.arange(0, cfg.optim.num_iters + 1):
            it(step)
    assert torch.equal(torch.get_rng_state(), want_rng)
    assert len(got) == len(want) == 2 * (cfg.optim.num_iters + 1)
    for n, (g, w) in enumerate(zip(got, want)):
        assert g[:4] == w[:4], (n, g, w)
        if w[4] is None:
            assert g[4] is None, n
        else:
            assert g[4] == loss.line_of_sight_consts(*w[4]), (n, g[4], w[4])
    # from step 1000 on, every sixth call of the proposal schedule asks for gradients; with two calls per iteration
    # that is always the pixel pass, so the lidar pass never updates the proposals once line of sight is on
    assert {(k, b) for k, b, *_ in got} == {("pixel", (False, False)), ("pixel", (True, False)),
                                            ("lidar", (False, False)), ("lidar", (True, False)),
                                            ("lidar", (False, True))}
    assert it.los.decay_weight == 0.5 ** 11


class _Opt:
    """A stand-in optimizer with a scheduler's ``param_groups``."""
    param_groups = [{"lr": 0.01}]


def _fused():
    from emernerf_b200.optim import FusedAdam

    return FusedAdam.__new__(FusedAdam)       # passes the type check; never stepped here


def _args(losses=None, opt=None, prop_opt=None, dataset=None):
    from emernerf_b200 import loss

    est = NS(optimizer=prop_opt if prop_opt is not None else _fused(), scheduler=None)
    losses = losses if losses is not None else {"rgb": loss.RealValueLoss()}
    return (None, dataset if dataset is not None else NS(), None, est, [], opt if opt is not None else _fused(), None,
            losses, lambda step: False)


def test_refusals(monkeypatch):
    import torch.distributed as dist

    from emernerf_b200 import loss
    from emernerf_b200.train import CapturedIteration

    with pytest.raises(ValueError, match="check_nan"):
        CapturedIteration(*_args(losses={"rgb": loss.RealValueLoss(check_nan=True)}))

    class ReferenceLoss(torch.nn.Module):          # what loss/base.py's classes are: not emernerf_b200.loss.Loss
        check_nan = False

    with pytest.raises(TypeError, match="boolean indexing"):
        CapturedIteration(*_args(losses={"rgb": loss.RealValueLoss(), "depth": ReferenceLoss()}))
    adam = torch.optim.Adam([torch.nn.Parameter(torch.zeros(1))])
    with pytest.raises(TypeError, match="FusedAdam"):
        CapturedIteration(*_args(opt=adam))
    with pytest.raises(TypeError, match="FusedAdam"):
        CapturedIteration(*_args(prop_opt=adam))
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(RuntimeError, match="2 ranks"):
        CapturedIteration(*_args())
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 1)
    src = NS(get_train_rays=lambda num_rays, candidate_indices=None: {})
    with pytest.raises(TypeError, match="PixelRaySampler"):
        CapturedIteration(*_args(dataset=NS(train_pixel_set=NS(datasource=src))))


@pytest.fixture
def em(monkeypatch):
    live_loss_emulator.install(monkeypatch)
    return cabi_emulator


def _rays(n=97, s=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(n, generator=g) * 60.0
    gt[::7] = 0.0
    t = torch.sort(torch.rand(n, s, generator=g) * 80.0, dim=-1).values
    w = torch.rand(n, s, generator=g) / s
    return w, t, gt


@pytest.mark.parametrize("eps", [6.0, 4.3, 2.5])
@pytest.mark.parametrize("decay", [1.0, 0.5, 0.125])
def test_live_entries_match_the_float_entries(em, eps, decay):
    from emernerf_b200 import loss

    w, t, gt = _rays()
    fn = loss.LineOfSightLoss(coef=0.1)
    w_f = w.clone().requires_grad_(True)
    v_f = fn(None, gt, w_f, t, eps, coef_decay=decay)["line_of_sight_my"]
    v_f.backward()
    del em.CALLS[:]
    w_l = w.clone().requires_grad_(True)
    consts = torch.tensor(loss.line_of_sight_consts(eps, decay), dtype=torch.float32)
    v_l = fn(None, gt, w_l, t, consts)["line_of_sight_my"]
    v_l.backward()
    assert em.CALLS == ["emer_ray_loss_live_fwd", "emer_ray_loss_live_bwd"]
    assert torch.equal(v_f, v_l) and torch.equal(w_f.grad, w_l.grad)


def test_line_of_sight_consts_round_as_the_float_call():
    from emernerf_b200 import _ops, loss

    for eps, decay in ((6.0, 1.0), (3.3, 0.5 ** 5), (2.5, 0.1)):
        want = [ctypes.c_float(v).value for v in (*_ops._sight_consts(eps), decay)]
        assert loss.line_of_sight_consts(eps, decay) == want


def test_live_form_refuses_a_second_decay_weight(em):
    from emernerf_b200 import loss

    w, t, gt = _rays()
    consts = torch.tensor(loss.line_of_sight_consts(4.0, 1.0))
    with pytest.raises(ValueError, match="coef_decay"):
        loss.LineOfSightLoss()(None, gt, w, t, consts, coef_decay=0.5)
    with pytest.raises(ValueError, match="4 values"):
        loss.LineOfSightLoss()(None, gt, w, t, consts[:3])

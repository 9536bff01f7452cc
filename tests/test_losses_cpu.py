"""emernerf_b200.loss through the C-ABI emulator on CPU: every class and option against the reference's own values
and gradients (tests/golden/losses.npz), the reference's signatures, defaults and returned keys, the options that
raise, and check_nan."""
import inspect
import json
import os

import numpy as np
import pytest
import torch

import cabi_emulator
import loss_cases as lc
import loss_emulator
from helpers import GOLDEN_DIR

Z = np.load(os.path.join(GOLDEN_DIR, "losses.npz"))
INPUTS = lc.make_inputs()
KEYS = json.loads(str(Z["meta/keys"]))
SIGNATURES = json.loads(str(Z["meta/signatures"]))


@pytest.fixture
def em(monkeypatch):
    loss_emulator.install(monkeypatch)
    return cabi_emulator


def test_regenerated_inputs_are_the_fixtures():
    got = lc.digest(INPUTS)
    assert set(got) == {k.split("/", 1)[1] for k in Z.files if k.startswith("in_digest/")}
    for k, v in got.items():
        assert np.allclose(v.numpy(), Z[f"in_digest/{k}"], rtol=1e-12, atol=0), k


def check_case(loss_mod, case, device="cpu", value_tol=1e-5, grad_tol=1e-6):
    name = case[0]
    key, value, grads = lc.run_case(loss_mod, INPUTS, case, device)
    assert key == KEYS[name]
    want = float(Z[f"{name}/value"])
    got = value.item()
    if np.isnan(want):
        assert np.isnan(got), (name, got)
    else:
        assert abs(got - want) <= value_tol * max(abs(want), 1e-30), (name, got, want)
    wanted = {k.split("/")[-1]: torch.from_numpy(Z[k]) for k in Z.files if k.startswith(f"{name}/grad/")}
    assert set(grads) == set(wanted), (name, set(grads) ^ set(wanted))
    for a, w in wanted.items():
        g = grads[a].detach().cpu().double()
        scale = w.abs().max().item()
        err = (g - w.double()).abs().max().item()
        assert err <= grad_tol * max(scale, 1e-30), (name, a, err, scale)
        # the masks decide the same samples: a gradient is zero exactly where the reference's is
        assert torch.equal(g == 0, w == 0), (name, a)


@pytest.mark.parametrize("case", lc.CASES, ids=[c[0] for c in lc.CASES])
def test_loss_matches_reference_golden(em, case):
    from emernerf_b200 import loss

    del em.CALLS[:]
    check_case(loss, case)
    assert em.CALLS and all("loss" in c for c in em.CALLS), em.CALLS


def test_one_launch_each_way(em):
    from emernerf_b200 import loss

    x = {k: v.clone().requires_grad_(k in lc.GRAD_INPUTS) for k, v in INPUTS.items()}
    del em.CALLS[:]
    v = loss.LineOfSightLoss(coef=0.1)(x["depth"], x["lidar_ranges"], x["weights"], x["t_vals"], epsilon=2.5)
    assert em.CALLS == ["emer_ray_loss_fwd"]
    v["line_of_sight_my"].backward()
    assert em.CALLS == ["emer_ray_loss_fwd", "emer_ray_loss_bwd"]
    del em.CALLS[:]
    v = loss.DynamicRegularizationLoss(loss_type="entropy")(x["dynamic_density"], x["static_density"])
    v["dynamic_entropy_loss"].backward()
    assert em.CALLS == ["emer_pointwise_loss_fwd", "emer_pointwise_loss_bwd"]


@pytest.mark.parametrize("eps", [6.0, 2.5])
def test_compute_line_of_sight_loss_matches_reference(em, eps):
    from emernerf_b200 import loss

    w = INPUTS["weights"].clone().requires_grad_()
    v = loss.compute_line_of_sight_loss(INPUTS["lidar_ranges"], w, INPUTS["t_vals"], eps)
    want = torch.from_numpy(Z[f"fn/los_{eps}/value"])
    assert v.shape == want.shape
    assert torch.allclose(v.detach(), want, rtol=1e-5, atol=0)
    (g,) = torch.autograd.grad(v.sum(), w)
    gw = torch.from_numpy(Z[f"fn/los_{eps}/grad/weights"])
    assert (g - gw).abs().max() <= 1e-6 * gw.abs().max()


def _sig(obj):
    return [[p.name, None if p.default is inspect.Parameter.empty else p.default]
            for p in inspect.signature(obj).parameters.values() if p.name != "self"]


def test_signatures_defaults_and_names_match_reference():
    from emernerf_b200 import loss

    for name in lc.CLASSES:
        cls = getattr(loss, name)
        for fn in ("__init__", "__call__"):
            assert _sig(getattr(cls, fn)) == SIGNATURES[name][fn], (name, fn)
    for name in lc.FUNCTIONS:
        assert _sig(getattr(loss, name)) == SIGNATURES[name], name
    assert loss.RealValueLoss().name == "rgb_loss_l2"
    assert loss.SkyLoss(loss_type="opacity_based").name == "sky_loss_opacity_based"
    assert loss.DepthLoss().name == "depth_loss_l2"
    assert loss.LineOfSightLoss().name == "line_of_sight_my"
    assert loss.DynamicRegularizationLoss(name="shadow").name == "shadow_sparsity_loss"
    l = loss.DepthLoss(coef=2.0)
    l.set_coef(0.25)
    assert l.coef == 0.25


def test_unsupported_options_raise():
    from emernerf_b200 import loss

    with pytest.raises(NotImplementedError, match="reduction"):
        loss.RealValueLoss(reduction="none")
    with pytest.raises(NotImplementedError, match="depth_error_percentile"):
        loss.DepthLoss(depth_error_percentile=0.9)
    with pytest.raises(NotImplementedError, match="depth_error_percentile"):
        loss.LineOfSightLoss(depth_error_percentile=0.9)
    with pytest.raises(NotImplementedError, match="mask"):
        loss.RealValueLoss()(INPUTS["rgb"], INPUTS["pixels"], mask=torch.ones(lc.R))
    with pytest.raises(NotImplementedError, match="mask"):
        loss.DynamicRegularizationLoss()(INPUTS["dynamic_density"], mask=torch.ones(lc.R))
    with pytest.raises(NotImplementedError, match="Unknown loss type"):
        loss.RealValueLoss(loss_type="huber")
    with pytest.raises(AssertionError):
        loss.SkyLoss(reduction="sum")


def test_check_nan(em):
    from emernerf_b200 import loss

    fn = loss.DepthLoss(check_nan=True)
    with pytest.raises(ValueError, match="lidar_range_loss is NaN"):
        fn(INPUTS["depth"], INPUTS["no_ranges"], name="lidar_range_loss")
    assert torch.isfinite(fn(INPUTS["depth"], INPUTS["lidar_ranges"])["depth_loss_l2"])
    # off by default: the NaN is returned
    assert torch.isnan(loss.DepthLoss()(INPUTS["depth"], INPUTS["no_ranges"])["depth_loss_l2"])

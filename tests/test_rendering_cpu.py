"""``render_rays`` with ``EMER_RENDERING=fused`` on CPU: the body of ``rendering`` goes through emer_render_fwd /
emer_render_bwd (answered by tests/render_emulator.py) and must reproduce the reference's golden outputs and parameter
gradients for every variant at the tolerances of tests/test_host_path_cpu.py, with one emer_render_fwd per pass and no
emer_accumulate_* in it; the switch-off outputs agree with the switch-on ones."""
import pytest
import torch

import cabi_emulator
import cases
import render_emulator
from helpers import assert_close_dict, rel_err
from oracle import adapters
from test_host_path_cpu import TOL, _build, _render


@pytest.fixture
def fused(monkeypatch):
    from emernerf_b200.radiance_fields import render_utils

    render_emulator.install(monkeypatch)
    monkeypatch.setattr(render_utils, "RENDERING", "fused")
    return cabi_emulator


def _tol():
    tol = {"*": TOL, "median_depth": 5e-2}
    for k in ("density", "static_density", "dynamic_density", "forward_flow", "backward_flow",
              "forward_pred_backward_flow", "backward_pred_forward_flow", "weights", "trans"):
        tol[k] = 1e-3
    return tol


@pytest.mark.parametrize("case", list(cases.CASES))
@pytest.mark.parametrize("mode", ["eval", "lidar", "train"])
def test_fused_rendering_matches_reference_outputs(fused, case, mode):
    g, field, props, est = _build(case)
    out = _render(g, field, props, est, mode)
    assert_close_dict(out, g.nested(f"{mode}/out"), _tol())
    calls = fused.CALLS
    if mode == "lidar":
        # densities only: nothing to blend or accumulate, the op-by-op path composites
        assert "emer_render_fwd" not in calls and "emer_composite_fwd" in calls
    else:
        assert calls.count("emer_render_fwd") == 1
        assert not any(c.startswith("emer_accumulate_") for c in calls)
        assert "emer_composite_fwd" not in calls


@pytest.mark.parametrize("case", list(cases.CASES))
def test_fused_rendering_parameter_gradients(fused, case):
    g, field, props, est = _build(case)
    out = _render(g, field, props, est, "train")
    loss = adapters.parity_loss(out)
    assert abs(loss.item() - g.scalar("train/loss")) < 1e-4
    del fused.CALLS[:]
    loss.backward()
    assert fused.CALLS.count("emer_render_bwd") == 1
    assert not any(c.startswith(("emer_accumulate_", "emer_composite_")) for c in fused.CALLS)
    want = g.tensors("train/grad/field")
    checked = 0
    for k, v in field.named_parameters():
        if k in want:
            assert v.grad is not None, k
            assert rel_err(v.grad, want[k]) < 5e-3, k
            checked += 1
    assert checked == len(want)


@pytest.mark.parametrize("case", list(cases.CASES))
@pytest.mark.parametrize("mode", ["eval", "train"])
def test_switch_on_and_off_agree(monkeypatch, case, mode):
    from emernerf_b200.radiance_fields import render_utils

    render_emulator.install(monkeypatch)
    outs = {}
    for how in ("torch", "fused"):
        monkeypatch.setattr(render_utils, "RENDERING", how)
        g, field, props, est = _build(case)
        outs[how] = _render(g, field, props, est, mode)
    assert_close_dict(outs["fused"], outs["torch"], 1e-5)


def test_decomposition_under_grad_takes_the_torch_path(fused):
    """The decomposition outputs have no backward in the kernel: asked for under grad, ``rendering`` falls back."""
    from emernerf_b200.radiance_fields.render_utils import render_rays

    g, field, props, est = _build("dynamic")
    batch = g.tensors("in/pixel")
    field.eval()
    out = render_rays(field, est, props, batch, cases.render_cfg(), return_decomposition=True)
    assert "static_rgb" in out and out["rgb"].requires_grad
    assert "emer_render_fwd" not in fused.CALLS and "emer_accumulate_fwd" in fused.CALLS


def test_render_checks_its_inputs(fused):
    from emernerf_b200 import _ops

    r, s = 3, 5
    t0 = torch.rand(r, s)
    t1 = t0 + 0.1
    sig = torch.rand(r, s)
    with pytest.raises(ValueError, match="come together"):
        _ops.render(t0, t1, {"sigma": sig, "sigma_s": sig})
    with pytest.raises(ValueError, match="must be"):
        _ops.render(t0, t1, {"sigma": sig, "rgb": torch.rand(r, s, 4)})
    with pytest.raises(ValueError, match="feature channels"):
        _ops.render(t0, t1, {"sigma": sig, "dino": torch.rand(r, s, 257)})
    with pytest.raises(ValueError, match="no gradient"):
        _ops.render(t0, t1, {"sigma": sig.requires_grad_(), "sigma_s": sig, "sigma_d": sig,
                             "rgb": torch.rand(r, s, 3)}, decomposition=True)

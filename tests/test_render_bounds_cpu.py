"""The per-element bounds of the render checks in test_gpu_composite_fp64 have teeth, on the CPU: on the same ray
families, the float64 reference rounded to fp32 passes every check, and each plausible slip in csrc/render.cu, computed
in float64 and rounded the same way, fails the check of the buffer it touches."""
import pytest
import torch

from oracle import nerfacc_ref as nf
from test_gpu_composite_fp64 import (COMBOS, _check, _hot, backward_checks, decomposition_checks, fwd_bounds,
                                     render_inputs)

R, C = 37, 33


def _fails(check, got, want, bound, mask=None):
    try:
        _check(check, got, want, bound, mask)
    except AssertionError:
        return True
    return False


def _backward(combo, S=33):
    t0, t1, ins, _ = render_inputs(combo, R, S, C, seed=4)
    want, _ = _hot(t0, t1, ins, None, False)
    W = want["extras"]["weights"][:, :S].float()
    names = {"dino": "dino_feat"}
    g = torch.Generator().manual_seed(9)
    ups = {"weights": W, "trans": W, "opacity": want["opacity"], "depth": want["depth"]}
    ups.update({k: want[names.get(k, k)] for k in ("rgb", "shadow_ratio", "dino", "dino_pe_free")
                if names.get(k, k) in want})
    ups = {k: torch.randn(v.shape, generator=g) for k, v in ups.items()}
    checks, leaves, ref = backward_checks(t0, t1, ins, ups, W)
    return ins, ups, checks, leaves, ref


@pytest.mark.parametrize("S", [1, 33])
@pytest.mark.parametrize("combo", list(COMBOS))
def test_rounded_reference_passes_backward(combo, S):
    _, _, checks, leaves, _ = _backward(combo, S)
    for k, (want, bound, mask) in checks.items():
        _check(f"cpu {combo} d_{k}", leaves[k].grad.float(), want, bound, mask)


def _slips(combo):
    """{(input, slip): float64 gradient with the slip} for the slips the combo's inputs allow."""
    ins, ups, checks, leaves, ref = _backward(combo)
    d = {k: v.double() for k, v in ins.items()}
    w = ref["weights"]
    grad = {k: v.grad.detach() for k, v in leaves.items()}
    gw = ups["rgb"].double()
    out = {}
    if "rgb_sky" in d:
        out[("rgb_sky", "the unclamped sum of the weights")] = gw * (1 - w.sum(-1, keepdim=True))
    if "sigma_s" in d:
        drs = grad["sigma_s"] * (d["sigma"] + 1e-6)
        out[("sigma_s", "den = sigma")] = drs / d["sigma"]
        rs = d["sigma_s"] / (d["sigma"] + 1e-6)
        out[("rgb_s", "no 1 - shadow")] = (w * rs)[..., None] * gw[:, None, :]
    if "shadow" in d:
        out[("shadow", "no 2 w g_shr sh")] = grad["shadow"] - 2 * w * ups["shadow_ratio"].double() * d["shadow"]
    if "dino_pe" in d:
        out[("dino_pe", "g_F")] = (ups["dino"] + ups["dino_pe_free"]).double()
    return out, checks


@pytest.mark.parametrize("combo", ["static_feat_sky_pe", "dynamic_shadow", "flow_feat"])
def test_backward_slips_are_rejected(combo):
    slips, checks = _slips(combo)
    assert len(slips) == {"static_feat_sky_pe": 2, "dynamic_shadow": 4, "flow_feat": 5}[combo]
    for (k, what), bad in slips.items():
        want, bound, mask = checks[k]
        finite = torch.isfinite(bad) if mask is None else torch.isfinite(bad) & mask
        assert _fails(f"cpu slip {k}", bad.float(), want, bound, finite), (combo, k, what)


def _forward(combo, S=33):
    t0, t1, ins, flows = render_inputs(combo, R, S, C, seed=6)
    want, _ = _hot(t0, t1, ins, flows, True)
    ref = nf.composite64(t0, t1, ins["sigma"], want["extras"]["weights"].float())
    return t0, t1, ins, flows, want, ref, fwd_bounds(ref)


@pytest.mark.parametrize("combo", ["flow", "flow_feat"])
def test_decomposition_bounds(combo):
    t0, t1, ins, flows, want, ref, fb = _forward(combo)
    checks = {k: (v, b) for k, v, b in decomposition_checks(t0, t1, ins, flows, want, ref, fb)}
    for k, (v, b) in checks.items():
        _check(f"cpu {combo} {k}", want[k].float(), v, b)
    # shadow_only_static_rgb's 1 - acc_sh taken over the static weights
    sw = nf.composite64(t0, t1, ins["sigma_s"])["weights"]
    sh = ins["shadow"].double()[..., None]
    bad = want["shadow_only_static_rgb"] + want["shadow"] - (sw[..., None] * sh).sum(1)
    assert _fails("cpu slip shadow_only_static_rgb", bad.float(), *checks["shadow_only_static_rgb"])
    if "dino_sky" in ins:
        # static_dino's sky term over the static opacity
        sky = ins["dino_sky"].double()
        bad = want["static_dino"] - sky * (1 - want["opacity"]) + sky * (1 - want["static_opacity"])
        assert _fails("cpu slip static_dino", bad.float(), *checks["static_dino"])

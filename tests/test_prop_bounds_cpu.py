"""The per-element bounds of test_gpu_prop_level_fp64 have teeth, on the CPU: on the same ray families and loss rows,
the float64 reference rounded to fp32 passes every check, and each plausible slip in csrc/prop_level.cu and
csrc/interlevel_loss.cu, computed in float64 and rounded the same way, fails the check of the buffer it touches."""
import math

import pytest
import torch

from oracle import nerfacc_ref as nf
from test_gpu_composite_fp64 import _check, fwd_bounds
from test_gpu_prop_level_fp64 import (E15, backward_inputs, check_cdf, interlevel64, interlevel_rows, level_bwd64,
                                      make_d_cdf)

R = 37


def _fails(fn, *args):
    try:
        fn(*args)
    except AssertionError:
        return True
    return False


def _forward(n):
    t, sigma = backward_inputs(R, n, seed=3 * n)
    ref = nf.composite64(t[:, :-1], t[:, 1:], sigma)
    return t, sigma, ref, fwd_bounds(ref)


@pytest.mark.parametrize("n", [1, 33, 64])
def test_rounded_reference_passes_forward(n):
    _, _, ref, fb = _forward(n)
    check_cdf("cpu", ref["cdf"].float(), ref, fb)


def test_forward_slips_are_rejected():
    n = 64
    _, _, ref, fb = _forward(n)
    x, E = ref["x"], ref["E"]
    # the old prefix carry + (incl - x): the inclusive sum rounded to fp32, then the own term taken off again
    incl = (E + x).float().double()
    bad = 1.0 - torch.exp(-(incl - x))
    bad = torch.cat([bad, torch.ones_like(bad[:, :1])], -1).float()
    assert _fails(check_cdf, "cpu slip prefix", bad, ref, fb)
    # no running minimum: one ulp down after a sample that adds nothing (the inversion of two scan trees)
    c = ref["cdf"].float()
    cand = torch.nonzero((x[:, :-1] == 0) & (c[:, :n - 1] > 0) & (c[:, :n - 1] < 0.5))
    assert len(cand), "no flat sample after a non-zero prefix"
    r, i = cand[0].tolist()
    c[r, i + 1] = torch.nextafter(c[r, i], torch.tensor(-math.inf))
    assert _fails(check_cdf, "cpu slip no minimum", c, ref, fb)
    # ... and the dip alone is within the per-sample bound: only the monotonicity check rejects it
    nan = torch.isnan(ref["cdf"][:, :n])
    _check("cpu dip per sample", c[:, :n], ref["cdf"][:, :n], fb["bT"] + 2 ** -24 * ref["cdf"][:, :n].abs(), ~nan)


def _backward(n=64):
    t, sigma = backward_inputs(R, n, seed=5 * n)
    d_cdf, kind = make_d_cdf(R, n, seed=n)
    return t, sigma, d_cdf, level_bwd64(t, sigma, d_cdf)


def _check_draw(tag, got, ref):
    ok = torch.isfinite(ref["d_raw"]) & torch.isfinite(ref["bound"])
    _check(tag, got, ref["d_raw"], ref["bound"], ok & torch.isfinite(got))
    assert torch.isfinite(got[ok]).all(), (tag, "non-finite")


@pytest.mark.parametrize("n", [1, 33, 64, 256])
def test_rounded_reference_passes_backward(n):
    _, _, _, ref = _backward(n)
    _check_draw("cpu d_raw", ref["d_raw"].float(), ref)


def test_backward_slips_are_rejected():
    t, sigma, d_cdf, ref = _backward()
    n = sigma.shape[-1]
    c64 = nf.composite64(t[:, :-1], t[:, 1:], sigma)
    T, delta = c64["trans"], c64["delta"]
    dc = d_cdf[:, :n].double()
    m = sigma.double().clamp(max=E15)
    S = ref["S"]
    slips = {
        "inclusive suffix": (S + dc * T) * delta * m,
        "min(sigma, e^15) dropped": S * delta * sigma.double(),
        "d_cdf[:, n] folded in": (S + (d_cdf[:, n:].double() * torch.exp(-(c64["E"][:, -1:] + c64["x"][:, -1:]))))
        * delta * m,
    }
    for what, bad in slips.items():
        assert _fails(_check_draw, f"cpu slip {what}", bad.float(), ref), what


@pytest.mark.parametrize("r", [0.03, 0.003, 2.0 ** -5])
def test_rounded_reference_passes_interlevel(r):
    s, cdf, ps, pc, _ = interlevel_rows(R, 65, 65, seed=1)
    ref = interlevel64(s, cdf, ps, pc, r)
    _check("cpu d_prop_cdf", ref["d"].float(), ref["d"], ref["bound_d"])


@pytest.mark.parametrize("r", [0.03, 0.003])
def test_interlevel_slip_is_rejected(r):
    """The gradient without its d^2 / den^2 term."""
    s, cdf, ps, pc, _ = interlevel_rows(R, 65, 65, seed=2)
    ref = interlevel64(s, cdf, ps, pc, r)
    g = -2 * ref["hinge"] / ref["den"]
    zero = torch.zeros_like(g[:, :1])
    bad = torch.cat([zero, g], -1) - torch.cat([g, zero], -1)
    assert _fails(_check, "cpu slip interlevel", bad.float(), ref["d"], ref["bound_d"])

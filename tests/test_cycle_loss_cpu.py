"""emernerf_b200.loss.flow_cycle_loss through the C-ABI emulator on CPU: value, flow statistics and gradients against
the reference's inline torch block (train_emernerf.py:700-740) in fp32 and fp64, on flows that are column slices of
[N, 6] and of padded-width rows (read in place, without a copy), a NaN row, the empty batch, and the parameter
gradients of the flow fixtures' parity loss with the cycle term computed by the library."""
import numpy as np
import pytest
import torch

import cabi_emulator
import cycle_loss_emulator
from helpers import rel_err
from oracle import adapters

FLOW_KEYS = ("forward_flow", "backward_flow", "forward_pred_backward_flow", "backward_pred_forward_flow")
STAT_KEYS = ("max_forward_flow_norm", "max_backward_flow_norm", "max_forward_pred_backward_flow_norm",
             "max_backward_pred_forward_flow_norm")
# (R, S): R * S = 1073 and 2039 are multiples of neither 32 nor the 256-thread CTA
SHAPES = [(37, 29), (1, 1), (2039, 1)]
# flow MLP output rows: [N, 6] as the flow head writes them, or padded to a wider row
WIDTHS = [6, 16]


@pytest.fixture
def em(monkeypatch):
    cycle_loss_emulator.install(monkeypatch)
    return cabi_emulator


def reference(ex, coef=0.01):
    """The reference's block, verbatim but for the names and the coefficient."""
    cycle = 0.5 * ((ex["forward_flow"].detach() + ex["forward_pred_backward_flow"]) ** 2
                   + (ex["backward_flow"].detach() + ex["backward_pred_forward_flow"]) ** 2).mean()
    stats = {"max_forward_flow_norm": ex["forward_flow"].detach().norm(dim=-1).max(),
             "max_backward_flow_norm": ex["backward_flow"].detach().norm(dim=-1).max(),
             "max_forward_pred_backward_flow_norm": ex["forward_pred_backward_flow"].norm(dim=-1).max(),
             "max_backward_pred_forward_flow_norm": ex["backward_pred_forward_flow"].norm(dim=-1).max()}
    return cycle * coef, stats


def make_flows(r, s, width, seed=0, device="cpu", dtype=torch.float32):
    """(leaf buffers, extras): the flows and the two predictions as 3-wide column slices of [R, S, width] rows, the
    predictions near the negated flows, as a trained flow field makes them."""
    g = torch.Generator().manual_seed(seed)
    flow = torch.randn(r, s, width, generator=g) * 2.0
    fwd_q = torch.randn(r, s, width, generator=g) * 0.3
    bwd_q = torch.randn(r, s, width, generator=g) * 0.3
    fwd_q[..., 3:6] -= flow[..., 3:6]
    bwd_q[..., 0:3] -= flow[..., 0:3]
    bufs = {k: v.to(device=device, dtype=dtype) for k, v in (("flow", flow), ("fwd_q", fwd_q), ("bwd_q", bwd_q))}
    bufs["fwd_q"].requires_grad_()
    bufs["bwd_q"].requires_grad_()
    return bufs, extras_of(bufs)


def extras_of(bufs):
    return {"forward_flow": bufs["flow"][..., 0:3], "backward_flow": bufs["flow"][..., 3:6],
            "forward_pred_backward_flow": bufs["fwd_q"][..., 3:6],
            "backward_pred_forward_flow": bufs["bwd_q"][..., 0:3]}


def check_against_reference(loss, bufs, ex, coef=0.01):
    """Value within 1e-5 relative and gradients within 1e-6 of their max-abs of the reference in fp32 and in fp64;
    statistics within 1e-6 relative; NaN where the reference's are."""
    got, stats = loss.flow_cycle_loss(ex, coef=coef)
    assert set(got) == {"cycle_loss"} and set(stats) == set(STAT_KEYS)
    value = got["cycle_loss"]
    assert value.dim() == 0 and value.requires_grad
    assert all(v.dim() == 0 and not v.requires_grad and v.device == value.device for v in stats.values())
    grads = torch.autograd.grad(value, [bufs["fwd_q"], bufs["bwd_q"]])
    for dtype in (torch.float32, torch.float64):
        ref_bufs = {k: v.detach().cpu().to(dtype).requires_grad_(v.requires_grad) for k, v in bufs.items()}
        want, want_stats = reference(extras_of(ref_bufs), coef)
        want_grads = torch.autograd.grad(want, [ref_bufs["fwd_q"], ref_bufs["bwd_q"]])
        w, v = want.item(), value.item()
        if np.isnan(w):
            assert np.isnan(v)
        else:
            assert abs(v - w) <= 1e-5 * abs(w), (dtype, v, w)
        for k in STAT_KEYS:
            w, v = want_stats[k].item(), stats[k].item()
            assert (np.isnan(v) and np.isnan(w)) or abs(v - w) <= 1e-6 * abs(w), (dtype, k, v, w)
        for gr, wg in zip(grads, want_grads):
            gr = gr.detach().cpu().double()
            assert torch.equal(torch.isnan(gr), torch.isnan(wg)), dtype
            fin = ~torch.isnan(wg)
            err = (gr[fin] - wg[fin].double()).abs().max().item() if fin.any() else 0.0
            scale = wg[fin].abs().max().item() if fin.any() else 0.0
            assert err <= 1e-6 * max(scale, 1e-30), (dtype, err, scale)
            # only the predicted columns of each buffer receive a gradient; the others stay exactly zero
            assert torch.equal(gr == 0, wg == 0), dtype
    return value, stats, grads


def _spy(monkeypatch):
    seen = []
    fwd = cycle_loss_emulator.emer_cycle_loss_fwd

    def spy(*args):
        seen.append(args)
        return fwd(*args)

    monkeypatch.setattr(cycle_loss_emulator, "emer_cycle_loss_fwd", spy)
    return seen


@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{r}x{s}" for r, s in SHAPES])
def test_cycle_loss_matches_reference_on_strided_slices(em, monkeypatch, shape, width):
    from emernerf_b200 import loss

    seen = _spy(monkeypatch)
    bufs, ex = make_flows(*shape, width)
    del em.CALLS[:]
    check_against_reference(loss, bufs, ex)
    assert em.CALLS == ["emer_cycle_loss_fwd", "emer_cycle_loss_bwd"]
    # the four views are read where they are: their own addresses, with the buffer's row stride
    (args,) = seen
    n = shape[0] * shape[1]
    want = [(ex[k].data_ptr(), width if n > 1 else 3) for k in FLOW_KEYS]
    assert [(a.value, ld) for a, ld in zip(args[0:8:2], args[1:8:2])] == want
    assert args[8] == n


@pytest.mark.parametrize("coef", [0.01, 1.0, 0.37])
def test_coefficient_and_name(em, coef):
    from emernerf_b200 import loss

    bufs, ex = make_flows(23, 11, 6, seed=1)
    check_against_reference(loss, bufs, ex, coef=coef)
    got, _ = loss.flow_cycle_loss(ex, coef=coef, name="flow_cycle")
    assert set(got) == {"flow_cycle"}


def test_other_layouts_are_copied(em):
    """Contiguous flows, a transposed buffer (unit stride on the wrong axis) and fp64 flows all give the same values
    as their fp32 strided originals."""
    from emernerf_b200 import loss

    bufs, ex = make_flows(19, 13, 6, seed=2)
    base, base_stats = loss.flow_cycle_loss(ex)
    contiguous = {k: v.contiguous() for k, v in ex.items()}
    transposed = {k: v.transpose(0, 2).contiguous().transpose(0, 2) for k, v in ex.items()}
    for other in (contiguous, transposed):
        got, stats = loss.flow_cycle_loss(other)
        assert torch.equal(got["cycle_loss"], base["cycle_loss"])
        for k in STAT_KEYS:
            assert torch.equal(stats[k], base_stats[k])
    b64 = {k: v.detach().double().requires_grad_(v.requires_grad) for k, v in bufs.items()}
    got, _ = loss.flow_cycle_loss(extras_of(b64))
    assert torch.equal(got["cycle_loss"], base["cycle_loss"])
    (g,) = torch.autograd.grad(got["cycle_loss"], [b64["fwd_q"]])
    assert g.dtype == torch.float64


@pytest.mark.parametrize("where", ["forward_flow", "forward_pred_backward_flow", "backward_pred_forward_flow"])
def test_nan_row_propagates(em, where):
    from emernerf_b200 import loss

    bufs, _ = make_flows(31, 9, 16, seed=3)
    with torch.no_grad():
        buf, col = {"forward_flow": ("flow", 1), "forward_pred_backward_flow": ("fwd_q", 4),
                    "backward_pred_forward_flow": ("bwd_q", 2)}[where]
        bufs[buf][17, 4, col] = float("nan")
    ex = extras_of(bufs)
    value, stats, _ = check_against_reference(loss, bufs, ex)
    assert torch.isnan(value)
    for k in STAT_KEYS:
        assert torch.isnan(stats[k]) == (k == "max_" + where + "_norm"), k


def test_empty_and_mismatched_inputs_raise(em):
    from emernerf_b200 import loss

    _, ex = make_flows(0, 16, 6)
    with pytest.raises(ValueError, match="no samples"):
        loss.flow_cycle_loss(ex)
    with pytest.raises(RuntimeError):                                   # what the reference raises
        reference(ex)
    _, ex = make_flows(4, 5, 6)
    with pytest.raises(ValueError, match="same"):
        loss.flow_cycle_loss({**ex, "backward_flow": ex["backward_flow"][:, :4]})


def test_emulator_refuses_what_the_library_refuses(em):
    from emernerf_b200 import _lib

    buf = torch.zeros(8, 6)
    p = buf.data_ptr()
    out = torch.zeros(6)
    with pytest.raises(RuntimeError, match="no rows"):
        _lib.call("emer_cycle_loss_fwd", p, 6, p, 6, p, 6, p, 6, 0, 1.0, out.data_ptr(), p, None)
    with pytest.raises(RuntimeError, match="row stride"):
        _lib.call("emer_cycle_loss_fwd", p, 6, p, 2, p, 6, p, 6, 8, 1.0, out.data_ptr(), p, None)
    with pytest.raises(RuntimeError, match="no gradient"):
        _lib.call("emer_cycle_loss_bwd", p, 6, p, 6, p, 6, p, 6, 8, 1.0, p, p, None, None, None)


# ---------------------------------------------------------------------------------------------- end to end
def parity_loss_with_library_cycle(out, loss):
    """``oracle.adapters.parity_loss`` with its cycle term (coefficient 1) computed by ``flow_cycle_loss``."""
    ex = out["extras"]
    rest = adapters.parity_loss({**out, "extras": {k: v for k, v in ex.items() if k not in FLOW_KEYS}})
    cycle, stats = loss.flow_cycle_loss(ex, coef=1.0)
    return rest + cycle["cycle_loss"], stats


@pytest.mark.parametrize("case", ["flow", "flow_feat"])
def test_flow_fixture_parameter_gradients(em, case):
    """The parameter gradients of the fixture's training pass match the reference's (train/grad/*) at the tolerances
    of tests/test_host_path_cpu.py, with the cycle term on the library."""
    from emernerf_b200 import loss
    from test_host_path_cpu import _build, _render

    g, field, props, est = _build(case)
    out = _render(g, field, props, est, "train")
    del em.CALLS[:]
    total, stats = parity_loss_with_library_cycle(out, loss)
    assert abs(total.item() - g.scalar("train/loss")) < 1e-4
    _, want_stats = reference(out["extras"])
    for k in STAT_KEYS:
        assert abs(stats[k].item() - want_stats[k].item()) <= 1e-6 * want_stats[k].item(), k
    total.backward()
    assert em.CALLS.count("emer_cycle_loss_fwd") == 1 and em.CALLS.count("emer_cycle_loss_bwd") == 1
    want = g.tensors("train/grad/field")
    checked = 0
    for k, v in field.named_parameters():
        if k in want:
            assert v.grad is not None, k
            assert rel_err(v.grad, want[k]) < 5e-3, k
            checked += 1
    assert checked == len(want)
    assert any(k.startswith("flow") for k in want)

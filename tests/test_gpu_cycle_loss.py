"""emernerf_b200.loss.flow_cycle_loss on the GPU: value, flow statistics and gradients against the reference's torch
block in fp32 and fp64 at training size (8192 x 64 samples) and ragged sizes, on strided column slices; a NaN row;
bit-identical repeats; exact scaling under a GradScaler factor; no host sync; capture and replay in a CUDA graph; one
library kernel and no copy in the forward; and the parameter gradients of the flow fixtures, miniature and full-size,
with the cycle term computed by the library."""
import pytest
import torch

from test_cycle_loss_cpu import (STAT_KEYS, check_against_reference, extras_of, make_flows,
                                 parity_loss_with_library_cycle, reference)

pytestmark = pytest.mark.gpu
DEV = "cuda"
SHAPES = [(8192, 64), (8191, 63), (37, 29), (1, 1)]


def _run(loss, bufs, coef=0.01, scale=None):
    for k in ("fwd_q", "bwd_q"):
        bufs[k].grad = None
    got, stats = loss.flow_cycle_loss(extras_of(bufs), coef=coef)
    value = got["cycle_loss"]
    (value if scale is None else value * scale).backward()
    return value, stats, bufs["fwd_q"].grad, bufs["bwd_q"].grad


@pytest.mark.parametrize("width", [6, 16])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{r}x{s}" for r, s in SHAPES])
def test_cycle_loss_on_cuda_matches_reference(shape, width):
    from emernerf_b200 import loss

    bufs, ex = make_flows(*shape, width, seed=4, device=DEV)
    check_against_reference(loss, bufs, ex)


@pytest.mark.parametrize("where", ["forward_flow", "backward_flow", "forward_pred_backward_flow",
                                   "backward_pred_forward_flow"])
def test_nan_row_on_cuda(where):
    from emernerf_b200 import loss

    bufs, _ = make_flows(4099, 7, 16, seed=5, device=DEV)
    buf, col = {"forward_flow": ("flow", 1), "backward_flow": ("flow", 5), "forward_pred_backward_flow": ("fwd_q", 4),
                "backward_pred_forward_flow": ("bwd_q", 2)}[where]
    with torch.no_grad():
        bufs[buf][4000, 3, col] = float("nan")
    value, stats, _ = check_against_reference(loss, bufs, extras_of(bufs))
    assert torch.isnan(value)
    for k in STAT_KEYS:
        assert bool(torch.isnan(stats[k])) == (k == "max_" + where + "_norm"), k


def test_bit_identical_repeats():
    from emernerf_b200 import loss

    bufs, _ = make_flows(8192, 64, 6, seed=6, device=DEV)
    first = [t.clone() for t in _run(loss, bufs)[2:]]
    a = _run(loss, bufs)
    b = _run(loss, bufs)
    assert torch.equal(a[0], b[0])
    for k in STAT_KEYS:
        assert torch.equal(a[1][k], b[1][k])
    for x, y, z in zip(first, a[2:], b[2:]):
        assert torch.equal(x, y) and torch.equal(y, z)


def test_scaled_upstream_scales_gradients_exactly():
    from emernerf_b200 import loss

    bufs, _ = make_flows(8191, 64, 16, seed=7, device=DEV)
    _, _, g_f, g_b = _run(loss, bufs)
    g_f, g_b = g_f.clone(), g_b.clone()
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
    for k in ("fwd_q", "bwd_q"):
        bufs[k].grad = None
    got, _ = loss.flow_cycle_loss(extras_of(bufs))
    scaler.scale(got["cycle_loss"]).backward()
    assert torch.equal(bufs["fwd_q"].grad, g_f * 2.0 ** 10)
    assert torch.equal(bufs["bwd_q"].grad, g_b * 2.0 ** 10)


def test_no_host_sync():
    from emernerf_b200 import loss

    bufs, _ = make_flows(8192, 64, 6, seed=8, device=DEV)
    _run(loss, bufs)                        # the device's loss workspace exists
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _run(loss, bufs)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_cuda_graph_capture_and_replay():
    from emernerf_b200 import loss

    static, _ = make_flows(2048, 48, 16, seed=9, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _run(loss, static)
    torch.cuda.current_stream().wait_stream(side)
    for k in ("fwd_q", "bwd_q"):
        static[k].grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got, stats = loss.flow_cycle_loss(extras_of(static))
        got["cycle_loss"].backward()
    for seed in (10, 11):
        fresh, _ = make_flows(2048, 48, 16, seed=seed, device=DEV)
        with torch.no_grad():
            for k in static:
                static[k].copy_(fresh[k])
        graph.replay()
        want = _run(loss, fresh)
        torch.cuda.synchronize()
        assert torch.equal(got["cycle_loss"], want[0])
        for k in STAT_KEYS:
            assert torch.equal(stats[k], want[1][k]), k
        assert torch.equal(static["fwd_q"].grad, want[2]) and torch.equal(static["bwd_q"].grad, want[3])


def test_forward_is_one_library_kernel_without_copies():
    from torch.profiler import ProfilerActivity, profile

    from emernerf_b200 import loss

    bufs, ex = make_flows(8192, 64, 16, seed=12, device=DEV)
    loss.flow_cycle_loss(ex)                # the device's loss workspace exists
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        loss.flow_cycle_loss(ex)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert len(names) == 1 and "cycle_loss_fwd_kernel" in names[0], names


@pytest.mark.parametrize("case", ["flow", "flow_feat"])
def test_flow_fixture_parameter_gradients_on_cuda(case):
    from emernerf_b200 import loss
    from helpers import rel_err
    from test_gpu_golden import _build, _render

    g, field, props, est = _build(case)
    out = _render(g, field, props, est, "train")
    total, stats = parity_loss_with_library_cycle(out, loss)
    assert abs(total.item() - g.scalar("train/loss")) < 1e-4
    _, want_stats = reference(out["extras"])
    for k in STAT_KEYS:
        assert abs(stats[k].item() - want_stats[k].item()) <= 1e-6 * want_stats[k].item(), k
    total.backward()
    want = g.tensors("train/grad/field")
    for k, v in field.named_parameters():
        if k in want:
            assert rel_err(v.grad, want[k]) < 5e-3, k
    assert sum(k in want for k, _ in field.named_parameters()) == len(want)


def test_full_size_flow_parameter_gradients():
    """The full-size flow fixture (tests/test_gpu_fullsize.py's bars, over its well-conditioned rays)."""
    import full_cases as fc
    from helpers import rel_err
    from test_gpu_fullsize import _build, _check_projection, _render

    from emernerf_b200 import loss

    g, field, props, est = _build("flow")
    out = _render(g, field, props, est, "train")
    keep = torch.from_numpy(g.z["train/stable"]).to(DEV)
    total, _ = parity_loss_with_library_cycle(fc.mask_rays(out, keep), loss)
    assert abs(total.item() - g.scalar("train/loss")) < 1e-4 * max(1.0, abs(g.scalar("train/loss")))
    total.backward()
    want, want_proj = g.tensors("train/grad/field"), g.tensors("train/gradproj/field")
    checked = 0
    for k, v in field.named_parameters():
        if k in want:
            tol_k = 3e-2 if "sky_head" in k else 5e-3
            assert rel_err(v.grad, want[k]) < tol_k, (k, rel_err(v.grad, want[k]))
            checked += 1
        elif k in want_proj:
            _check_projection(v.grad, want_proj[k], k)
            checked += 1
    assert checked == len(want) + len(want_proj)

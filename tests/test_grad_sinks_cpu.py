"""Gradient sinks on CPU (C ABI answered by tests/cabi_emulator.py): the registry's lookup and touched bookkeeping,
and the library backward passes that accumulate into the sinks -- the fused flow branch's chain, the stacked-row grid
encoding and the proposal level's table zeroing -- against the same passes without sinks, bit for bit."""
import gc
import weakref

import pytest
import torch

import cabi_emulator
import flow_branch_emulator
from test_flow_branch_cpu import R, S, _inputs, _model


@pytest.fixture
def restore_sinks():
    """The registry is global: each test starts without sinks, and whatever was registered before is put back."""
    from emernerf_b200 import _ops

    saved = dict(_ops._GRAD_SINKS)
    _ops.clear_grad_sinks()
    yield
    _ops._GRAD_SINKS.clear()
    _ops._GRAD_SINKS.update(saved)


@pytest.fixture
def one_thread():
    """The emulated table scatter is autograd of a CPU gather, whose sums are ordered only on one thread."""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


def _grads(params):
    return {k: None if p.grad is None else p.grad.clone() for k, p in params}


def _check_sinks(plain, sunk, opt, params):
    """Sinks hold what autograd got without them, bit for bit; exactly the parameters that got a gradient are
    touched, and ``.grad`` is the sink view."""
    from emernerf_b200 import _ops

    assert any(v is not None for v in plain.values())
    for k, p in params:
        assert torch.equal(sunk[k], plain[k]) if plain[k] is not None else not sunk[k].any(), k
        assert (id(p) in opt._touched) == (plain[k] is not None), k
        assert p.grad.data_ptr() == _ops._grad_sink(p).buf.data_ptr(), k


@pytest.mark.parametrize("feature", [False, True])
def test_flow_chain_into_sinks_matches_autograd(feature, monkeypatch, restore_sinks, one_thread):
    """EMER_FLOW_BRANCH=fused training pass (_FlowWarp, _GridEncodeRows, _FlowFieldChain with the colour head) with and
    without FusedAdam."""
    from emernerf_b200 import _ops
    from emernerf_b200.optim import FusedAdam

    flow_branch_emulator.install(monkeypatch)
    monkeypatch.setattr(_ops, "FLOW_BRANCH", "fused")
    runs = {}
    for sinks in (False, True):
        field = _model(feature)
        field._noise_override = torch.rand(R, S, 1, generator=torch.Generator().manual_seed(2))
        params = list(field.named_parameters())
        opt = FusedAdam([p for _, p in params], lr=1e-3) if sinks else None
        pos, d, data = _inputs()
        field.train()
        del cabi_emulator.CALLS[:]
        out = field(pos, d, data, query_pe_head=False)
        sum((v ** 2).mean() for v in out.values() if torch.is_tensor(v) and v.requires_grad).backward()
        assert {"emer_flow_field_bwd", "emer_field_wgrad"} <= set(cabi_emulator.CALLS)
        runs[sinks] = _grads(params)
    _check_sinks(runs[False], runs[True], opt, params)


def test_grid_encode_rows_into_sink_matches_autograd(monkeypatch, restore_sinks, one_thread):
    """The table gradient of grid_encode_rows lands in the sink as autograd would have it; x_var's input gradient is
    the same either way."""
    from emernerf_b200 import _ops
    from emernerf_b200.optim import FusedAdam
    from emernerf_b200.radiance_fields.encodings import HashEncoder

    cabi_emulator.install(monkeypatch)
    g = torch.Generator().manual_seed(3)
    x_fixed, x_var0 = torch.rand(37, 4, generator=g), torch.rand(50, 4, generator=g)
    up = None
    runs, dx = {}, {}
    for sinks in (False, True):
        torch.manual_seed(0)
        enc = HashEncoder(n_input_dims=4, n_levels=8, base_resolution=4, max_resolution=64, log2_hashmap_size=10,
                          n_features_per_level=4, verbose=False)
        table = enc.tcnn_encoding.params
        opt = FusedAdam([table], lr=1e-3) if sinks else None
        x_var = x_var0.clone().requires_grad_()
        y = _ops.grid_encode_rows(x_fixed, x_var, table, enc.desc)
        if up is None:
            up = torch.randn(y.shape, generator=g)
        del cabi_emulator.CALLS[:]
        (y * up).sum().backward()
        assert cabi_emulator.CALLS == ["emer_grid_bwd", "emer_grid_bwd"]
        runs[sinks], dx[sinks] = _grads([("table", table)]), x_var.grad
    assert torch.equal(dx[True], dx[False])
    _check_sinks(runs[False], runs[True], opt, [("table", table)])


def test_registry_lookup_and_touched(monkeypatch, restore_sinks):
    """A sink is found by the address of the tensor handed in, only while the registered parameter still lives there
    with the same shape; ``touched()`` follows ``mark`` and is cleared by FusedAdam's step and zero_grad."""
    from emernerf_b200 import _ops
    from emernerf_b200.optim import FusedAdam

    cabi_emulator.install(monkeypatch)
    storage = torch.zeros(64)
    p = torch.nn.Parameter(storage[:16])
    opt = FusedAdam([p], lr=1e-3)
    s = _ops._grad_sink(storage[:16])
    assert s is not None and s.buf.data_ptr() == p.grad.data_ptr()
    assert _ops._grad_sink(storage[:16].view(4, 4)) is None          # same address, another shape
    assert not s.touched()
    s.touch()
    assert s.touched() and id(p) in opt._touched
    opt.step()
    assert not s.touched()
    s.touch()
    opt.zero_grad()
    assert not s.touched()

    marked = set()                                                    # ids, as FusedAdam keeps them
    q = torch.nn.Parameter(storage[16:32])
    _ops.register_grad_sink(q, torch.zeros(16), lambda t: marked.add(id(t)), lambda t: id(t) in marked)
    found = lambda t: _ops._grad_sink(t) is not None
    s = _ops._grad_sink(storage[16:32])
    assert not s.touched()
    s.touch()
    assert s.touched() and marked == {id(q)}
    q.data = torch.zeros(16)                                          # the parameter moved: its old address has no sink
    assert not found(storage[16:32])
    q.data = storage[16:32]
    assert found(storage[16:32])
    ref = weakref.ref(q)
    del q, s
    gc.collect()
    assert ref() is None and not found(storage[16:32])                # freed, the address reused by another tensor


def test_prop_level_table_sink_cleared_only_when_untouched(monkeypatch, restore_sinks, one_thread):
    """_PropLevelTrain accumulates into pre-filled sinks of a registrant that does not report ``touched`` (they count
    as touched: nothing is cleared), and zeroes an untouched FusedAdam table slice -- garbage included -- before its
    scatter; either way the sinks end up holding what autograd got without them, added to what was there."""
    from emernerf_b200 import _ops
    from emernerf_b200.optim import FusedAdam
    from oracle import hotpath
    from test_gpu_prop_level_grad import FAR, KIND, NEAR, _density_field, _params, _rays

    cabi_emulator.install(monkeypatch)
    R, n = 37, 16
    net = _density_field(8, True, 5, "cpu", max_resolution=64, log2_hashmap_size=12)
    desc = net.xyz_encoder.desc
    assert _ops.prop_level_train_usable(desc)
    origins, dirs = _rays(R, 6, "cpu")
    s_min, s_max = hotpath.s_bounds(KIND, NEAR, FAR)
    first = torch.arange(2, dtype=torch.float32).repeat(R, 1)
    g = torch.Generator().manual_seed(7)
    bias, d_cdf = torch.rand(R, generator=g), torch.randn(R, n + 1, generator=g)

    def backward(params):
        _, _, cdf = _ops.prop_level_train(first, first.clone(), n, bias, s_min, s_max, KIND, origins, dirs, net.aabb,
                                          True, desc, *params)
        del cabi_emulator.CALLS[:]
        (cdf * d_cdf).sum().backward()
        assert cabi_emulator.CALLS == ["emer_prop_level_bwd", "emer_grid_bwd"]

    plain = [p.detach().clone().requires_grad_() for p in _params(net)]
    backward(plain)
    want = [p.grad for p in plain]
    assert all(w.any() for w in want)

    pre = [torch.randn(p.shape, generator=g) for p in plain]
    sinks = [x.clone() for x in pre]
    params = [p.detach().clone().requires_grad_() for p in plain]
    marked = set()
    for p, s in zip(params, sinks):
        _ops.register_grad_sink(p, s, lambda t: marked.add(id(t)))
    backward(params)
    assert all(p.grad is None for p in params) and marked == {id(p) for p in params}
    for s, x, w in zip(sinks, pre, want):
        assert torch.equal(s, x + w)

    _ops.clear_grad_sinks()
    params = [p.detach().clone().requires_grad_() for p in plain]
    opt = FusedAdam(params, lr=1e-3)
    params[0].grad.fill_(7.0)
    backward(params)
    assert all(id(p) in opt._touched for p in params)
    for p, w in zip(params, want):
        assert torch.equal(p.grad, w)

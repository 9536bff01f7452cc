"""The product's HOST side on CPU: the drop-in modules (``render_rays``, ``RadianceField``, ``DensityField``,
``PropNetEstimator``) and the autograd wrappers of ``emernerf_b200/_ops.py`` run unmodified on CPU tensors, with
the shared library's entry points answered by ``tests/cabi_emulator.py`` (oracle arithmetic behind the same
pointers / strides / sizes), and are compared with the golden vectors produced by the reference's own Python
(tests/golden/make_golden.py) -- the same comparisons tests/test_gpu_golden.py makes on the GPU, at the same
tolerances.  What this pins without a GPU: closure plumbing, per-sample expand views, fused-path selection,
weight-column permutations of the colour head, buffer / stride / padding bookkeeping, gradient routing, the
proposal cache and the interlevel loss.
"""
import types

import pytest
import torch

import cabi_emulator
import cases
from helpers import Golden, assert_close_dict, rel_err
from oracle import adapters

TOL = 1e-4


@pytest.fixture
def emulated(monkeypatch):
    cabi_emulator.install(monkeypatch)
    return cabi_emulator


def _build(case):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder
    from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    field, props = cases.build_models(ns, case)
    g = Golden(case)
    field.load_state_dict(g.tensors("sd/field"))
    for i, p in enumerate(props):
        p.load_state_dict(g.tensors(f"sd/prop{i}"))
    return g, field, props, PropNetEstimator(None, None)


def _render(g, field, props, est, mode):
    from emernerf_b200.radiance_fields.render_utils import render_rays

    lidar = mode == "lidar"
    batch = g.tensors("in/lidar" if lidar else "in/pixel")
    train = mode != "eval"
    field.train(train); est.train(train)
    [p.train(train) for p in props]
    est._jitter_override = g.jitters(mode) if train else None
    field._noise_override = g.noise(mode) if train else None
    est.prop_cache.clear()
    with torch.set_grad_enabled(train):
        return render_rays(field, est, props, batch, cases.render_cfg(), proposal_requires_grad=(mode == "train"),
                           return_decomposition=(mode == "eval"), prefix="lidar_" if lidar else "")


@pytest.mark.parametrize("case", list(cases.CASES))
@pytest.mark.parametrize("mode", ["eval", "lidar", "train"])
def test_host_path_matches_reference_outputs(emulated, case, mode):
    g, field, props, est = _build(case)
    out = _render(g, field, props, est, mode)
    want = g.nested(f"{mode}/out")
    tol = {"*": TOL, "median_depth": 5e-2}
    for k in ("density", "static_density", "dynamic_density", "forward_flow", "backward_flow",
              "forward_pred_backward_flow", "backward_pred_forward_flow", "weights", "trans"):
        tol[k] = 1e-3
    assert_close_dict(out, want, tol)
    hit = set(emulated.CALLS)
    assert {"emer_grid_fwd", "emer_pdf_resample", "emer_composite_fwd", "emer_contract_fwd"} <= hit
    assert "emer_prop_level" in hit                      # the fused level, with or without proposal gradients
    if mode != "lidar":
        assert {"emer_field_tail_fwd", "emer_accumulate_fwd"} <= hit


@pytest.mark.parametrize("prop_train", ["fused", "layers"])
@pytest.mark.parametrize("case", list(cases.CASES))
def test_host_path_gradients_and_proposal_loss(emulated, monkeypatch, case, prop_train):
    """``prop_train``: the proposal levels of an update step as emer_prop_level + emer_prop_level_bwd and the
    interlevel loss as emer_interlevel_loss (default), or both through the modular autograd paths (contract, grid,
    layers, trunc_exp, composite; blur_stepfun / sorted_interp_quad in torch)."""
    from emernerf_b200 import _ops
    monkeypatch.setattr(_ops, "PROP_TRAIN", prop_train)
    monkeypatch.setattr(_ops, "INTERLEVEL", "fused" if prop_train == "fused" else "torch")
    g, field, props, est = _build(case)
    out = _render(g, field, props, est, "train")
    ploss = est.compute_loss(out["extras"]["trans"], 1024.0)
    want_ploss = g.scalar("train/prop_loss")
    assert abs(ploss.item() - want_ploss) <= 1e-3 * max(1.0, abs(want_ploss))
    pnames = [k for k, _ in props[1].named_parameters()]
    pgrads = torch.autograd.grad(ploss, [v for _, v in props[1].named_parameters()])
    assert ("emer_prop_level_bwd" in emulated.CALLS) == (prop_train == "fused")
    assert ("emer_interlevel_loss" in emulated.CALLS) == (prop_train == "fused")
    want_p = g.tensors("train/grad/prop1")
    for k, gr in zip(pnames, pgrads):
        assert rel_err(gr, want_p[k]) < 5e-3, k
    assert all(p.grad is None for p in props[0].parameters())      # network 0 is never evaluated (Q21)

    loss = adapters.parity_loss(out)
    assert abs(loss.item() - g.scalar("train/loss")) < 1e-4
    loss.backward()
    want = g.tensors("train/grad/field")
    checked = 0
    for k, v in field.named_parameters():
        if k in want:
            assert v.grad is not None, k
            assert rel_err(v.grad, want[k]) < 5e-3, k
            checked += 1
    assert checked == len(want)
    hit = set(emulated.CALLS)
    assert {"emer_grid_bwd", "emer_composite_bwd", "emer_accumulate_bwd", "emer_field_tail_bwd",
            "emer_contract_bwd"} & hit >= {"emer_grid_bwd", "emer_composite_bwd", "emer_accumulate_bwd",
                                           "emer_field_tail_bwd"}


def test_host_path_image_shaped_batches_round_trip(emulated):
    """[H, W, 3] inputs are flattened and every output reshaped back (render_utils.py:303-312,385-387)."""
    from emernerf_b200.radiance_fields.render_utils import render_rays

    g, field, props, est = _build("static")
    batch = g.tensors("in/pixel")
    field.eval()
    with torch.no_grad():
        flat = render_rays(field, est, props, batch, cases.render_cfg())
        img = {k: v.reshape(6, 8, *v.shape[1:]) for k, v in batch.items()}
        out = render_rays(field, est, props, img, cases.render_cfg())
    assert out["rgb"].shape == (6, 8, 3) and out["depth"].shape == (6, 8, 1)
    assert torch.equal(out["rgb"].reshape(-1, 3), flat["rgb"])


def test_host_path_chunked_eval_equals_one_chunk(emulated):
    """Evaluation renders in chunks of cfg.render.render_chunk_size rays (render_utils.py:350-383): rays are
    independent, so chunking changes nothing beyond the host BLAS's batch-size-dependent rounding."""
    from emernerf_b200.radiance_fields.render_utils import render_rays

    g, field, props, est = _build("dynamic")
    batch = g.tensors("in/pixel")
    field.eval()
    cfg_one, cfg_many = cases.render_cfg(), cases.render_cfg()
    cfg_many.render.render_chunk_size = 7               # 48 rays -> 7 chunks, the last one ragged
    with torch.no_grad():
        one = render_rays(field, est, props, batch, cfg_one, return_decomposition=True)
        many = render_rays(field, est, props, batch, cfg_many, return_decomposition=True)
    assert set(one) == set(many)
    for k in one:
        if k != "extras":
            assert one[k].shape == many[k].shape and rel_err(many[k], one[k]) < 2e-6, k


def test_host_path_query_flow_and_attributes_agree_with_forward(emulated):
    """The point-query entry points the evaluation code uses (train_emernerf.py:266-272,
    datasets/metrics.py:276-300) return the same tensors as ``forward`` on the same points."""
    g, field, props, est = _build("flow_feat")
    field.eval()
    gen = torch.Generator().manual_seed(4)
    pos = torch.rand(257, 3, generator=gen) * torch.tensor([100.0, 80.0, 20.0]) + torch.tensor([-20.0, -40.0, 0.0])
    t = torch.rand(257, generator=gen)
    with torch.no_grad():
        full = field(pos, None, {"normed_timestamps": t}, combine_static_dynamic=True, query_pe_head=False)
        flow = field.query_flow(pos, t)
        attr = field.query_attributes(pos, t)
    assert torch.equal(flow["forward_flow"], full["forward_flow"])
    assert torch.equal(flow["backward_flow"], full["backward_flow"])
    for k in ("density", "static_density", "dynamic_density", "static_dino_feat", "dynamic_dino_feat"):
        assert torch.equal(attr[k], full[k]), k
    want = (full["static_density"].unsqueeze(-1) * full["static_dino_feat"]
            + full["dynamic_density"].unsqueeze(-1) * full["dynamic_dino_feat"]) / (full["density"].unsqueeze(-1) + 1e-6)
    assert rel_err(attr["dino_feat"], want) < 1e-6
    assert flow["dynamic_density"].shape == (257,)


def test_host_path_generic_proposal_call_matches_fused_level(emulated):
    """DensityField.forward on explicit points (the closure path) and the fused proposal-level entry point see
    the same network and the same bookkeeping of their arguments."""
    from emernerf_b200 import _ops
    from emernerf_b200.third_party.nerfacc_prop_net import s_bounds

    g, field, props, est = _build("static")
    batch = g.tensors("in/pixel")
    net = props[1]
    R, n = batch["origins"].shape[0], 32
    base = torch.arange(2, dtype=torch.float32).repeat(R, 1)
    s_min, s_max = s_bounds("uniform_lindisp", cases.NEAR, cases.FAR)
    lin = [m for m in net.base_mlp if isinstance(m, torch.nn.Linear)]
    with torch.no_grad():
        s, t, cdf = _ops.prop_level(base, base, n, None, s_min, s_max, "uniform_lindisp", batch["origins"],
                                    batch["viewdirs"], net.aabb, True, net.xyz_encoder.desc,
                                    net.xyz_encoder.tcnn_encoding.params, lin[0].weight, lin[0].bias, lin[1].weight,
                                    lin[1].bias)
        pos = batch["origins"][:, None, :] + batch["viewdirs"][:, None, :] * (t[:, :-1] + t[:, 1:])[..., None] / 2.0
        sigma = net(pos)["density"].squeeze(-1)
        cdf2 = _ops.composite(t[:, :-1].contiguous(), t[:, 1:].contiguous(), sigma, want_cdf=True)[5]
    assert rel_err(cdf, cdf2) < 2e-5


def test_host_path_without_emulator_refuses_cpu():
    """The emulator is opt-in test infrastructure: the product itself has no CPU path."""
    g, field, props, est = _build("static")
    with pytest.raises(RuntimeError, match="CUDA"):
        _render(g, field, props, est, "eval")

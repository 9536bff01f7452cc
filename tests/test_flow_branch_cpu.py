"""EMER_FLOW_BRANCH=fused on CPU tensors through the C-ABI emulators (cabi_emulator + flow_branch_emulator): the host
wiring of the fused flow branch -- _FlowWarp, _GridEncodeRows, _FlowFieldChain and RadianceField._flow_branch -- against
the per-layer path of the same model: every output key, every parameter gradient, the density-only (lidar) and eval
passes, and the generator state."""
import pytest
import torch

import cabi_emulator
import flow_branch_emulator
from helpers import rel_err

R, S = 4, 32
AABB = [-20.0, -40.0, 0.0, 80.0, 40.0, 20.0]


def _model(feature: bool):
    from emernerf_b200.radiance_fields import RadianceField
    from emernerf_b200.radiance_fields.encodings import HashEncoder

    torch.manual_seed(0)
    enc = lambda d, lv: HashEncoder(n_input_dims=d, n_levels=lv, base_resolution=4, max_resolution=32,
                                    log2_hashmap_size=10, n_features_per_level=4, verbose=False)
    field = RadianceField(xyz_encoder=enc(3, 8), dynamic_xyz_encoder=enc(4, 10), flow_xyz_encoder=enc(4, 10), aabb=AABB,
                          unbounded=True, geometry_feature_dim=64, base_mlp_layer_width=64, head_mlp_layer_width=64,
                          enable_shadow_head=True, enable_feature_head=feature, semantic_feature_dim=64,
                          feature_mlp_layer_width=64, feature_embedding_dim=64, enable_learnable_pe=False,
                          num_train_timesteps=10)
    field.register_normalized_training_timesteps(torch.linspace(0, 1, 10), time_diff=0.1)
    with torch.no_grad():
        for k, v in field.named_parameters():
            if k.endswith("tcnn_encoding.params"):
                v.copy_(torch.randn(v.shape, generator=torch.Generator().manual_seed(v.numel())) * 0.3)
    return field


def _inputs():
    g = torch.Generator().manual_seed(1)
    lo, hi = torch.tensor(AABB[:3]), torch.tensor(AABB[3:])
    pos = lo + (hi - lo) * (torch.rand(R, S, 3, generator=g) * 1.6 - 0.3)
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)[:, None, :].expand(R, S, 3)
    t = torch.rand(R, generator=g)[:, None].expand(R, S)
    return pos, d, {"normed_timestamps": t}


def _run(field, mode):
    pos, d, data = _inputs()
    field.train(mode != "eval")
    with torch.set_grad_enabled(mode != "eval"):
        out = field(pos, d, data, return_density_only=(mode == "lidar"), query_pe_head=False)
    grads = {}
    if mode != "eval":
        loss = sum((v ** 2).mean() for v in out.values() if torch.is_tensor(v) and v.requires_grad)
        params = [(k, p) for k, p in field.named_parameters() if p.requires_grad]
        gr = torch.autograd.grad(loss, [p for _, p in params], allow_unused=True)
        grads = {k: v for (k, _), v in zip(params, gr) if v is not None}
    return out, grads


@pytest.mark.parametrize("feature", [False, True])
@pytest.mark.parametrize("mode", ["train", "lidar", "eval"])
def test_fused_flow_branch_matches_the_per_layer_path(feature, mode, monkeypatch):
    from emernerf_b200 import _ops

    flow_branch_emulator.install(monkeypatch)
    field = _model(feature)
    field._noise_override = torch.rand(R, S, 1, generator=torch.Generator().manual_seed(2))
    res = {}
    for sw in ("layers", "fused"):
        monkeypatch.setattr(_ops, "FLOW_BRANCH", sw)
        del cabi_emulator.CALLS[:]
        res[sw] = _run(field, mode)
        fused = {"emer_flow_warp_fwd", "emer_flow_field_fwd"} <= set(cabi_emulator.CALLS)
        assert fused == (sw == "fused"), sorted(set(cabi_emulator.CALLS))
        if sw == "fused" and mode != "eval":
            assert {"emer_flow_warp_bwd", "emer_flow_field_bwd"} <= set(cabi_emulator.CALLS)
    (a, ga), (b, gb) = res["layers"], res["fused"]
    assert list(a) == list(b)
    for k in a:
        if torch.is_tensor(a[k]):
            assert a[k].shape == b[k].shape, k
            assert rel_err(b[k].detach(), a[k].detach()) < 1e-5, (k, rel_err(b[k].detach(), a[k].detach()))
    assert ga.keys() == gb.keys()
    for k in ga:
        assert rel_err(gb[k], ga[k]) < 1e-4, (k, rel_err(gb[k], ga[k]))


def test_fused_flow_branch_draws_the_reference_noise(monkeypatch):
    """Without a noise override both paths make the same rand_like call: same outputs, same generator state."""
    from emernerf_b200 import _ops

    flow_branch_emulator.install(monkeypatch)
    field = _model(False)
    outs, states = {}, {}
    for sw in ("layers", "fused"):
        monkeypatch.setattr(_ops, "FLOW_BRANCH", sw)
        torch.manual_seed(5)
        outs[sw] = _run(field, "train")[0]
        states[sw] = torch.get_rng_state()
    assert torch.equal(states["layers"], states["fused"])
    assert rel_err(outs["fused"]["dynamic_density"].detach(), outs["layers"]["dynamic_density"].detach()) < 1e-5

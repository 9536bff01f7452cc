"""CPU-side checks: the C-ABI library loads and exports every symbol include/emer_b200.h declares,
host-side level tables agree with the oracle, the drop-in modules carry the reference's state-dict
keys, and the host logic (requires-grad schedule, s-bounds) matches the oracle."""
import ctypes
import os
import re
import types

import pytest
import torch

import cases
from helpers import Golden
from oracle import hotpath, tcnn_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "emer_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(emer_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_loads_and_exports_every_declared_symbol():
    from emernerf_b200 import _lib
    from emernerf_b200.build import build_library

    path = build_library()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    declared = _declared_symbols()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in emer_b200.h but not exported"
    assert sorted(_lib.EXPORTS) == declared
    _lib.load()
    assert _lib.load().emer_version() >= 1


def test_struct_layout_matches_header():
    from emernerf_b200.grid_desc import EmerGridDesc

    # 4 int32 + 16 float + 16 u32 + 17 u32 + 16 u32
    assert ctypes.sizeof(EmerGridDesc) == 4 * (4 + 16 + 16 + 17 + 16)


@pytest.mark.parametrize("name,D,args", [
    ("static", 3, (10, 16, 8192, 20, 4)), ("dynamic", 4, (10, 32, 8192, 18, 4)),
    ("flow", 4, (10, 16, 4096, 18, 4)), ("prop0", 3, (8, 16, 512, 20, 1)), ("prop1", 3, (8, 16, 2048, 20, 1)),
    ("tiny", 3, (4, 8, 64, 10, 4)), ("tiny4", 4, (4, 4, 32, 10, 2)),
])
def test_host_level_table_matches_oracle(name, D, args):
    from emernerf_b200.grid_desc import GridDesc

    cfg = hotpath.hash_encoder_config(*args)
    g = GridDesc(D, cfg)
    o = tcnn_ref.grid_geometry(D, cfg)
    assert g.offsets == o.offsets and g.resolutions == o.resolutions and g.hashed == o.hashed
    assert g.scales == o.scales
    assert [g.c.offset[i] for i in range(g.n_levels + 1)] == o.offsets
    assert g.bytes_per_point() == {"static": 1452, "dynamic": 2736, "flow": 2736, "prop0": 300, "prop1": 300}.get(
        name, g.bytes_per_point())


@pytest.mark.parametrize("case", list(cases.CASES))
def test_dropin_state_dict_keys_match_reference(case):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    field, props = cases.build_models(ns, case)
    g = Golden(case)
    want = g.tensors("sd/field")
    have = field.state_dict()
    assert set(want) == set(have)
    for k in want:
        assert tuple(want[k].shape) == tuple(have[k].shape), k
    field.load_state_dict(want)
    for i, p in enumerate(props):
        p.load_state_dict(g.tensors(f"sd/prop{i}"))


def test_install_dropin_aliases_reference_module_names():
    import sys
    import emernerf_b200

    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in ("radiance_fields", "third_party")}
    try:
        emernerf_b200.install_dropin()
        from radiance_fields import DensityField, RadianceField, build_density_field, build_radiance_field_from_cfg  # noqa
        from radiance_fields.render_utils import render_rays  # noqa
        from third_party.nerfacc_prop_net import PropNetEstimator, get_proposal_requires_grad_fn  # noqa
        import third_party.tcnn_modules as tcnn
        assert RadianceField.__module__.startswith("emernerf_b200")
        assert hasattr(tcnn, "Encoding")
    finally:
        for k in list(sys.modules):
            if k.split(".")[0] in ("radiance_fields", "third_party"):
                del sys.modules[k]
        sys.modules.update(saved)


def test_requires_grad_schedule_and_s_bounds():
    from emernerf_b200.third_party.nerfacc_prop_net import get_proposal_requires_grad_fn, s_bounds

    fn = get_proposal_requires_grad_fn()
    seq = [fn(s) for s in [0, 0, 1, 1, 2, 2, 500, 500, 500, 500, 500, 2000, 2000, 2000, 2000, 2000, 2000, 2000]]
    # reference closure semantics (nerfacc_prop_net.py:280-296), advanced twice per training step (Q16)
    steps_since, want = 0, []
    for s in [0, 0, 1, 1, 2, 2, 500, 500, 500, 500, 500, 2000, 2000, 2000, 2000, 2000, 2000, 2000]:
        tgt = min(s / 1000, 1.0) * 5.0
        r = steps_since > tgt
        if r:
            steps_since = 0
        steps_since += 1
        want.append(r)
    assert seq == want
    for kind in ("uniform", "lindisp", "sqrt", "log", "uniform_lindisp", "uniform_lindisp_0"):
        assert s_bounds(kind, 0.1, 1000.0) == hotpath.s_bounds(kind, 0.1, 1000.0)
    lo, hi = s_bounds("uniform_lindisp", 0.1, 1000.0)
    assert abs(lo - 2.5e-4) < 1e-9 and abs(hi - 0.9) < 1e-7


def test_ops_refuse_cpu_tensors():
    from emernerf_b200 import _ops
    from emernerf_b200.grid_desc import GridDesc

    g = GridDesc(3, hotpath.hash_encoder_config(4, 8, 64, 10, 4))
    with pytest.raises(RuntimeError, match="CUDA"):
        _ops.grid_encode(torch.rand(4, 3), torch.zeros(g.n_params), g)
    with pytest.raises(RuntimeError, match="CUDA"):
        _ops.linear(torch.rand(4, 8), torch.rand(3, 8), None)


def test_sorted_interp_quad_searchsorted_equals_dense_mask():
    """The searchsorted formulation of the zip-nerf interpolation equals the reference's dense-mask
    formulation (and the oracle's restatement of it) on blurred step functions, values and gradients."""
    from emernerf_b200.third_party import nerfacc_prop_net as pn

    g = torch.Generator().manual_seed(0)
    R = 40
    s = torch.sort(torch.rand(R, 65, generator=g), -1).values
    w = torch.rand(R, 64, generator=g)
    w[:, ::7] = 0.0
    for r in (0.03, 0.003):
        c, wv = pn.blur_stepfun(s, w, r)
        area = 0.5 * (wv[..., 1:] + wv[..., :-1]) * (c[..., 1:] - c[..., :-1])
        cdf = torch.cat([torch.zeros_like(area[..., :1]), torch.cumsum(area, -1)], -1)
        for n in (129, 65):
            # queries inside the knot range, as in compute_loss (proposal edges lie in [0, 1], the blurred
            # knots span [min - r, max + r]); beyond the last knot the reference's masked arg-max picks an
            # arbitrary tied index and the two forms may differ by an ulp
            x = torch.sort(torch.rand(R, n, generator=g), -1).values
            x = x * (s[:, -1:] - s[:, :1]) + s[:, :1]
            a = pn.sorted_interp_quad(x, c, wv, cdf)
            b = pn.sorted_interp_quad_dense(x, c, wv, cdf)
            d = hotpath.sorted_interp_quad(x, c, wv, cdf)
            assert torch.equal(b, d)
            assert torch.allclose(a, b, rtol=0, atol=1e-7)
            # (no gradient check: compute_loss feeds detached tensors, gradients reach the proposal
            #  network only through w_prop)


def test_tensor_core_eligibility_mirrors_the_library_limits():
    """_ops only sends a layer to the tensor-core kernels when the library can take it (csrc/linear_tc.cu launch<>,
    emer_linear_tc_bwd_weight); the emulator carries an independent restatement of the same limits, so a
    disagreement between the two shows up here before it can on the GPU."""
    import ctypes

    import cabi_emulator as em
    from emernerf_b200 import _ops

    # the shipped layer shapes all run on the tensor cores
    for k, n_out in ((40, 64), (64, 64), (64, 128), (113, 64), (177, 64), (49, 64), (32, 64)):
        assert _ops._tc_fits(k, n_out) and _ops._tc_fits(n_out, k) and _ops._tc_wgrad_fits(k, n_out), (k, n_out)
    assert _ops._tc_fits(128, 113)                       # stacked skip gradient [dZ0 | dZ1] [W0 ; W1[:, h:]]
    # layers the resident weight panels / accumulators cannot hold
    assert not _ops._tc_fits(256, 256) and not _ops._tc_fits(113, 256) and not _ops._tc_fits(64, 384)
    assert not _ops._tc_wgrad_fits(256, 128) and not _ops._tc_wgrad_fits(64, 256) and not _ops._tc_wgrad_fits(369, 64)

    buf = (ctypes.c_float * 64)()
    ptr = ctypes.c_void_p((ctypes.addressof(buf) + 15) // 16 * 16)
    for k in range(8, 400, 24):
        for n_out in range(8, 400, 24):
            if _ops._tc_fits(k, n_out):
                em._check_tc(k, n_out, "fwd")            # raises if the library would refuse
            else:
                with pytest.raises(RuntimeError):
                    em._check_tc(k, n_out, "fwd")
            try:
                em._check_tc_wgrad(ptr, _ops._pad4(k), ptr, _ops._pad4(n_out), k, n_out)
                lib_ok = True
            except RuntimeError:
                lib_ok = False
            assert lib_ok == _ops._tc_wgrad_fits(k, n_out), (k, n_out)


def test_blur_stepfun_merge_equals_the_reference_sort():
    """The merge formulation of blur_stepfun (two searchsorted ranks + scatter) gives the reference's sort-based result
    (nerfacc_prop_net.py:22-34), ties included."""
    import torch

    from emernerf_b200.third_party.nerfacc_prop_net import blur_stepfun

    def reference(x, y, r):
        xr, xr_idx = torch.sort(torch.cat([x - r, x + r], dim=-1))
        y1 = (torch.cat([y, torch.zeros_like(y[..., :1])], dim=-1) - torch.cat([torch.zeros_like(y[..., :1]), y], dim=-1)) / (2 * r)
        y2 = torch.cat([y1, -y1], dim=-1).take_along_dim(xr_idx[..., :-1], dim=-1)
        yr = torch.cumsum((xr[..., 1:] - xr[..., :-1]) * torch.cumsum(y2, dim=-1), dim=-1).clamp_min(0)
        return xr, torch.cat([torch.zeros_like(yr[..., :1]), yr], dim=-1)

    g = torch.Generator().manual_seed(0)
    x = torch.sort(torch.rand(33, 65, generator=g), dim=-1).values
    x[:, 10] = x[:, 9]                      # repeated edges
    x[0] = torch.linspace(0, 1, 65)         # regular spacing: x_i - r == x_j + r ties for r = k / 128
    y = torch.rand(33, 64, generator=g)
    for r in (0.03, 0.003, 1.0 / 128):
        e0, h0 = reference(x, y, r)
        e1, h1 = blur_stepfun(x, y, r)
        assert torch.equal(e0, e1)
        assert torch.allclose(h0, h1, rtol=1e-6, atol=1e-7)

"""The hash grid's level-group schedule: forward gather and table-only scatter on ray-coherent points, at the
small test grids (odd level counts included) and at the real configs (static 10x4 2^20, 4-D 10x4 2^18, the 3-D 8x1
proposal grids).  The forward is checked against the CPU oracle, the table gradient against an fp64 scatter built
from the kernel's own corner indices and the oracle's interpolation weights."""
import pytest
import torch

from helpers import rel_err
from oracle import hotpath, tcnn_ref
from test_gpu_kernels import GRIDS

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = dict(GRIDS)
CASES["3d_f4_odd"] = (3, (5, 8, 64, 10, 4))          # F = 4 with a trailing level group of one level
CASES["prop_512"] = (3, (8, 16, 512, 20, 1))         # the proposal grids (configs.py)
CASES["prop_2048"] = (3, (8, 16, 2048, 20, 1))
SMALL = ["3d_f4", "4d_f4", "3d_f1", "4d_f2", "3d_f4_odd"]
REAL = ["3d_f4_cfg", "4d_f4_cfg", "prop_512", "prop_2048"]


def _grid(name):
    from emernerf_b200.grid_desc import GridDesc

    D, args = CASES[name]
    cfg = hotpath.hash_encoder_config(*args)
    return D, GridDesc(D, cfg), tcnn_ref.grid_geometry(D, cfg)


def _ray_points(rays, samples, D, seed=0):
    """Ray-major [rays * samples, D] in [0, 1]: consecutive rows are consecutive samples of one ray (what the
    renderer feeds the grid), with short rays whose samples share cells even at fine levels, long rays that cross
    many cells, and some rows on the cube's faces."""
    g = torch.Generator().manual_seed(seed)
    o = torch.rand(rays, 1, 3, generator=g)
    d = torch.nn.functional.normalize(torch.randn(rays, 1, 3, generator=g), dim=-1)
    length = torch.rand(rays, 1, 1, generator=g) ** 3 * 1.5
    t = torch.sort(torch.rand(rays, samples, 1, generator=g), dim=1).values * length
    x = (o + d * t).clamp(0.0, 1.0)
    if D == 4:
        x = torch.cat([x, torch.rand(rays, 1, 1, generator=g).expand(rays, samples, 1)], -1)
    x = x.reshape(-1, D).contiguous()
    x[-7:] = torch.rand(7, D, generator=g).round()
    return x


def _table_grad_fp64(x, dy, desc, geom):
    """fp64 scatter of dy through the corner indices the kernels use and the oracle's fp32 interpolation weights."""
    from emernerf_b200 import _ops

    F = geom.n_feat
    idx = _ops.grid_indices(x.to(DEV), desc).long()                  # [N, L, 2^D] absolute entries
    out = torch.zeros(geom.n_params // F, F, dtype=torch.float64, device=DEV)
    dyl = dy.to(DEV).double().view(x.shape[0], geom.n_levels, F)
    for lvl in range(geom.n_levels):
        _, w, _, _ = tcnn_ref.corner_indices_and_weights(x, geom, lvl)
        w = w.to(DEV).double()
        for c in range(w.shape[1]):
            out.index_add_(0, idx[:, lvl, c], w[:, c : c + 1] * dyl[:, lvl])
    return out.view(-1)


@pytest.mark.parametrize("name", SMALL + REAL)
def test_grid_forward_level_groups_vs_oracle(name):
    from emernerf_b200 import _ops

    D, desc, geom = _grid(name)
    x = _ray_points(256, 64, D, seed=1)
    g = torch.Generator().manual_seed(2)
    params = torch.randn(geom.n_params, generator=g) * 0.3
    want = tcnn_ref.grid_forward(x, params, geom)
    for n in (1, 31, 257, x.shape[0] - 3, x.shape[0]):
        got = _ops.grid_encode(x[:n].to(DEV), params.to(DEV), desc).cpu()
        assert got.shape == (n, geom.n_output_dims)
        assert (got - want[:n]).abs().max().item() <= 1e-6 * want[:n].abs().max().item(), n
        assert (got == want[:n]).float().mean().item() > 0.999, n


@pytest.mark.parametrize("name", SMALL + REAL)
def test_grid_table_only_backward_vs_fp64(name):
    from emernerf_b200 import _ops

    D, desc, geom = _grid(name)
    x = _ray_points(256, 64, D, seed=3)
    g = torch.Generator().manual_seed(4)
    params = (torch.randn(geom.n_params, generator=g) * 0.3).to(DEV)
    dy = torch.randn(x.shape[0], geom.n_output_dims, generator=g)
    dy[::5] = 0.0                                      # rows without upstream gradient
    for n in (1, 31, 257, x.shape[0] - 3, x.shape[0]):
        p = params.clone().requires_grad_(True)
        y = _ops.grid_encode(x[:n].to(DEV), p, desc)   # x without requires_grad: the table-only scatter
        y.backward(dy[:n].to(DEV))
        want = _table_grad_fp64(x[:n], dy[:n], desc, geom)
        assert rel_err(p.grad, want) < 2e-5, n
        assert torch.equal(p.grad == 0, want == 0), n     # no entry is touched that no corner reaches


@pytest.mark.parametrize("name", ["3d_f4", "3d_f4_odd", "3d_f4_cfg", "4d_f4_cfg", "prop_2048"])
def test_grid_table_backward_adds_into_fused_adam_sink(name):
    """The scatter adds into the optimizer's gradient buffer in place and keeps what is already there."""
    from emernerf_b200 import _ops
    from emernerf_b200.optim import FusedAdam

    D, desc, geom = _grid(name)
    x = _ray_points(128, 64, D, seed=5)
    g = torch.Generator().manual_seed(6)
    p = torch.nn.Parameter((torch.randn(geom.n_params, generator=g) * 0.3).to(DEV))
    FusedAdam([p], lr=1e-3)
    sink = p.grad
    g0 = torch.randn(geom.n_params, generator=g).to(DEV)
    sink.copy_(g0)
    dy = torch.randn(x.shape[0], geom.n_output_dims, generator=g)
    _ops.grid_encode(x.to(DEV), p, desc).backward(dy.to(DEV))
    assert p.grad.data_ptr() == sink.data_ptr()
    want = g0.double() + _table_grad_fp64(x, dy, desc, geom)
    assert rel_err(p.grad, want) < 2e-5


@pytest.mark.parametrize("name", SMALL + ["3d_f4_cfg", "4d_f4_cfg"])
def test_grid_both_gradients_match_single_gradient_calls(name):
    from emernerf_b200 import _ops

    D, desc, geom = _grid(name)
    x = _ray_points(64, 64, D, seed=7)[:-5].to(DEV)
    g = torch.Generator().manual_seed(8)
    params = (torch.randn(geom.n_params, generator=g) * 0.3).to(DEV)
    dy = torch.randn(x.shape[0], geom.n_output_dims, generator=g).to(DEV)

    xb, pb = x.clone().requires_grad_(True), params.clone().requires_grad_(True)
    _ops.grid_encode(xb, pb, desc).backward(dy)
    xs = x.clone().requires_grad_(True)
    _ops.grid_encode(xs, params, desc).backward(dy)
    ps = params.clone().requires_grad_(True)
    _ops.grid_encode(x, ps, desc).backward(dy)
    assert torch.equal(xb.grad, xs.grad)              # dx has no atomics: bit-identical
    want = _table_grad_fp64(x.cpu(), dy.cpu(), desc, geom)
    assert rel_err(pb.grad, want) < 2e-5 and rel_err(ps.grad, want) < 2e-5

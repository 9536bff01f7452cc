"""The hash-grid gather fetches the two x-neighbour corners of a cell (c, c ^ 1) in one load instruction: a lane pair
shares the loads of its two rows for F = 4, and one 16-byte load covers both corners where they share a block for
F = 1.  These cases are the ones that pairing creates: odd N and N below one lane pair (a lane whose partner row does
not exist), points on the far faces (a dense x + 1 corner that wraps and is not adjacent), and cells whose x has long
runs of trailing one bits (a hashed pair that lands in different lines).  The forward must equal the grid evaluated
one level at a time bit for bit and the fp64 interpolation of the same corners; the table scatter must match fp64."""
import pytest
import torch

from helpers import rel_err
from oracle import hotpath, tcnn_ref
from test_gpu_grid_schedule import _table_grad_fp64
from test_gpu_grid_sectors import _bwd_table, _fwd, _level_at_a_time

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (D, (n_levels, base_resolution, max_resolution, log2_hashmap_size, F)): dense and hashed levels, even and odd L
CASES = {
    f"{d}d_f{f}_{tag}": (d, (nl, 4, res, 12, f))
    for d, res in ((3, 512), (4, 96))
    for f in (1, 2, 4)
    for tag, nl in (("even", 8), ("odd", 7))
}
SIZES = (1, 3, 33, 1001, 64 * 257 + 1)


def _grid(name):
    from emernerf_b200.grid_desc import GridDesc

    D, args = CASES[name]
    cfg = hotpath.hash_encoder_config(*args)
    return GridDesc(D, cfg), tcnn_ref.grid_geometry(D, cfg)


def _points(geom, n, seed):
    """[n, D] in [0, 1]: a third random, a third on the cube's faces (0 or 1 in some dimensions), a third whose x
    falls in cell 2^k - 1 of a random level (k trailing one bits), centred in the cell."""
    g = torch.Generator().manual_seed(seed)
    D = geom.n_dims
    x = torch.rand(n, D, generator=g)
    kind = torch.arange(n) % 3
    face = torch.rand(n, D, generator=g) < 0.5
    x = torch.where((kind == 1)[:, None] & face, torch.rand(n, D, generator=g).round(), x)
    for i in torch.nonzero(kind == 2).flatten().tolist():
        lvl = int(torch.randint(geom.n_levels, (1,), generator=g))
        s = geom.scales[lvl]
        kmax = max(1, int(s + 0.5).bit_length() - 1)
        k = int(torch.randint(1, kmax + 1, (1,), generator=g))
        v = ((1 << k) - 1) / s                      # pos = s * x + 0.5: cell 2^k - 1, plus one half
        x[i, 0] = min(max(v, 0.0), 1.0)
    return x.contiguous()


def _forward_fp64(x, table, desc, geom):
    from emernerf_b200 import _ops

    F = geom.n_feat
    idx = _ops.grid_indices(x.to(DEV), desc).long()
    t = table.double().view(-1, F)
    cols = []
    for lvl in range(geom.n_levels):
        _, w, _, _ = tcnn_ref.corner_indices_and_weights(x, geom, lvl)
        w = w.to(DEV).double()
        cols.append((w[:, :, None] * t[idx[:, lvl]]).sum(1))
    return torch.cat(cols, 1)


@pytest.mark.parametrize("name", list(CASES))
def test_forward_pairs_bit_identical_and_vs_fp64(name):
    desc, geom = _grid(name)
    for n in SIZES:
        x = _points(geom, n, seed=n).to(DEV)
        g = torch.Generator().manual_seed(n + 1)
        table = (torch.randn(geom.n_params, generator=g) * 0.3).to(DEV)
        y = torch.full((n, geom.n_output_dims), float("nan"), device=DEV)
        _fwd(desc.c, x, table, y, n)
        assert torch.equal(y, _level_at_a_time(desc, x, table)), n
        want = _forward_fp64(x.cpu(), table, desc, geom)
        assert (y.double() - want).abs().max().item() <= 1e-6 * max(want.abs().max().item(), 1.0), n


@pytest.mark.parametrize("name", list(CASES))
def test_table_scatter_pairs_vs_fp64(name):
    desc, geom = _grid(name)
    for n in SIZES:
        x = _points(geom, n, seed=n + 5).to(DEV)
        g = torch.Generator().manual_seed(n + 6)
        dy = torch.randn(n, geom.n_output_dims, generator=g).to(DEV)
        dt = torch.zeros(geom.n_params, device=DEV)
        _bwd_table(desc.c, x, dy, dt, n)
        want = _table_grad_fp64(x.cpu(), dy.cpu(), desc, geom)
        assert torch.isfinite(dt).all(), n
        assert rel_err(dt, want) < 2e-5, n

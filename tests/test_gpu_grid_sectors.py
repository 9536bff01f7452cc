"""The hash grid's whole-sector level pairs: the forward, which pairs levels (2k, 2k+1) and writes each row's 32-byte
sector with one store of a lane pair, is bit-identical to the grid evaluated one level at a time; the table scatter,
which pairs levels only while both tables are small, matches an fp64 scatter; neither writes past the N*L*F outputs
nor reads past the N*L*F upstream gradients; and both replay in a CUDA graph."""
import ctypes

import pytest
import torch

from helpers import rel_err
from oracle import hotpath, tcnn_ref
from test_gpu_grid_schedule import _ray_points, _table_grad_fp64

pytestmark = pytest.mark.gpu
DEV = "cuda"

# name -> (D, (n_levels, base_resolution, max_resolution, log2_hashmap_size, F)); every <D, F> instantiation, even
# and odd level counts, dense level pairs and hashed levels whose partner is hashed
CASES = {
    "3d_f4_even": (3, (6, 8, 256, 12, 4)),
    "3d_f4_odd": (3, (7, 8, 256, 12, 4)),
    "3d_f2_even": (3, (6, 8, 256, 12, 2)),
    "3d_f1_odd": (3, (9, 8, 256, 12, 1)),
    "4d_f4_even": (4, (6, 4, 64, 12, 4)),
    "4d_f4_odd": (4, (5, 4, 64, 12, 4)),
    "4d_f2_odd": (4, (5, 4, 64, 12, 2)),
    "4d_f1_even": (4, (8, 4, 64, 12, 1)),
    "static_cfg": (3, (10, 16, 8192, 20, 4)),      # 2^20-entry hashed pairs: the scatter keeps them apart
}
SIZES = (1, 2, 1001, 64 * 1023 + 1)                 # the last spans many CTAs per level group, odd like 1 and 1001


def _grid(name):
    from emernerf_b200.grid_desc import GridDesc

    D, args = CASES[name]
    cfg = hotpath.hash_encoder_config(*args)
    return D, GridDesc(D, cfg), tcnn_ref.grid_geometry(D, cfg)


def _one_level(desc, l):
    """A descriptor of level l alone, addressing the same table storage."""
    c = type(desc.c)()
    c.n_dims, c.n_levels, c.n_feat = desc.n_dims, 1, desc.n_feat
    c.scale[0], c.resolution[0], c.hashed[0] = desc.scales[l], desc.resolutions[l], int(desc.hashed[l])
    c.offset[0], c.offset[1] = desc.offsets[l], desc.offsets[l + 1]
    return c


def _ptr(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _fwd(c, x, table, y, n):
    from emernerf_b200 import _lib

    _lib.call("emer_grid_fwd", ctypes.byref(c), _ptr(x), _ptr(table), _ptr(y), n,
              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def _bwd_table(c, x, dy, dtable, n):
    from emernerf_b200 import _lib

    _lib.call("emer_grid_bwd", ctypes.byref(c), _ptr(x), None, _ptr(dy), _ptr(dtable), None, n,
              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def _level_at_a_time(desc, x, table):
    n, F = x.shape[0], desc.n_feat
    cols = []
    for l in range(desc.n_levels):
        yl = torch.empty(n, F, device=DEV)
        _fwd(_one_level(desc, l), x, table, yl, n)
        cols.append(yl)
    return torch.cat(cols, 1)


def _inputs(name, n, seed):
    D, desc, geom = _grid(name)
    rays = (n + 63) // 64
    x = _ray_points(rays, 64, D, seed=seed)[:n].contiguous().to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    table = (torch.randn(geom.n_params, generator=g) * 0.3).to(DEV)
    dy = torch.randn(n, geom.n_output_dims, generator=g).to(DEV)
    return D, desc, geom, x, table, dy


@pytest.mark.parametrize("name", list(CASES))
def test_forward_bit_identical_to_level_at_a_time(name):
    for n in SIZES:
        _, desc, geom, x, table, _ = _inputs(name, n, seed=n)
        y = torch.empty(n, geom.n_output_dims, device=DEV)
        _fwd(desc.c, x, table, y, n)
        assert torch.equal(y, _level_at_a_time(desc, x, table)), n


@pytest.mark.parametrize("name", list(CASES))
def test_forward_writes_nothing_past_the_outputs(name):
    n = 1001
    _, desc, geom, x, table, _ = _inputs(name, n, seed=3)
    m = n * geom.n_output_dims
    buf = torch.full((m + 1024,), float("nan"), device=DEV)
    _fwd(desc.c, x, table, buf[:m], n)
    torch.cuda.synchronize()
    assert torch.isnan(buf[m:]).all()
    assert torch.equal(buf[:m].view(n, -1), _level_at_a_time(desc, x, table))


@pytest.mark.parametrize("name", list(CASES))
def test_table_scatter_vs_fp64_and_reads_nothing_past_dy(name):
    for n in SIZES:
        _, desc, geom, x, _, dy = _inputs(name, n, seed=n + 7)
        m = n * geom.n_output_dims
        buf = torch.full((m + 1024,), float("nan"), device=DEV)    # a read past dy would spread NaN into the grads
        buf[:m] = dy.view(-1)
        grads = []
        for _ in range(2):
            dt = torch.zeros(geom.n_params, device=DEV)
            _bwd_table(desc.c, x, buf[:m], dt, n)
            grads.append(dt)
        want = _table_grad_fp64(x.cpu(), dy.cpu(), desc, geom)
        assert torch.isfinite(grads[0]).all(), n
        assert rel_err(grads[0], want) < 2e-5, n
        assert torch.equal(grads[0] == 0, want == 0), n
        assert rel_err(grads[1], grads[0].double()) < 1e-6, n       # launches differ only in atomic order


@pytest.mark.parametrize("name", ["3d_f4_even", "4d_f4_odd", "3d_f1_odd", "static_cfg"])
def test_graph_replay_with_changing_inputs(name):
    n = 64 * 1023 + 1
    _, desc, geom, x, table, dy = _inputs(name, n, seed=11)
    y = torch.empty(n, geom.n_output_dims, device=DEV)
    dt = torch.zeros(geom.n_params, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                       # warm-up launch outside the capture
        _fwd(desc.c, x, table, y, n)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _fwd(desc.c, x, table, y, n)
        _bwd_table(desc.c, x, dy, dt, n)
    for seed in (12, 13):
        _, _, _, x2, table2, dy2 = _inputs(name, n, seed=seed)
        x.copy_(x2)
        table.copy_(table2)
        dy.copy_(dy2)
        dt.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, _level_at_a_time(desc, x2, table2)), seed
        want = _table_grad_fp64(x2.cpu(), dy2.cpu(), desc, geom)
        assert rel_err(dt, want) < 2e-5, seed

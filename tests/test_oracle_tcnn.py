"""Hash-grid restatement: level tables (SURVEY.md §8a) and structural properties."""
import torch

from oracle import hotpath, tcnn_ref

TABLE = {  # name: (D, HashEncoder args, entries, resolutions of first/last level, n dense levels)
    "static": (3, (10, 16, 8192, 20, 4), 7_639_040, (16, 8192), 3),
    "dynamic": (4, (10, 32, 8192, 18, 4), 2_621_440, (32, 8192), 0),
    "flow": (4, (10, 16, 4096, 18, 4), 2_424_832, (16, 4096), 1),
    "prop0": (3, (8, 16, 512, 20, 1), 4_661_184, (16, 512), 4),
    "prop1": (3, (8, 16, 2048, 20, 1), 5_541_888, (16, 2048), 3),
}


def test_level_tables_match_survey():
    for name, (D, args, entries, (r0, r1), n_dense) in TABLE.items():
        g = tcnn_ref.grid_geometry(D, hotpath.hash_encoder_config(*args))
        assert g.offsets[-1] == entries, name
        assert (g.resolutions[0], g.resolutions[-1]) == (r0, r1), name
        assert sum(not h for h in g.hashed) == n_dense, name
        assert all(o % 8 == 0 for o in g.offsets), name


def test_weights_partition_of_unity_and_linear_reproduction():
    cfg = hotpath.hash_encoder_config(3, 4, 16, 12, 2)   # all levels dense (res<=16^3<=4096)
    g = tcnn_ref.grid_geometry(3, cfg)
    assert not any(g.hashed)
    x = torch.rand(257, 3) * 0.7 + 0.05      # keep cell+1 < res at level 0 (no dense wrap-around)
    for lvl in range(g.n_levels):
        idx, w, frac, cell = tcnn_ref.corner_indices_and_weights(x, g, lvl)
        assert torch.allclose(w.sum(-1), torch.ones(257), atol=1e-6)
        assert (idx >= g.offsets[lvl]).all() and (idx < g.offsets[lvl + 1]).all()
    # a table that stores an affine function of the vertex coordinate is reproduced exactly
    lvl = 0
    res, scale = g.resolutions[0], g.scales[0]
    params = torch.zeros(g.n_params)
    table = params.view(-1, 2)
    ii = torch.arange(res)
    vx, vy, vz = torch.meshgrid(ii, ii, ii, indexing="ij")
    lin = (vx + 2 * vy + 3 * vz).float()
    flat_idx = (vx + vy * res + vz * res * res).reshape(-1)
    table[g.offsets[0] + flat_idx, 0] = lin.reshape(-1)
    y = tcnn_ref.grid_forward(x, params, g)[:, 0]
    pos = x * scale + 0.5
    want = pos[:, 0] + 2 * pos[:, 1] + 3 * pos[:, 2]
    assert torch.allclose(y, want, atol=2e-4)


def test_input_gradient_is_scale_times_finite_difference():
    cfg = hotpath.hash_encoder_config(2, 8, 16, 10, 4)
    g = tcnn_ref.grid_geometry(4, cfg)
    params = torch.randn(g.n_params, dtype=torch.float32)
    x = (torch.rand(33, 4) * 0.8 + 0.1).requires_grad_(True)
    y = tcnn_ref.grid_forward(x, params, g)
    (gx,) = torch.autograd.grad(y.sum(), x)
    eps = 1e-4
    for d in range(4):
        xp = x.detach().clone(); xp[:, d] += eps
        xm = x.detach().clone(); xm[:, d] -= eps
        fd = (tcnn_ref.grid_forward(xp, params, g).sum(-1) - tcnn_ref.grid_forward(xm, params, g).sum(-1)) / (2 * eps)
        ok = (fd - gx[:, d]).abs() < 5e-2 * gx[:, d].abs().clamp_min(1.0)
        assert ok.float().mean() > 0.9     # cells crossed by the +-eps stencil are the exceptions


def test_fp64_grid_gradients_match_autograd():
    """grid_input_grad64 / grid_table_grad64, the float64 references of the GPU input-gradient tests, against float64
    autograd of the interpolation at the same cells and fractions, on a dense + hashed 4-D grid, a 3-D F = 1 grid and
    the dynamic grid; levels with a zero upstream gradient included."""
    for D, args in ((4, (3, 4, 24, 9, 2)), (3, (4, 16, 96, 12, 1)), (4, (10, 32, 8192, 18, 4))):
        geom = tcnn_ref.grid_geometry(D, hotpath.hash_encoder_config(*args))
        L, F = geom.n_levels, geom.n_feat
        gen = torch.Generator().manual_seed(D * 100 + L)
        x = torch.rand(500, D, generator=gen)
        x[:50] = x[:50].round()
        params = torch.randn(geom.n_params, generator=gen)
        dy = torch.randn(500, L * F, generator=gen)
        dy[::3, :F] = 0.0
        dx, mag = tcnn_ref.grid_input_grad64(x, params, dy, geom)
        tab, tmag, count = tcnn_ref.grid_table_grad64(x, dy, geom)

        table = params.double().view(-1, F).requires_grad_(True)
        dyl = dy.double().view(500, L, F)
        loss, fracs = 0.0, []
        for lvl in range(L):
            idx, _, frac, _ = tcnn_ref.corner_indices_and_weights(x, geom, lvl)
            fr = frac.double().requires_grad_(True)
            fracs.append(fr)
            for c in range(1 << D):
                w = torch.ones_like(fr[:, 0])
                for d in range(D):
                    w = w * (fr[:, d] if (c >> d) & 1 else 1.0 - fr[:, d])
                loss = loss + (w[:, None] * table[idx[:, c]] * dyl[:, lvl]).sum()
        g_table, *g_frac = torch.autograd.grad(loss, [table] + fracs)
        want = sum(geom.scales[lvl] * g for lvl, g in enumerate(g_frac))
        assert (dx - want).abs().max() <= 1e-12 * want.abs().max()
        assert (mag >= dx.abs()).all() and (mag > 0).all()
        # the table reference weights with the kernels' fp32 corner weights: 2^-24 relative of the products
        assert (tab - g_table.view(-1)).abs().max() <= 1e-6 * g_table.abs().max()
        assert (tmag >= tab.abs()).all()
        live = sum(int((dyl[:, lvl] != 0).any(-1).sum()) for lvl in range(L))
        assert count.sum() == live * (1 << D) * F

"""The voxel-lifting kernels (csrc/voxels.cu) and emernerf_b200.voxels on the H100.

* emer_voxel_mark against a torch restatement of the reference's formula on the same device, bit for bit, from 1 to
  2^21 + 5 rays, with strided rows, NaN and +-inf, q exactly an integer, exactly res and in (-1, 0), depth exactly 80;
* emer_voxel_compact against ``min + nonzero(grid) * voxel_size``, bit for bit, several grids per launch, an empty and a
  full one;
* emer_voxel_select: the same kept rows as torch's ``stack(d).mean(0) > thr`` at exact thresholds and with NaN, colours
  within 1e-6 of torch's formula (``max == min`` included), bit-identical repeats;
* visualize_voxels end to end against the reference's golden (the checks of test_voxels_cpu.py), and its host syncs:
  none in the marking loop, and as many for 2 images as for 8.
"""
import warnings

import numpy as np
import pytest
import torch

import voxel_cases as vc
from test_voxels_cpu import GOLDEN, check_case, dropin_models, golden_pca

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


@pytest.fixture(scope="module")
def voxels():
    from emernerf_b200 import voxels

    return voxels


def restated_marks(o, d, t, lo, vs, res, depth_test):
    """The reference's marking in torch on the device: linear indices of the marked voxels."""
    p = o + d * t[:, None]
    q = (p - lo) / vs
    ok = ((q > -1) & (q.double() < res.double())).all(-1)
    if depth_test:
        ok &= t < 80
    ql = q[ok].long()
    return torch.unique((ql[:, 0] * res[1] + ql[:, 1]) * res[2] + ql[:, 2])


def bits_of(lin, words):
    want = torch.zeros(words * 32, dtype=torch.bool, device=DEV)
    want[lin] = True
    return want


def grid_bits(g):
    b = g.bits.view(torch.uint8).cpu().numpy()
    return torch.from_numpy(np.unpackbits(b, bitorder="little").astype(bool)).to(DEV)


def ray_case(n, seed, lo, vs, res):
    g = torch.Generator(device=DEV).manual_seed(seed)
    base = torch.rand(n, 6, generator=g, device=DEV)           # rows of 6: the origins are a strided view
    ext = vs * res.float()
    base[:, :3] = lo - 0.3 * ext + base[:, :3] * 1.6 * ext
    o = base[:, :3]
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g, device=DEV), dim=-1)
    t = torch.rand(n, generator=g, device=DEV) * 100
    k = min(n, 12)
    if k >= 12:
        # exact cases: p = o (d * 0 = 0) at chosen q
        t[:k] = 0.0
        q = torch.tensor([[0.0, 1.0, 2.0], [-0.5, 0.25, 0.5], [res[0].item(), 1.0, 1.0], [-1.0, 1, 1],
                          [res[0].item() - 1e-3, 0, 0], [float("nan"), 1, 1], [float("inf"), 1, 1],
                          [1, float("-inf"), 1], [3.0, 4.0, 5.0], [-0.999, -0.001, 0.0], [2, 2, 2], [1, 1, 1]],
                         device=DEV)
        o[:k] = lo + q * vs
        t[10:12] = 80.0
        t[11] = torch.nextafter(torch.tensor(80.0), torch.tensor(0.0)).item()
        d[9] = float("nan")
    return o, d, t


@pytest.mark.parametrize("n", [1, 13, 1000, 2 ** 21 + 5])
def test_mark_is_the_reference_formula(voxels, n):
    lo = torch.tensor([-20.0, -41.0, -1.0], device=DEV)
    res = torch.tensor([51, 41, 11], device=DEV)
    vs = torch.tensor([101.0, 82.0, 22.0], device=DEV) / res
    vs_d = torch.tensor([101.0, 82.0, 22.0], device=DEV) / torch.tensor([41, 33, 9], device=DEV)
    res_d = torch.tensor([41, 33, 9], device=DEV)
    o, d, t = ray_case(n, n, lo, vs, res)
    td = torch.rand(n, 2, device=DEV)[:, 1] * 120                # a strided depth column
    s = voxels.BitGrid(lo.tolist(), vs.tolist(), res.tolist(), DEV)
    dy = voxels.BitGrid(lo.tolist(), vs_d.tolist(), res_d.tolist(), DEV)
    voxels.mark(s, o, d, t[:, None], dy, td[:, None])
    torch.cuda.synchronize()
    assert torch.equal(grid_bits(s), bits_of(restated_marks(o, d, t, lo, vs, res, True), s.words))
    assert torch.equal(grid_bits(dy), bits_of(restated_marks(o, d, td, lo, vs_d, res_d, False), dy.words))


def test_compact_is_nonzero(voxels):
    shapes = [(7, 5, 3), (33, 17, 65), (1, 1, 1), (4, 4, 4), (64, 64, 64)]
    grids, dense = [], []
    g = torch.Generator(device=DEV).manual_seed(3)
    for k, res in enumerate(shapes):
        lo = [-1.5 * k, 2.0, -0.25]
        vs = (torch.tensor([3.7, 1.1, 0.3]) / torch.tensor(res)).tolist()
        bg = voxels.BitGrid(lo, vs, list(res), DEV)
        n = res[0] * res[1] * res[2]
        occ = torch.rand(n, generator=g, device=DEV) < [0.3, 0.01, 0.0, 1.0, 0.05][k]     # grid 2 empty, 3 full
        w = torch.zeros(bg.words * 32, dtype=torch.bool, device=DEV)
        w[:n] = occ
        packed = np.packbits(w.cpu().numpy(), bitorder="little").view(np.int32)
        bg.bits.copy_(torch.from_numpy(packed))
        grids.append(bg)
        dense.append((torch.tensor(lo, device=DEV), torch.tensor(vs, device=DEV), occ.view(*res)))
    coords, counts = voxels.compact(grids)
    row = 0
    for (lo, vs, occ), c in zip(dense, counts):
        want = lo + torch.nonzero(occ) * vs
        assert c == want.shape[0]
        assert torch.equal(coords[row:row + c], want)
        row += c
    again, _ = voxels.compact(grids)
    assert torch.equal(coords, again)


def select_case(n, k, c, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    d = [torch.rand(n, generator=g, device=DEV) for _ in range(k)]
    thr = 0.5
    # rows whose mean lands exactly on, just above and just below the threshold, and NaN
    for j in range(min(n, 16)):
        d[0][j] = thr
        for col in d[1:]:
            col[j] = thr
    if n > 20:
        d[0][16] = float("nan")
        d[-1][17] = torch.nextafter(torch.tensor(thr), torch.tensor(1.0)).item()
        d[0][18] = 1.0 / 3
    feat = torch.randn(n, c + 4, generator=g, device=DEV)[:, :c] / 4       # strided rows
    m = torch.randn(c, 3, generator=g, device=DEV) / c ** 0.5
    pts = torch.randn(n, 3, generator=g, device=DEV)
    return d, thr, feat, m, pts


@pytest.mark.parametrize("n,k,c", [(1, 1, 4), (5000, 3, 64), (2 ** 18, 3, 64), (2 ** 18 + 77, 2, 128),
                                   (100003, 1, 256)])
def test_select_is_torch(voxels, n, k, c):
    d, thr, feat, m, pts = select_case(n, k, c, n + k)
    lo, hi = torch.tensor([-1.0, -0.5, 0.2], device=DEV), torch.tensor([1.0, 0.5, 0.2], device=DEV)   # hi == lo
    out_p = torch.full((n + 5, 3), -7.0, device=DEV)
    out_c = torch.full((n + 5, 3), -7.0, device=DEV)
    count = torch.full((1,), 5, dtype=torch.int64, device=DEV)                   # appends behind 5 rows
    voxels.select(d, thr, pts, feat, m, lo, hi, out_p, out_c, count)
    keep = torch.stack(d, 0).mean(0) > thr
    kept = int(keep.sum())
    assert int(count) == 5 + kept
    assert torch.equal(out_p[5:5 + kept], pts[keep])
    want = torch.clamp((feat[keep].double() @ m.double()).float().sub(lo).div(hi - lo), 0, 1)
    got = out_c[5:5 + kept]
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    ok = ~torch.isnan(want)
    assert (got[ok] - want[ok]).abs().max().item() <= 1e-6 if kept else True
    torch_colors = torch.clamp((feat[keep] @ m - lo) / (hi - lo), 0, 1)
    assert ((got[ok] - torch_colors[ok]).abs().max().item() <= 1e-5) if kept else True
    p2, c2 = out_p.clone(), out_c.clone()
    count.fill_(5)
    voxels.select(d, thr, pts, feat, m, lo, hi, out_p, out_c, count)
    assert torch.equal(out_p, p2) and torch.equal(out_c.view(torch.int32), c2.view(torch.int32))


def dataset_on_device(case, n=None):
    ds = vc.dataset(case, DEV)
    if n is not None:
        ds.full_pixel_set = vc._Items(list.__getitem__(ds.full_pixel_set, slice(0, n)))
    return ds


@pytest.mark.parametrize("case", list(vc.CASES))
def test_against_reference_golden(voxels, monkeypatch, case):
    z = np.load(GOLDEN)
    field, props, est = dropin_models(z, case, DEV)
    monkeypatch.setattr(voxels, "robust_pca", lambda features, m=2.5: golden_pca(z, case, features.device))
    got = voxels.visualize_voxels(vc.render_cfg(), field, est, props, dataset_on_device(case), device="cuda",
                                  is_dynamic=vc.CASES[case]["dynamic"])
    check_case(z, case, got)


def test_marking_loop_does_not_sync(voxels):
    z = np.load(GOLDEN)
    field, props, est = dropin_models(z, "dynamic_3cam", DEV)
    geo = voxels.VoxelGeometry(field.aabb, vc.VOXEL_SIZE)
    ds = dataset_on_device("dynamic_3cam")
    voxels.mark_images(vc.render_cfg(), field, est, props, ds, geo, True)      # warm-up: workspaces, first launches
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        voxels.mark_images(vc.render_cfg(), field, est, props, ds, geo, True)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_syncs_do_not_grow_with_images(voxels):
    z = np.load(GOLDEN)
    field, props, est = dropin_models(z, "static_1cam", DEV)

    def syncs(n):
        ds = dataset_on_device("static_1cam", n)
        voxels.visualize_voxels(vc.render_cfg(), field, est, props, ds)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                voxels.visualize_voxels(vc.render_cfg(), field, est, props, ds)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        return sum("synchroniz" in str(x.message) for x in w)

    assert syncs(2) == syncs(8)

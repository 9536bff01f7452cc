"""The lidar scene-flow evaluation on the GPU: emer_lidar_flow_accumulate against an fp64 torch restatement for 0 to
2^20 + 17 points, reading the prediction in place from [n, 6] rows and from dense [n, 3] rows, with and without the
ground removal, with NaN and -0 inputs and densities of exactly 0.2f and NaN; bit-identical repeats; agreement with
emer_scene_flow_metrics, bit for bit, on points that are all counted and ungated; the drop-ins against the reference's
own results (tests/golden/lidar_flow.npz) with the bars of the CPU suite; no host sync once the frame table exists and
one per call; and, on the benchmark drive and field (tools/bench_lidar_flow.py), the result against the oracle."""
import math
import os
import sys
import warnings

import numpy as np
import pytest
import torch

import lidar_flow_cases as lc
from oracle import lidar_flow_ref
from test_lidar_flow_cpu import check_against_golden, dropin_field

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import bench_lidar_flow  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lidar_flow.npz")
SIZES = [0, 1, 255, (1 << 20) + 17]


def make_inputs(n, ld, seed=0):
    g = torch.Generator().manual_seed(seed)
    wide = torch.randn(n, ld, generator=g) * 0.3
    pred = wide[:, :3]
    pred[5::17] = -pred[5::17].abs()                  # negative flows, gated to -0 where the density is low
    pred[7::29, 1] = float("nan")
    labels = pred + torch.randn(n, 3, generator=g) * torch.rand(n, 1, generator=g) * 0.3
    labels[3::13] = 0.0                               # no motion: not in the angle mean
    labels[4::31] = -0.0
    labels[11::37, 2] = float("nan")
    density = torch.rand(n, generator=g) * 0.4
    density[::9] = 0.2                                # exactly 0.2f: kept
    density[2::23] = float("nan")                     # kept
    classes = torch.randint(0, 4, (n,), generator=g)
    classes[torch.rand(n, generator=g) < 0.2] = -1
    ground = torch.rand(n, generator=g) < 0.3
    return wide, pred, density, labels, classes, ground


def ref_sums(pred, density, labels, classes, ground):
    """The kernel's row in fp64: oracle.metrics_ref's formulas over the counted points."""
    valid = classes != -1
    counted = valid & ~ground if ground is not None else valid
    p = pred.clone()
    p[density < 0.2] *= 0                             # fp32, as the reference
    p, lab = p[counted].double(), labels[counted].double()
    l2 = (p - lab).pow(2).sum(-1).sqrt()
    ln = lab.pow(2).sum(-1).sqrt()
    rel = l2 / (ln + 1e-20)
    moving = ln > 0.1
    dot = ((lab / (ln[:, None] + 1e-7)) * (p / (p.pow(2).sum(-1).sqrt()[:, None] + 1e-7))).sum(-1)[moving]
    dot_max = float(np.float32(1 - 1e-7))
    dot = torch.where(dot != dot, torch.zeros_like(dot), dot.clamp(-dot_max, dot_max))
    return torch.tensor([l2.sum(), ((l2 < 0.05) | (rel < 0.05)).sum(), ((l2 < 0.1) | (rel < 0.1)).sum(),
                         ((l2 > 0.3) | (rel > 0.1)).sum(), torch.acos(dot).sum(), moving.sum(), counted.sum(),
                         valid.sum()], dtype=torch.float64)


def launch(wide, ld, density, labels, classes, ground, sums):
    from emernerf_b200 import _lib, _ops, metrics

    n = labels.shape[0]
    ws = _ops._workspace(metrics._WS, wide.device, metrics.WORKSPACE_BYTES, "metrics")
    g = None if ground is None else ground.contiguous().view(torch.uint8)
    _ops._need_cuda(wide, density, labels, classes, g, sums)
    _lib.call("emer_lidar_flow_accumulate", _ops._ptr(wide), ld, _ops._ptr(density), _ops._ptr(labels),
              _ops._ptr(classes), _ops._ptr(g), n, 0.2, _ops._ptr(sums), _ops._ptr(ws), _ops._stream())


@pytest.mark.parametrize("with_ground", [False, True], ids=["keep_ground", "remove_ground"])
@pytest.mark.parametrize("ld", [3, 6])
@pytest.mark.parametrize("n", SIZES)
def test_kernel_matches_fp64(n, ld, with_ground):
    wide, pred, density, labels, classes, ground = make_inputs(n, ld, seed=n + ld)
    ground = ground if with_ground else None
    sums = torch.full((8,), 0.5, dtype=torch.float64, device=DEV)            # the kernel ADDS
    launch(wide.to(DEV), ld, density.to(DEV), labels.to(DEV), classes.to(DEV),
           None if ground is None else ground.to(DEV), sums)
    got = sums.cpu() - 0.5
    want = ref_sums(pred, density, labels, classes, ground)
    idx = [1, 2, 3, 5, 6, 7]
    assert torch.equal(got[idx], want[idx]), (got, want)
    for k in (0, 4):                                  # NaN labels make the EPE sum NaN; the angle sum stays finite
        if math.isnan(want[k]):
            assert math.isnan(got[k])
        else:
            assert abs(got[k] - want[k]) <= 1e-12 * max(1.0, abs(want[k])), (k, got[k], want[k])
    if n > 255:                                       # every kind of input is present
        assert math.isnan(want[0]) and want[4] > 0 and 0 < want[6] <= want[7] <= n
        assert (want[6] < want[7]) == with_ground


def test_bit_identical_repeats():
    n = (1 << 20) + 17
    wide, _, density, labels, classes, ground = (t.to(DEV) for t in make_inputs(n, 6, seed=3))
    wide, labels = torch.nan_to_num(wide), torch.nan_to_num(labels)
    rows = [torch.zeros(8, dtype=torch.float64, device=DEV) for _ in range(3)]
    for r in rows:
        launch(wide, 6, density, labels, classes, ground, r)
    assert not rows[0].isnan().any()
    assert all(torch.equal(rows[0].view(torch.int64), r.view(torch.int64)) for r in rows[1:])


@pytest.mark.parametrize("n", [255, (1 << 20) + 17])
def test_same_terms_as_scene_flow_metrics(n):
    """On points that are all counted and ungated, the row is emer_scene_flow_metrics' sums bit for bit: both kernels
    call the same per-point code and reduce in the same order."""
    from emernerf_b200 import metrics

    g = torch.Generator(device=DEV).manual_seed(n)
    pred = torch.randn(n, 3, generator=g, device=DEV) * 0.3
    labels = pred + torch.randn(n, 3, generator=g, device=DEV) * 0.1
    sums = torch.zeros(8, dtype=torch.float64, device=DEV)
    launch(pred, 3, torch.ones(n, device=DEV), labels, torch.zeros(n, dtype=torch.int64, device=DEV), None, sums)
    out = metrics._pair_launch("emer_scene_flow_metrics", pred[None], labels[None], 7).cpu()
    s = sums.cpu()
    assert s[6].item() == n and s[5].item() == out[5].item()
    assert torch.equal(s[:4] / n, out[:4]) and torch.equal(s[4:5] / s[5:6], out[4:5])


@pytest.mark.parametrize("case", list(lc.CASES))
def test_against_reference_golden(case):
    from emernerf_b200 import metrics

    z = np.load(GOLDEN)
    check_against_golden(metrics, z, case, dropin_field(z).to(DEV), device=DEV)


def test_one_sync_per_call_and_none_once_the_table_exists():
    from emernerf_b200 import metrics

    z = np.load(GOLDEN)
    field = dropin_field(z).to(DEV)
    lidar_set = lc.SplitSet(lc.load(z, "unsorted", device=DEV), range(lc.N_SCANS))
    metrics.eval_lidar_flow(lidar_set, field)        # warm-up: the frame table, workspaces, modules
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        metrics._lidar_flow_sums(lidar_set, field, True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            metrics.eval_lidar_flow(lidar_set, field)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert sum("synchroniz" in str(w.message) for w in caught) == 1


def test_bound_sampler_is_used():
    """A source whose get_render_rays is bound to a LidarRaySampler is served from that sampler's table."""
    from emernerf_b200 import metrics
    from emernerf_b200.raygen import LidarRaySampler

    z = np.load(GOLDEN)
    src = lc.load(z, "drive", device=DEV)
    sampler = LidarRaySampler(src)
    src.get_render_rays = sampler.get_render_rays
    lidar_set = lc.SplitSet(src, lc.CASES["drive"][2])
    got = metrics.eval_lidar_flow(lidar_set, dropin_field(z).to(DEV))
    assert sampler._frames is not None
    want = z["drive/result"]
    assert all(abs(got[k] - w) <= 1e-6 * abs(w) for k, w in zip(lidar_flow_ref.KEYS, want))


def test_bench_drive_against_oracle():
    """The benchmark's drive and field: the fp64 sums against the reference's fp32 formulation.  Points that flip at a
    threshold between fp32 and fp64 are the only difference allowed: 1e-5 relative on the EPE and the angle, 1e-4
    absolute on the fractions."""
    from emernerf_b200 import metrics

    field = bench_lidar_flow.flow_field()
    drive = bench_lidar_flow.Split(bench_lidar_flow.SyntheticDrive(200, 100_000), range(200))
    want = lidar_flow_ref.eval_lidar_flow(drive, field, True)
    got = metrics.eval_lidar_flow(drive, field, True)
    assert list(got) == list(want)
    for k in ("EPE3D", "angle_error"):
        assert abs(got[k] - want[k]) <= 1e-5 * abs(want[k]), (k, got[k], want[k])
    for k in ("acc3d_strict", "acc3d_relax", "outlier"):
        assert abs(got[k] - want[k]) <= 1e-4, (k, got[k], want[k])

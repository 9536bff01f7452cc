"""The few-shot occupancy evaluation on the GPU: emer_occ_accumulate and emer_occ_classify against an fp64 torch
restatement from 1 to 1 000 003 voxels, at 4, 64 and 256 channels and 1, 15 and 32 classes, with densities of exactly
0.2 and NaN, zero feature rows, zero centroids, exact ties, labels outside the classes and strided inputs; bit-identical
repeats; the drop-ins against the reference's own results (tests/golden/occupancy.npz) with the bars of the CPU suite;
no host sync between frames and one per call; and the peak memory of collect_centroids against the frame count."""
import os
import warnings

import numpy as np
import pytest
import torch

import occ_cases as oc
from test_occupancy_cpu import check_against_golden, dropin_field

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "occupancy.npz")
SHAPES = [(1, 15, 64), (31, 15, 64), (1_000_003, 15, 64), (31, 15, 4), (1_000_003, 15, 4), (31, 15, 256),
          (1_000_003, 15, 256), (4099, 32, 64), (4099, 1, 8)]


def make_inputs(n, k, c, seed=0, ld=None):
    g = torch.Generator().manual_seed(seed)
    ld = ld or c
    wide = torch.randn(n, ld, generator=g)
    feat = wide[:, :c]
    feat[::7] = 0.0                                   # zero rows
    dens2 = torch.rand(n, 2, generator=g) * 0.4      # density is column 0: read with stride 2
    density = dens2[:, 0]
    density[::5] = 0.2                               # not measured: the filter is strict
    density[3::11] = float("nan")                    # not measured
    labels = torch.randint(0, k, (n,), generator=g)
    labels[2::13] = k                                # outside the classes
    labels[6::17] = -1
    centroids = torch.randn(k, c, generator=g)
    if k > 2:
        centroids[1] = 0.0                           # a zero centroid
        centroids[k - 1] = centroids[0]              # a duplicate of class 0: every such tie goes to 0
    return wide, feat, dens2, density, labels, centroids


def ref_accumulate(feat, density, labels, k):
    keep = (density > np.float32(0.2)) & (labels >= 0) & (labels < k)
    f, lab = feat.double()[keep], labels[keep]
    sums = torch.zeros(k, feat.shape[1], dtype=torch.float64).index_add_(0, lab, f)
    return sums, torch.bincount(lab, minlength=k)


def ref_classify(feat, density, labels, centroids, bank):
    k = centroids.shape[0]
    measured = density > np.float32(0.2)
    inside = measured & (labels >= 0) & (labels < k)
    c = centroids.double()
    chat = c / (c.norm(dim=-1, keepdim=True) + 1e-7)
    q = feat.double()[inside]
    sims = torch.stack([q @ chat[j] for j in range(k)], -1)   # per class: duplicate rows give identical columns
    pred = bank[torch.argmax(sims, dim=-1)]                   # the first maximum
    true = labels[inside]
    counts = torch.zeros(2 * k + 2, dtype=torch.int64)
    counts[:k] = torch.bincount(true, minlength=k)
    counts[k:2 * k] = torch.bincount(true[pred == true], minlength=k)
    counts[2 * k] = int(measured.sum())
    counts[2 * k + 1] = int((measured & ~inside).sum())
    return counts


def launch(metrics, name, wide, ld, c, dens2, labels, k, sums=None, counts=None, centroids=None, bank=None):
    from emernerf_b200 import _lib, _ops

    n = labels.numel()
    common = (_ops._ptr(wide), ld, c, _ops._ptr(dens2), 2, _ops._ptr(labels), n)
    ws = _ops._ptr(metrics._occ_workspace(wide.device))
    _ops._need_cuda(wide)
    if name == "emer_occ_accumulate":
        _lib.call(name, *common, k, 0.2, _ops._ptr(sums), _ops._ptr(counts), ws, _ops._stream())
    else:
        _lib.call(name, *common, _ops._ptr(centroids), k, _ops._ptr(bank), 0.2, _ops._ptr(counts), ws,
                  _ops._stream())


@pytest.mark.parametrize("shape", SHAPES, ids=[f"n{n}_k{k}_c{c}" for n, k, c in SHAPES])
def test_kernels_match_fp64(shape):
    from emernerf_b200 import metrics

    n, k, c = shape
    ld = c + 4 if c < 256 else c                     # strided rows where the width allows
    wide, feat, dens2, density, labels, centroids = make_inputs(n, k, c, seed=n + c, ld=ld)
    d_wide, d_dens2, d_labels = wide.to(DEV), dens2.to(DEV), labels.to(DEV)
    sums = torch.full((k, c), 0.5, dtype=torch.float64, device=DEV)      # the kernels ADD
    counts = torch.full((k,), 3, dtype=torch.int64, device=DEV)
    launch(metrics, "emer_occ_accumulate", d_wide, ld, c, d_dens2, d_labels, k, sums=sums, counts=counts)
    want_s, want_n = ref_accumulate(feat, density, labels, k)
    assert torch.equal(counts.cpu(), want_n + 3)
    scale = want_s.abs().amax().clamp_min(1.0)
    assert ((sums.cpu() - 0.5 - want_s).abs().max() / scale) <= 1e-12
    bank = torch.arange(k, dtype=torch.int64) * 2 % max(k, 1)              # a permuted label bank
    cc = torch.full((2 * k + 2,), 1, dtype=torch.int64, device=DEV)
    launch(metrics, "emer_occ_classify", d_wide, ld, c, d_dens2, d_labels, k, counts=cc,
           centroids=centroids.to(DEV), bank=bank.to(DEV))
    assert torch.equal(cc.cpu(), ref_classify(feat, density, labels, centroids, bank) + 1)


def test_bit_identical_repeats():
    from emernerf_b200 import metrics

    n, k, c = 1_000_003, 15, 64
    wide, _, dens2, _, labels, centroids = (t.to(DEV) for t in make_inputs(n, k, c, seed=5))
    bank = torch.arange(k, device=DEV)
    first = None
    for _ in range(3):
        sums = torch.zeros(k, c, dtype=torch.float64, device=DEV)
        counts = torch.zeros(k, dtype=torch.int64, device=DEV)
        cc = torch.zeros(2 * k + 2, dtype=torch.int64, device=DEV)
        launch(metrics, "emer_occ_accumulate", wide, c, c, dens2, labels, k, sums=sums, counts=counts)
        launch(metrics, "emer_occ_classify", wide, c, c, dens2, labels, k, counts=cc, centroids=centroids, bank=bank)
        if first is None:
            first = (sums, counts, cc)
        else:
            assert all(torch.equal(a, b) for a, b in zip(first, (sums, counts, cc)))


@pytest.mark.parametrize("model", oc.MODELS)
def test_against_reference_golden(model):
    from emernerf_b200 import metrics

    z = np.load(GOLDEN)
    field = dropin_field(z, model).to(DEV)
    dataset = oc.OccDataset(oc.load_frames(z, model), device=DEV)
    check_against_golden(metrics, z, model, field, dataset, torch.device(DEV))


class SeededFrames:
    """Frames of ``n`` seeded voxels generated on the device at each get_occ (nothing held between frames)."""

    def __init__(self, n):
        self.n = n
        self.label_mapping = dict(oc.LABEL_MAPPING)

    def get_occ(self, index):
        g = torch.Generator(device=DEV).manual_seed(index)
        u = torch.rand(self.n, 3, generator=g, device=DEV)
        coords = torch.stack([u[:, 0] * 40.0, u[:, 1] * 40.0 - 20.0, u[:, 2] * 6.0], -1)
        labels = torch.randint(0, oc.N_CLASSES, (self.n,), generator=g, device=DEV)
        return coords, labels, torch.full((self.n,), index / 9.0, device=DEV)


def _field():
    z = np.load(GOLDEN)
    return dropin_field(z, "flow_feat").to(DEV)


def test_no_host_sync_between_frames_and_one_per_call():
    from emernerf_b200 import metrics

    field, ds = _field(), SeededFrames(50_000)
    centroids, bank = metrics.collect_centroids([0], ds, field, DEV)      # warm-up: workspaces, modules
    metrics.eval_few_shot_occ([1], ds, field, DEV, centroids, bank)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        centroids, bank = metrics.collect_centroids([0, 2, 3], ds, field, DEV)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            got = metrics.eval_few_shot_occ([1, 4, 5, 6], ds, field, DEV, centroids, bank)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert sum("synchroniz" in str(w.message) for w in caught) == 1
    assert got["num_total_points"] == 200_000


def test_collect_centroids_memory_does_not_grow_with_frames():
    from emernerf_b200 import metrics

    field, ds = _field(), SeededFrames(300_000)
    metrics.collect_centroids([0], ds, field, DEV)
    peaks = []
    for frames in (2, 8):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        c, _ = metrics.collect_centroids(list(range(frames)), ds, field, DEV)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
        del c
    # one frame's kept features alone are ~38 MB (150 000 rows x 256 B): a concatenation over frames would add six
    # of them; the allocator's block rounding moves the peak by about 1 MB
    assert peaks[1] <= peaks[0] + (16 << 20), peaks

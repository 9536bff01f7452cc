"""emernerf_b200.metrics on the GPU: image_metrics against the fp64 oracle (oracle/metrics_ref.py) from the smallest
image the SSIM window allows to a full 640 x 960 evaluation image, with empty, sparse and full masks and 64-channel
features; against the reference's float32 SSIM path; identical, constant and NaN images; bit-identical repeats; no host
sync; CUDA-graph capture and replay; one library launch per image; and the PSNR, depth-RMSE and scene-flow functions
against the reference's goldens and the fp64 oracle, up to a lidar-frame-sized flow evaluation."""
import math
import os

import numpy as np
import pytest
import torch

import metric_cases as mc
from oracle import metrics_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz")
SSIM_ABS = 1e-7              # against the fp64 oracle
PSNR_DB = 1e-6
REL = 1e-6
SSIM_FP32 = 1e-5             # against the reference's float32 path
PSNR_FP32_DB = 1e-4
ANGLE_FP32_REL = 1e-4        # the reference's angles carry fp32 unit vectors (see test_metrics_cpu.py)
SIZES = [(7, 7), (7, 1001), (37, 53), (160, 240), (640, 960)]
MASKS = ["empty", "sparse", "full"]


def make_case(h, w, seed, mask_kind="sparse", cf=64, noise=0.05):
    g = torch.Generator().manual_seed(seed)
    y = torch.rand(h, w, 3, generator=g)
    x = (y + noise * torch.randn(h, w, 3, generator=g)).clamp(0, 1)
    m = {"empty": torch.zeros(h, w), "full": torch.ones(h, w),
         "sparse": (torch.rand(h, w, generator=g) < 0.05).float()}[mask_kind]
    fy = torch.randn(h, w, cf, generator=g)
    fx = fy + 0.1 * torch.randn(h, w, cf, generator=g)
    return x, y, m, fx, fy


def check_close(got, want, what):
    for k, v in got.items():
        g, w = float(v), want[k]
        if math.isnan(w) or math.isinf(w):
            assert (math.isnan(g) and math.isnan(w)) or g == w, (what, k, g, w)
            continue
        tol = {"ssim": SSIM_ABS, "masked_ssim": SSIM_ABS, "mask_count": 0.0}.get(k, PSNR_DB)
        assert abs(g - w) <= tol, (what, k, g, w, abs(g - w))


@pytest.mark.parametrize("size", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_image_metrics_match_fp64_oracle(size):
    from emernerf_b200 import metrics

    h, w = size
    for i, kind in enumerate(MASKS):
        x, y, m, fx, fy = make_case(h, w, seed=10 * h + i, mask_kind=kind)
        got = metrics.image_metrics(x.to(DEV), y.to(DEV), m.to(DEV), fx.to(DEV), fy.to(DEV))
        want = metrics_ref.image_metrics(x.numpy(), y.numpy(), m.numpy(), fx.numpy(), fy.numpy())
        check_close(got, want, f"{h}x{w} {kind}")
        assert float(got["mask_count"]) == float(m.sum())


@pytest.mark.parametrize("size", [(37, 53), (160, 240)], ids=["37x53", "160x240"])
def test_image_metrics_match_reference_fp32_path(size):
    from emernerf_b200 import metrics

    x, y, m, _, _ = make_case(*size, seed=3)
    got = metrics.image_metrics(x.to(DEV), y.to(DEV), m.to(DEV))
    want = metrics_ref.image_metrics(x.numpy(), y.numpy(), m.numpy(), mode="fp32")
    for k in ("ssim", "masked_ssim"):
        assert abs(float(got[k]) - want[k]) <= SSIM_FP32, k
    for k in ("psnr", "masked_psnr"):
        assert abs(float(got[k]) - want[k]) <= PSNR_FP32_DB, k


def test_strided_features_and_channel_counts():
    from emernerf_b200 import metrics

    for c in (1, 2, 4):
        g = torch.Generator().manual_seed(c)
        y = torch.rand(33, 41, c, generator=g)
        x = (y + 0.1 * torch.randn(33, 41, c, generator=g)).clamp(0, 1)
        m = (torch.rand(33, 41, generator=g) < 0.2).float()
        wide = torch.randn(33, 41, 300, generator=g)
        fx, fy = wide[..., 10:266], wide[..., 40:296]          # 256 channels, row stride 300
        got = metrics.image_metrics(x.to(DEV), y.to(DEV), m.to(DEV), fx.to(DEV), fy.to(DEV))
        check_close(got, metrics_ref.image_metrics(x, y, m, fx, fy), f"C={c}")


def test_identical_constant_and_nan_images():
    from emernerf_b200 import metrics

    x, _, m, _, _ = make_case(37, 53, seed=5)
    got = metrics.image_metrics(x.to(DEV), x.to(DEV), m.to(DEV), x.to(DEV), x.to(DEV))
    assert float(got["ssim"]) == 1.0 and float(got["masked_ssim"]) == 1.0
    for k in ("psnr", "masked_psnr", "feat_psnr", "masked_feat_psnr"):
        assert float(got[k]) == math.inf, k
    a, b = torch.full((20, 30, 3), 0.25), torch.full((20, 30, 3), 0.75)     # zero variance everywhere
    got = metrics.image_metrics(a.to(DEV), b.to(DEV), m[:20, :30].to(DEV))
    check_close(got, metrics_ref.image_metrics(a, b, m[:20, :30]), "constant")
    bad = x.clone()
    bad[17, 20, 1] = float("nan")
    got = metrics.image_metrics(bad.to(DEV), x.to(DEV), m.to(DEV))
    assert math.isnan(float(got["psnr"])) and math.isnan(float(got["ssim"]))
    with pytest.raises(AssertionError, match="prediction must be"):
        metrics.compute_ssim(bad.to(DEV), x.to(DEV))


def test_bit_identical_repeats_and_one_launch():
    from emernerf_b200 import _lib, metrics

    x, y, m, fx, fy = (t.to(DEV) for t in make_case(640, 960, seed=6))
    first = metrics.image_metrics(x, y, m, fx, fy)
    n0 = _lib.LAUNCHES
    for _ in range(3):
        again = metrics.image_metrics(x, y, m, fx, fy)
        for k in first:
            assert torch.equal(first[k], again[k]) or (first[k].isnan() and again[k].isnan()), k
    assert _lib.LAUNCHES - n0 == 3


def test_no_host_sync():
    from emernerf_b200 import metrics

    x, y, m, fx, fy = (t.to(DEV) for t in make_case(160, 240, seed=7))
    metrics.image_metrics(x, y, m, fx, fy)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        per = [metrics.image_metrics(x, y, m, fx, fy) for _ in range(3)]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert metrics.summarize(per)["psnr"] > 0


def test_cuda_graph_capture_and_replay():
    from emernerf_b200 import metrics

    x, y, m, fx, fy = (t.to(DEV) for t in make_case(160, 240, seed=8))
    metrics.image_metrics(x, y, m, fx, fy)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = metrics.image_metrics(x, y, m, fx, fy)
    for seed in (9, 10):
        nx, ny, nm, nfx, nfy = (t.to(DEV) for t in make_case(160, 240, seed=seed))
        for dst, src in ((x, nx), (y, ny), (m, nm), (fx, nfx), (fy, nfy)):
            dst.copy_(src)
        graph.replay()
        eager = metrics.image_metrics(nx, ny, nm, nfx, nfy)
        torch.cuda.synchronize()
        for k in eager:
            assert torch.equal(captured[k], eager[k]) or (captured[k].isnan() and eager[k].isnan()), k


@pytest.mark.parametrize("case", [c[0] for c in mc.CASES])
def test_against_reference_goldens(case):
    from emernerf_b200 import metrics

    gold = np.load(GOLDEN)
    _, fn, keys = next(c for c in mc.CASES if c[0] == case)
    x = mc.make_inputs()
    got = getattr(metrics, fn)(*(x[k].to(DEV) for k in keys))
    if fn == "compute_scene_flow_metrics":
        n = x[keys[0]].shape[1]
        want64, counts = metrics_ref.scene_flow_metrics(x[keys[0]], x[keys[1]])
        for k in mc.FLOW_KEYS:
            want = float(gold[f"{case}/{k}"])
            if k in ("acc3d_strict", "acc3d_relax", "outlier"):
                assert round(got[k] * n) == round(want * n) == counts[k], k
                continue
            if math.isnan(want):
                assert math.isnan(got[k]) and math.isnan(want64[k])
                continue
            assert abs(got[k] - want64[k]) <= REL * abs(want64[k]), k
            assert abs(got[k] - want) <= (ANGLE_FP32_REL if k == "angle_error" else REL) * abs(want), k
    elif fn == "compute_psnr":
        want = float(gold[f"{case}/value"])
        want64 = metrics_ref.psnr(x[keys[0]], x[keys[1]])
        assert got == want == want64 or (abs(got - want64) <= PSNR_DB and abs(got - want) <= PSNR_FP32_DB)
    else:
        want = float(gold[f"{case}/value"])
        want64, _ = metrics_ref.valid_depth_rmse(x[keys[0]], x[keys[1]])
        if math.isnan(want):
            assert math.isnan(got) and math.isnan(want64)
        else:
            assert abs(got - want64) <= REL * want64 and abs(got - want) <= REL * want


def test_lidar_frame_scene_flow():
    from emernerf_b200 import metrics

    g = torch.Generator().manual_seed(11)
    labels = torch.randn(1, 150001, 3, generator=g) * 0.4
    labels[0, ::17] = 0.0
    pred = labels + torch.randn(1, 150001, 3, generator=g) * 0.05
    pred[0, ::5] = 0.0                                   # static points: the prediction is zeroed
    got = metrics.compute_scene_flow_metrics(pred.to(DEV), labels.to(DEV))
    want, counts = metrics_ref.scene_flow_metrics(pred, labels)
    for k in ("acc3d_strict", "acc3d_relax", "outlier"):
        assert round(got[k] * 150001) == counts[k], k
    for k in ("EPE3D", "angle_error"):
        assert abs(got[k] - want[k]) <= REL * abs(want[k]), k


def test_depth_rmse_and_psnr_at_training_size():
    from emernerf_b200 import metrics

    g = torch.Generator().manual_seed(12)
    t = torch.rand(8192, generator=g) * 80
    t[::3] = 0.0
    p = t + torch.randn(8192, generator=g)
    want, _ = metrics_ref.valid_depth_rmse(p, t)
    assert abs(metrics.compute_valid_depth_rmse(p.to(DEV)[:, None], t.to(DEV)) - want) <= REL * want
    rgb, pix = torch.rand(8192, 3, generator=g), torch.rand(8192, 3, generator=g)
    assert abs(metrics.compute_psnr(rgb.to(DEV), pix.to(DEV)) - metrics_ref.psnr(rgb, pix)) <= PSNR_DB
    assert abs(metrics.compute_psnr(rgb.numpy(), pix.numpy()) - metrics_ref.psnr(rgb, pix)) <= PSNR_DB

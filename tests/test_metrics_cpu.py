"""emernerf_b200.metrics on the host (CPU suite): the module runs through tests/metrics_emulator.py, the fp64 restatement
of csrc/metrics.cu's entry points, and is checked against the reference's own datasets/metrics.py (tests/golden/
metrics.npz) and against oracle.metrics_ref; the oracle's box filter against scipy's; the aggregation against the
reference's ``non_zero_mean``; the argument errors."""
import math
import os

import numpy as np
import pytest
import torch

import metric_cases as mc
import metrics_emulator
from oracle import metrics_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz")
PSNR_FP32_DB = 1e-4          # against the reference's float32 path (its own rounding)
SSIM_FP32 = 1e-5
REL = 1e-6                   # depth RMSE and flow statistics
# the reference forms each angle from fp32 unit vectors: near the clamp (parallel vectors) acos amplifies that
# rounding by 1 / sqrt(1 - dot^2), so its mean is held to the fp32 rounding it carries, not to fp64's
ANGLE_FP32_REL = 1e-4


@pytest.fixture
def metrics(monkeypatch):
    metrics_emulator.install(monkeypatch)
    from emernerf_b200 import metrics

    return metrics


def noisy_image(h, w, c=3, seed=0, noise=0.05):
    g = torch.Generator().manual_seed(seed)
    y = torch.rand(h, w, c, generator=g)
    x = (y + noise * torch.randn(h, w, c, generator=g)).clamp(0, 1)
    return x, y


def non_zero_mean(x):        # radiance_fields/video_utils.py:45-47
    return sum(x) / len(x) if len(x) > 0 else -1


def close(a, b, rel=0.0, abs_=0.0):
    if math.isnan(b) or math.isinf(b):
        return (math.isnan(a) and math.isnan(b)) or a == b
    return abs(a - b) <= max(abs_, rel * abs(b))


# ----------------------------------------------------------------------------- goldens
@pytest.mark.parametrize("case", [c[0] for c in mc.CASES])
def test_against_reference_goldens(metrics, case):
    gold = np.load(GOLDEN)
    _, fn, keys = next(c for c in mc.CASES if c[0] == case)
    x = mc.make_inputs()
    for k in keys:
        assert np.array_equal(gold[f"in/{k}"], x[k].numpy(), equal_nan=True), k
    got = getattr(metrics, fn)(*(x[k] for k in keys))
    if fn == "compute_scene_flow_metrics":
        n = x[keys[0]].shape[1]
        for k in mc.FLOW_KEYS:
            want = float(gold[f"{case}/{k}"])
            assert isinstance(got[k], float)
            if k in ("acc3d_strict", "acc3d_relax", "outlier"):
                assert round(got[k] * n) == round(want * n), k          # the same count of points
            elif k == "angle_error":
                assert close(got[k], want, rel=ANGLE_FP32_REL), (k, got[k], want)
            else:
                assert close(got[k], want, rel=REL), (k, got[k], want)
    else:
        want = float(gold[f"{case}/value"])
        assert isinstance(got, float)
        if fn == "compute_psnr":
            assert close(got, want, abs_=PSNR_FP32_DB), (got, want)
        else:
            assert close(got, want, rel=REL), (got, want)


def test_flow_counts_match_the_fp64_oracle(metrics):
    x = mc.make_inputs()
    for p, l in (("flow_pred", "flow_labels"), ("flow_pred_zeros", "flow_labels_zeros")):
        got = metrics.compute_scene_flow_metrics(x[p], x[l])
        want, counts = metrics_ref.scene_flow_metrics(x[p], x[l])
        n = x[p].shape[1]
        for k in ("acc3d_strict", "acc3d_relax", "outlier"):
            assert round(got[k] * n) == counts[k]
        for k in ("EPE3D", "angle_error"):
            assert close(got[k], want[k], rel=REL)


# ----------------------------------------------------------------------------- the oracle
def test_box_filter_matches_scipy_uniform_filter():
    from scipy.ndimage import uniform_filter

    g = np.random.default_rng(0)
    for h, w in ((7, 7), (7, 31), (37, 53)):
        a = g.random((h, w))
        np.testing.assert_allclose(metrics_ref.box7(a), uniform_filter(a, size=7, mode="reflect"), rtol=0, atol=1e-14)


@pytest.mark.parametrize("shape", [(7, 7), (37, 53), (64, 48)])
def test_fp32_path_agrees_with_fp64(shape):
    x, y = noisy_image(*shape, seed=1)
    mask = np.zeros(shape, bool)
    mask[2:5, 3:9] = True
    s64, m64 = metrics_ref.ssim(x.numpy(), y.numpy(), "fp64", mask)
    s32, m32 = metrics_ref.ssim(x.numpy(), y.numpy(), "fp32", mask)
    assert abs(s64 - s32) <= SSIM_FP32 and abs(m64 - m32) <= SSIM_FP32
    assert abs(metrics_ref.psnr(x, y, "fp64") - metrics_ref.psnr(x, y, "fp32")) <= PSNR_FP32_DB


def test_ssim_of_identical_images_is_one():
    x, _ = noisy_image(16, 16)
    assert metrics_ref.ssim(x.numpy(), x.numpy(), "fp64", np.ones((16, 16)))[0] == 1.0


# ----------------------------------------------------------------------------- the module
def test_image_metrics_keys_and_values(metrics):
    x, y = noisy_image(37, 53, seed=2)
    mask = torch.rand(37, 53, generator=torch.Generator().manual_seed(3)) < 0.05
    fx, fy = torch.randn(37, 53, 80), torch.randn(37, 53, 80)
    fx, fy = fx[..., 8:72], fy[..., :64]                  # column slices: read in place with their row stride
    got = metrics.image_metrics(x, y, mask, fx, fy)
    assert set(got) == {"psnr", "ssim", "masked_psnr", "masked_ssim", "mask_count", "feat_psnr", "masked_feat_psnr"}
    assert all(v.dim() == 0 and v.dtype == torch.float64 for v in got.values())
    want = metrics_ref.image_metrics(x, y, mask.numpy(), fx.numpy(), fy.numpy())
    for k, v in got.items():
        assert close(float(v), want[k], rel=1e-12), k
    assert set(metrics.image_metrics(x, y)) == {"psnr", "ssim"}
    assert set(metrics.image_metrics(x, y, mask)) == {"psnr", "ssim", "masked_psnr", "masked_ssim", "mask_count"}
    assert set(metrics.image_metrics(x, y, None, fx, fy)) == {"psnr", "ssim", "feat_psnr"}
    assert set(metrics.image_metrics(x, y, None, fx, None)) == {"psnr", "ssim"}


def test_empty_mask_gives_nan_and_a_zero_count(metrics):
    x, y = noisy_image(9, 11)
    got = metrics.image_metrics(x, y, torch.zeros(9, 11), torch.rand(9, 11, 4), torch.rand(9, 11, 4))
    assert float(got["mask_count"]) == 0.0
    for k in ("masked_psnr", "masked_ssim", "masked_feat_psnr"):
        assert math.isnan(float(got[k]))


def test_summarize_follows_the_reference_aggregation(metrics):
    images = [noisy_image(16, 20, seed=s) for s in range(4)]
    masks = [None, torch.zeros(16, 20), torch.rand(16, 20) < 0.3, torch.ones(16, 20, 1)]
    feats = [(torch.rand(16, 20, 8), torch.rand(16, 20, 8)) if s % 2 else (None, None) for s in range(4)]
    per = [metrics.image_metrics(x, y, m, *f) for (x, y), m, f in zip(images, masks, feats)]
    lists = {k: [] for k in metrics.SUMMARY_KEYS}
    for (x, y), m, (fx, fy) in zip(images, masks, feats):     # video_utils.py:205-247 with the oracle's metrics
        ref = metrics_ref.image_metrics(x, y, m, fx, fy)
        lists["psnr"].append(ref["psnr"])
        lists["ssim"].append(ref["ssim"])
        if fx is not None:
            lists["feat_psnr"].append(ref["feat_psnr"])
        if m is not None and m.sum() > 0:
            lists["masked_psnr"].append(ref["masked_psnr"])
            lists["masked_ssim"].append(ref["masked_ssim"])
            if fx is not None:
                lists["masked_feat_psnr"].append(ref["masked_feat_psnr"])
    got = metrics.summarize(per)
    assert set(got) == set(metrics.SUMMARY_KEYS)
    for k, v in lists.items():
        assert close(got[k], non_zero_mean(v), rel=1e-12), k
    assert lists["masked_feat_psnr"] and lists["masked_psnr"]


def test_summarize_of_nothing_is_minus_one(metrics):
    assert metrics.summarize([]) == {k: -1 for k in metrics.SUMMARY_KEYS}
    x, y = noisy_image(8, 8)
    got = metrics.summarize([metrics.image_metrics(x, y, torch.zeros(8, 8))])
    assert got["masked_psnr"] == got["masked_ssim"] == got["feat_psnr"] == got["masked_feat_psnr"] == -1
    assert got["psnr"] > 0 and 0 < got["ssim"] < 1


def test_compute_ssim_and_its_range_assertions(metrics):
    x, y = noisy_image(12, 10)
    assert close(metrics.compute_ssim(x, y), metrics_ref.ssim(y.numpy(), x.numpy())[0], rel=1e-12)
    assert isinstance(metrics.compute_ssim(x.numpy(), y.numpy()), float)
    with pytest.raises(AssertionError, match="target must be"):
        metrics.compute_ssim(x + 2, y + 2)                   # both out of range: the target is checked first
    with pytest.raises(AssertionError, match="prediction must be"):
        metrics.compute_ssim(x - 1, y)
    bad = y.clone()
    bad[3, 4, 1] = float("nan")                            # numpy's max of a NaN image is NaN: the check fails
    with pytest.raises(AssertionError, match="target must be"):
        metrics.compute_ssim(x, bad)


def test_compute_psnr_accepts_numpy_and_any_shape(metrics):
    x, y = noisy_image(5, 3, c=2)
    want = metrics_ref.psnr(x, y)
    assert close(metrics.compute_psnr(x.numpy(), y.numpy()), want, rel=1e-12)
    assert close(metrics.compute_psnr(x.reshape(-1, 2), y.reshape(-1, 2)), want, rel=1e-12)
    assert metrics.compute_psnr(x, x) == math.inf


@pytest.mark.parametrize("bad", ["small_h", "small_w", "shape", "channels", "features", "feature_shape", "mask",
                                 "two_dims"])
def test_argument_errors(metrics, bad):
    x, y = noisy_image(8, 9)
    args = dict(rgb=x, pixels=y)
    if bad == "small_h":
        args = dict(rgb=x[:6], pixels=y[:6])
    elif bad == "small_w":
        args = dict(rgb=x[:, :6], pixels=y[:, :6])
    elif bad == "shape":
        args["pixels"] = y[:, :8]
    elif bad == "channels":
        args = dict(rgb=torch.rand(8, 9, 5), pixels=torch.rand(8, 9, 5))
    elif bad == "features":
        args.update(dino_feat=torch.rand(8, 9, 257), features=torch.rand(8, 9, 257))
    elif bad == "feature_shape":
        args.update(dino_feat=torch.rand(8, 9, 64), features=torch.rand(8, 8, 64))
    elif bad == "mask":
        args.update(dynamic_mask=torch.ones(8, 8))
    else:
        args = dict(rgb=x[..., 0], pixels=y[..., 0])
    with pytest.raises(ValueError):
        metrics.image_metrics(**args)


def test_other_errors(metrics):
    with pytest.raises(ValueError):
        metrics.compute_psnr(torch.rand(4, 3), torch.rand(3, 4))
    with pytest.raises(ValueError):
        metrics.compute_valid_depth_rmse(torch.rand(4), torch.rand(5))
    with pytest.raises(ValueError):
        metrics.compute_scene_flow_metrics(torch.rand(10, 3), torch.rand(10, 3))
    with pytest.raises(ValueError):
        metrics.compute_ssim(torch.rand(6, 9, 3), torch.rand(6, 9, 3))


def test_cpu_tensors_are_refused():
    from emernerf_b200 import metrics

    x, y = noisy_image(8, 8)
    for call in (lambda: metrics.image_metrics(x, y), lambda: metrics.compute_ssim(x, y),
                 lambda: metrics.compute_psnr(x, y), lambda: metrics.compute_valid_depth_rmse(x[..., 0], y[..., 0]),
                 lambda: metrics.compute_scene_flow_metrics(x, y)):
        with pytest.raises(RuntimeError, match="CUDA"):
            call()

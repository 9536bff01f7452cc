"""The render rays and the error-map update of emernerf_b200.raygen on the host (CPU suite): ``PixelRaySampler``'s
``get_render_rays`` and ``update_pixel_error_maps``, with emer_image_rays, emer_error_map and
emer_error_map_normalize run through tests/errormap_emulator.py, against the reference's own methods
(tests/golden/errormap.npz, make_golden_errormap.py).  Every key in the reference's order, with its dtype and shape;
values with torch.equal, except view directions and norms (within 1e-6, the bar of the ray kernels) and the resized
image, which is torch's own op.  The maps bit for bit, NaN where the reference's are NaN.  oracle/errormap_ref.py is
held to the same fixture."""
import os

import numpy as np
import pytest
import torch

import cabi_emulator
import errormap_cases as ec
import errormap_emulator
from helpers import rel_err
from oracle import errormap_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "errormap.npz")
CLOSE = ("viewdirs", "direction_norm")
RAY_CASES = [(c, d, i) for c in ec.SOURCES for d in ec.DOWNSCALES for i in ec.IMAGES[d]]


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


@pytest.fixture
def raygen(monkeypatch):
    errormap_emulator.install(monkeypatch)
    from emernerf_b200 import raygen

    return raygen


def check_rays(z, prefix, rays, resized_exact):
    assert list(rays) == z[f"{prefix}/keys"].tolist()
    for k, v in rays.items():
        want = torch.from_numpy(z[f"{prefix}/{k}"])
        assert v.dtype == want.dtype and v.shape == want.shape, (prefix, k, v.dtype, v.shape)
        if k in CLOSE:
            assert rel_err(v, want) < 1e-6, (prefix, k)
        elif k != "pixels" or resized_exact:
            assert torch.equal(v, want), (prefix, k)


@pytest.mark.parametrize("case,d,img", RAY_CASES)
def test_render_rays_match_reference(z, raygen, case, d, img):
    src = ec.fill(ec.PixelSource(), case, ec.DOWNSCALES[d])
    del cabi_emulator.CALLS[:]
    rays = raygen.PixelRaySampler(src).get_render_rays(img)
    check_rays(z, f"rays/{case}/{d}/{img}", rays, d == "1")
    assert cabi_emulator.CALLS == ["emer_image_rays"]
    # the image is torch's bicubic resize, here of all images at once
    want = torch.from_numpy(z[f"rays/{case}/{d}/{img}/pixels"])
    assert (rays["pixels"] - want).abs().max() <= 1e-6


@pytest.mark.parametrize("case,d,img", RAY_CASES)
def test_render_rays_oracle_matches_reference(z, case, d, img):
    src = ec.fill(ec.PixelSource(), case, ec.DOWNSCALES[d])
    check_rays(z, f"rays/{case}/{d}/{img}", errormap_ref.get_render_rays(src, img), True)


def check_map(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    assert torch.equal(torch.nan_to_num(got), torch.nan_to_num(want))


@pytest.mark.parametrize("case", list(ec.UPDATES))
def test_update_matches_reference(z, raygen, case):
    src = ec.fill(ec.PixelSource(), "full")
    src.pixel_error_buffered = False
    old = src.pixel_error_maps
    raygen.PixelRaySampler(src).update_pixel_error_maps(ec.render_results(case))
    check_map(src.pixel_error_maps, torch.from_numpy(z[f"update/{case}"]))
    assert src.pixel_error_maps is not old and src.pixel_error_buffered
    assert not raygen._MAP_WS[torch.device("cpu")].any()


@pytest.mark.parametrize("case", list(ec.UPDATES))
def test_update_from_tensor_lists_matches_reference(z, raygen, case):
    src = ec.fill(ec.PixelSource(), "full")
    rr = {k: [torch.from_numpy(a) for a in v] for k, v in ec.render_results(case).items()}
    raygen.PixelRaySampler(src).update_pixel_error_maps(rr)
    check_map(src.pixel_error_maps, torch.from_numpy(z[f"update/{case}"]))


@pytest.mark.parametrize("case", list(ec.UPDATES))
def test_update_oracle_matches_reference(z, case):
    src = ec.fill(ec.PixelSource(), "full")
    errormap_ref.update_pixel_error_maps(src, ec.render_results(case))
    check_map(src.pixel_error_maps, torch.from_numpy(z[f"update/{case}"]))


def test_update_without_a_map_does_nothing(raygen):
    src = ec.fill(ec.PixelSource(), "full")
    src.pixel_error_maps, src.pixel_error_buffered = None, False
    raygen.PixelRaySampler(src).update_pixel_error_maps(ec.render_results("plain"))
    assert src.pixel_error_maps is None and not src.pixel_error_buffered


@pytest.mark.parametrize("case", ["constant", "nan"])
def test_next_draw_raises_the_reference_error(raygen, case):
    src = ec.fill(ec.PixelSource(), "full")
    want_src = ec.fill(ec.PixelSource(), "full")
    errormap_ref.update_pixel_error_maps(want_src, ec.render_results(case))
    from oracle import raybatch_ref

    with pytest.raises(RuntimeError) as want:
        raybatch_ref.pixel_train_rays(want_src, 96, None)
    sampler = raygen.PixelRaySampler(src)
    sampler.get_train_rays(96, None)                       # the old map, validated
    sampler.update_pixel_error_maps(ec.render_results(case))
    with pytest.raises(RuntimeError) as got:
        sampler.get_train_rays(96, None)
    assert str(got.value) == str(want.value)

"""The render rays and the error-map refresh on the GPU, against oracle/errormap_ref.py (the reference's torch path).

(a) get_render_rays on a 600-image 640 x 960 source and on the fixture sources, at downscales 1, 1/4, 1/16 and 1/3:
    the oracle's keys, dtypes and shapes; every value bit-identical except viewdirs / direction_norm (within 1e-6, the
    bar of test_gen_rays_matches_the_reference_formula).
(b) update_pixel_error_maps from numpy lists and from device tensors: the oracle's map bit for bit; a constant map and
    a NaN pixel give the oracle's NaN map, and the next get_train_rays raises torch.multinomial's message (pinned
    against the reference on the CPU in test_errormap_cpu.py; on CUDA torch checks the weights with a device-side
    assert, so the oracle's draw is not run on such a map here).
(c) refresh_pixel_error_maps with a small static and a small dynamic field: the map of the oracle's cache step bit for
    bit when the oracle renders the same rays, and the next get_train_rays draws the oracle's batch from it.  With the
    oracle's own rays, whose view directions differ in the last bits, the maps agree to 1e-4 on 99 % of the pixels.
(d) A second refresh runs under torch.cuda.set_sync_debug_mode("error"); the first draw after it validates the new map
    (its one sync), and the draws after that run under "error" too.
The error-map workspace is zero after every call."""
import types

import pytest
import torch

import cases
import errormap_cases as ec
import raybatch_cases as rc
from helpers import rel_err
from oracle import errormap_ref, raybatch_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
CLOSE = ("viewdirs", "direction_norm")


def big_source():
    """A Waymo-sized source drawn on the device, as in test_gpu_raybatch.py."""
    src = ec.fill(ec.PixelSource(), "full")
    n, (h, w) = 600, (640, 960)
    g = torch.Generator(device=DEV).manual_seed(11)
    src.data_cfg.load_size = [h, w]
    src.images = torch.rand(n, h, w, 3, device=DEV, generator=g)
    src.sky_masks = (torch.rand(n, h, w, device=DEV, generator=g) > 0.7).float()
    src.dynamic_masks = (torch.rand(n, h, w, device=DEV, generator=g) > 0.9).float()
    src.features = torch.rand(n, 46, 69, 64, device=DEV, generator=g)
    src.featmap_downscale_factor = (46 / h, 69 / w)
    src.pixel_error_maps = torch.rand(n, h // rc.DOWNSCALE, w // rc.DOWNSCALE, device=DEV, generator=g)
    src._normalized_timestamps = torch.rand(n, device=DEV, generator=g)
    src.cam_ids = torch.arange(n, device=DEV) % 3
    reps = (n + rc.N_IMAGES - 1) // rc.N_IMAGES
    src.cam_to_worlds = src.cam_to_worlds.repeat(reps, 1, 1)[:n]
    K = src.intrinsics.repeat(reps, 1, 1)[:n].clone()
    K[:, 0, 0] *= 10
    K[:, 1, 1] *= 10
    K[:, 0, 2], K[:, 1, 2] = w / 2, h / 2
    src.intrinsics = K
    return rc.to_device(src, DEV)


@pytest.fixture(scope="module")
def big():
    return big_source()


def check_rays(got, want):
    assert list(got) == list(want)
    for k, v in want.items():
        g = got[k]
        assert g.is_cuda and g.dtype == v.dtype and g.shape == v.shape, k
        if k in CLOSE:
            assert rel_err(g, v.to(DEV)) < 1e-6, k
        else:
            assert torch.equal(g, v.to(DEV)), k


def map_ws_is_zero():
    from emernerf_b200 import raygen

    return not raygen._map_workspace(torch.device(DEV, torch.cuda.current_device())).any()


@pytest.mark.parametrize("d", list(ec.DOWNSCALES))
def test_render_rays_match_oracle_on_a_waymo_sized_source(big, d):
    from emernerf_b200 import raygen

    big._downscale_factor = ec.DOWNSCALES[d]
    sampler = raygen.PixelRaySampler(big)
    for i in (0, 299, 599):
        check_rays(sampler.get_render_rays(i), errormap_ref.get_render_rays(big, i))


@pytest.mark.parametrize("case", ec.SOURCES)
@pytest.mark.parametrize("d", list(ec.DOWNSCALES))
def test_render_rays_match_oracle_on_fixture_sources(case, d):
    from emernerf_b200 import raygen

    src = rc.to_device(ec.fill(ec.PixelSource(), case, ec.DOWNSCALES[d]), DEV)
    sampler = raygen.PixelRaySampler(src)
    for i in range(rc.N_IMAGES):
        check_rays(sampler.get_render_rays(i), errormap_ref.get_render_rays(src, i))


def render_results(shape, kind, seed=0):
    """Device tensors shaped as render_pixels' per-image outputs."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    n, h, w = shape
    gt = torch.rand(n, h, w, 3, device=DEV, generator=g)
    rgb = torch.rand(n, h, w, 3, device=DEV, generator=g)
    out = {"gt_rgbs": list(gt), "rgbs": list(rgb)}
    if kind == "constant":
        out = {"gt_rgbs": list(torch.full_like(gt, 0.5)), "rgbs": list(torch.full_like(rgb, 0.25))}
    elif kind == "nan":
        rgb[n // 2, 3, 4, 1] = float("nan")
    elif kind == "dynamic":
        out["dynamic_opacities"] = list(torch.rand(n, h, w, device=DEV, generator=g))
    return out


def check_map(got, want):
    assert got.is_cuda and got.dtype == want.dtype and got.shape == want.shape
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    assert torch.equal(torch.nan_to_num(got), torch.nan_to_num(want))


@pytest.mark.parametrize("kind", ["plain", "dynamic", "constant", "nan"])
def test_update_matches_oracle(big, kind):
    from emernerf_b200 import raygen

    rr = render_results(big.pixel_error_maps.shape, kind)
    as_numpy = {k: [t.cpu().numpy() for t in v] for k, v in rr.items()}
    ref = types.SimpleNamespace(pixel_error_maps=big.pixel_error_maps, device=torch.device(DEV))
    errormap_ref.update_pixel_error_maps(ref, as_numpy)
    sampler = raygen.PixelRaySampler(big)
    for results in (as_numpy, rr):
        big.pixel_error_buffered = False
        sampler.update_pixel_error_maps(results)
        assert big.pixel_error_buffered
        check_map(big.pixel_error_maps, ref.pixel_error_maps)
        assert map_ws_is_zero()
    if kind in ("constant", "nan"):
        assert torch.isnan(big.pixel_error_maps).all()
        big.data_cfg.sampler.buffer_ratio = 0.25
        with pytest.raises(RuntimeError, match="probability tensor contains either `inf`, `nan` or element < 0"):
            sampler.get_train_rays(8192, None)


def small_models(kind):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder
    from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    field, props = cases.build_models(ns, kind)
    return field.to(DEV), [p.to(DEV) for p in props], PropNetEstimator(None, None).to(DEV)


@pytest.mark.parametrize("kind", ["static", "dynamic"])
def test_refresh_matches_oracle_cache_step(kind):
    from emernerf_b200 import raygen
    from emernerf_b200.radiance_fields.render_utils import render_rays

    field, props, est = small_models(kind)
    cfg = cases.render_cfg()
    src = rc.to_device(ec.fill(ec.PixelSource(), "full", 1.0), DEV)
    ref = rc.to_device(ec.fill(ec.PixelSource(), "full", 1.0), DEV)
    sampler = raygen.PixelRaySampler(src)
    own = rc.to_device(ec.fill(ec.PixelSource(), "full", 1.0), DEV)
    errormap_ref.cache_step(own, field, est, props, cfg, render_rays)
    errormap_ref.cache_step(ref, field, est, props, cfg, render_rays, lambda i, d: sampler._render_rays_at(i, d))
    src.pixel_error_buffered = False
    sampler.refresh_pixel_error_maps(field, est, props, cfg)
    check_map(src.pixel_error_maps, ref.pixel_error_maps)
    close = torch.isclose(src.pixel_error_maps, own.pixel_error_maps, rtol=0, atol=1e-4)
    assert close.float().mean() > 0.99
    assert src.pixel_error_buffered and src.downscale_factor == 1.0 and map_ws_is_zero()
    assert not torch.isnan(src.pixel_error_maps).any()
    # the sampler's bit-identity carries through: the draw from the new map is the oracle's draw from its map
    cand = rc.pixel_candidates("full")
    torch.cuda.manual_seed(5)
    want = raybatch_ref.pixel_train_rays(ref, 96, cand)
    torch.cuda.manual_seed(5)
    got = sampler.get_train_rays(96, cand)
    assert list(got) == list(want)
    for k, v in want.items():
        if k in ("viewdirs", "direction_norms"):
            assert rel_err(got[k], v) < 1e-6, k
        else:
            assert torch.equal(got[k], v), k


def test_refresh_is_sync_free_after_the_first():
    from emernerf_b200 import raygen

    field, props, est = small_models("dynamic")
    cfg = cases.render_cfg()
    src = rc.to_device(ec.fill(ec.PixelSource(), "full", 1.0), DEV)
    cand = rc.pixel_candidates("full")
    sampler = raygen.PixelRaySampler(src)
    sampler.refresh_pixel_error_maps(field, est, props, cfg)
    first = src.pixel_error_maps
    sampler.get_train_rays(96, cand)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sampler.refresh_pixel_error_maps(field, est, props, cfg)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert src.pixel_error_maps is not first
    sampler.get_train_rays(96, cand)                       # validates the new map: its one sync
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            sampler.get_train_rays(96, cand)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(src.pixel_error_maps, first)       # same field, same map
    assert map_ws_is_zero()


def test_kernels_write_the_map_in_chunks():
    """emer_error_map folds several chunks into one normalisation: the map of one chunk per image equals the map of
    one chunk for all images."""
    from emernerf_b200 import _lib, _ops, raygen

    rr = render_results((40, 40, 60), "dynamic", seed=3)
    gt, rgb, op = (torch.stack(rr[k]) for k in ("gt_rgbs", "rgbs", "dynamic_opacities"))
    ws = raygen._map_workspace(gt.device)
    p = _ops._ptr
    maps = []
    for chunks in (1, 40, 7):
        m = torch.empty(op.shape, device=DEV)
        _ops._need_cuda(m)
        for idx in torch.arange(40).tensor_split(chunks):
            a, b = int(idx[0]), int(idx[-1]) + 1
            _lib.call("emer_error_map", p(gt[a:b]), p(rgb[a:b]), p(op[a:b]), (b - a) * 2400, p(m[a:b]), p(ws),
                      _ops._stream())
        _lib.call("emer_error_map_normalize", p(m), m.numel(), p(ws), _ops._stream())
        assert not ws.any()
        maps.append(m)
    assert torch.equal(maps[0], maps[1]) and torch.equal(maps[0], maps[2])
    e = (gt - rgb).abs()
    e = ((e[..., 0] + e[..., 1]) + e[..., 2]).cpu() / 3
    e = torch.where(op.cpu() > 0.1, e * 5, e)
    assert torch.equal(maps[0].cpu(), (e - e.min()) / (e.max() - e.min()))

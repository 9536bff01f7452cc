"""The training-batch samplers of emernerf_b200.raygen on the host (CPU suite): ``PixelRaySampler`` with
``emer_topk_ratio`` and ``emer_pixel_batch`` run through tests/raybatch_emulator.py, and ``LidarRaySampler``, against
the reference's own ``get_train_rays`` (tests/golden/raybatch.npz, make_golden_raybatch.py) under the CPU generator:
every key of every call with torch.equal, in the reference's key order, and the generator left where the reference
leaves it.  oracle/raybatch_ref.py is held to the same fixture.  Invalid error maps and too many importance rays raise
torch.multinomial's messages, and the map is validated again after it is replaced or modified in place."""
import os

import numpy as np
import pytest
import torch

import cabi_emulator
import raybatch_cases as rc
import raybatch_emulator
from oracle import raybatch_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "raybatch.npz")


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


@pytest.fixture
def raygen(monkeypatch):
    raybatch_emulator.install(monkeypatch)
    from emernerf_b200 import raygen

    return raygen


def check_batch(z, prefix, batch):
    assert list(batch) == z[f"{prefix}/keys"].tolist()
    for k, v in batch.items():
        want = torch.from_numpy(z[f"{prefix}/{k}"])
        assert v.dtype == want.dtype and v.shape == want.shape, (prefix, k, v.dtype, v.shape)
        assert torch.equal(v, want), (prefix, k)


def run_pixel(z, case, get_train_rays):
    _, _, _, _, rays, calls, seed = rc.PIXEL_CASES[case]
    torch.manual_seed(seed)
    for c in range(calls):
        check_batch(z, f"pixel/{case}/{c}", get_train_rays(rays, rc.pixel_candidates(case)))
    assert torch.equal(torch.rand(8), torch.from_numpy(z[f"pixel/{case}/after"]))


def run_lidar(z, case, get_train_rays):
    sets, rays, seed = rc.LIDAR_CASES[case]
    torch.manual_seed(seed)
    for c in range(len(sets)):
        check_batch(z, f"lidar/{case}/{c}", get_train_rays(rays, rc.lidar_candidates(case, c)))
    assert torch.equal(torch.rand(8), torch.from_numpy(z[f"lidar/{case}/after"]))


@pytest.mark.parametrize("case", list(rc.PIXEL_CASES))
def test_pixel_sampler_matches_reference(z, raygen, case):
    src = rc.fill_pixel(rc.PixelSource(), case)
    del cabi_emulator.CALLS[:]
    run_pixel(z, case, raygen.PixelRaySampler(src).get_train_rays)
    importance = rc.PIXEL_CASES[case][0] > 0 and rc.PIXEL_CASES[case][1]
    assert ("emer_topk_ratio" in cabi_emulator.CALLS) == importance
    assert "emer_pixel_batch" in cabi_emulator.CALLS


@pytest.mark.parametrize("case", list(rc.PIXEL_CASES))
def test_pixel_oracle_matches_reference(z, case):
    src = rc.fill_pixel(rc.PixelSource(), case)
    run_pixel(z, case, lambda n, c: raybatch_ref.pixel_train_rays(src, n, c))


@pytest.mark.parametrize("case", list(rc.LIDAR_CASES))
def test_lidar_sampler_and_oracle_match_reference(z, raygen, case):
    src = rc.fill_lidar(rc.LidarSource(), case)
    run_lidar(z, case, raygen.LidarRaySampler(src).get_train_rays)
    cache = raybatch_ref.LidarCache()
    run_lidar(z, case, lambda n, c: raybatch_ref.lidar_train_rays(src, n, c, cache))


def _message(fn):
    with pytest.raises(RuntimeError) as e:
        fn()
    return str(e.value)


@pytest.mark.parametrize("bad", ["nan", "inf", "negative", "zero_over_candidates", "too_many_rays"])
def test_invalid_maps_raise_torch_messages(raygen, bad):
    src = rc.fill_pixel(rc.PixelSource(), "full")
    cand = rc.pixel_candidates("full")
    rays = 96
    if bad == "nan":
        src.pixel_error_maps[cand[1], 1, 2] = float("nan")
    elif bad == "inf":
        src.pixel_error_maps[cand[0], 0, 0] = float("inf")
    elif bad == "negative":
        src.pixel_error_maps[cand[-1], 3, 5] = -1e-3
    elif bad == "zero_over_candidates":
        src.pixel_error_maps[cand] = 0.0
        src.pixel_error_maps[1] = 1.0                       # positive, but not a candidate
    else:
        rays = 4 * len(cand) * 24 + 4                       # a quarter of them is more than the weights
    torch.manual_seed(0)
    want = _message(lambda: raybatch_ref.pixel_train_rays(src, rays, cand))
    state = torch.get_rng_state()
    torch.manual_seed(0)
    got = _message(lambda: raygen.PixelRaySampler(src).get_train_rays(rays, cand))
    assert got == want
    assert torch.equal(torch.get_rng_state(), state)


def test_no_importance_rays_raises_as_torch(raygen):
    src = rc.fill_pixel(rc.PixelSource(), "full")
    torch.manual_seed(0)
    want = _message(lambda: raybatch_ref.pixel_train_rays(src, 1, None))
    assert want == _message(lambda: raygen.PixelRaySampler(src).get_train_rays(1, None))


def test_map_is_validated_again_after_it_changes(raygen):
    src = rc.fill_pixel(rc.PixelSource(), "full")
    cand = rc.pixel_candidates("full")
    sampler = raygen.PixelRaySampler(src)
    sampler.get_train_rays(96, cand)
    calls = []
    real = sampler._validate.__func__

    def counting(self, *a):
        calls.append(1)
        return real(self, *a)

    sampler._validate = counting.__get__(sampler)
    sampler.get_train_rays(96, cand)
    assert sampler._valid is not None and sampler._valid[0] is src.pixel_error_maps
    src.pixel_error_maps[cand[2], 0, 1] = float("nan")      # in place: _version moves
    with pytest.raises(RuntimeError, match="probability tensor contains"):
        sampler.get_train_rays(96, cand)
    src.pixel_error_maps = torch.rand_like(src.pixel_error_maps)      # replaced
    sampler.get_train_rays(96, cand)
    valid = sampler._valid
    sampler.get_train_rays(96, cand)
    assert sampler._valid is valid and valid[0] is src.pixel_error_maps
    sampler.get_train_rays(96, cand[:-1])                   # another candidate set
    assert sampler._valid[2] != valid[2]
    assert len(calls) == 5


def test_samplers_refuse_cpu_tensors_without_the_emulator():
    from emernerf_b200 import raygen

    src = rc.fill_pixel(rc.PixelSource(), "full")
    with pytest.raises(RuntimeError, match="CUDA"):
        raygen.PixelRaySampler(src).get_train_rays(96, rc.pixel_candidates("full"))

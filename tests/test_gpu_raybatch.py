"""The training-batch samplers on the GPU.

(a) emer_topk_ratio against a sort by (-key, index) of torch's p[cand] / q, and its values against torch.topk, for
    M in {1, 1000, 540 * 2400, 2^21 + 17} and every k in {1, 7, 2048, 8192, 16384} up to M, on random maps, on maps
    with forced ties and on a map with zeros.
(b) PixelRaySampler and LidarRaySampler against oracle/raybatch_ref.py (the reference's torch path) on the device after
    torch.cuda.manual_seed: every key bit-identical except viewdirs / direction_norms (within 1e-6, the bar of
    test_gen_rays_matches_the_reference_formula), and the CUDA generator left where the oracle leaves it.
(c) After the first call, both samplers run under torch.cuda.set_sync_debug_mode("error").
(d) A CUDA graph of the two kernels on fixed draws replays to the eager results and leaves the workspace zeroed.
(e) The error map is validated again after it is replaced or modified in place."""
import re

import pytest
import torch

import raybatch_cases as rc
from helpers import rel_err
from oracle import raybatch_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
MS = [(1, 1, 1), (10, 100, 10), (600, 2400, 540), (1, 2 ** 21 + 17, 1)]   # (images, plane, candidates)
KS = [1, 7, 2048, 8192, 16384]
EXACT = ["img_idx", "cam_idx", "pixels", "sky_masks", "dynamic_masks", "features", "normed_timestamps", "origins",
         "pixel_coords"]


def topk(p, cand, q, k):
    from emernerf_b200 import _lib, _ops, raygen

    out = torch.empty(k, dtype=torch.int64, device=DEV)
    _ops._need_cuda(p, cand, q)
    _lib.call("emer_topk_ratio", _ops._ptr(p), p[0].numel(), _ops._ptr(cand), len(cand), _ops._ptr(q), k,
              _ops._ptr(out), _ops._ptr(raygen._workspace(p.device)), _ops._stream())
    return out


def expected_order(p, cand, q, k):
    keys = p[cand].reshape(-1) / q
    return keys, torch.sort(keys, descending=True, stable=True).indices[:k]


@pytest.mark.parametrize("kind", ["random", "ties", "zeros"])
@pytest.mark.parametrize("n,plane,nc", MS)
def test_topk_ratio_matches_sorted_keys(n, plane, nc, kind):
    from emernerf_b200 import raygen

    g = torch.Generator(device=DEV).manual_seed(n * 7 + plane)
    p = torch.rand(n, plane, device=DEV, generator=g)
    cand = torch.randperm(n, device=DEV, generator=g)[:nc]
    q = torch.empty(nc * plane, device=DEV).exponential_(1, generator=g)
    if kind == "ties":
        p = torch.floor(p * 8) / 8                        # eight distinct weights and a constant q: long runs of ties
        q.fill_(1.0)
    elif kind == "zeros":
        p[p < 0.5] = 0.0
        p[cand[0], 0] = -0.0                               # a negative zero weighs as much as a zero
    m = nc * plane
    for k in sorted({k for k in KS if k <= m} | ({m} if m <= 16384 else set())):
        got = topk(p, cand, q, k)
        keys, want = expected_order(p, cand, q, k)
        assert torch.equal(got, want), (m, k, kind)
        assert torch.equal(keys[got], torch.topk(keys, k).values), (m, k, kind)
    assert not raygen._workspace(p.device).any()


def pixel_source(case, n_images=None, size=None):
    src = rc.fill_pixel(rc.PixelSource(), case)
    if n_images is not None:                               # a Waymo-sized source, drawn on the device
        g = torch.Generator(device=DEV).manual_seed(11)
        h, w = size
        ds = rc.DOWNSCALE
        src.data_cfg.load_size = [h, w]
        src.images = torch.rand(n_images, h, w, 3, device=DEV, generator=g)
        src.sky_masks = (torch.rand(n_images, h, w, device=DEV, generator=g) > 0.7).float()
        src.dynamic_masks = (torch.rand(n_images, h, w, device=DEV, generator=g) > 0.9).float()
        src.features = torch.rand(n_images, 46, 69, 64, device=DEV, generator=g)
        src.featmap_downscale_factor = (46 / h, 69 / w)
        src.pixel_error_maps = torch.rand(n_images, h // ds, w // ds, device=DEV, generator=g)
        src._normalized_timestamps = torch.rand(n_images, device=DEV, generator=g)
        src.cam_ids = torch.arange(n_images, device=DEV) % 5
        reps = (n_images + rc.N_IMAGES - 1) // rc.N_IMAGES
        src.cam_to_worlds = src.cam_to_worlds.repeat(reps, 1, 1)[:n_images]
        K = src.intrinsics.repeat(reps, 1, 1)[:n_images].clone()
        K[:, 0, 0] *= 10
        K[:, 1, 1] *= 10
        K[:, 0, 2], K[:, 1, 2] = w / 2, h / 2
        src.intrinsics = K
    return rc.to_device(src, DEV)


def check_against_oracle(got, want):
    assert list(got) == list(want)
    for k, v in want.items():
        assert got[k].dtype == v.dtype and got[k].shape == v.shape, k
        if k in EXACT:
            assert torch.equal(got[k], v), k
        else:
            assert rel_err(got[k], v) < 1e-6, k


def candidates(kind, n_images):
    if kind == "none":
        return None
    idx = [i for i in range(n_images) if i % 10 != 3]
    return idx if kind == "list" else torch.tensor(idx, device=DEV)


# (ratio, buffered, candidates, rays)
PIXEL = [(0.25, True, "list", 8192), (0.25, True, "none", 8205), (0.25, True, "tensor", 8192), (0.0, True, "list", 8192),
         (1.0, True, "list", 8192), (0.25, False, "list", 8205), (1.0, True, "tensor", 1), (0.0, True, "none", 1),
         (0.25, True, "list", 1)]


@pytest.fixture(scope="module")
def big_source():
    return pixel_source("full", 600, (640, 960))


@pytest.mark.parametrize("ratio,buffered,cand_kind,rays", PIXEL)
def test_pixel_sampler_matches_oracle(big_source, ratio, buffered, cand_kind, rays):
    from emernerf_b200 import raygen

    src = big_source
    src.data_cfg.sampler.buffer_ratio, src.pixel_error_buffered = ratio, buffered
    cand = candidates(cand_kind, len(src.images))
    sampler = raygen.PixelRaySampler(src)
    for seed in (0, 1):
        torch.cuda.manual_seed(seed)
        try:
            want = raybatch_ref.pixel_train_rays(src, rays, cand)
        except RuntimeError as e:                          # 1 ray at ratio 0.25: no importance ray, torch refuses
            state = torch.cuda.get_rng_state()
            torch.cuda.manual_seed(seed)
            with pytest.raises(RuntimeError, match=re.escape(str(e))):
                sampler.get_train_rays(rays, cand)
            assert torch.equal(torch.cuda.get_rng_state(), state)
            continue
        state = torch.cuda.get_rng_state()
        torch.cuda.manual_seed(seed)
        got = sampler.get_train_rays(rays, cand)
        assert torch.equal(torch.cuda.get_rng_state(), state)
        check_against_oracle(got, want)


@pytest.mark.parametrize("case", list(rc.PIXEL_CASES))
def test_pixel_sampler_matches_oracle_on_fixture_cases(case):
    from emernerf_b200 import raygen

    src = pixel_source(case)
    _, _, _, _, rays, calls, seed = rc.PIXEL_CASES[case]
    sampler = raygen.PixelRaySampler(src)
    torch.cuda.manual_seed(seed)
    want = [raybatch_ref.pixel_train_rays(src, rays, rc.pixel_candidates(case, DEV)) for _ in range(calls)]
    state = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(seed)
    got = [sampler.get_train_rays(rays, rc.pixel_candidates(case, DEV)) for _ in range(calls)]
    assert torch.equal(torch.cuda.get_rng_state(), state)
    for a, b in zip(got, want):
        check_against_oracle(a, b)


def lidar_source():
    src = rc.fill_lidar(rc.LidarSource(), "lists")
    g = torch.Generator().manual_seed(3)
    n = 1_000_003
    src.origins = torch.randn(n, 3, generator=g)
    src.directions = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    src.ranges = torch.rand(n, 1, generator=g) * 80
    src._timesteps = torch.sort(torch.randint(0, 200, (n,), generator=g)).values
    src._normalized_timestamps = src._timesteps.float() / 199
    return rc.to_device(src, DEV)


def test_lidar_sampler_matches_oracle():
    from emernerf_b200 import raygen

    src = lidar_source()
    sets = [list(range(0, 200, 2)), list(range(0, 200, 2)), torch.arange(50, 150, device=DEV), list(range(7, 90))]
    sampler, cache = raygen.LidarRaySampler(src), raybatch_ref.LidarCache()
    torch.cuda.manual_seed(4)
    want = [raybatch_ref.lidar_train_rays(src, 8192, c, cache) for c in sets]
    state = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(4)
    got = [sampler.get_train_rays(8192, c) for c in sets]
    assert torch.equal(torch.cuda.get_rng_state(), state)
    for a, b in zip(got, want):
        assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in b)


def test_no_host_sync_after_the_first_call(big_source):
    from emernerf_b200 import raygen

    src = big_source
    src.data_cfg.sampler.buffer_ratio, src.pixel_error_buffered = 0.25, True
    cand = candidates("list", len(src.images))
    lsrc = lidar_source()
    lcand = list(range(0, 200, 3))
    pix, lid = raygen.PixelRaySampler(src), raygen.LidarRaySampler(lsrc)
    pix.get_train_rays(8192, cand)
    lid.get_train_rays(8192, lcand)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            pix.get_train_rays(8192, cand)
            lid.get_train_rays(8192, lcand)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_graph_replays_to_eager_and_leaves_workspace_zeroed(big_source):
    from emernerf_b200 import _lib, _ops, raygen

    src = big_source
    maps = src.pixel_error_maps
    n_img, mh, mw = maps.shape
    H, W, ds = src.HEIGHT, src.WIDTH, src.buffer_downscale
    cand = torch.arange(0, n_img, 2, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(9)
    n_u, n_i = 6144, 2048
    u_pick = torch.randint(0, len(cand), (n_u,), device=DEV, generator=g)
    u_x = torch.randint(0, W, (n_u,), device=DEV, generator=g)
    u_y = torch.randint(0, H, (n_u,), device=DEV, generator=g)
    q = torch.empty(len(cand) * mh * mw, device=DEV).exponential_(1, generator=g)
    i_dy = torch.randint(0, ds, (n_i,), device=DEV, generator=g)
    i_dx = torch.randint(0, ds, (n_i,), device=DEV, generator=g)
    sampler = raygen.PixelRaySampler(src)

    def run():
        sel = torch.empty(n_i, dtype=torch.int64, device=DEV)
        _ops._need_cuda(maps)
        _lib.call("emer_topk_ratio", _ops._ptr(maps), mh * mw, _ops._ptr(cand), len(cand), _ops._ptr(q), n_i,
                  _ops._ptr(sel), _ops._ptr(raygen._workspace(maps.device)), _ops._stream())
        out = sampler._assemble(n_u, n_i, cand, u_pick, u_x, u_y, sel, i_dy, i_dx, mh, mw, ds, H, W, src.images,
                                src.sky_masks, src.dynamic_masks, src.features, src.normalized_timestamps, src.cam_ids,
                                src.cam_to_worlds, src.intrinsics)
        return sel, out

    eager_sel, eager = run()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()                                              # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sel, out = run()
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(sel, eager_sel)
    for k in eager:
        assert torch.equal(out[k], eager[k]), k
    assert not raygen._workspace(maps.device).any()


def test_map_is_validated_again_after_it_changes():
    from emernerf_b200 import raygen

    src = pixel_source("full")
    cand = rc.pixel_candidates("full")
    sampler = raygen.PixelRaySampler(src)
    sampler.get_train_rays(96, cand)
    first = sampler._valid
    sampler.get_train_rays(96, cand)
    assert sampler._valid is first
    src.pixel_error_maps[cand[1], 2, 3] = -1.0             # in place
    with pytest.raises(RuntimeError, match="probability tensor contains"):
        sampler.get_train_rays(96, cand)
    src.pixel_error_maps = torch.rand_like(src.pixel_error_maps)     # replaced
    sampler.get_train_rays(96, cand)
    assert sampler._valid is not first and sampler._valid[0] is src.pixel_error_maps
    src.pixel_error_maps.mul_(0.0)
    with pytest.raises(RuntimeError, match="sum of probabilities"):
        sampler.get_train_rays(96, cand)

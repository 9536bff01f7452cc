"""``raygen.CameraTrajectory`` on the GPU: emer_trajectory_rays against get_render_rays, the golden file and the
fp64 oracle (oracle/trajectory_ref.py, run on the device's tables).

(a) Keyframes (zero offset) are ``torch.equal`` to ``get_render_rays`` of their image on every shared key, at
    downscales 1, 1/2 and 1/3.
(b) Frames between keyframes match tests/golden/trajectory.npz and the oracle within 1e-5 on view directions and
    norms, 1e-5 max(1, |o|) on origins and 1e-7 on timestamps, at 24 x 40 and on a 640 x 960 source; the pixel
    coordinates match the oracle exactly and the file (host division) within 1e-7.
(c) An item is one library launch and runs under ``torch.cuda.set_sync_debug_mode("error")``.
(d) ``render_rays`` of a keyframe equals ``render_rays`` of ``get_render_rays`` bit for bit for a static, a dynamic
    and a flow field; a mid-segment frame with an offset renders finite outputs of the frame's shape."""
import os

import numpy as np
import pytest
import torch

import trajectory_cases as tc
from oracle import trajectory_ref
from test_trajectory_cpu import DOWNSCALES, check_close, flat, golden, small_models

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trajectory.npz")


def on_device(src):
    for k, v in list(vars(src).items()):
        if isinstance(v, torch.Tensor):
            setattr(src, k, v.to(DEV))
    src.device = torch.device(DEV)
    return src


def source(name, d=1.0):
    return on_device(tc.source(name, d))


def big_source():
    """The "main" poses on a Waymo-sized frame (640 x 960), intrinsics scaled to match."""
    src = tc.source("main")
    h, w = 640, 960
    s = h / tc.HEIGHT
    src.data_cfg.load_size = [h, w]
    g = torch.Generator().manual_seed(12)
    n = len(src.cam_to_worlds)
    src.images = torch.rand(n, h, w, 3, generator=g)
    src.sky_masks = torch.zeros(n, h, w)
    src.intrinsics[:, :2, :] *= s
    return on_device(src)


@pytest.mark.parametrize("d", list(DOWNSCALES))
def test_keyframes_equal_render_rays(d):
    from emernerf_b200 import raygen

    sampler = raygen.PixelRaySampler(source("main", DOWNSCALES[d]))
    traj = raygen.CameraTrajectory(sampler, frames_per_keyframe=3)
    for k in range(len(traj)):
        a, _, i, _ = traj.segment(k)
        if i:
            continue
        got, want = traj[k], sampler.get_render_rays(a)
        assert list(got) == [key for key in want if key in got]
        for key, v in got.items():
            assert v.is_cuda
            if key == "sky_masks":
                assert v.shape == want[key].shape and not v.any()
            else:
                assert v.dtype == want[key].dtype and torch.equal(v, want[key]), (k, key)


@pytest.mark.parametrize("case", list(tc.CASES))
def test_frames_match_golden_and_oracle(case):
    from emernerf_b200 import raygen

    z = np.load(GOLDEN)
    name, d, m, offset = tc.CASES[case]
    src = source(name, d)
    traj = raygen.CameraTrajectory(raygen.PixelRaySampler(src), frames_per_keyframe=m, offset=offset)
    for k in tc.golden_items(case):
        got = traj[k]
        # the file's pixel coordinates are y / h as torch divides on the host; on CUDA torch, as the kernel,
        # multiplies by the rounded reciprocal (rays.cuh, pixel_coord), which the oracle run here pins exactly
        check_close(got, golden(z, case, k), (case, k), rounded=("pixel_coords",))
        a, b, i, c = tc.segment(name, m, k)
        check_close(got, {key: v.cpu() for key, v in trajectory_ref.frame_rays(src, a, b, i, m, c, offset).items()},
                    (case, k, "oracle"))


def test_waymo_sized_frames_match_oracle():
    from emernerf_b200 import raygen

    src = big_source()
    for d in (1.0, 0.5):
        src._downscale_factor = d
        traj = raygen.CameraTrajectory(raygen.PixelRaySampler(src), frames_per_keyframe=4, offset=tc.OFFSET)
        for k in (5, 8, 15, 28, 31, len(traj) - 1):
            a, b, i, c = tc.segment("main", 4, k)
            want = {key: v.cpu() for key, v in trajectory_ref.frame_rays(src, a, b, i, 4, c, tc.OFFSET).items()}
            assert want["origins"].shape == (int(640 * d), int(960 * d), 3)
            check_close(traj[k], want, (d, k))


def test_one_launch_without_a_host_sync():
    from emernerf_b200 import _lib, raygen

    traj = raygen.CameraTrajectory(raygen.PixelRaySampler(source("main", 0.5)), frames_per_keyframe=4,
                                   offset=tc.OFFSET)
    traj[0]                                            # the resize of get_render_rays' images, once per downscale
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for k in (1, 8, 30, len(traj) - 1):
            before = _lib.LAUNCHES
            traj[k]
            assert _lib.LAUNCHES - before == 1
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.parametrize("kind", ["static", "dynamic", "flow"])
def test_render_keyframe_equals_render_of_render_rays(kind):
    from emernerf_b200 import raygen
    from emernerf_b200.radiance_fields.render_utils import render_rays
    import cases

    field, props, est = small_models(kind)
    field, props, est = field.to(DEV), [p.to(DEV) for p in props], est.to(DEV)
    sampler = raygen.PixelRaySampler(source("main", 0.5))
    traj = raygen.CameraTrajectory(sampler, frames_per_keyframe=2, offset=tc.OFFSET)
    plain = raygen.CameraTrajectory(sampler, frames_per_keyframe=2)
    render = lambda data: flat(render_rays(radiance_field=field, proposal_estimator=est, proposal_networks=props,
                                           data_dict=data, cfg=cases.render_cfg(), return_decomposition=True))
    with torch.no_grad():
        for k, img in ((2 * tc.N_CAMS + 1, 4), (len(plain) - 1, 14)):
            got, want = render(plain[k]), render(sampler.get_render_rays(img))
            assert list(got) == list(want)
            for key, v in want.items():
                assert torch.equal(got[key], v), (k, key)
        mid = render(traj[3 * tc.N_CAMS + 2])
    h, w = plain[0]["origins"].shape[:2]
    for key in want:
        if "/" not in key:
            assert mid[key].shape[:2] == (h, w) and torch.isfinite(mid[key]).all(), key

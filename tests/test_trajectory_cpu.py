"""``raygen.CameraTrajectory`` on the host (CPU suite), with emer_trajectory_rays run through
tests/trajectory_emulator.py.

- Keyframes (zero offset) are ``torch.equal`` to ``PixelRaySampler.get_render_rays`` of their image on every shared
  key, at downscales 1, 1/2 and 1/3.
- Frames between keyframes match tests/golden/trajectory.npz (the reference's ``get_rays`` on the fp64-interpolated
  poses) within 1e-5 on view directions and norms, 1e-5 max(1, |o|) on origins and 1e-7 on timestamps; the oracle
  matches the file bit for bit, and its poses take the short way round.
- The item layout, the appearance index, the sky masks, the errors, and one library call per item.
- ``render_rays`` of a keyframe equals ``render_rays`` of ``get_render_rays`` bit for bit, and a mid-segment frame with
  an offset renders finite outputs of the frame's shape."""
import os
import types

import numpy as np
import pytest
import torch

import cabi_emulator
import cases
import trajectory_cases as tc
import trajectory_emulator
from oracle import trajectory_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trajectory.npz")
DOWNSCALES = {"1": 1.0, "1_2": 0.5, "1_3": 1 / 3}


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


@pytest.fixture
def raygen(monkeypatch):
    trajectory_emulator.install(monkeypatch)
    from emernerf_b200 import raygen

    return raygen


def check_close(got, want, where, rounded=()):
    """1e-5 on directions and norms, 1e-5 max(1, |o|) on origins, 1e-7 on timestamps and on the keys in
    ``rounded``; the rest exactly."""
    assert list(got) == list(want), where
    for k, v in want.items():
        g = got[k].cpu()
        assert g.dtype == v.dtype and g.shape == v.shape, (where, k, g.dtype, g.shape)
        if k in ("viewdirs", "direction_norm"):
            assert (g - v).abs().max() <= 1e-5, (where, k)
        elif k == "origins":
            assert ((g - v).abs() <= 1e-5 * v.abs().clamp(min=1)).all(), (where, k)
        elif k == "normed_timestamps" or k in rounded:
            assert (g - v).abs().max() <= 1e-7, (where, k)
        else:
            assert torch.equal(g, v), (where, k)


def golden(z, case, k):
    keys = z[f"{case}/{k}/keys"].tolist()
    return {key: torch.from_numpy(z[f"{case}/{k}/{key}"]) for key in keys}


@pytest.mark.parametrize("d", list(DOWNSCALES))
@pytest.mark.parametrize("m", [1, 3])
def test_keyframes_equal_render_rays(raygen, d, m):
    src = tc.source("main", DOWNSCALES[d])
    sampler = raygen.PixelRaySampler(src)
    traj = raygen.CameraTrajectory(sampler, frames_per_keyframe=m)
    seen = 0
    for k in range(len(traj)):
        a, _, i, _ = traj.segment(k)
        if i:
            continue
        got, want = traj[k], sampler.get_render_rays(a)
        assert list(got) == [key for key in want if key in got]
        for key, v in got.items():
            if key == "sky_masks":
                assert v.shape == want[key].shape and not v.any()
            else:
                assert v.dtype == want[key].dtype and torch.equal(v, want[key]), (k, key)
        seen += 1
    assert seen == tc.N_CAMS * tc.N_TIMESTEPS


@pytest.mark.parametrize("case", list(tc.CASES))
def test_frames_match_golden(z, raygen, case):
    name, d, m, offset = tc.CASES[case]
    traj = raygen.CameraTrajectory(raygen.PixelRaySampler(tc.source(name, d)), frames_per_keyframe=m, offset=offset)
    for k in tc.golden_items(case):
        check_close(traj[k], golden(z, case, k), (case, k))


@pytest.mark.parametrize("case", list(tc.CASES))
def test_oracle_matches_golden(z, case):
    name, d, m, offset = tc.CASES[case]
    src = tc.source(name, d)
    for k in tc.golden_items(case):
        a, b, i, c = tc.segment(name, m, k)
        got, want = trajectory_ref.frame_rays(src, a, b, i, m, c, offset), golden(z, case, k)
        assert list(got) == list(want)
        for key, v in want.items():
            assert torch.equal(got[key], v), (case, k, key)


def test_oracle_poses_take_the_short_way():
    src = tc.source("main")
    c2w = src.cam_to_worlds.numpy()

    def pair(seg):
        c, t = seg
        return c2w[t * tc.N_CAMS + c], c2w[(t + 1) * tc.N_CAMS + c]

    assert trajectory_ref.quat_dot(*pair(tc.NLERP_SEGMENT)) > trajectory_ref.NLERP_DOT
    assert trajectory_ref.quat_dot(*pair(tc.FLIP_SEGMENT)) < -0.99
    assert abs(trajectory_ref.quat_dot(*pair(tc.YAW_SEGMENT))) < trajectory_ref.NLERP_DOT
    mid = lambda seg: trajectory_ref.frame_pose(*pair(seg), 1, 2)[:3, :3]
    assert np.abs(mid(tc.FLIP_SEGMENT) - tc.rot(tc.X, -120)).max() < 1e-6
    assert np.abs(mid(tc.YAW_SEGMENT) - tc.rot(tc.Z, 85) @ tc.FORWARD).max() < 1e-6
    assert np.abs(mid(tc.NLERP_SEGMENT) - pair(tc.NLERP_SEGMENT)[0][:3, :3]).max() < 1e-6
    # the offset moves the origin along the frame's own axes
    A, B = pair(tc.YAW_SEGMENT)
    P = trajectory_ref.frame_pose(A, B, 1, 2, (1.0, 0.0, 0.0))
    assert np.abs(P[:3, 3] - (A[:3, 3] + B[:3, 3]) / 2 - P[:3, 0]).max() < 1e-6


@pytest.mark.parametrize("name,m", [("main", 1), ("main", 3), ("main", 4), ("single", 3)])
def test_layout(raygen, name, m):
    src = tc.source(name)
    traj = raygen.CameraTrajectory(raygen.PixelRaySampler(src), frames_per_keyframe=m)
    assert traj.split == "trajectory" and traj.cams == [0, 1, 2]
    assert len(traj) == tc.num_items(name, m) and traj.num_frames * len(traj.cams) == len(traj)
    for k in range(len(traj)):
        a, b, i, c = tc.segment(name, m, k)
        assert traj.segment(k) == (a, b, i, m)
        r = traj[k]
        assert (r["cam_idx"] == c).all()
        assert (r["img_idx"] == (a if 2 * i <= m else b)).all()
        assert ("sky_masks" in r) == (name == "main") and ("normed_timestamps" in r) == (name == "main")
        if "sky_masks" in r:
            assert r["sky_masks"].shape == (tc.HEIGHT, tc.WIDTH) and not r["sky_masks"].any()
    with pytest.raises(IndexError):
        traj[len(traj)]
    assert torch.equal(traj[-1]["origins"], traj[len(traj) - 1]["origins"])


def test_appearance_index_switches_at_the_midpoint(raygen):
    traj = raygen.CameraTrajectory(raygen.PixelRaySampler(tc.source("main")), frames_per_keyframe=4)
    idx = [int(traj[f * tc.N_CAMS + 1]["img_idx"][0, 0]) for f in range(5)]
    assert idx == [1, 1, 1, 4, 4]                     # frames 0..4 of camera 1: i / 4 <= 0.5 keeps keyframe a


def test_camera_subset(raygen):
    traj = raygen.CameraTrajectory(raygen.PixelRaySampler(tc.source("main")), cams=[2, 0], frames_per_keyframe=2)
    assert len(traj) == 9 * 2
    for k in range(len(traj)):
        assert (traj[k]["cam_idx"] == [2, 0][k % 2]).all()
    assert traj.segment(2) == (2, 5, 1, 2)            # frame 1 of camera 2: timesteps 0 -> 1 at 1/2
    assert traj.segment(5) == (3, 6, 0, 2)            # frame 2 of camera 0: keyframe 1


def test_errors(raygen):
    src = tc.source("main")
    sampler = raygen.PixelRaySampler(src)
    for m in (0, -1, 1.5):
        with pytest.raises(ValueError):
            raygen.CameraTrajectory(sampler, frames_per_keyframe=m)
    for off in ((float("nan"), 0, 0), (0, float("inf"), 0), (0, 0)):
        with pytest.raises(ValueError):
            raygen.CameraTrajectory(sampler, offset=off)
    with pytest.raises(ValueError, match="no camera 3"):
        raygen.CameraTrajectory(sampler, cams=[0, 3])
    src.num_cams = 4
    with pytest.raises(ValueError, match="camera 3 has no image"):
        raygen.CameraTrajectory(sampler, cams=[3])
    with pytest.raises(ValueError, match="no camera 4"):
        raygen.CameraTrajectory(sampler, cams=[4])
    src.cam_ids = torch.tensor([0, 1, 2] * 4 + [0, 1, 1])
    with pytest.raises(ValueError, match="different numbers of images"):
        raygen.CameraTrajectory(sampler)


def test_one_library_call_per_item(raygen):
    traj = raygen.CameraTrajectory(raygen.PixelRaySampler(tc.source("main", 0.5)), frames_per_keyframe=3)
    traj[0]                                            # the resize of get_render_rays' images, once per downscale
    for k in (4, 20, len(traj) - 1):
        del cabi_emulator.CALLS[:]
        traj[k]
        assert cabi_emulator.CALLS == ["emer_trajectory_rays"]


def flat(out, prefix=""):
    """render_rays' outputs with the nested dicts (extras) flattened."""
    res = {}
    for k, v in out.items():
        if isinstance(v, dict):
            res.update(flat(v, f"{prefix}{k}/"))
        elif isinstance(v, torch.Tensor):
            res[prefix + k] = v
    return res


def small_models(kind):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder
    from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    field, props = cases.build_models(ns, kind)
    est = PropNetEstimator(None, None)
    for mod in [field, est] + props:
        mod.eval()
    return field, props, est


@pytest.mark.parametrize("kind", ["static", "dynamic", "flow"])
def test_render_keyframe_equals_render_of_render_rays(raygen, kind):
    from emernerf_b200.radiance_fields.render_utils import render_rays

    field, props, est = small_models(kind)
    sampler = raygen.PixelRaySampler(tc.source("main", 1 / 4))
    traj = raygen.CameraTrajectory(sampler, frames_per_keyframe=2, offset=tc.OFFSET)
    plain = raygen.CameraTrajectory(sampler, frames_per_keyframe=2)
    render = lambda data: flat(render_rays(radiance_field=field, proposal_estimator=est, proposal_networks=props,
                                           data_dict=data, cfg=cases.render_cfg(), return_decomposition=True))
    k = 2 * tc.N_CAMS + 1                              # frame 2 of camera 1: keyframe image 4
    with torch.no_grad():
        got, want = render(plain[k]), render(sampler.get_render_rays(4))
        assert list(got) == list(want)
        for key, v in want.items():
            assert torch.equal(got[key], v), key
        mid = render(traj[3 * tc.N_CAMS + 2])            # frame 3 of camera 2: between timesteps 1 and 2
    h, w = plain[k]["origins"].shape[:2]
    for key in want:
        if "/" not in key:                             # the per-sample extras are [h, w, samples]
            assert mid[key].shape[:2] == (h, w) and torch.isfinite(mid[key]).all(), key

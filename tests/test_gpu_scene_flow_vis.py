"""The scene-flow figure on the H100 (csrc/flow_vis.cu through emernerf_b200.flow_vis):

* golden: ``visualize_scene_flow`` against the reference's own (tests/golden/scene_flow_vis.npz), with the checks of
  tests/test_scene_flow_vis_cpu.py;
* colour kernel: ``scene_flow_to_rgb`` bit for bit against the torch restatement of the reference's function on the
  GPU (oracle.scene_flow_vis_ref) on 2^20 + 3 finite flows, with angles on the wheel's boundaries and radii 0, 1 and
  2 exactly, for both backgrounds, with a given radius and with None; NaN and inf flows against the CPU emulator only;
* select kernel: kept set, order, counts and label colours bit for bit against the oracle's boolean indexes at
  2^21 + 5 points and 3 cameras, the points near an image edge or depth 0 left out;
* end to end: the colours bit for bit against the oracle's loop on the fixture's frames;
* no host sync in the frame loop, the same sync count for 3 drawn frames as for 30, bit-identical repeats, and
  ``scene_flow_to_rgb`` with a given radius in one launch without a sync, and one CUDA kernel (counted by torch.profiler
  in a fresh process).
"""
import math
import os
import types
import warnings

import numpy as np
import pytest
import torch

import lidar_flow_cases as lc
import scene_flow_vis_cases as sc
import scene_flow_vis_emulator as emu
from oracle import scene_flow_vis_ref
from test_scene_flow_vis_cpu import GOLDEN, LIDAR_GOLDEN, check_case, dropin_field

pytestmark = pytest.mark.gpu
DEV = "cuda"


def bits(x):
    return np.ascontiguousarray(np.asarray(x, np.float32)).view(np.int32)


def fixture(case="drive"):
    zl, zs = np.load(LIDAR_GOLDEN), np.load(GOLDEN)
    ds, src = sc.load(zl, zs, case, DEV)
    return zs, ds, src, dropin_field(zl, zs, DEV).eval()


@pytest.mark.parametrize("case", list(sc.CASES))
def test_against_reference_golden(case):
    from emernerf_b200 import flow_vis

    zs, ds, _, field = fixture(case)
    check_case(zs, case, flow_vis.visualize_scene_flow(types.SimpleNamespace(), field, ds, device=DEV))


def crafted_flows(n=(1 << 20) + 3, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    f = torch.randn(n, 3, generator=g, device=DEV) * torch.rand(n, 1, generator=g, device=DEV) * 4.0
    k = torch.arange(4096, device=DEV)
    ang = (k % 55).double() * (2 * math.pi / 54) + (k // 55 % 3 - 1).double() * 1e-7
    rad = torch.tensor([0.5, 1.0, 2.0, 2.5, 7.0], device=DEV, dtype=torch.float64)[k % 5]
    f[:4096, 0] = (rad * torch.cos(ang)).float()
    f[:4096, 1] = (rad * torch.sin(ang)).float()
    edge = torch.tensor([[0.0, 0.0], [-0.0, 0.0], [0.0, -0.0], [1.0, 0.0], [2.0, 0.0], [0.0, 2.0], [-2.0, 0.0],
                         [-2.0, -0.0], [0.0, -2.0], [4.0, 0.0], [-1.0, -0.0], [2.0, -0.0]], device=DEV)
    f[4096:4096 + len(edge), :2] = edge
    return f


@pytest.mark.parametrize("background", ["bright", "dark"])
@pytest.mark.parametrize("radius", [2.0, 0.7, None])
def test_colour_kernel_bit_for_bit(background, radius):
    from emernerf_b200 import flow_vis

    flows = crafted_flows()
    got = flow_vis.scene_flow_to_rgb(flows, flow_max_radius=radius, background=background)
    want = scene_flow_vis_ref.scene_flow_to_rgb(flows.clone(), radius, background)
    torch.cuda.synchronize()
    assert got.dtype == torch.float32 and got.shape == want.shape
    diff = (got.view(torch.int32) != want.view(torch.int32)).any(-1)
    assert not bool(diff.any()), (int(diff.sum()), flows[diff][:4].tolist(), got[diff][:4].tolist(),
                                  want[diff][:4].tolist())


def test_colour_kernel_on_nan_and_inf():
    from emernerf_b200 import flow_vis

    nan, inf = float("nan"), float("inf")
    vals = [nan, inf, -inf, 0.0, -0.0, 1.5, -3.0]
    flows = torch.tensor([[x, y, 0.0] for x in vals for y in vals], device=DEV)
    dens = torch.tensor([0.1, 0.5, nan] * (len(flows) // 3 + 1), device=DEV)[:len(flows)]
    for bg in ("bright", "dark"):
        got = flow_vis.scene_flow_to_rgb(flows, flow_max_radius=2.0, background=bg).cpu().numpy()
        want = emu.flow_rgb(flows[:, 0].cpu().numpy(), flows[:, 1].cpu().numpy(), emu.SCALE_HOST, np.float32(0.5),
                            bg == "bright")
        assert np.array_equal(np.isnan(got), np.isnan(want))
        assert np.nanmax(np.abs(got - want)) <= 3e-6
    out = torch.empty(len(flows), 3, device=DEV)
    flow_vis.color(flows, out, density=dens)
    f = flows.cpu().numpy().copy()
    f[dens.cpu().numpy() < np.float32(0.2)] *= np.float32(0)
    want = emu.flow_rgb(f[:, 0], f[:, 1], emu.SCALE_HOST, np.float32(0.5), True)
    got = out.cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.nanmax(np.abs(got - want)) <= 3e-6


class Cams:
    def __init__(self, n_pos):
        self.num_cams, self.WIDTH, self.HEIGHT = sc.NUM_CAMS, sc.WIDTH, sc.HEIGHT
        self.intrinsics = torch.stack([sc.intrinsics(i % len(sc.SPLIT), c) for i in range(n_pos)
                                       for c in range(sc.NUM_CAMS)]).to(DEV)
        self.cam_to_worlds = torch.stack([sc.cam_to_world(i % len(sc.SPLIT), c) for i in range(n_pos)
                                          for c in range(sc.NUM_CAMS)]).to(DEV)


def test_select_kernel_bit_for_bit():
    from emernerf_b200 import flow_vis

    n = (1 << 21) + 5
    g = torch.Generator(device=DEV).manual_seed(7)
    pix = Cams(1)
    c0 = pix.cam_to_worlds[0, :3, 3]
    origins = c0 + 0.1 * torch.randn(n, 3, generator=g, device=DEV)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g, device=DEV) *
                                         torch.tensor([1.0, 1.0, 0.3], device=DEV), dim=-1)
    ranges = 1.0 + 40.0 * torch.rand(n, 1, generator=g, device=DEV)
    pts64 = (origins + ranges * dirs).double()
    firm = torch.ones(n, dtype=torch.bool, device=DEV)
    for c in range(sc.NUM_CAMS):
        k4 = torch.nn.functional.pad(pix.intrinsics[c].double(), (0, 1, 0, 1))
        k4[3, 3] = 1.0
        l2i = k4 @ torch.linalg.inv(pix.cam_to_worlds[c].double())
        proj = pts64 @ l2i[:3, :3].T + l2i[:3, 3]
        d = proj[:, 2]
        u, v = proj[:, 0] / d, proj[:, 1] / d
        m = 1e-4
        near = (d.abs() <= m * ranges[:, 0]) | (d > 0) & ((u.abs() <= m * sc.WIDTH) | ((u - sc.WIDTH).abs() <= m *
                                                          sc.WIDTH) | (v.abs() <= m * sc.HEIGHT) |
                                                         ((v - sc.HEIGHT).abs() <= m * sc.HEIGHT))
        firm &= ~near
    frame = {"lidar_origins": origins[firm], "lidar_viewdirs": dirs[firm], "lidar_ranges": ranges[firm]}
    m = int(firm.sum())
    frame["lidar_normed_timestamps"] = torch.rand(m, generator=g, device=DEV)
    frame["lidar_flow"] = torch.randn(m, 3, generator=g, device=DEV) * 2.0
    cls = torch.randint(0, 4, (m,), generator=g, device=DEV)
    cls[torch.rand(m, generator=g, device=DEV) < 0.2] = -1
    frame["lidar_flow_class"] = cls
    # the oracle: boolean indexes, the reference's camera mask and colour
    data = {k: v[cls != -1] for k, v in frame.items()}
    mask = scene_flow_vis_ref.get_valid_lidar_mask(pix, 0, data)
    data = {k: v[mask] for k, v in data.items()}
    want_pts = data["lidar_origins"] + data["lidar_ranges"] * data["lidar_viewdirs"]
    want_rgb = scene_flow_vis_ref.scene_flow_to_rgb(data["lidar_flow"], 2.0, "bright")
    points, times, rows9 = (torch.full((m, k), float("nan"), device=DEV) for k in (3, 1, 9))
    counts = torch.zeros(3, dtype=torch.int64, device=DEV)
    counts[2] = 0
    flow_vis.select(frame, flow_vis.lidar2img(pix, 0, sc.NUM_CAMS), sc.WIDTH, sc.HEIGHT, points, times, rows9,
                    counts[2:], counts[:2])
    k = len(want_pts)
    assert counts.tolist() == [int((cls != -1).sum()), k, k]
    assert k > 1000 and k < int((cls != -1).sum())
    assert torch.equal(points[:k].view(torch.int32), want_pts.view(torch.int32))
    assert torch.equal(rows9[:k, :3].view(torch.int32), want_pts.view(torch.int32))
    assert torch.equal(rows9[:k, 6:].view(torch.int32), want_rgb.view(torch.int32))
    assert torch.equal(times[:k, 0].view(torch.int32), data["lidar_normed_timestamps"].view(torch.int32))
    assert bool(torch.isnan(points[k:]).all())


def test_end_to_end_bit_for_bit_and_repeats():
    from emernerf_b200 import flow_vis

    for case in sc.CASES:
        _, ds, _, field = fixture(case)
        got = flow_vis.visualize_scene_flow(types.SimpleNamespace(), field, ds, device=DEV)
        again = flow_vis.visualize_scene_flow(types.SimpleNamespace(), field, ds, device=DEV)
        want = scene_flow_vis_ref.visualize_scene_flow(types.SimpleNamespace(), field, ds, device=DEV)
        for part in ("pred", "gt"):
            assert got[part]["vis_aabb"] == want[part]["vis_aabb"]
            assert [got[part][k] for k in ("x_ratio", "y_ratio", "z_ratio")] == \
                [want[part][k] for k in ("x_ratio", "y_ratio", "z_ratio")]
            for key in ("dynamic_coords", "dynamic_colors"):
                assert len(got[part][key]) == len(want[part][key]) == len(again[part][key])
                for a, b, c in zip(got[part][key], want[part][key], again[part][key]):
                    assert np.array_equal(bits(a), bits(b)), (case, part, key)
                    assert np.array_equal(bits(a), bits(c)), (case, part, key)


def long_drive(n_split):
    zl, zs = np.load(LIDAR_GOLDEN), np.load(GOLDEN)
    _, src = sc.load(zl, zs, "drive", DEV)
    split = [s % lc.N_SCANS for s in range(n_split)]
    ds = types.SimpleNamespace(full_lidar_set=lc.SplitSet(src, split), pixel_source=Cams(n_split))
    return ds, dropin_field(zl, zs, DEV).eval()


def syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message) for w in caught)


def test_no_sync_in_the_frame_loop_and_a_fixed_sync_count():
    from emernerf_b200 import flow_vis, metrics

    ds, field = long_drive(301)
    cfg = types.SimpleNamespace()
    flow_vis.visualize_scene_flow(cfg, field, ds, device=DEV)               # the frame table exists from here on
    src = ds.full_lidar_set.datasource
    sampler = metrics._lidar_sampler(src)
    cap = len(src.timesteps)
    points, times, rows9 = torch.empty(cap, 3, device=DEV), torch.empty(cap, device=DEV), torch.empty(cap, 9,
                                                                                                       device=DEV)
    counts = torch.zeros(2 * 30 + 1, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for f, i in enumerate(range(0, 300, 10)):
            frame = sampler.get_render_rays(ds.full_lidar_set.split_indices[i])
            flow_vis.select(frame, flow_vis.lidar2img(ds.pixel_source, i, sc.NUM_CAMS), sc.WIDTH, sc.HEIGHT,
                            points, times, rows9, counts[60:], counts[2 * f:2 * f + 2])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    few, _ = long_drive(31)
    flow_vis.visualize_scene_flow(cfg, field, few, device=DEV)
    n_few = syncs(lambda: flow_vis.visualize_scene_flow(cfg, field, few, device=DEV))
    n_many = syncs(lambda: flow_vis.visualize_scene_flow(cfg, field, ds, device=DEV))
    assert n_few == n_many


def test_scene_flow_to_rgb_is_one_launch_without_a_sync():
    from emernerf_b200 import _lib, flow_vis

    flows = crafted_flows(5000)
    flow_vis.scene_flow_to_rgb(flows, flow_max_radius=2.0)
    torch.cuda.synchronize()
    before = _lib.LAUNCHES
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = flow_vis.scene_flow_to_rgb(flows, flow_max_radius=2.0, background="bright")
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _lib.LAUNCHES - before == 1, _lib.LAUNCHES - before
    assert out.shape == (5000, 3)


# The kernels a call runs, counted by torch.profiler in a process of its own: after other profiler sessions in a
# long-lived process, CUPTI can hand the profiler no GPU activity at all, which would make any count meaningless.
_COUNT_KERNELS = """
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
from emernerf_b200 import flow_vis
flows = torch.randn(5000, 3, device="cuda")
flow_vis.scene_flow_to_rgb(flows, flow_max_radius=2.0)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    flow_vis.scene_flow_to_rgb(flows, flow_max_radius=2.0, background="bright")
    torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                  and not e.name.startswith(("Memcpy", "Memset"))]))
"""


def test_scene_flow_to_rgb_runs_one_kernel():
    import json
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _COUNT_KERNELS, root], cwd=root, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    kernels = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(kernels) == 1 and "flow_vis_color" in kernels[0], kernels

"""The scene-flow figure of emernerf_b200.flow_vis on the host (CPU suite): ``visualize_scene_flow`` runs the drop-in
field through tests/cabi_emulator.py and the two kernels through tests/scene_flow_vis_emulator.py, and is checked
against the reference's own ``visualize_scene_flow`` (tests/golden/scene_flow_vis.npz, make_golden_scene_flow_vis.py):
the box and ratios exactly, the drawn frames' points kept and ordered as the reference keeps them, their coordinates
bit for bit, the label colours within COLOR_TOL = 3e-6 (the reference's CPU path divides where torch's CUDA path
multiplies by a reciprocal, and glibc's hypot and atan2 may differ from libdevice's by an ulp or two, which the wheel's
lerp amplifies: the bound is derived below), and the predicted colours within 1e-5 (the drop-in field's flows agree
with the reference field's to fp32 rounding).  Also ``scene_flow_to_rgb`` against the
reference's function, NaN and inf flows, empty frames, and the errors.
"""
import logging
import os
import types

import numpy as np
import pytest
import torch

import lidar_flow_cases as lc
import scene_flow_vis_cases as sc
import scene_flow_vis_emulator as emu
from oracle import scene_flow_vis_ref

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "scene_flow_vis.npz")
LIDAR_GOLDEN = os.path.join(HERE, "golden", "lidar_flow.npz")
ULPS = 2
# a 2-ulp difference in atan2 moves the scaled angle by at most 2 ulp(54) = 7.6e-6 and the hue by 63.75 times that (the
# steepest wheel transition, 255 over 4 entries), 1.9e-6 after / 255; a 2-ulp radius moves a colour by 2.4e-7
COLOR_TOL = 3e-6
PRED_TOL = 1e-5


@pytest.fixture
def flow_vis(monkeypatch):
    emu.install(monkeypatch)
    from emernerf_b200 import flow_vis

    return flow_vis


def dropin_field(zl, zs, device="cpu"):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    field = lc.fixture_field(ns, float(zl["density_shift"]))
    assert sorted(k for k, _ in field.named_parameters()) == zs["parameters"].tolist()
    return field.to(device)


def close_colors(got, want, tol=None):
    """Within COLOR_TOL of the reference's colours (or ``tol``), NaN where the reference has NaN."""
    close_abs(np.asarray(got, np.float32), np.asarray(want, np.float32), COLOR_TOL if tol is None else tol)


def close_ulps(got, want, ulps=ULPS):
    """Within ``ulps`` fp32 spacings of the larger magnitude, NaN where the reference has NaN."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    tol = ulps * np.spacing(np.maximum(np.abs(got), np.abs(want)).astype(np.float32))
    bad = np.abs(got[~nan].astype(np.float64) - want[~nan]) > tol[~nan]
    assert not bad.any(), (got[~nan][bad][:5], want[~nan][bad][:5])


def close_abs(got, want, tol):
    assert got.shape == want.shape and np.array_equal(np.isnan(got), np.isnan(want))
    assert np.nanmax(np.abs(got.astype(np.float64) - want), initial=0) <= tol


def check_case(zs, case, got):
    pred, gt = got["pred"], got["gt"]
    assert pred["dynamic_coords"] is gt["dynamic_coords"]
    for kw in (pred, gt):
        assert kw["vis_aabb"] == zs[f"{case}/vis_aabb"].tolist()
        assert [kw["x_ratio"], kw["y_ratio"], kw["z_ratio"]] == zs[f"{case}/ratios"].tolist()
    n = int(zs[f"{case}/frames"])
    assert len(pred["dynamic_coords"]) == len(pred["dynamic_colors"]) == len(gt["dynamic_colors"]) == n
    for f in range(n):
        c = pred["dynamic_coords"][f]
        assert c.dtype == np.float32 and pred["dynamic_colors"][f].dtype == np.float32
        assert np.array_equal(c.view(np.int32), zs[f"{case}/frame{f}/coords"].view(np.int32)), (case, f)
        close_colors(gt["dynamic_colors"][f], zs[f"{case}/frame{f}/gt"])
        # the prediction comes from the drop-in field, whose flows agree with the reference field's to fp32 rounding
        close_abs(pred["dynamic_colors"][f], zs[f"{case}/frame{f}/pred"], PRED_TOL)


def run(flow_vis, case, device="cpu"):
    zl, zs = np.load(LIDAR_GOLDEN), np.load(GOLDEN)
    ds, _ = sc.load(zl, zs, case, device)
    return zs, flow_vis.visualize_scene_flow(types.SimpleNamespace(), dropin_field(zl, zs, device), ds,
                                             device=device)


@pytest.mark.parametrize("case", list(sc.CASES))
def test_against_reference_golden(flow_vis, case):
    zs, got = run(flow_vis, case)
    check_case(zs, case, got)


def test_skipped_frame_is_logged(flow_vis, caplog):
    """Position 10 of the drive is its scan without labels: skipped before the camera mask, with the reference's
    message."""
    with caplog.at_level(logging.INFO):
        zs, got = run(flow_vis, "drive")
    assert "no valid points, skipping..." in caplog.text
    assert len(got["pred"]["dynamic_coords"]) == 2


def test_frames_in_chunks(flow_vis, monkeypatch):
    from emernerf_b200 import metrics

    monkeypatch.setattr(metrics, "FLOW_CHUNK_POINTS", 37)
    zs, got = run(flow_vis, "unsorted")
    check_case(zs, "unsorted", got)


def test_wheel_is_the_references():
    zs = np.load(GOLDEN)
    assert np.array_equal(scene_flow_vis_ref.WHEEL.numpy(), zs["wheel"])


@pytest.mark.parametrize("background", ["bright", "dark"])
@pytest.mark.parametrize("radius", ["r2", "quantile"])
def test_scene_flow_to_rgb_is_the_references(flow_vis, background, radius):
    zs = np.load(GOLDEN)
    flows = torch.from_numpy(zs["rgb/flows"])
    got = flow_vis.scene_flow_to_rgb(flows, flow_max_radius=2.0 if radius == "r2" else None, background=background)
    assert got.dtype == torch.float32 and got.shape == flows.shape
    close_colors(got.numpy(), zs[f"rgb/{background}/{radius}"])
    # the torch restatement of the oracle is the reference's function as well
    want = scene_flow_vis_ref.scene_flow_to_rgb(flows.clone(), 2.0 if radius == "r2" else None, background)
    close_ulps(want.numpy(), zs[f"rgb/{background}/{radius}"], 0)


def test_scene_flow_to_rgb_shapes_and_radii(flow_vis):
    g = torch.Generator().manual_seed(3)
    flows = torch.randn(4, 5, 3, generator=g)
    for r in (0.5, 3.0, torch.tensor(1.5), 0.0, -1.0):
        got = flow_vis.scene_flow_to_rgb(flows, flow_max_radius=r, background="bright")
        want = scene_flow_vis_ref.scene_flow_to_rgb(flows.clone(), r, "bright")
        assert got.shape == (4, 5, 3)
        close_colors(got.numpy(), want.numpy())


def test_nan_and_inf_flows(flow_vis):
    nan, inf = float("nan"), float("inf")
    flows = torch.tensor([[nan, 0.0, 0.0], [0.0, nan, 0.0], [inf, 0.0, 0.0], [-inf, 0.0, 0.0], [0.0, inf, 0.0],
                          [inf, inf, 0.0], [1.0, 1.0, nan]])
    got = flow_vis.scene_flow_to_rgb(flows, flow_max_radius=2.0, background="bright").numpy()
    assert np.isnan(got[[0, 1, 4, 5]]).all()           # a NaN angle (an infinite y makes the real part NaN)
    # an infinite x: radius inf, angle 0 or pi, 1 / inf = 0, so V-axis colours of 0
    assert np.array_equal(got[2], [0, 0, 0]) and np.array_equal(got[3], [0, 0, 0])
    assert not np.isnan(got[6]).any()                  # z does not enter the colour
    dark = flow_vis.scene_flow_to_rgb(flows, flow_max_radius=2.0, background="dark").numpy()
    assert np.array_equal(dark[2], [1, 1, 1])          # 255 - 0 * (255 - hue)


def test_gate_on_nan_and_inf(flow_vis):
    """pred[density < 0.2] *= 0: NaN stays NaN, inf becomes NaN, a NaN density does not gate."""
    nan, inf = float("nan"), float("inf")
    flows = torch.tensor([[nan, 1.0, 0.0], [inf, 0.0, 0.0], [1.0, 1.0, 0.0], [1.0, 1.0, 0.0], [-1.0, 0.5, 0.0]])
    dens = torch.tensor([0.1, 0.1, 0.1, nan, 0.1])
    out = torch.empty(5, 3)
    flow_vis.color(flows, out, density=dens)
    got = out.numpy()
    assert np.isnan(got[0]).all() and np.isnan(got[1]).all()
    assert np.array_equal(got[2], [1, 1, 1]) and np.array_equal(got[4], [1, 1, 1])   # gated to zero: white
    want = flow_vis.scene_flow_to_rgb(flows[3:4], flow_max_radius=2.0, background="bright").numpy()
    assert np.array_equal(got[3:4], want)


def test_frame_without_points_in_view(flow_vis, monkeypatch):
    """Labelled points that no camera sees give empty (0, 3) arrays (the reference's query_flow fails there)."""
    zl, zs = np.load(LIDAR_GOLDEN), np.load(GOLDEN)
    ds, _ = sc.load(zl, zs, "drive")
    ds.pixel_source.cam_to_worlds[:, :3, 3] += 1e4          # every camera far away, looking past the points
    got = flow_vis.visualize_scene_flow(types.SimpleNamespace(), dropin_field(zl, zs), ds, device="cpu")
    assert len(got["pred"]["dynamic_coords"]) == 2
    for c, p, g in zip(got["pred"]["dynamic_coords"], got["pred"]["dynamic_colors"], got["gt"]["dynamic_colors"]):
        assert c.shape == p.shape == g.shape == (0, 3)


def test_argument_errors(flow_vis):
    with pytest.raises(ValueError, match="background should be one the following"):
        flow_vis.scene_flow_to_rgb(torch.zeros(3, 3), background="grey")
    with pytest.raises(ValueError):
        flow_vis.scene_flow_to_rgb(torch.zeros(3, 1))
    zl, zs = np.load(LIDAR_GOLDEN), np.load(GOLDEN)
    ds, src = sc.load(zl, zs, "drive")
    src.flows = None
    with pytest.raises(ValueError, match="flows"):
        flow_vis.visualize_scene_flow(types.SimpleNamespace(), dropin_field(zl, zs), ds)
    field = dropin_field(zl, zs)
    field.flow_xyz_encoder = None
    with pytest.raises(ValueError, match="flow branch"):
        flow_vis.visualize_scene_flow(types.SimpleNamespace(), field, sc.load(zl, zs, "drive")[0])


def test_cpu_tensors_are_refused():
    from emernerf_b200 import flow_vis

    with pytest.raises(ValueError, match="CUDA"):
        flow_vis.scene_flow_to_rgb(torch.zeros(4, 3))

"""The voxel lifting of emernerf_b200.voxels on the host (CPU suite): ``visualize_voxels`` runs the drop-in field and
renderer through tests/cabi_emulator.py and the voxel kernels through tests/voxels_emulator.py, and is checked against
the reference's own ``visualize_voxels`` (tests/golden/voxels.npz, make_golden_voxels.py) with the reference's PCA:
the box and ratios exactly; per grid, every voxel produced is one the reference's rays can reach, every firm voxel
away from the density threshold is kept exactly when the reference keeps it, in the reference's order, with its
colour to 1e-4.  Also ``robust_pca`` against the reference's ``get_robust_pca``, the dynamic grouping, and the errors.
"""
import os
import types

import numpy as np
import pytest
import torch

import voxel_cases as vc
import voxels_emulator

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxels.npz")
COLOR_TOL = 1e-4


@pytest.fixture
def voxels(monkeypatch):
    voxels_emulator.install(monkeypatch)
    from emernerf_b200 import voxels

    return voxels


def dropin_models(z, case, device="cpu", shifts=None):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder
    from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    shifts = tuple(z[f"{case}/shifts"].tolist()) if shifts is None else shifts
    field, props = vc.build_models(ns, vc.CASES[case]["model"], shifts)
    assert sorted(k for k, _ in field.named_parameters()) == z[f"{case}/parameters"].tolist()
    return field.to(device), [p.to(device) for p in props], PropNetEstimator(None, None).to(device)


def golden_pca(z, case, device):
    p = torch.from_numpy(z[f"{case}/pca"]).to(device)
    return p[:-2], p[-2], p[-1]


def run(voxels, monkeypatch, z, case, device="cpu"):
    field, props, est = dropin_models(z, case, device)
    monkeypatch.setattr(voxels, "robust_pca", lambda features, m=2.5: golden_pca(z, case, features.device))
    return voxels.visualize_voxels(vc.render_cfg(), field, est, props, vc.dataset(case, device), device=device,
                                   is_dynamic=vc.CASES[case]["dynamic"])


def check_grid(z, key, coords, colors, thr):
    """The checks of one grid's produced points against the golden's voxels of that grid."""
    vox, firm, gate = z[f"{key}/vox"], z[f"{key}/firm"], z[f"{key}/gate"]
    band, want_colors = z[f"{key}/band"], z[f"{key}/colors"]
    where = {tuple(c.tolist()): i for i, c in enumerate(z[f"{key}/coords"].astype(np.float32))}
    rows = []
    for c in coords.astype(np.float32):
        assert tuple(c.tolist()) in where, f"{key}: voxel {c} is one no reference ray reaches"
        rows.append(where[tuple(c.tolist())])
    rows = np.array(rows, np.int64)
    assert (np.diff(vox[rows]) > 0).all(), f"{key}: not in linear-index order"
    assert ((gate[rows] > thr) | band[rows]).all(), f"{key}: a voxel at or below the threshold was kept"
    must = np.nonzero(firm & (gate > thr) & ~band)[0]
    assert set(must.tolist()) <= set(rows.tolist()), f"{key}: a firm voxel above the threshold is missing"
    assert np.abs(colors - want_colors[rows]).max(initial=0) <= COLOR_TOL
    return rows


def check_case(z, case, got):
    assert got["vis_aabb"] == z[f"{case}/vis_aabb"].tolist()
    assert [got["x_ratio"], got["y_ratio"], got["z_ratio"]] == z[f"{case}/ratios"].tolist()
    assert got["coords"].dtype == np.float32 and got["colors"].shape == got["coords"].shape
    check_grid(z, f"{case}/static", got["coords"], got["colors"], 0.5)
    if not vc.CASES[case]["dynamic"]:
        assert got["dynamic_coords"] is None and got["dynamic_colors"] is None
        return
    live = []
    for j in z[f"{case}/groups"].tolist():
        key = f"{case}/group{j}"
        gate, band, firm = z[f"{key}/gate"], z[f"{key}/band"], z[f"{key}/firm"]
        if (firm & (gate > 0.1) & ~band).any():
            live.append(key)
        else:
            assert not ((gate > 0.1) | band).any(), f"{key}: whether the group is empty is not pinned"
    assert len(got["dynamic_coords"]) == len(live) == int(z[f"{case}/ref_dynamic_groups"])
    for key, c, col in zip(live, got["dynamic_coords"], got["dynamic_colors"]):
        check_grid(z, key, c, col, 0.1)


@pytest.mark.parametrize("case", list(vc.CASES))
def test_against_reference_golden(voxels, monkeypatch, case):
    z = np.load(GOLDEN)
    got = run(voxels, monkeypatch, z, case)
    check_case(z, case, got)
    # the reference's own kept points, where they are pinned, are produced bit for bit
    assert np.isin(z[f"{case}/ref_coords"].view(np.int32).reshape(-1, 3)[:, 0],
                   got["coords"].view(np.int32)[:, 0]).mean() > 0.9


def test_static_chunks_keep_the_order(voxels, monkeypatch):
    """Static candidates split into chunks that divide nothing: the same points, in the same order."""
    z = np.load(GOLDEN)
    monkeypatch.setattr(voxels, "CHUNK", 37)
    check_case(z, "dynamic_3cam", run(voxels, monkeypatch, z, "dynamic_3cam"))


def test_robust_pca_is_the_references():
    from emernerf_b200.voxels import robust_pca

    z = np.load(GOLDEN)
    for case in vc.CASES:
        torch.manual_seed(int(z[f"{case}/pca_seed"]))
        basis, lo, hi = robust_pca(torch.from_numpy(z[f"{case}/pca_features"]), m=2.5)
        want = torch.from_numpy(z[f"{case}/pca"])
        assert torch.equal(basis, want[:-2]) and torch.equal(lo, want[-2]) and torch.equal(hi, want[-1])


@pytest.mark.parametrize("n_images,cams", [(1, 1), (2, 1), (12, 1), (13, 1), (34, 3), (35, 3), (4, 3), (3, 3),
                                           (62, 3), (200, 5)])
def test_groups_follow_the_reference_loop(n_images, cams):
    from emernerf_b200.voxels import group_of, queried_groups

    groups, current = [], []
    for i in range(n_images):                      # the reference's flush rule, restated
        current.append(i)
        if i % cams == 0 and i > 0:
            groups.append(current)
            current = []
    assert queried_groups(n_images, cams) == [j for j in range(len(groups)) if j % 10 == 0]
    for j, imgs in enumerate(groups):
        assert all(group_of(i, cams) == j for i in imgs)
    assert all(group_of(i, cams) >= len(groups) for i in current)


def test_no_kept_static_voxel_raises(voxels, monkeypatch):
    z = np.load(GOLDEN)
    field, props, est = dropin_models(z, "static_1cam", shifts=(40.0, 0.0))
    monkeypatch.setattr(voxels, "robust_pca", lambda features, m=2.5: golden_pca(z, "static_1cam", "cpu"))
    with pytest.raises(RuntimeError, match="torch.cat"):
        voxels.visualize_voxels(vc.render_cfg(), field, est, props, vc.dataset("static_1cam"), device="cpu")


@pytest.mark.parametrize("bad", ["voxel_size", "too_many_voxels", "channels", "wide"])
def test_argument_errors(voxels, bad):
    z = np.load(GOLDEN)
    field, props, est = dropin_models(z, "static_1cam")
    cfg = vc.render_cfg()
    if bad in ("voxel_size", "too_many_voxels"):
        if bad == "voxel_size":
            del cfg.render.vis_voxel_size
        else:
            cfg.render.vis_voxel_size = 0.01        # 10100 x 8200 x 2200 voxels
        with pytest.raises(ValueError):
            voxels.visualize_voxels(cfg, field, est, props, vc.dataset("static_1cam"), device="cpu")
        return
    c = 6 if bad == "channels" else 260
    n = 5
    pts, out = torch.zeros(n, 3), torch.zeros(n, 3)
    with pytest.raises(ValueError):
        voxels.select([torch.ones(n)], 0.5, pts, torch.zeros(n, c), torch.zeros(c, 3), torch.zeros(3), torch.ones(3),
                      out, out.clone(), torch.zeros(1, dtype=torch.int64))


def test_cpu_tensors_are_refused():
    from emernerf_b200 import voxels

    z = np.load(GOLDEN)
    field, props, est = dropin_models(z, "static_1cam")
    with pytest.raises(ValueError, match="CUDA"):
        voxels.visualize_voxels(vc.render_cfg(), field, est, props, vc.dataset("static_1cam"), device="cpu")

"""Generate tests/golden/scene_flow_vis.npz by running the REFERENCE's own ``visualize_scene_flow`` and
``scene_flow_to_rgb`` on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_scene_flow_vis.py

``utils/visualization_tools.py`` is loaded unmodified by ``make_golden_voxels.load_visualization_tools``, with its
``vis_occ_plotly`` replaced by a recorder of its arguments.  The lidar source and split wrapper are the reference's
(``make_golden_lidar_flow``), and the dataset's ``get_valid_lidar_mask`` is the reference's Waymo method, compiled on
its own from datasets/waymo.py (that module needs video libraries) and bound to the fixture dataset.  For each case of
``scene_flow_vis_cases`` the generator first marks the candidates within 1e-4 relative of an image edge or of depth 0
in a camera of a drawn position (fp64 projection of the fp32 points) as not firm, drops them, and runs the reference.
It stores per case the firm masks, the box and ratios, and per drawn frame the reference's coordinates, predicted and
label colours; and ``scene_flow_to_rgb`` of a set of flows for both backgrounds, with radius 2 and with None.
"""
from __future__ import annotations

import ast
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden_lidar_flow as mglf  # noqa: E402  (installs oracle.ref_shims, imports the reference's field)
import make_golden_occ as mgo  # noqa: E402
import make_golden_voxels as mgv  # noqa: E402

import lidar_flow_cases as lc  # noqa: E402
import scene_flow_vis_cases as sc  # noqa: E402
from oracle import ref_shims  # noqa: E402

FRAMES = list(range(0, len(sc.SPLIT) - 1, 10))


def reference_valid_lidar_mask():
    """The reference's WaymoDataset.get_valid_lidar_mask, compiled from its source on its own."""
    path = os.path.join(ref_shims.REFERENCE_ROOT, "datasets", "waymo.py")
    tree = ast.parse(open(path).read())
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name == "get_valid_lidar_mask":
            mod = ast.Module(body=[node], type_ignores=[])
            ns = {"torch": torch}
            exec(compile(mod, path, "exec"), ns)
            return ns["get_valid_lidar_mask"]
    raise AssertionError("get_valid_lidar_mask not found")


def firm_masks(keeps, labels, source, pix):
    """Per scan, per kept candidate: False when it lies within MARGIN of an image edge or of depth 0 in a camera of
    a drawn position that shows its scan."""
    out = {}
    for s in range(lc.N_SCANS):
        c = lc.candidates(source, s)
        k = keeps[s]
        pts = (c["origins"][k] + c["ranges"][k] * c["directions"][k]).double()
        firm = torch.ones(len(pts), dtype=torch.bool)
        for i in FRAMES:
            if sc.SPLIT[i] != s:
                continue
            for cam in range(sc.NUM_CAMS):
                img = i * sc.NUM_CAMS + cam
                k4 = torch.nn.functional.pad(pix.intrinsics[img].double(), (0, 1, 0, 1))
                k4[3, 3] = 1.0
                l2i = k4 @ torch.linalg.inv(pix.cam_to_worlds[img].double())
                proj = (l2i[:3, :3] @ pts.T + l2i[:3, 3:4]).T
                d = proj[:, 2]
                u, v = proj[:, 0] / d, proj[:, 1] / d
                near = (d.abs() <= sc.MARGIN * pts.norm(dim=-1)) | (d > 0) & (
                    (u.abs() <= sc.MARGIN * sc.WIDTH) | ((u - sc.WIDTH).abs() <= sc.MARGIN * sc.WIDTH)
                    | (v.abs() <= sc.MARGIN * sc.HEIGHT) | ((v - sc.HEIGHT).abs() <= sc.MARGIN * sc.HEIGHT))
                firm &= ~near
        out[s] = firm.numpy()
    return out


def coverage(pix, src, store, case):
    """Counts of the camera outcomes the fixture must contain, from the reference's own arithmetic."""
    behind = outside = twice = 0
    for i in FRAMES:
        d = src.get_render_rays(sc.SPLIT[i])
        d = {k: v[d["lidar_flow_class"] != -1] for k, v in d.items()}
        if not len(d["lidar_origins"]):
            continue
        pts = d["lidar_origins"] + d["lidar_ranges"] * d["lidar_viewdirs"]
        seen = torch.zeros(len(pts), dtype=torch.int64)
        for cam in range(sc.NUM_CAMS):
            img = i * sc.NUM_CAMS + cam
            k4 = torch.nn.functional.pad(pix.intrinsics[img], (0, 1, 0, 1))
            k4[3, 3] = 1.0
            l2i = k4 @ pix.cam_to_worlds[img].inverse()
            proj = (l2i[:3, :3] @ pts.T + l2i[:3, 3:4]).T
            behind += int((proj[:, 2] <= 0).sum())
            uv = proj[:, :2] / (proj[:, 2:] + 1e-6)
            ok = (uv[:, 0] >= 0) & (uv[:, 0] < sc.WIDTH) & (uv[:, 1] >= 0) & (uv[:, 1] < sc.HEIGHT) & (proj[:, 2] > 0)
            outside += int(((proj[:, 2] > 0) & ~ok).sum())
            seen += ok.long()
        twice += int((seen >= 2).sum())
    store[f"{case}/coverage"] = np.array([behind, outside, twice], np.int64)
    return behind, outside, twice


def rgb_flows() -> torch.Tensor:
    """Flows for scene_flow_to_rgb: both signs of x and y, radius 0, the branch cut, x only, long and short."""
    g = torch.Generator().manual_seed(11)
    f = torch.randn(997, 3, generator=g) * torch.rand(997, 1, generator=g) * 4.0
    f[:9, :2] = torch.tensor([[0.0, 0.0], [-0.0, 0.0], [-1.0, 0.0], [-1.0, -0.0], [2.0, 0.0], [0.0, 2.0],
                              [-3.0, -0.0], [0.5, -0.0], [0.0, -0.7]])
    return f


def main():
    assert ref_shims.reference_available(), "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
    torch.set_num_threads(1)
    vt = mgv.load_visualization_tools()
    ls, sw = mglf.load_base("lidar_source"), mglf.load_base("split_wrapper")
    zl = np.load(os.path.join(HERE, "lidar_flow.npz"))
    field = lc.fixture_field(mgo.REF, float(zl["density_shift"]))
    mask_fn = reference_valid_lidar_mask()
    store = {"parameters": np.array(sorted(k for k, _ in field.named_parameters())),
             "wheel": vt.WHEEL.numpy()}
    for case, source in sc.CASES.items():
        keeps, labels = sc.base_scans(zl, source)
        pix = sc.PixelSource()
        firm = firm_masks(keeps, labels, source, pix)
        for s in range(lc.N_SCANS):
            store[f"{case}/scan{s}/firm"] = firm[s]
        keeps, labels = sc.drop(keeps, labels, firm)
        src = lc.fill(mglf.waymo_source(ls), source, keeps, labels)
        ds = types.SimpleNamespace(full_lidar_set=sw.SplitWrapper(src, split_indices=sc.SPLIT, split="full"),
                                   pixel_source=pix)
        ds.get_valid_lidar_mask = types.MethodType(mask_fn, ds)
        calls = []

        def plot(**kw):
            calls.append(kw)
            return types.SimpleNamespace(write_html=lambda path: None)

        vt.vis_occ_plotly = plot
        vt.visualize_scene_flow(types.SimpleNamespace(log_dir="."), field, ds, device="cpu", save_html=False)
        pred, gt = calls
        assert pred["dynamic_coords"] is gt["dynamic_coords"]
        store[f"{case}/vis_aabb"] = np.array(pred["vis_aabb"], np.float64)
        store[f"{case}/ratios"] = np.array([pred["x_ratio"], pred["y_ratio"], pred["z_ratio"]], np.float64)
        store[f"{case}/frames"] = np.array(len(pred["dynamic_coords"]))
        for f, (c, p, g) in enumerate(zip(pred["dynamic_coords"], pred["dynamic_colors"], gt["dynamic_colors"])):
            store[f"{case}/frame{f}/coords"] = c
            store[f"{case}/frame{f}/pred"] = p
            store[f"{case}/frame{f}/gt"] = g
        b = coverage(pix, src, store, case)
        print(f"{case}: {len(pred['dynamic_coords'])} frames of {[len(c) for c in pred['dynamic_coords']]} points; "
              f"dropped {sum(int((~firm[s]).sum()) for s in firm)}; behind / outside / twice {b}")
        assert min(b) > 0
    flows = rgb_flows()
    store["rgb/flows"] = flows.numpy()
    for bg in ("bright", "dark"):
        for r, name in ((2.0, "r2"), (None, "quantile")):
            store[f"rgb/{bg}/{name}"] = vt.scene_flow_to_rgb(flows.clone(), flow_max_radius=r, background=bg).numpy()
    path = os.path.join(HERE, "scene_flow_vis.npz")
    np.savez_compressed(path, **store)
    print(f"wrote {path}: {len(store)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()

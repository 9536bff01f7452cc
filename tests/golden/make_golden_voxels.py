"""Generate tests/golden/voxels.npz by running the REFERENCE's own ``visualize_voxels`` on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_voxels.py

``utils/visualization_tools.py`` is loaded unmodified with the stand-ins of ``oracle.ref_shims`` and stubs for plotly,
matplotlib and pyquaternion (which the lifting does not use).  Its ``vis_occ_plotly`` is replaced by a recorder that
keeps the arguments and stops the run before the figure; ``get_robust_pca`` and ``render_rays`` are wrapped to record
the PCA and each image's depths.  For every case of ``voxel_cases`` the generator picks the density shifts (the static
gate's median at 0.5, the dynamic density's at 1, or far below 0.1), runs the reference, and writes per grid (the
static grid, then each queried dynamic group):

  * ``vox``: the linear indices of the voxels a drop-in may produce, ``firm``: whether a ray whose q lies more than
    1e-4 from an integer on every axis (and, static, whose depth is not within 1e-4 relative of 80) hits it; the other
    voxels are the ones such a ray could reach on either side of its near boundaries;
  * ``gate``: the reference's gated density there (the static mean over the proposal networks and the field in the
    reference's chunks, or the dynamic density at the group's timestamp), ``band``: within 1e-4 relative of the
    threshold, ``colors``: the reference's PCA colours there;

and the reference's own ``vis_occ_plotly`` arguments, its PCA output with the features and seed it came from, and
each image's depths.
"""
from __future__ import annotations

import importlib.util
import math
import os
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

warnings.filterwarnings("ignore")

from oracle import ref_shims  # noqa: E402

ref_shims.install()

import voxel_cases as vc  # noqa: E402
from radiance_fields import RadianceField, build_density_field  # noqa: E402  (reference)
from radiance_fields.encodings import HashEncoder  # noqa: E402  (reference)
from third_party.nerfacc_prop_net import PropNetEstimator  # noqa: E402  (reference)

REF = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                            build_density_field=build_density_field)
PCA_SEED = 1234
DYNAMIC_MEDIAN = 1.0         # thinner dynamic fields put every dynamic depth outside the box


class _Stop(Exception):
    pass


def load_visualization_tools():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    mpl = mod("matplotlib")
    mpl.__path__ = []
    mpl.cm = mod("matplotlib.cm", get_cmap=lambda name: None)
    plotly = mod("plotly")
    plotly.__path__ = []
    plotly.graph_objects = mod("plotly.graph_objects", Figure=object)
    mod("pyquaternion", Quaternion=object)
    ds = mod("datasets", SceneDataset=object)
    ds.__path__ = [os.path.join(ref_shims.REFERENCE_ROOT, "datasets")]
    ut = mod("utils")
    ut.__path__ = [os.path.join(ref_shims.REFERENCE_ROOT, "utils")]
    spec = importlib.util.spec_from_file_location(
        "reference_visualization_tools", os.path.join(ref_shims.REFERENCE_ROOT, "utils", "visualization_tools.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def box(field, voxel_size):
    """The reference's box, resolutions, voxel sizes (as visualize_voxels / world_coords_to_voxel_coords compute
    them on CPU)."""
    a = torch.tensor(field.aabb)
    a[1:3] -= 1
    a[3:] += 1
    lo, hi = torch.split(a, 3, dim=-1)
    res_s = torch.ceil((hi - lo) / voxel_size).long()
    res_d = torch.ceil((hi - lo) / voxel_size * 0.8).long()
    return a, lo, hi, res_s, res_d


def static_gate(field, props, pts):
    """The reference's static gate values, chunk by chunk of 2^18."""
    out = []
    with torch.no_grad():
        for s in range(0, len(pts), 2 ** 18):
            x = pts[s:s + 2 ** 18]
            d = [p(x)["density"].squeeze(-1) for p in props] + [field.forward(x, query_feature_head=False)["density"]]
            out.append(torch.stack(d, 0).mean(0))
    return torch.cat(out) if out else torch.zeros(0)


def dynamic_gate(field, pts, t):
    with torch.no_grad():
        r = field.forward(pts, data_dict={"normed_timestamps": t.repeat(len(pts), 1)}, query_feature_head=False)
    return r["dynamic_density"].squeeze(-1)


def calibrate(field_fn, target, lo_s=-30.0, hi_s=30.0):
    """The shift s for which the median of field_fn(s) is target (bisection; field_fn decreases in s)."""
    for _ in range(40):
        mid = 0.5 * (lo_s + hi_s)
        if float(field_fn(mid).median()) > target:
            lo_s = mid
        else:
            hi_s = mid
    return 0.5 * (lo_s + hi_s)


def _axis_options(q: float, res: int):
    """The voxels trunc(q') in [0, res) for q' within MARGIN of q (the band reaches at most one boundary)."""
    return {int(math.trunc(x)) for x in (q - vc.MARGIN, q, q + vc.MARGIN) if -1 < x < res}


def ray_voxels(o, d, t, lo, vs, res, depth_test):
    """Per ray, with the reference's fp32 arithmetic: (the voxel it marks or -1, whether the outcome is firm, the
    voxels a ray within MARGIN of it could mark)."""
    p = o + d * t[:, None]
    q = (p - lo) / vs
    ql = q.long()
    marks = ((ql >= 0) & (ql < res)).all(-1) & torch.isfinite(q).all(-1)
    near_depth = torch.zeros_like(marks)
    if depth_test:
        marks &= t < 80
        near_depth = (t - 80).abs() <= vc.MARGIN * 80
    lin = (ql[:, 0] * res[1] + ql[:, 1]) * res[2] + ql[:, 2]
    near = ((q - q.round()).abs() <= vc.MARGIN).any(-1) | near_depth
    out = []
    for r in range(len(t)):
        hit = int(lin[r]) if bool(marks[r]) else -1
        if not bool(near[r]) or not bool(torch.isfinite(q[r]).all()):
            out.append((hit, True, set()))
            continue
        opts = [_axis_options(float(q[r, a]), int(res[a])) for a in range(3)]
        reach = {(x * int(res[1]) + y) * int(res[2]) + z for x in opts[0] for y in opts[1] for z in opts[2]}
        out.append((hit, False, reach))
    return out


def grid_record(store, key, rays, lo, vs, res, depth_test, gate_fn, thr, pca, feat_fn):
    firm, loose = set(), set()
    for o, d, t in rays:
        for lin, is_firm, reach in ray_voxels(o, d, t, lo, vs, res, depth_test):
            if is_firm and lin >= 0:
                firm.add(lin)
            elif not is_firm:
                loose |= reach | ({lin} if lin >= 0 else set())
    loose -= firm
    vox = np.array(sorted(firm | loose), np.int64)
    r = res.tolist()
    ijk = torch.from_numpy(np.stack([vox // (r[1] * r[2]), (vox // r[2]) % r[1], vox % r[2]], 1))
    pts = lo + ijk * vs
    gate = gate_fn(pts) if len(vox) else torch.zeros(0)
    M, cmin, cmax = pca
    feats = feat_fn(pts) if len(vox) else torch.zeros(0, M.shape[0])
    colors = torch.clamp((feats @ M - cmin) / (cmax - cmin), 0, 1)
    store[f"{key}/vox"] = vox
    store[f"{key}/firm"] = np.array([v in firm for v in vox.tolist()], bool)
    store[f"{key}/coords"] = pts.numpy()
    store[f"{key}/gate"] = gate.numpy()
    store[f"{key}/band"] = ((gate - thr).abs() <= vc.MARGIN * thr).numpy()
    store[f"{key}/colors"] = colors.numpy()
    return pts, gate


def run_case(vt, case, store):
    c = vc.CASES[case]
    ds = vc.dataset(case)
    cfg = vc.render_cfg()
    cfg.data = types.SimpleNamespace(pixel_source=types.SimpleNamespace(feature_model_type="dino"))
    cfg.nerf.model = types.SimpleNamespace(head=types.SimpleNamespace(enable_learnable_pe=True))
    cfg.log_dir = "."
    g = torch.Generator().manual_seed(5)
    probe = torch.tensor([-20.0, -40.0, 0.0]) + torch.rand(4000, 3, generator=g) * torch.tensor([100.0, 80.0, 20.0])

    def static_median(s):
        f, p = vc.build_models(REF, c["model"], (s, 0.0))
        return static_gate(f, p, probe)

    s_shift = calibrate(static_median, 0.5)
    if not c["dynamic"]:
        d_shift = 0.0
    elif case.endswith("closed"):
        d_shift = vc.CLOSED_SHIFT
    else:
        d_shift = calibrate(lambda s: dynamic_gate(vc.build_models(REF, c["model"], (s_shift, s))[0], probe,
                                                   torch.tensor(0.0)), DYNAMIC_MEDIAN)
    field, props = vc.build_models(REF, c["model"], (s_shift, d_shift))
    est = PropNetEstimator(None, None)
    store[f"{case}/shifts"] = np.array([s_shift, d_shift], np.float64)
    store[f"{case}/parameters"] = np.array(sorted(k for k, _ in field.named_parameters()))

    rec = {"depths": [], "features": []}
    orig_render, orig_pca = vt.render_rays, vt.get_robust_pca

    def render(**kw):
        out = orig_render(**kw)
        if kw.get("prefix") == "lidar_":
            rec["depths"].append({k: out[k].reshape(-1).clone() for k in ("depth", "static_depth", "dynamic_depth")
                                  if k in out})
        return out

    def pca(features, m=2):
        rec["features"].append(features.clone())
        torch.manual_seed(PCA_SEED)
        rec["pca"] = orig_pca(features, m)
        return rec["pca"]

    def plot(**kw):
        rec["kw"] = kw
        raise _Stop

    vt.render_rays, vt.get_robust_pca, vt.vis_occ_plotly = render, pca, plot
    try:
        vt.visualize_voxels(cfg, field, est, props, ds, device="cpu", is_dynamic=c["dynamic"])
        raise AssertionError("vis_occ_plotly was not reached")
    except _Stop:
        pass
    finally:
        vt.render_rays, vt.get_robust_pca = orig_render, orig_pca
    kw = rec["kw"]
    M, cmin, cmax = rec["pca"]
    store[f"{case}/pca_features"] = rec["features"][0].numpy()
    store[f"{case}/pca_seed"] = np.array(PCA_SEED)
    store[f"{case}/pca"] = torch.cat([M, cmin[None], cmax[None]], 0).numpy()      # [C + 2, 3]
    store[f"{case}/vis_aabb"] = np.array(kw["vis_aabb"], np.float64)
    store[f"{case}/ratios"] = np.array([kw["x_ratio"], kw["y_ratio"], kw["z_ratio"]], np.float64)
    store[f"{case}/ref_coords"] = kw["coords"]
    store[f"{case}/ref_colors"] = kw["colors"]
    store[f"{case}/ref_dynamic_groups"] = np.array(len(kw["dynamic_coords"]) if kw["dynamic_coords"] is not None
                                                   else -1)
    for j, (a, b) in enumerate(zip(kw["dynamic_coords"] or [], kw["dynamic_colors"] or [])):
        store[f"{case}/ref_dynamic_coords{j}"] = a
        store[f"{case}/ref_dynamic_colors{j}"] = b
    for i, dep in enumerate(rec["depths"]):
        for k, v in dep.items():
            store[f"{case}/depth{i}/{k}"] = v.numpy()

    _, lo, hi, res_s, res_d = box(field, vc.VOXEL_SIZE)
    vs_s, vs_d = (hi - lo) / res_s, (hi - lo) / res_d
    items = [vc.image_rays(case, i) for i in range(c["images"])]
    rays = lambda i, key: (items[i]["origins"].reshape(-1, 3), items[i]["viewdirs"].reshape(-1, 3),  # noqa: E731
                           rec["depths"][i][key])
    static_key = "static_depth" if c["dynamic"] else "depth"
    pca_t = (M, cmin, cmax)
    feat_s = lambda x: field.forward(x, query_feature_head=True, query_pe_head=False)["dino_feat"]  # noqa: E731
    with torch.no_grad():
        pts, gate = grid_record(store, f"{case}/static", [rays(i, static_key) for i in range(c["images"])], lo, vs_s,
                                res_s, True, lambda x: static_gate(field, props, x), 0.5, pca_t, feat_s)
        kept = pts[gate > 0.5]
        want = torch.from_numpy(kw["coords"])
        assert all(bool((want == p).all(-1).any()) for p in kept), "the recorded kept voxels"
        groups = []
        if c["dynamic"]:
            n_closed = (c["images"] - 1) // c["cams"]
            unq = ds.pixel_source.unique_normalized_timestamps
            for j in range(0, n_closed, 10):
                imgs = [i for i in range(c["images"]) if (0 if i == 0 else (i - 1) // c["cams"]) == j]
                t = unq[j]
                feat_d = lambda x: field.forward(x, data_dict={"normed_timestamps": t.repeat(len(x), 1)},  # noqa
                                                 query_feature_head=True, query_pe_head=False)["dynamic_dino_feat"]
                grid_record(store, f"{case}/group{j}", [rays(i, "dynamic_depth") for i in imgs], lo, vs_d, res_d,
                            False, lambda x: dynamic_gate(field, x, t), 0.1, pca_t, feat_d)
                groups.append(j)
        store[f"{case}/groups"] = np.array(groups, np.int64)
    n_firm = int(store[f"{case}/static/firm"].sum())
    print(f"{case}: shifts {s_shift:.3f} {d_shift:.3f}; static {len(store[f'{case}/static/vox'])} voxels "
          f"({n_firm} firm), kept {len(kw['coords'])}; groups {groups}, kept per group "
          f"{[len(a) for a in kw['dynamic_coords'] or []]}")


def coverage(store, case):
    """Rays that leave the box, cross the (-1, 0) band and reach depth 80 or more, over a case's images."""
    c = vc.CASES[case]
    key = "static_depth" if c["dynamic"] else "depth"
    a = torch.from_numpy(store[f"{case}/vis_aabb"]).float()
    lo, hi = a[:3], a[3:]
    res = torch.ceil((hi - lo) / vc.VOXEL_SIZE).long()
    vs = (hi - lo) / res
    band = out = far = 0
    for i in range(c["images"]):
        r = vc.image_rays(case, i)
        t = torch.from_numpy(store[f"{case}/depth{i}/{key}"])
        q = (r["origins"].reshape(-1, 3) + r["viewdirs"].reshape(-1, 3) * t[:, None] - lo) / vs
        band += int(((q > -1) & (q < 0)).any(-1).sum())
        out += int(((q <= -1) | (q >= res)).any(-1).sum())
        far += int((t >= 80).sum())
    return band, out, far


def main():
    assert ref_shims.reference_available(), "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
    vt = load_visualization_tools()
    store = {}
    for case in vc.CASES:
        run_case(vt, case, store)
        band, out, far = coverage(store, case)
        print(f"  rays in the (-1, 0) band {band}, outside the box {out}, at depth >= 80 {far}")
        assert band > 0 and out > 0
    path = os.path.join(HERE, "voxels.npz")
    np.savez_compressed(path, **store)
    print(f"wrote {path}: {len(store)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()

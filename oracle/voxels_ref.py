"""Op-for-op restatement of the reference's ``visualize_voxels`` (utils/visualization_tools.py:456-726) without the
figure -- TEST AND BENCHMARK INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

The same torch calls in the same order, on whatever device the models and data are: the boolean indexes per image,
dense float voxel grids, ``torch.nonzero`` per grid, two field passes per chunk of 2^18 voxels.  ``render_rays`` and
``robust_pca`` are arguments, so the benchmark can run this loop on the drop-in renderer beside
``emernerf_b200.voxels.visualize_voxels``.  Returns the keyword arguments of the reference's ``vis_occ_plotly`` call.
"""
from __future__ import annotations

import torch


def _to_voxel(points, lo, hi, res):
    return ((points - lo) / ((hi - lo) / res)).long()


def _to_world(lo, hi, res, idx):
    return lo + idx * ((hi - lo) / res)


def _mark(grid, points, lo, hi, res):
    v = _to_voxel(points, lo, hi, res)
    sel = ((v[..., 0] >= 0) & (v[..., 0] < res[0]) & (v[..., 1] >= 0) & (v[..., 1] < res[1]) & (v[..., 2] >= 0)
           & (v[..., 2] < res[2]))
    grid[v[..., 0][sel], v[..., 1][sel], v[..., 2][sel]] = 1


def visualize_voxels(cfg, model, proposal_estimator, proposal_networks, dataset, device, is_dynamic, render_rays,
                     robust_pca):
    model.eval()
    if proposal_estimator is not None:
        proposal_estimator.eval()
    for p in proposal_networks:
        p.eval()
    aabb = model.aabb.detach().reshape(-1).clone().to(device)
    aabb[1:3] -= 1
    aabb[3:] += 1
    lo, hi = torch.split(aabb, 3, dim=-1)
    length = hi - lo
    res_s = torch.ceil((hi - lo) / cfg.render.vis_voxel_size).long()
    static_grid = torch.zeros(*res_s, device=device)
    if is_dynamic:
        res_d = torch.ceil((hi - lo) / cfg.render.vis_voxel_size * 0.8).long()
        groups = []
        dynamic_grid = torch.zeros(*res_d, device=device)
    patches = []
    for i in range(len(dataset.full_pixel_set)):
        data = dataset.full_pixel_set[i]
        for k, v in data.items():
            data[k] = v.to(device)
        if i < dataset.num_cams:
            with torch.no_grad():
                out = render_rays(radiance_field=model, proposal_estimator=proposal_estimator,
                                  proposal_networks=proposal_networks, data_dict=data, cfg=cfg,
                                  proposal_requires_grad=False)
            f = out["dino_pe_free"] if "dino_pe_free" in out else out["dino_feat"]
            patches.append(f.reshape(-1, f.shape[-1]))
        data["lidar_origins"] = data["origins"].to(device)
        data["lidar_viewdirs"] = data["viewdirs"].to(device)
        data["lidar_normed_timestamps"] = data["normed_timestamps"].to(device)
        with torch.no_grad():
            out = render_rays(radiance_field=model, proposal_estimator=proposal_estimator,
                              proposal_networks=proposal_networks, data_dict=data, cfg=cfg,
                              proposal_requires_grad=False, prefix="lidar_", return_decomposition=True)
        depth = out["static_depth"] if is_dynamic else out["depth"]
        points = data["lidar_origins"] + data["lidar_viewdirs"] * depth
        _mark(static_grid, points[depth.squeeze() < 80], lo, hi, res_s)
        if is_dynamic:
            _mark(dynamic_grid, data["lidar_origins"] + data["lidar_viewdirs"] * out["dynamic_depth"], lo, hi, res_d)
            if i % dataset.num_cams == 0 and i > 0:
                groups.append(_to_world(lo, hi, res_d, torch.nonzero(dynamic_grid)))
                dynamic_grid = torch.zeros(*res_d, device=device)
    basis, cmin, cmax = robust_pca(torch.cat(patches, dim=0).to(device), m=2.5)
    static_points = _to_world(lo, hi, res_s, torch.nonzero(static_grid))
    chunk = 2 ** 18
    colors, kept = [], []
    for s in range(0, static_points.shape[0], chunk):
        pts = static_points[s:s + chunk]
        dens = [p(pts)["density"].squeeze(-1) for p in proposal_networks]
        with torch.no_grad():
            dens.append(model.forward(pts, query_feature_head=False)["density"])
        pts = pts[torch.stack(dens, dim=0).mean(dim=0) > 0.5]
        if len(pts) == 0:
            continue
        with torch.no_grad():
            feats = model.forward(pts, query_feature_head=True, query_pe_head=False)["dino_feat"]
        colors.append(torch.clamp((feats @ basis - cmin) / (cmax - cmin), 0, 1))
        kept.append(pts)
    colors, kept = torch.cat(colors, dim=0), torch.cat(kept, dim=0)
    dynamic_coords = dynamic_colors = None
    if is_dynamic:
        dynamic_coords, dynamic_colors = [], []
        unq = dataset.pixel_source.unique_normalized_timestamps.to(device)
        for j in range(0, len(groups), 10):
            pts = groups[j]
            with torch.no_grad():
                r = model.forward(pts, data_dict={"normed_timestamps": unq[j].repeat(pts.shape[0], 1)},
                                  query_feature_head=False)
            pts = pts[r["dynamic_density"].squeeze() > 0.1]
            if len(pts) == 0:
                continue
            with torch.no_grad():
                feats = model.forward(pts, data_dict={"normed_timestamps": unq[j].repeat(pts.shape[0], 1)},
                                      query_feature_head=True, query_pe_head=False)["dynamic_dino_feat"]
            dynamic_colors.append(torch.clamp((feats @ basis - cmin) / (cmax - cmin), 0, 1).cpu().numpy())
            dynamic_coords.append(pts.cpu().numpy())
    return {"vis_aabb": aabb.cpu().numpy().tolist(), "coords": kept.cpu().numpy(), "colors": colors.cpu().numpy(),
            "dynamic_coords": dynamic_coords, "dynamic_colors": dynamic_colors, "x_ratio": 1,
            "y_ratio": (length[1] / length[0]).item(), "z_ratio": (length[2] / length[0]).item()}

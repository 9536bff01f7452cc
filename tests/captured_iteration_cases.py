"""Small training setups for ``emernerf_b200.train.CapturedIteration`` and an independent eager restatement of the
reference's loop body (train_emernerf.py:612-855) on the package's objects, with the float line-of-sight path.

A setup is the reference's ``main`` in miniature: a ``make_cfg(small=True)`` field with FusedAdam for the field and the
proposal networks, the reference's two ``ChainedScheduler``s (builders.py:67-89, 129-142), the losses of
``emernerf_b200.loss`` with the default configs' coefficients, and the raybatch fixture sources (12 images of 64 x 96,
500 lidar points) drawn by the device samplers."""
from __future__ import annotations

import types

import torch

import errormap_cases as ec
import raybatch_cases as rc

NS = types.SimpleNamespace
DEV = "cuda"
PIXEL_RAYS, LIDAR_RAYS = 512, 512
LIDAR_CANDIDATES = [1, 3, 4, 8]


def scheduler(opt, num_iters):
    """builders.py:67-89."""
    milestones = [num_iters // 2, num_iters * 3 // 4, num_iters * 9 // 10]
    if num_iters >= 10000:
        milestones.insert(0, num_iters // 4)
    return torch.optim.lr_scheduler.ChainedScheduler([
        torch.optim.lr_scheduler.LinearLR(opt, start_factor=0.01, total_iters=num_iters // 10),
        torch.optim.lr_scheduler.MultiStepLR(opt, milestones=milestones, gamma=0.33)])


def make_cfg(variant, num_iters=60, start_iter=10, decay_steps=7, small=True):
    """``small=False``: the benchmark's field (2^20-entry tables, 64 samples, proposal samples [128, 64])."""
    from emernerf_b200 import configs

    sizes = dict(num_samples=16, prop_samples=(32, 16)) if small else dict(num_samples=64, prop_samples=(128, 64))
    cfg = configs.make_cfg(variant, num_timesteps=rc.N_IMAGES, small=small, **sizes)
    cfg.optim.num_iters = num_iters
    cfg.optim.check_nan = False
    cfg.data.pixel_source = NS(load_rgb=True)
    cfg.data.lidar_source = NS(load_lidar=True)
    cfg.supervision = NS(
        depth=NS(enable=True, line_of_sight=NS(enable=True, start_iter=start_iter, decay_steps=decay_steps,
                                               decay_rate=0.5, start_epsilon=6.0, end_epsilon=2.5)),
        sky=NS(loss_type="opacity_based"))
    return cfg


class Split:
    """The reference's SplitWrapper, train split."""

    def __init__(self, source, split_indices, ray_batch_size):
        self.datasource, self.split_indices, self.ray_batch_size = source, split_indices, ray_batch_size

    def __getitem__(self, idx):
        return self.datasource.get_train_rays(num_rays=self.ray_batch_size, candidate_indices=self.split_indices)

    def __len__(self):
        return 1000000


def make_dataset(feature_dim=None, pixel_rays=PIXEL_RAYS, lidar_rays=LIDAR_RAYS):
    from emernerf_b200 import raygen

    pix = ec.fill(ec.PixelSource(), "full", 1.0)
    if feature_dim is not None:
        g = torch.Generator().manual_seed(3)
        pix.features = torch.rand(rc.N_IMAGES, rc.FEAT_H, rc.FEAT_W, feature_dim, generator=g)
    pix = rc.to_device(pix, DEV)
    lid = rc.to_device(rc.fill_lidar(rc.LidarSource(), "lists"), DEV)
    pixel_sampler = raygen.PixelRaySampler(pix)
    pix.get_train_rays = pixel_sampler.get_train_rays
    lid.get_train_rays = raygen.LidarRaySampler(lid).get_train_rays
    return NS(pixel_source=pix, lidar_source=lid, pixel_sampler=pixel_sampler,
              train_pixel_set=Split(pix, rc.pixel_candidates("full"), pixel_rays),
              train_lidar_set=Split(lid, LIDAR_CANDIDATES, lidar_rays))


def make_losses(cfg):
    from emernerf_b200 import loss

    head = cfg.nerf.model.head
    return {
        "rgb": loss.RealValueLoss(loss_type="l2", coef=1.0),
        "sky": loss.SkyLoss(loss_type="opacity_based", coef=0.001),
        "feature": loss.RealValueLoss(loss_type="l2", coef=0.5, name="feature") if head.enable_feature_head else None,
        "dynamic_reg": loss.DynamicRegularizationLoss(loss_type="sparsity", coef=0.01)
        if head.enable_dynamic_branch else None,
        "shadow": loss.DynamicRegularizationLoss(name="shadow", loss_type="sparsity", coef=0.01)
        if head.enable_shadow_head else None,
        "depth": loss.DepthLoss(loss_type="l2", coef=1.0),
        "line_of_sight": loss.LineOfSightLoss(loss_type="my", name="line_of_sight", coef=0.1),
    }


def make_req_fn():
    """The reference's proposal schedule with its ramp shortened from 1000 to 10 steps, so that short runs see proposal
    updates on some passes and not on others."""
    from emernerf_b200.third_party.nerfacc_prop_net import get_proposal_requires_grad_fn

    return get_proposal_requires_grad_fn(target=5.0, num_steps=10)


def req_cell(fn):
    """The cell of the schedule's counter (snapshots restore it)."""
    return fn.__closure__[fn.__code__.co_freevars.index("since_last")]


def make_setup(variant, seed=0, pixel_rays=PIXEL_RAYS, lidar_rays=LIDAR_RAYS, **cfg_kw):
    from emernerf_b200 import configs

    cfg = make_cfg(variant, **cfg_kw)
    field, props, est, opt = configs.build_hot_path(cfg, DEV, table_std=0.3, seed=seed, optimizer="fused")
    est.scheduler = scheduler(est.optimizer, cfg.optim.num_iters)
    sched = scheduler(opt, cfg.optim.num_iters)
    feats = cfg.nerf.model.head.feature_embedding_dim if cfg.nerf.model.head.enable_feature_head else None
    return NS(cfg=cfg, model=field, props=props, est=est, opt=opt, sched=sched, dataset=make_dataset(feats, pixel_rays, lidar_rays),
              losses=make_losses(cfg), req_fn=make_req_fn(), decay=1.0)


def captured(s):
    from emernerf_b200.train import CapturedIteration

    return CapturedIteration(s.cfg, s.dataset, s.model, s.est, s.props, s.opt, s.sched, s.losses, s.req_fn)


def reference_iteration(s, step):
    """One pass of train_emernerf.py:612-855, eager, float line-of-sight path; returns what the loop logs."""
    from emernerf_b200 import loss as L
    from emernerf_b200 import metrics
    from emernerf_b200.radiance_fields.render_utils import render_rays

    cfg, los = s.cfg, s.cfg.supervision.depth.line_of_sight
    for m in [s.model, s.est] + s.props:
        m.train()
    if step > los.start_iter and (step - los.start_iter) % los.decay_steps == 0:
        s.decay *= los.decay_rate
    fn = s.losses
    logged, epsilon, stats = {}, None, None
    pixel_loss_dict, lidar_loss_dict = {}, {}

    prg = s.req_fn(int(step))
    i = torch.randint(0, len(s.dataset.train_pixel_set), (1,)).item()
    pdata = s.dataset.train_pixel_set[i]
    res = render_rays(radiance_field=s.model, proposal_estimator=s.est, proposal_networks=s.props, data_dict=pdata,
                      cfg=cfg, proposal_requires_grad=prg)
    s.est.update_every_n_steps(res["extras"]["trans"], prg, loss_scaler=1024)
    pixel_loss_dict.update(fn["rgb"](res["rgb"], pdata["pixels"]))
    pixel_loss_dict.update(fn["sky"](res["opacity"], pdata["sky_masks"]))
    if fn["feature"] is not None:
        pixel_loss_dict.update(fn["feature"](res["dino_feat"], pdata["features"]))
    if fn["dynamic_reg"] is not None:
        pixel_loss_dict.update(fn["dynamic_reg"](dynamic_density=res["extras"]["dynamic_density"],
                                                 static_density=res["extras"]["static_density"]))
    if fn["shadow"] is not None:
        pixel_loss_dict.update(fn["shadow"](res["shadow_ratio"]))
    if "forward_flow" in res["extras"]:
        cycle, stats = L.flow_cycle_loss(res["extras"])
        pixel_loss_dict.update(cycle)
    total_pixel_loss = sum(v for v in pixel_loss_dict.values())
    s.opt.zero_grad()
    (total_pixel_loss * 1024.0).backward()
    s.opt.step()
    s.sched.step()

    prg = s.req_fn(int(step))
    i = torch.randint(0, len(s.dataset.train_lidar_set), (1,)).item()
    ldata = s.dataset.train_lidar_set[i]
    lres = render_rays(radiance_field=s.model, proposal_estimator=s.est, proposal_networks=s.props, data_dict=ldata,
                       cfg=cfg, proposal_requires_grad=prg, prefix="lidar_")
    s.est.update_every_n_steps(lres["extras"]["trans"], prg, loss_scaler=1024)
    lidar_loss_dict.update(fn["depth"](lres["depth"], ldata["lidar_ranges"], name="lidar_range_loss"))
    if step > los.start_iter:
        m = (los.end_epsilon - los.start_epsilon) / (cfg.optim.num_iters - los.start_iter)
        b = los.start_epsilon - m * los.start_iter
        epsilon = m * step + b if los.start_iter <= step <= cfg.optim.num_iters else (
            los.start_epsilon if step < los.start_iter else los.end_epsilon)
        d = fn["line_of_sight"](pred_depth=lres["depth"], gt_depth=ldata["lidar_ranges"],
                                weights=lres["extras"]["weights"], t_vals=lres["extras"]["t_vals"], epsilon=epsilon,
                                name="lidar_line_of_sight", coef_decay=s.decay)
        lidar_loss_dict["lidar_line_of_sight"] = d["lidar_line_of_sight"].mean()
    if fn["dynamic_reg"] is not None:
        lidar_loss_dict.update(fn["dynamic_reg"](dynamic_density=lres["extras"]["dynamic_density"],
                                                 static_density=lres["extras"]["static_density"],
                                                 name="lidar_dynamic"))
    total_lidar_loss = sum(v for v in lidar_loss_dict.values())
    s.opt.zero_grad()
    (total_lidar_loss * 1024.0).backward()
    s.opt.step()
    s.sched.step()

    logged["psnr"] = metrics.compute_psnr(res["rgb"], pdata["pixels"])
    logged["total_pixel_loss"] = total_pixel_loss.item()
    logged["total_lidar_loss"] = total_lidar_loss.item()
    logged["range_rmse"] = metrics.compute_valid_depth_rmse(lres["depth"], ldata["lidar_ranges"])
    logged.update({k: v.item() for k, v in pixel_loss_dict.items()})
    logged.update({k: v.item() for k, v in lidar_loss_dict.items()})
    logged["lr"] = s.opt.param_groups[0]["lr"]
    if stats is not None:
        logged.update({k: v.item() for k, v in stats.items()})
    if epsilon is not None:
        logged["epsilon"] = epsilon
    return logged

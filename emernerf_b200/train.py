"""``CapturedIteration``: the body of the reference's training loop (train_emernerf.py:612-855) replayed as CUDA graphs.

The loop users run launches every kernel from Python and reads about a dozen values back per iteration.  Here one call
``it(step)`` does what one pass of that loop body does -- the same host-side state changes, in the same order -- and,
once a branch of the pass has been seen twice, replays it as a captured CUDA graph: no Python-side library launch and
no host sync.  The logged values stay on the device until ``drain()``.

    it = CapturedIteration(cfg, dataset, model, proposal_estimator, proposal_networks, optimizer, scheduler, losses,
                           proposal_requires_grad_fn)
    for step in metric_logger.log_every(all_iters, cfg.logging.print_freq):
        it(step)
        if <the logger prints this step, or wandb logs every step>:
            for row in it.drain():
                metric_logger.update(**row)

How it works (DESIGN.md, "Training iterations as CUDA graphs"):

* A pass's branch and the memory it reads are its key: ``("pixel", (proposal_requires_grad, importance sampling
  live), (error map, candidates))`` and ``("lidar", (proposal_requires_grad, line of sight on), (candidates,))``,
  the error map and a candidate tensor by ``(data_ptr, _version)``.  The first occurrence of a key runs eagerly on a
  side stream and is that step's training work; the second is captured, then replayed once for its step; after that
  the key is only replayed.  Every step trains exactly once.
* The eager run and the capture execute one body, which does not sync.  Host decisions (the proposal schedule, the
  CPU generator's draw, the schedulers, the line-of-sight decay) are made outside it, before or after each pass.
* Values that change per step reach the graph through device memory: the learning rates through
  ``FusedAdam.sync_lr()`` before every replay and once right before every capture; the line-of-sight constants
  through one small host-to-device copy from pageable memory before each lidar pass (the copy has consumed the host
  buffer when it returns, so no later step can overwrite it in flight).
* A changed error map or candidate set makes a new key and drops the graphs of the old one, which hold the old map
  alive until then: no graph can replay on freed memory.
* Every graph allocates from one memory pool.  Nothing a graph allocates is read outside it: the logged scalars are
  copied inside the graph into a ring buffer allocated before any capture, at a slot held in a device counter.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple

import torch
from torch import Tensor

from . import loss as _loss
from . import metrics as _metrics
from .optim import FusedAdam
from .raygen import LidarRaySampler, PixelRaySampler, _candidate_key

__all__ = ["CapturedIteration", "LineOfSightSchedule"]

LOSS_KEYS = ("rgb", "sky", "feature", "dynamic_reg", "shadow", "depth", "line_of_sight")
RING_SLOTS = 1024           # iterations between two drains before one extra sync empties the ring
RING_WIDTH = 16             # scalars one pass may log


class LineOfSightSchedule:
    """The host arithmetic of the reference's line-of-sight schedule (train_emernerf.py:615-631, 779-792): the decay
    weight, multiplied by ``decay_rate`` every ``decay_steps`` steps after ``start_iter``, and ``epsilon``, linear from
    ``start_epsilon`` at ``start_iter`` to ``end_epsilon`` at ``num_iters``."""

    def __init__(self, cfg):
        los = cfg.supervision.depth.line_of_sight
        self.start_iter, self.decay_steps, self.decay_rate = los.start_iter, los.decay_steps, los.decay_rate
        self.start, self.final, self.num_iters = los.start_epsilon, los.end_epsilon, cfg.optim.num_iters
        self.decay_weight = 1.0

    def begin(self, step) -> None:
        if step > self.start_iter and (step - self.start_iter) % self.decay_steps == 0:
            self.decay_weight *= self.decay_rate

    def active(self, step) -> bool:
        return step > self.start_iter

    def epsilon(self, step) -> float:
        m = (self.final - self.start) / (self.num_iters - self.start_iter)
        b = self.start - m * self.start_iter
        if step < self.start_iter:
            return self.start
        if step > self.num_iters:
            return self.final
        return m * step + b


def _identity(t: Optional[Tensor]):
    return None if t is None else (t.data_ptr(), t._version)


def _candidates(split) -> tuple:
    idx = getattr(split, "split_indices", None)
    if isinstance(idx, Tensor):
        return ("tensor", _identity(idx))
    return _candidate_key(idx)


class _Graph:
    """One key: how often it has run, and, once captured, the graph, the names of the scalars it logs and the tensors
    whose memory it reads (held until the key is dropped)."""

    def __init__(self, held: tuple):
        self.runs, self.graph, self.names, self.held = 0, None, None, held


class CapturedIteration:
    def __init__(self, cfg, dataset, model, proposal_estimator, proposal_networks, optimizer, scheduler, losses,
                 proposal_requires_grad_fn: Callable[[int], bool]):
        self.cfg, self.dataset, self.model = cfg, dataset, model
        self.est, self.props = proposal_estimator, list(proposal_networks)
        self.optimizer, self.scheduler = optimizer, scheduler
        self.losses = {k: losses.get(k) for k in LOSS_KEYS}
        self.req_fn = proposal_requires_grad_fn
        self._refuse()
        self.pixel_on = bool(cfg.data.pixel_source.load_rgb)
        self.lidar_on = bool(cfg.data.lidar_source.load_lidar and cfg.supervision.depth.enable)
        self.los = LineOfSightSchedule(cfg) if self.losses["line_of_sight"] is not None else None
        self._graphs: Dict[tuple, _Graph] = {}
        self._device_state(next(model.parameters()).device)
        self._written = 0                    # iterations whose scalars went to the ring
        self._pending: List[dict] = []       # host part of the iterations not drained yet
        self._drained: List[dict] = []       # rows moved off the ring when it filled up
        self.events: List[Tuple[str, tuple]] = []     # ("eager" | "capture" | "replay" | "drop", key), in order

    def _device_state(self, dev: torch.device) -> None:
        """The memory every graph shares, allocated before any capture: the pool, the warm-up stream, the staged
        line-of-sight constants, the ring of logged values and its slot counter."""
        self.device = dev
        self._pool = torch.cuda.graph_pool_handle()
        self._side = torch.cuda.Stream(dev)
        self._sight = torch.zeros(4, dtype=torch.float32, device=dev)
        self._ring = {p: torch.zeros(RING_SLOTS * RING_WIDTH, dtype=torch.float64, device=dev)
                      for p in ("pixel", "lidar")}
        self._cols = torch.arange(RING_WIDTH, dtype=torch.int64, device=dev)
        self._slot = torch.zeros(1, dtype=torch.int64, device=dev)

    def _stage_sight(self, vals: List[float]) -> None:
        """One 16-byte copy from pageable memory: it has consumed the host buffer when it returns."""
        self._sight.copy_(torch.tensor(vals, dtype=torch.float32), non_blocking=True)

    # ------------------------------------------------------------------ refusals
    def _refuse(self) -> None:
        for k, fn in self.losses.items():
            if fn is None:
                continue
            if not isinstance(fn, _loss.Loss):
                raise TypeError(f"CapturedIteration: losses[{k!r}] is a {type(fn).__module__}.{type(fn).__name__}; "
                                "the reference's loss/base.py classes sync the host through boolean indexing. Build "
                                "the losses from emernerf_b200.loss")
            if fn.check_nan:
                raise ValueError(f"CapturedIteration: losses[{k!r}] has check_nan=True, which reads every value on "
                                 "the host; set cfg.optim.check_nan = False")
        if self.losses["rgb"] is None:
            raise ValueError("CapturedIteration: losses['rgb'] is required")
        for what, opt in (("optimizer", self.optimizer), ("proposal optimizer", self.est.optimizer)):
            if not isinstance(opt, FusedAdam):
                raise TypeError(f"CapturedIteration: the {what} is a {type(opt).__name__}; graph capture needs "
                                "emernerf_b200.optim.FusedAdam (INTEGRATION.md §4)")
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            raise RuntimeError("CapturedIteration: runs on one process; a process group of "
                               f"{dist.get_world_size()} ranks is initialised")
        for what, split, cls in (("pixel", "train_pixel_set", PixelRaySampler),
                                 ("lidar", "train_lidar_set", LidarRaySampler)):
            s = getattr(self.dataset, split, None)
            src = getattr(s, "datasource", None)
            if src is not None and not isinstance(getattr(src.get_train_rays, "__self__", None), cls):
                raise TypeError(f"CapturedIteration: the {what} source draws its batches with the reference's "
                                f"get_train_rays, which syncs the host; bind raygen.{cls.__name__} (INTEGRATION.md "
                                "§11)")

    # ------------------------------------------------------------------ one iteration
    def __call__(self, step) -> None:
        for m in [self.model, self.est] + self.props:
            m.train()
        if self.los is not None:
            self.los.begin(step)
        row: dict = {"pixel": None, "lidar": None, "epsilon": None}
        if self.pixel_on:
            prg = self.req_fn(int(step))
            i = torch.randint(0, len(self.dataset.train_pixel_set), (1,)).item()
            src = self.dataset.train_pixel_set.datasource
            importance = bool(src.buffer_ratio > 0 and src.pixel_error_buffered)
            maps = src.pixel_error_maps if importance else None
            key = ("pixel", (prg, importance), (_identity(maps), _candidates(self.dataset.train_pixel_set)))
            row["pixel"] = self._run(key, lambda: self._pixel_body(prg, i), held=(maps,))
            self._after_pass()
        if self.lidar_on:
            prg = self.req_fn(int(step))
            i = torch.randint(0, len(self.dataset.train_lidar_set), (1,)).item()
            los_on = self.los is not None and self.los.active(step)
            if los_on:
                row["epsilon"] = self.los.epsilon(step)
                self._stage_sight(_loss.line_of_sight_consts(row["epsilon"], self.los.decay_weight))
            key = ("lidar", (prg, los_on), (_candidates(self.dataset.train_lidar_set),))
            row["lidar"] = self._run(key, lambda: self._lidar_body(prg, i, los_on), held=())
            self._after_pass()
        row["lr"] = self.optimizer.param_groups[0]["lr"]
        self._pending.append(row)
        self._written += 1
        if len(self._pending) >= RING_SLOTS:
            self._drained.extend(self._read_ring())

    def _after_pass(self) -> None:
        # update_every_n_steps steps the proposal scheduler in both of its branches; the loop then steps the main one
        if self.est.scheduler is not None:
            self.est.scheduler.step()
        self.scheduler.step()

    def _drop_stale(self, key: tuple) -> None:
        """A pass whose error map or candidate set changed: the graphs of the old state go (and release it)."""
        for k in [k for k in self._graphs if k[0] == key[0] and k[2] != key[2]]:
            if self._graphs[k].graph is not None:
                self.events.append(("drop", k))
            del self._graphs[k]

    def _run(self, key: tuple, body: Callable[[], List[str]], held: tuple) -> List[str]:
        self._drop_stale(key)
        g = self._graphs.setdefault(key, _Graph(held))
        self.optimizer.sync_lr()
        self.est.optimizer.sync_lr()
        if g.runs == 0:
            # warm-up: this step's training work, eager, on a side stream (lazy workspaces and caches are made here)
            self.events.append(("eager", key))
            cur = torch.cuda.current_stream(self.device)
            self._side.wait_stream(cur)
            with torch.cuda.stream(self._side):
                g.names = body()
            cur.wait_stream(self._side)
        else:
            if g.graph is None:
                self.events.append(("capture", key))
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, pool=self._pool):
                    names = body()
                if names != g.names:
                    raise RuntimeError(f"CapturedIteration: the pass {key} logged {names} when captured and "
                                       f"{g.names} when run eagerly")
                g.graph = graph
            self.events.append(("replay", key))
            g.graph.replay()
        g.runs += 1
        return g.names

    # ------------------------------------------------------------------ the bodies (no host sync in them)
    def _log(self, ring: str, scalars: List[Tuple[str, Tensor]], advance: bool) -> List[str]:
        if len(scalars) > RING_WIDTH:
            raise ValueError(f"CapturedIteration: {len(scalars)} scalars in one pass; the ring holds {RING_WIDTH}")
        vals = torch.stack([v.detach().reshape(()).to(torch.float64) for _, v in scalars])
        idx = self._slot * RING_WIDTH + self._cols[:len(scalars)]
        self._ring[ring].index_copy_(0, idx, vals)
        if advance:
            self._slot.add_(1).remainder_(RING_SLOTS)
        return [k for k, _ in scalars]

    def _backward_and_step(self, total: Tensor) -> None:
        self.optimizer.zero_grad()
        (total * 1024.0).backward()          # the loop's GradScaler(2**10).scale(loss), never unscaled
        self.optimizer.step()

    def _pixel_body(self, prg: bool, i: int) -> List[str]:
        from .radiance_fields.render_utils import render_rays

        L = self.losses
        data = self.dataset.train_pixel_set[i]
        res = render_rays(radiance_field=self.model, proposal_estimator=self.est, proposal_networks=self.props,
                          data_dict=data, cfg=self.cfg, proposal_requires_grad=prg)
        if prg:
            self.est.update_tensor(res["extras"]["trans"], loss_scaler=1024)
        d = dict(L["rgb"](res["rgb"], data["pixels"]))
        if L["sky"] is not None:
            pred = res["extras"]["weights"] if L["sky"].loss_type == "weights_based" else res["opacity"]
            d.update(L["sky"](pred, data["sky_masks"]))
        if L["feature"] is not None:
            d.update(L["feature"](res["dino_feat"], data["features"]))
        if L["dynamic_reg"] is not None:
            d.update(L["dynamic_reg"](dynamic_density=res["extras"]["dynamic_density"],
                                      static_density=res["extras"]["static_density"]))
        if L["shadow"] is not None:
            d.update(L["shadow"](res["shadow_ratio"]))
        stats = {}
        if "forward_flow" in res["extras"]:
            cycle, stats = _loss.flow_cycle_loss(res["extras"])
            d.update(cycle)
        total = sum(v for v in d.values())
        self._backward_and_step(total)
        psnr = _metrics._pair_launch("emer_depth_rmse", res["rgb"], data["pixels"], 3)[2]
        scalars = [("psnr", psnr), ("total_pixel_loss", total)] + list(d.items()) + list(stats.items())
        return self._log("pixel", scalars, advance=not self.lidar_on)

    def _lidar_body(self, prg: bool, i: int, los_on: bool) -> List[str]:
        from .radiance_fields.render_utils import render_rays

        L = self.losses
        data = self.dataset.train_lidar_set[i]
        res = render_rays(radiance_field=self.model, proposal_estimator=self.est, proposal_networks=self.props,
                          data_dict=data, cfg=self.cfg, proposal_requires_grad=prg, prefix="lidar_")
        if prg:
            self.est.update_tensor(res["extras"]["trans"], loss_scaler=1024)
        d = dict(L["depth"](res["depth"], data["lidar_ranges"], name="lidar_range_loss"))
        if los_on:
            sight = L["line_of_sight"](pred_depth=res["depth"], gt_depth=data["lidar_ranges"],
                                       weights=res["extras"]["weights"], t_vals=res["extras"]["t_vals"],
                                       epsilon=self._sight, name="lidar_line_of_sight")
            d["lidar_line_of_sight"] = sight["lidar_line_of_sight"].mean()
        if L["dynamic_reg"] is not None:
            d.update(L["dynamic_reg"](dynamic_density=res["extras"]["dynamic_density"],
                                      static_density=res["extras"]["static_density"], name="lidar_dynamic"))
        total = sum(v for v in d.values())
        self._backward_and_step(total)
        rmse = _metrics._pair_launch("emer_depth_rmse", res["depth"].squeeze(), data["lidar_ranges"].squeeze(), 3)[0]
        scalars = [("total_lidar_loss", total), ("range_rmse", rmse)] + list(d.items())
        return self._log("lidar", scalars, advance=True)

    # ------------------------------------------------------------------ logged values
    def _read_ring(self) -> List[dict]:
        """The pending iterations' rows: one device-to-host copy of the ring and one sync."""
        n = len(self._pending)
        if n == 0:
            return []
        host = torch.stack([self._ring["pixel"], self._ring["lidar"]]).cpu().view(2, RING_SLOTS, RING_WIDTH).tolist()
        first = (self._written - n) % RING_SLOTS
        rows = []
        for j, p in enumerate(self._pending):
            slot = (first + j) % RING_SLOTS
            pix = dict(zip(p["pixel"], host[0][slot])) if p["pixel"] is not None else {}
            lid = dict(zip(p["lidar"], host[1][slot])) if p["lidar"] is not None else {}
            # the keys in the order the loop hands them to metric_logger.update
            row = {}
            if pix:
                row["psnr"], row["total_pixel_loss"] = pix["psnr"], pix["total_pixel_loss"]
            if lid:
                row["total_lidar_loss"], row["range_rmse"] = lid["total_lidar_loss"], lid["range_rmse"]
            stats = {k: v for k, v in pix.items() if k in _loss.FLOW_STAT_KEYS}
            row.update({k: v for k, v in pix.items() if k not in row and k not in stats})
            row.update({k: v for k, v in lid.items() if k not in row})
            row["lr"] = p["lr"]
            row.update(stats)
            if p["epsilon"] is not None:
                row["epsilon"] = p["epsilon"]
            rows.append(row)
        self._pending = []
        return rows

    def drain(self) -> List[dict]:
        """One dict per iteration since the last drain, with the keys and values the loop passes to
        ``metric_logger.update``; costs one device-to-host copy and one sync."""
        rows = self._drained + self._read_ring()
        self._drained = []
        return rows

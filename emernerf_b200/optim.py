"""``FusedAdam``: torch.optim.Adam's arithmetic (the optimizer the reference builds, builders.py:50-61,114-120:
lr 0.01, eps 1e-15, weight_decay 1e-5, betas (0.9, 0.99)) with the hot path's gradient plumbing:

* every parameter's gradient lives in ONE persistent flat fp32 buffer per parameter group (``p.grad`` are views of it);
  the library's backward kernels -- hash-grid scatter, weight-gradient kernels -- accumulate straight into those views
  (``_ops.register_grad_sink``): no ``zeros_like`` of a 122 MB table per backward, no AccumulateGrad copy;
* ``step()`` is one launch per group (``emer_adam_step``, csrc/optim.cu): Adam update of every block + zeroing of the
  gradient it consumed (replaces ``optimizer.zero_grad()`` and tiny-cuda-nn's table memset);
* the flat gradient buffer is what ``emernerf_b200.distributed`` reduces: one collective per group instead of one per
  tensor, or reduce-scatter -> Adam on this rank's shard -> all-gather of the flat parameters.

Semantics kept from torch: parameters that received no gradient since the last step are skipped (the reference's
proposal network 0 is never evaluated -- DESIGN.md Q21 -- and must stay at its initial values, weight decay included);
``state_dict()`` / ``load_state_dict()`` carry ``step`` / ``exp_avg`` / ``exp_avg_sq`` per parameter like torch's, so
checkpoints written by either optimizer load into the other.

A maintainer swaps it in with one line in builders.py:50-61 (``torch.optim.Adam`` -> ``emernerf_b200.optim.FusedAdam``);
with the reference's own torch optimizer nothing here is active and the ordinary autograd path runs.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

from . import _lib, _ops

ALIGN = 64          # floats: every block starts on a 256-byte boundary of the flat buffers
SHARD_ALIGN = ALIGN * 8


class _Group:
    """Flat state of one param group."""

    def __init__(self, params: List[Tensor], lr: float, flatten_params: bool):
        dev = params[0].device
        self.params = params
        self.offsets, off = [], 0
        for p in params:
            if not (_ops.on_device(p) and p.dtype == torch.float32 and p.is_contiguous() and p.device == dev):
                raise ValueError("FusedAdam takes contiguous fp32 CUDA parameters on one device")
            self.offsets.append(off)
            off += (p.numel() + ALIGN - 1) // ALIGN * ALIGN
        off = (off + SHARD_ALIGN - 1) // SHARD_ALIGN * SHARD_ALIGN      # splits evenly over 1, 2, 4 or 8 ranks
        self.total = off
        z = lambda: torch.zeros(off, dtype=torch.float32, device=dev)
        self.grad, self.exp_avg, self.exp_avg_sq = z(), z(), z()
        self.flat_params: Optional[Tensor] = None
        if flatten_params:
            # the parameters become views of one flat buffer too (same values, same state-dict keys): what the sharded
            # data-parallel step all-gathers
            self.flat_params = z()
            for p, o in zip(params, self.offsets):
                self.flat_params[o:o + p.numel()].copy_(p.detach().reshape(-1))
                p.data = self.flat_params[o:o + p.numel()].view(p.shape)
        self.hyper = torch.tensor([0.0, lr], dtype=torch.float32, device=dev)      # [step, lr], read by the kernel
        self.lr_host = lr
        self.desc: Dict[Tuple, Tuple[Tensor, Tensor, int, int]] = {}

    def view(self, flat: Tensor, i: int) -> Tensor:
        p, o = self.params[i], self.offsets[i]
        return flat[o:o + p.numel()].view(p.shape)

    def descriptor(self, active: Tuple[int, ...], lo: int = 0, hi: Optional[int] = None):
        """Device arrays for ``emer_adam_step`` over the active blocks clipped to flat range [lo, hi)."""
        hi = self.total if hi is None else hi
        key = (active, lo, hi)
        if key not in self.desc:
            rows, prefix, acc = [], [0], 0
            for i in active:
                p, o = self.params[i], self.offsets[i]
                a, b = max(o, lo), min(o + p.numel(), hi)
                if a >= b:
                    continue
                s = a - o                                   # first element of the block inside the range
                rows.append([p.data_ptr() + 4 * s, self.grad.data_ptr() + 4 * a, self.exp_avg.data_ptr() + 4 * a,
                             self.exp_avg_sq.data_ptr() + 4 * a, b - a])
                acc += (b - a + 3) // 4 * 4
                prefix.append(acc)
                if (p.data_ptr() + 4 * s) % 16:
                    raise ValueError("FusedAdam: parameter storage must be 16-byte aligned")
            dev = self.grad.device
            blocks = torch.tensor(rows or [[0] * 5], dtype=torch.int64, device=dev)
            self.desc[key] = (blocks, torch.tensor(prefix, dtype=torch.int64, device=dev), len(rows), acc)
        return self.desc[key]


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, flatten_params: bool = False, **ignored):
        # (``fused`` / ``capturable`` / ``foreach`` of torch.optim.Adam are accepted and ignored: this IS the fused,
        # capturable implementation)
        for k in ignored:
            if k not in ("fused", "capturable", "foreach", "amsgrad", "maximize", "differentiable"):
                raise TypeError(f"FusedAdam: unexpected argument {k}")
        if ignored.get("amsgrad") or ignored.get("maximize"):
            raise NotImplementedError("FusedAdam: amsgrad / maximize are not used by the reference and not implemented")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._touched = set()
        self._groups: List[_Group] = []
        self._flatten = flatten_params
        self.shard: Optional[Tuple[int, int]] = None          # (rank, world): step() updates this rank's slice only
        for group in self.param_groups:
            g = _Group(list(group["params"]), group["lr"], flatten_params)
            self._groups.append(g)
            for i, p in enumerate(g.params):
                sink = g.view(g.grad, i)
                p.grad = sink
                _ops.register_grad_sink(p, sink, self._mark, self._is_touched)
                p.register_post_accumulate_grad_hook(self._mark)          # gradients that arrive through torch autograd
                self.state[p] = {"step": g.hyper[0], "exp_avg": g.view(g.exp_avg, i), "exp_avg_sq": g.view(g.exp_avg_sq, i)}

    # ------------------------------------------------------------------ bookkeeping
    def _mark(self, p: Tensor) -> None:
        self._touched.add(id(p))

    def _is_touched(self, p: Tensor) -> bool:
        return id(p) in self._touched

    def flat_grads(self) -> List[Tensor]:
        """One flat gradient buffer per param group (what data parallelism reduces)."""
        return [g.grad for g in self._groups]

    def flat_params(self) -> List[Optional[Tensor]]:
        return [g.flat_params for g in self._groups]

    def mark_all_touched(self) -> None:
        for g in self._groups:
            for p in g.params:
                self._touched.add(id(p))

    def zero_grad(self, set_to_none: bool = True) -> None:
        """Gradients are zeroed by ``step()``.  Called with gradients pending (backward without a step), it discards
        them like torch's."""
        for g in self._groups:
            for i, p in enumerate(g.params):
                if id(p) in self._touched:
                    g.view(g.grad, i).zero_()
                if p.grad is None or p.grad.data_ptr() != g.view(g.grad, i).data_ptr():
                    p.grad = g.view(g.grad, i)                 # someone set it to None: re-attach the sink
        self._touched.clear()

    # ------------------------------------------------------------------ the step
    @staticmethod
    def _sync_group_lr(group, g: _Group) -> None:
        if group["lr"] != g.lr_host:
            g.hyper[1].fill_(group["lr"])
            g.lr_host = group["lr"]

    @torch.no_grad()
    def sync_lr(self) -> None:
        """Write every group's ``lr`` to the device where the Adam kernel reads it, if it changed since the last write.
        ``step()`` does this itself; a CUDA graph that captured ``step()`` does not (the write is a host decision), so
        call this before each replay, and once before the capture, so that the capture records no write."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("FusedAdam.sync_lr: call it outside graph capture")
        for group, g in zip(self.param_groups, self._groups):
            self._sync_group_lr(group, g)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        _ops.join_side_streams()                 # weight gradients that ran beside the rest of the backward pass
        for group, g in zip(self.param_groups, self._groups):
            active = tuple(i for i, p in enumerate(g.params) if id(p) in self._touched)
            if not active:
                continue
            self._sync_group_lr(group, g)
            g.hyper[0].add_(1.0)
            lo, hi = 0, g.total
            if self.shard is not None:
                rank, world = self.shard
                per = g.total // world if g.total % (ALIGN * world) == 0 else (g.total // ALIGN + world - 1) // world * ALIGN
                lo, hi = min(rank * per, g.total), min((rank + 1) * per, g.total)
            blocks, prefix, n_blocks, total = g.descriptor(active, lo, hi)
            beta1, beta2 = group["betas"]
            _lib.DEVICE = g.grad.device.index
            _lib.call("emer_adam_step", ctypes.c_void_p(blocks.data_ptr()), ctypes.c_void_p(prefix.data_ptr()), n_blocks, total,
                      ctypes.c_void_p(g.hyper.data_ptr()), float(beta1), float(beta2), float(group["eps"]),
                      float(group["weight_decay"]), 1, _ops._stream())
            if self.shard is not None and hi - lo < g.total:
                # the part of the gradient this rank did not consume still has to be cleared
                if lo > 0:
                    g.grad[:lo].zero_()
                if hi < g.total:
                    g.grad[hi:].zero_()
        self._touched.clear()
        return loss

    # ------------------------------------------------------------------ checkpoints (torch.optim.Adam's layout)
    def state_dict(self):
        sd = super().state_dict()
        for st in sd["state"].values():                       # detach from the flat buffers
            for k, v in st.items():
                if torch.is_tensor(v):
                    st[k] = v.detach().clone()
        return sd

    def load_state_dict(self, state_dict) -> None:
        ids = [i for grp in state_dict["param_groups"] for i in grp["params"]]
        params = [p for grp in self.param_groups for p in grp["params"]]
        if len(ids) != len(params):
            raise ValueError("FusedAdam.load_state_dict: parameter count differs")
        for pid, p in zip(ids, params):
            src = state_dict["state"].get(pid)
            if src is None:
                continue
            st = self.state[p]
            st["exp_avg"].copy_(src["exp_avg"])
            st["exp_avg_sq"].copy_(src["exp_avg_sq"])
            st["step"].fill_(float(src["step"]))             # one step counter per group (they all advance together)
        for grp, src in zip(self.param_groups, state_dict["param_groups"]):
            for k, v in src.items():
                if k != "params":
                    grp[k] = v

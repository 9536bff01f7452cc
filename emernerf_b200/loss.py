"""The training losses of the reference's ``loss/base.py`` on the device: same class names, constructor arguments and
defaults, ``__call__`` signatures and returned ``{name: value}`` keys, each loss one CUDA launch forward and one
backward (csrc/losses.cu), with no host synchronisation and no data-dependent shapes.

Drop-in for ``train_emernerf.py``: replace ``import loss`` with ``from emernerf_b200 import loss``.  The flow variants'
cycle loss and flow statistics, inline in ``train_emernerf.py:700-740`` rather than in ``loss/base.py``, are
``flow_cycle_loss`` here.

Differences from the op-by-op reference, all deliberate:
  * ``DepthLoss`` averages over the valid rays (0.01 < gt < upper_bound) with a count kept on the device instead of
    boolean indexing, so there is no ``nonzero`` / device-to-host sync between the lidar forward and its backward, and
    the lidar losses can be captured in a CUDA graph.  A batch with no valid ray still gives NaN.
  * Targets, masks, ``t_vals`` and ground-truth depths are constants: only predictions, weights and densities (and
    the static density of the entropy loss) receive gradients.
  * Options that no shipped configuration reaches raise ``NotImplementedError``: ``reduction="none"``,
    ``depth_error_percentile``, and the optional ``mask`` arguments.
  * ``check_nan=True`` keeps the reference's NaN check, which reads the value on the host (a sync); the default
    configuration has it off.
  * A CUDA graph that captures a loss call bakes in its Python scalars (``coef``, ``coef_decay``, ``epsilon``): recapture
    when they change, or give ``LineOfSightLoss`` its ``epsilon`` and ``coef_decay`` as device constants
    (``line_of_sight_consts``), which the kernels read when they run.
"""
from __future__ import annotations

import math
from typing import Dict, Literal, Tuple

import torch
import torch.nn as nn
from torch import Tensor

from . import _ops

__all__ = ["normalize_depth", "Loss", "RealValueLoss", "SkyLoss", "DepthLoss", "LineOfSightLoss",
           "DynamicRegularizationLoss", "line_of_sight_consts", "dirac_delta_approx", "compute_line_of_sight_loss", "flow_cycle_loss"]


def _unsupported(what: str):
    return NotImplementedError(f"emernerf_b200.loss: {what} is not supported (no shipped configuration uses it)")


def normalize_depth(depth: Tensor, max_depth: float = 80.0):
    return torch.clamp(depth / max_depth, 0.0, 1.0)


class Loss(nn.Module):
    """Base class: ``coef`` scales the loss, ``check_nan`` raises ``ValueError`` on a NaN value (a host sync)."""

    def __init__(self, coef: float = 1.0, check_nan: bool = False, reduction="mean"):
        super(Loss, self).__init__()
        self.coef = coef
        self.check_nan = check_nan
        assert reduction in ["mean", "none"]
        if reduction != "mean":
            raise _unsupported('reduction="none"')
        self.reduction = reduction

    def __call__(self, *args, name: str, **kwargs):
        raise NotImplementedError()

    def set_coef(self, coef: float):
        self.coef = coef

    def return_loss(self, name: str, loss: Tensor):
        """The reference's reduction of an unreduced loss tensor (for subclasses that compute their own)."""
        return self._result(name, loss.mean() * self.coef)

    def _result(self, name: str, value: Tensor):
        if self.check_nan:
            if torch.isnan(value):
                raise ValueError(f"Loss {name} is NaN.")
        return {name: value}


class RealValueLoss(Loss):
    """``coef * mean(call_coef * loss_fn(predicted, gt))`` with loss_fn l1 / l2 / smooth_l1 (beta 1)."""

    def __init__(
        self,
        loss_type: Literal["l1", "l2", "smooth_l1"] = "l2",
        coef: float = 1.0,
        name="rgb",
        reduction="mean",
        check_nan=False,
    ):
        super(RealValueLoss, self).__init__(coef, check_nan, reduction)
        self.loss_type = loss_type
        if self.loss_type not in ("l1", "l2", "smooth_l1"):
            raise NotImplementedError(f"Unknown loss type: {loss_type}")
        self.name = f"{name}_loss_{self.loss_type}"

    def __call__(
        self,
        predicted: Tensor,
        gt: Tensor,
        mask: Tensor = None,
        name: str = None,
        coef: float = 1.0,
    ):
        if mask is not None:
            raise _unsupported("RealValueLoss's mask")
        name = self.name if name is None else name
        value = _ops.pointwise_loss(self.loss_type, predicted, gt.detach(), pre=coef, post=self.coef)
        return self._result(name, value)


class SkyLoss(Loss):
    """``weights_based``: ``coef * mean_r(sum_s weights^2 * sky_mask)``; ``opacity_based``:
    ``coef * mean(BCE(opacity, 1 - sky_mask))``."""

    def __init__(
        self,
        loss_type: Literal["weights_based", "opacity_based"] = "weights_based",
        coef: float = 0.01,
        reduction="mean",
        check_nan=False,
    ):
        super(SkyLoss, self).__init__(coef, check_nan, reduction)
        self.loss_type = loss_type
        if self.loss_type not in ("weights_based", "opacity_based"):
            raise NotImplementedError(f"Unknown loss type: {loss_type}")
        self.name = f"sky_loss_{self.loss_type}"

    def __call__(
        self,
        predictions: Tensor,
        sky_mask: Tensor,
    ):
        # predictions are the weights [R, S] (weights_based) or the opacity [R, 1] (opacity_based)
        if self.loss_type == "weights_based":
            value = _ops.sky_weights_loss(predictions, sky_mask, post=self.coef)
        else:
            value = _ops.pointwise_loss("sky_bce", predictions, sky_mask.detach(), post=self.coef)
        return self._result(self.name, value)


class DepthLoss(Loss):
    """``coef * mean over the rays with 0.01 < gt < upper_bound of loss_fn(normalize_depth(pred), normalize_depth(gt))``,
    depths normalised by ``upper_bound``."""

    def __init__(
        self,
        loss_type: Literal[
            "l1",
            "l2",
            "smooth_l1",
        ] = "l2",
        name: str = "depth_loss",
        normalize: bool = True,
        depth_error_percentile: float = None,
        coef: float = 1.0,
        upper_bound: float = 80,
        reduction="mean",
        check_nan=False,
    ):
        super(DepthLoss, self).__init__(coef, check_nan, reduction)
        self.loss_type = loss_type
        if self.loss_type not in ("l1", "l2", "smooth_l1"):
            raise NotImplementedError(f"Unknown loss type: {self.loss_type}")
        if depth_error_percentile is not None:
            raise _unsupported("depth_error_percentile")
        self.normalize = normalize
        self.name = f"{name}_{self.loss_type}"
        self.upper_bound = upper_bound
        self.depth_error_percentile = depth_error_percentile

    def __call__(
        self,
        pred_depth: Tensor,
        gt_depth: Tensor,
        name: str = None,
    ):
        name = self.name if name is None else name
        value = _ops.pointwise_loss("depth_" + self.loss_type, pred_depth, gt_depth.detach(),
                                    p0=float(self.upper_bound), post=self.coef)
        return self._result(name, value)


class LineOfSightLoss(Loss):
    """``coef * mean(coef_decay * compute_line_of_sight_loss(gt_depth, weights, t_vals, epsilon))``; ``pred_depth``
    gets no gradient and ``t_vals`` is detached, as in the reference.

    ``epsilon`` may also be a float32 CUDA tensor holding ``line_of_sight_consts(epsilon, coef_decay)`` (then leave
    ``coef_decay`` at 1): the kernels read the four values when they run, so a captured CUDA graph follows whatever
    was last written there.  Value and gradient are bit-identical to the float call with the same two numbers."""

    def __init__(
        self,
        loss_type: Literal[
            "my",
        ] = "my",
        name: str = "line_of_sight",
        depth_error_percentile: float = None,
        coef: float = 1.0,
        upper_bound: float = 80,
        reduction="mean",
        check_nan=False,
    ):
        super(LineOfSightLoss, self).__init__(coef, check_nan, reduction)
        self.loss_type = loss_type
        if depth_error_percentile is not None:
            raise _unsupported("depth_error_percentile")
        self.name = f"{name}_{self.loss_type}"
        self.upper_bound = upper_bound
        self.depth_error_percentile = depth_error_percentile

    def __call__(
        self,
        pred_depth: Tensor,
        gt_depth: Tensor,
        weights: Tensor,
        t_vals: Tensor,
        epsilon: float,
        name: str = None,
        coef_decay: float = 1.0,
    ):
        if self.loss_type != "my":
            raise NotImplementedError(f"Unknown loss type: {self.loss_type}")
        name = self.name if name is None else name
        if torch.is_tensor(epsilon):
            if coef_decay != 1.0:
                raise ValueError("LineOfSightLoss: with device constants, coef_decay is their last value")
            value = _ops.line_of_sight_loss(weights, t_vals, gt_depth, epsilon, post=self.coef)
        else:
            value = _ops.line_of_sight_loss(weights, t_vals, gt_depth, epsilon, pre=coef_decay, post=self.coef)
        return self._result(name, value)


class DynamicRegularizationLoss(Loss):
    """``sparsity``: ``coef * mean(dynamic_density)``; ``entropy``: ``coef * mean`` of the binary entropy of
    ``clamp((dynamic / (dynamic + static + 1e-7)) ** entropy_skewness, 1e-6, 1 - 1e-6)``.  The shadow regulariser is
    this class with ``name="shadow"``, fed the shadow ratio."""

    def __init__(
        self,
        name: str = "dynamic",
        loss_type: Literal["sparsity", "entropy"] = "sparsity",
        coef: float = 1.0,
        entropy_skewness: float = 2.0,
        reduction="mean",
        check_nan=False,
    ):
        super(DynamicRegularizationLoss, self).__init__(coef, check_nan, reduction)
        if loss_type not in ("sparsity", "entropy"):
            raise NotImplementedError(f"Unknown loss type: {loss_type}")
        self.loss_type = loss_type
        self.entropy_skewness = entropy_skewness
        self.name = f"{name}_{self.loss_type}_loss"

    def __call__(
        self,
        dynamic_density: Tensor,
        static_density: Tensor = None,
        mask: Tensor = None,
        name: str = None,
    ):
        if mask is not None:
            raise _unsupported("DynamicRegularizationLoss's mask")
        name = self.name if name is None else name
        if self.loss_type == "sparsity":
            value = _ops.pointwise_loss("sparsity", dynamic_density, None, post=self.coef)
        else:
            k = float(self.entropy_skewness)
            value = _ops.pointwise_loss("entropy", dynamic_density, static_density, p0=k, p1=k - 1, post=self.coef)
        return self._result(name, value)


FLOW_STAT_KEYS = ("max_forward_flow_norm", "max_backward_flow_norm", "max_forward_pred_backward_flow_norm",
                  "max_backward_pred_forward_flow_norm")


def flow_cycle_loss(extras: Dict[str, Tensor], coef: float = 0.01,
                    name: str = "cycle_loss") -> Tuple[Dict[str, Tensor], Dict[str, Tensor]]:
    """The flow variants' cycle-consistency loss and flow statistics of the reference's pixel pass
    (train_emernerf.py:700-740), in one launch each way:

        {name: coef * 0.5 * mean((forward_flow + forward_pred_backward_flow) ** 2
                                 + (backward_flow + backward_pred_forward_flow) ** 2)},
        {"max_forward_flow_norm": max |forward_flow|, ... for the four flows}

    ``extras`` is ``render_results["extras"]``, each flow ``[R, S, 3]``.  Only the two predicted flows receive a
    gradient; the statistics are 0-d device tensors without one, NaN when a row of their flow is.  An empty batch
    raises ``ValueError``, as the reference's ``.max()`` does."""
    value, stats = _ops.cycle_loss(extras["forward_flow"], extras["backward_flow"],
                                   extras["forward_pred_backward_flow"], extras["backward_pred_forward_flow"], coef)
    return {name: value}, dict(zip(FLOW_STAT_KEYS, stats.unbind(0)))


def line_of_sight_consts(epsilon: float, coef_decay: float = 1.0) -> list:
    """The four fp32 values a live ``LineOfSightLoss`` call reads, ``[epsilon, 2 sigma^2, 1 / sqrt(2 pi sigma^2),
    coef_decay]`` with ``sigma = epsilon / 3``, derived in double and rounded once, as the float call rounds them.
    Copy them into a float32 CUDA tensor of 4 and pass that as ``epsilon``."""
    return _ops.sight_consts(epsilon, coef_decay)


def dirac_delta_approx(x, mu=0, sigma=1e-5):
    """A Gaussian of standard deviation ``sigma`` around ``mu`` (the reference's helper, elementwise torch)."""
    return (1 / (math.sqrt(2 * torch.pi * sigma**2))) * torch.exp(
        -((x - mu) ** 2) / (2 * sigma**2)
    )


def compute_line_of_sight_loss(
    gt_depth: Tensor,
    weights: Tensor,
    t_vals: Tensor,
    epsilon: float = 2.0,
):
    """Per ray: ``(mean_r empty_r + mean_r near_r) * (gt_depth > 0)``, the reference's [R] result; the sums run in one
    launch (``LineOfSightLoss`` folds the final mean in as well)."""
    gt = gt_depth.squeeze()
    sight = _ops.line_of_sight_sum(weights, t_vals, gt, epsilon)
    return sight * (gt > 0)

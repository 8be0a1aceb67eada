"""Depth evaluation on the device: a replacement for the metric block of validate() (test_MaGNet.py:52-79,
train_MaGNet.py:153-180) and its ``utils.RunningAverageDict`` (utils/utils.py:160-174)."""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib, dist, ops
from .ops import METRIC_KEYS


class DepthMetrics:
    """Running average over images of the per-image metrics of ``ops.depth_metrics``, kept on the device.

    ``update`` adds every image of the batch (the reference scores only image 0 of each batch; its test loaders use
    batch 1) without a host read, so it can be captured in a CUDA graph once the accumulator exists (after the first
    update, or ``reset``).  ``value`` reads the accumulator once and returns the reference's dict.  Sums and the
    average are float64; an image without a valid pixel contributes NaN, as it does to the reference's average.

    An instance scores one of three forms: Gaussian predictions [mu, sigma] (full resolution or fused upsampling; nll
    is the Gaussian NLL), with ``nearest=True`` F-Net depth maps (train_FNet.py's validate(); nll is 0.0), or with
    ``variance=True`` D-Net's [mu, var] (test_DNet.py's validate(); nll of the variance itself).  The form is fixed at
    the first update and the others are refused, because the nll column means something different in each."""

    _FORMS = {"gaussian": "Gaussian predictions (nearest=False, variance=False)",
              "nearest": "F-Net depth maps (nearest=True)", "variance": "D-Net [mu, var] predictions (variance=True)"}

    def __init__(self, min_depth: float, max_depth: float, crop: Optional[str] = None):
        ops.crop_box(crop, 1, 1)                       # reject an unknown crop now, not at the first update
        self.min_depth, self.max_depth, self.crop = float(min_depth), float(max_depth), crop
        # (P, 14) float64: images seen, then the sums over images of the 13 columns of ops.depth_metrics
        self._acc: Optional[torch.Tensor] = None
        self._form: Optional[str] = None               # the form of the first update (a key of _FORMS)

    def reset(self) -> None:
        """Zero the running sums in place (a captured update keeps accumulating into the same memory)."""
        if self._acc is not None:
            self._acc.zero_()

    def update(self, pred_or_list, gt: torch.Tensor, up_mask: Optional[torch.Tensor] = None,
               k: Optional[int] = None, nearest: bool = False, variance: bool = False) -> torch.Tensor:
        """Score one batch: ``pred_or_list`` is (a list of up to 8) full-resolution (B,2,H,W) [mu, sigma], or with
        ``up_mask`` and ``k`` the quarter-resolution Gaussians of ``MagnetHead.forward_quarter``, or with
        ``nearest=True`` the (B,1,h,w) depth maps of ``MagnetF.predict`` / ``ops.plane_depth``, nearest-upsampled to
        the GT size, or with ``variance=True`` the full-resolution (B,2,H,W) [mu, var] of ``DnetHead`` (D-Net).
        Returns the (P,B,13) per-image rows of ``ops.depth_metrics``.  Half-precision predictions / masks
        (torch.autocast) are upcast."""
        nearest, variance = bool(nearest), bool(variance)
        form = "variance" if variance else "nearest" if nearest else "gaussian"
        if self._form is not None and form != self._form:
            raise _lib.MagnetError(f"this DepthMetrics scores {self._FORMS[self._form]}; use another instance for "
                                   "another form (its nll column differs)")
        preds = [pred_or_list] if isinstance(pred_or_list, torch.Tensor) else list(pred_or_list)
        pred_or_list = [p.float() for p in preds]
        up_mask = None if up_mask is None else up_mask.float()
        rows = ops.depth_metrics(pred_or_list, gt.float(), min_depth=self.min_depth, max_depth=self.max_depth, crop=self.crop,
                                 up_mask=up_mask, k=k, nearest=nearest, variance=variance)
        self._form = form
        P, B = rows.shape[0], rows.shape[1]
        if self._acc is None:
            self._acc = torch.zeros(P, 1 + _lib.MAGNET_METRICS_COLS, device=rows.device, dtype=torch.float64)
        elif self._acc.shape[0] != P or self._acc.device != rows.device:
            raise _lib.MagnetError(f"this DepthMetrics accumulates {self._acc.shape[0]} predictions on "
                                   f"{self._acc.device}, got {P} on {rows.device}")
        self._acc[:, 0] += B
        self._acc[:, 1:] += rows.sum(dim=1)
        return rows

    def all_reduce(self) -> None:
        """Sum the running sums over the ranks of ``torch.distributed`` (sharded evaluation); afterwards ``value`` is the
        average over every rank's images.  Call it once, after the last update."""
        if self._acc is None:
            raise _lib.MagnetError("DepthMetrics.all_reduce before any update")
        dist.sum_tensor_over_ranks_(self._acc)

    def images(self) -> int:
        """Number of images accumulated (one host read)."""
        return 0 if self._acc is None else int(self._acc[0, 0].item())

    def value(self, all_predictions: bool = False):
        """The reference's ``RunningAverageDict.get_value()`` (keys in METRIC_KEYS order) for the last prediction, or a
        list with one such dict per prediction.  One host read."""
        if self._acc is None:
            raise _lib.MagnetError("DepthMetrics.value before any update")
        acc = self._acc.cpu()
        out = [{key: float(acc[p, 2 + i] / acc[p, 0]) for i, key in enumerate(METRIC_KEYS)} for p in range(acc.shape[0])]
        return out if all_predictions else out[-1]

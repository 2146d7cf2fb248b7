"""MMDMetric (reference: generative/metrics/mmd.py) on b200_mmd."""
from __future__ import annotations

from collections.abc import Callable

import torch

from .. import ops
from .metric import Metric, require_cuda
from .ssim import device_of


class MMDMetric(Metric):
    """Maximum Mean Discrepancy with the linear kernel (Gretton et al., JMLR 13, 2012, eq. 3 with beta = 1 and
    gamma = 2): mean(Y Y^T) + mean(P P^T) - 2 mean(P Y^T) over the flattened samples, Y Y^T / V etc. the Gram matrices
    of the B rows of length V.  Smaller is closer.

    The three Gram means collapse to sum_v (ybar_v - pbar_v)^2 / V (ybar, pbar: the means over the batch), which the
    kernel sums in fp64 from the fp32 differences: the result is the difference of the terms without their
    cancellation, never negative, where the reference's three fp32 GEMMs can lose every digit when y is close to y_pred.

    Args:
        y_transform: callable applied to ``y`` first (e.g. a filter or a feature extractor), or None.
        y_pred_transform: callable applied to ``y_pred`` first, or None.

    ``metric(y, y_pred)`` (note the order) returns a 0-dim tensor in ``y``'s dtype.
    """

    def __init__(self, y_transform: Callable | None = None, y_pred_transform: Callable | None = None) -> None:
        super().__init__()
        self.y_transform = y_transform
        self.y_pred_transform = y_pred_transform

    def __call__(self, y: torch.Tensor, y_pred: torch.Tensor) -> torch.Tensor:
        if self.y_transform is not None:
            y = self.y_transform(y)
        if self.y_pred_transform is not None:
            y_pred = self.y_pred_transform(y_pred)
        if y_pred.shape != y.shape:
            raise ValueError("y_pred and y shapes dont match after being processed "
                             f"by their transforms, received y_pred: {y_pred.shape} and y: {y.shape}")
        for d in range(len(y.shape) - 1, 1, -1):
            y = y.squeeze(dim=d)
            y_pred = y_pred.squeeze(dim=d)
        require_cuda(y, y_pred)
        with device_of(y):
            out = ops.mmd(y, y_pred)
        return out if out.dtype == y.dtype else out.to(y.dtype)

"""MultiScaleSSIMMetric (reference: generative/metrics/ms_ssim.py): per scale one b200_ssim pass, an fp32 2x average
pooling (b200_avgpool2_f32, floor) between scales, and one b200_ssim_combine for prod_s relu(cs_s) ** w_s with the
last scale's SSIM in place of its CS: 3 * len(weights) - 1 launches per call, no host synchronisation."""
from __future__ import annotations

from collections.abc import Sequence

import torch

from .. import ops
from .metric import MetricReduction, RegressionMetric, require_cuda
from .ssim import (KernelType, _per_axis, as_5d, check_extent, check_image_dims, device_of,  # noqa: F401
                   separable_kernel)


class MultiScaleSSIMMetric(RegressionMetric):
    """Multi-Scale Structural Similarity (Wang, Simoncelli and Bovik, Asilomar 2003) per batch item.

    Args: those of :class:`SSIMMetric`, plus ``weights``, one per scale.  The image must be larger than
    ``(kernel_size - 1) * max(1, len(weights) - 1) ** 2`` along every axis (the reference's size check, kept as is).
    ``metric(y_pred, y)`` returns fp32 [B, 1] on the inputs' CUDA device.
    """

    def __init__(
        self,
        spatial_dims: int,
        data_range: float = 1.0,
        kernel_type: KernelType | str = KernelType.GAUSSIAN,
        kernel_size: int | Sequence[int] = 11,
        kernel_sigma: float | Sequence[float] = 1.5,
        k1: float = 0.01,
        k2: float = 0.03,
        weights: Sequence[float] = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333),
        reduction: MetricReduction | str = MetricReduction.MEAN,
        get_not_nans: bool = False,
    ) -> None:
        super().__init__(reduction=reduction, get_not_nans=get_not_nans)
        self.spatial_dims = spatial_dims
        self.data_range = data_range
        self.kernel_type = kernel_type
        self.kernel_size = _per_axis(kernel_size, spatial_dims)
        self.kernel_sigma = _per_axis(kernel_sigma, spatial_dims)
        self.k1 = k1
        self.k2 = k2
        self.weights = weights

    def _compute_metric(self, y_pred: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        check_image_dims(self.spatial_dims, y_pred.ndimension())
        weights_div = max(1, (len(self.weights) - 1)) ** 2
        spatial = y_pred.shape[2:]
        for i in range(len(spatial)):
            if spatial[i] // weights_div <= self.kernel_size[i] - 1:
                raise ValueError(
                    f"For a given number of `weights` parameters {len(self.weights)} and kernel size "
                    f"{self.kernel_size[i]}, the image height must be larger than "
                    f"{(self.kernel_size[i] - 1) * weights_div}.")
        taps, scale = separable_kernel(self.spatial_dims, self.kernel_type, self.kernel_size, self.kernel_sigma)
        require_cuda(y_pred, y)
        x5, y5 = as_5d(y_pred, self.spatial_dims), as_5d(y, self.spatial_dims)
        # the reference pools after every scale, the last included: an extent that would pool to nothing fails there
        shape = list(x5.shape)
        for s in range(len(self.weights)):
            check_extent(shape, taps)
            shape = shape[:2] + [n // 2 for n in shape[2:]] if self.spatial_dims == 3 else \
                shape[:3] + [n // 2 for n in shape[3:]]
        if min(shape[2:]) < 1:
            raise RuntimeError(f"avg_pool: output size is too small after {len(self.weights)} scales")
        c1, c2 = (self.k1 * self.data_range) ** 2, (self.k2 * self.data_range) ** 2
        scales = []
        with device_of(y_pred):
            for s in range(len(self.weights)):
                part, _, _ = ops.ssim_pass(x5, y5, taps, scale, c1, c2)
                scales.append(part)
                if s + 1 < len(self.weights):
                    x5, y5 = ops.avgpool2_f32(x5, self.spatial_dims), ops.avgpool2_f32(y5, self.spatial_dims)
            _, _, ms = ops.ssim_combine(scales, y_pred.shape[0], self.weights)
        return ms.view(-1, 1)

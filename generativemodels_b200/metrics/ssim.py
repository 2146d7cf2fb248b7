"""SSIMMetric and compute_ssim_and_cs (reference: generative/metrics/ssim.py) on b200_ssim: one fused pass filters
x, y, x^2, y^2 and xy with the separable kernel (W, then H, then D) and forms SSIM and CS per valid voxel; the metric
classes take the per-item means from b200_ssim_combine and never write the maps."""
from __future__ import annotations

import contextlib
from collections.abc import Sequence

import torch

from .. import ops
from ..utils.enums import _StrEnum
from .metric import MetricReduction, RegressionMetric, require_cuda


class KernelType(_StrEnum):
    GAUSSIAN = "gaussian"
    UNIFORM = "uniform"


def _per_axis(v, spatial_dims: int) -> tuple:
    return tuple(v) if isinstance(v, Sequence) else (v,) * spatial_dims


def gaussian_taps(kernel_size: int, sigma: float) -> list[float]:
    """Normalised 1-D Gaussian in fp32 at offsets (1 - k) / 2 .. (k - 1) / 2, as the reference builds each axis."""
    dist = torch.arange(start=(1 - kernel_size) / 2, end=(1 + kernel_size) / 2, step=1)
    g = torch.exp(-torch.pow(dist / sigma, 2) / 2)
    return (g / g.sum()).tolist()


def separable_kernel(spatial_dims: int, kernel_type, kernel_size, kernel_sigma) -> tuple[list, float]:
    """((taps_d, taps_h, taps_w), scale) for b200_ssim: the Gaussian's per-axis taps with scale 1, or all-ones taps
    with the uniform kernel's fp32 1 / prod(kernel_size) applied once."""
    ks = _per_axis(kernel_size, spatial_dims)[:spatial_dims]
    if kernel_type == KernelType.GAUSSIAN:
        sig = _per_axis(kernel_sigma, spatial_dims)
        taps = [gaussian_taps(k, s) for k, s in zip(ks, sig)]
        scale = 1.0
    elif kernel_type == KernelType.UNIFORM:
        taps = [[1.0] * k for k in ks]
        scale = (torch.ones(()) / torch.prod(torch.tensor(ks))).item()
    else:    # the reference reaches its convolutions with no kernel bound
        raise UnboundLocalError(f"kernel_type must be 'gaussian' or 'uniform', got {kernel_type!r}")
    if spatial_dims == 2:
        taps = [[1.0]] + taps
    return taps, scale


def as_5d(t: torch.Tensor, spatial_dims: int) -> torch.Tensor:
    return t.unsqueeze(2) if spatial_dims == 2 else t


def device_of(t: torch.Tensor):
    return torch.cuda.device(t.device) if t.is_cuda else contextlib.nullcontext()


def check_extent(shape: Sequence[int], taps: Sequence[Sequence[float]]) -> None:
    for n, t in zip(shape[2:], taps):
        if len(t) > n:
            raise RuntimeError(f"Kernel size can't be greater than actual input size: kernel "
                               f"{tuple(len(t) for t in taps)} on an input of spatial size {tuple(shape[2:])}")


def compute_ssim_and_cs(
    y_pred: torch.Tensor,
    y: torch.Tensor,
    spatial_dims: int,
    data_range: float = 1.0,
    kernel_type: KernelType | str = KernelType.GAUSSIAN,
    kernel_size: int | Sequence[int] = 11,
    kernel_sigma: float | Sequence[float] = 1.5,
    k1: float = 0.01,
    k2: float = 0.03,
) -> tuple[torch.Tensor, torch.Tensor]:
    """The SSIM and contrast-sensitivity maps [B, C, *(spatial - kernel_size + 1)] (fp32, valid convolution) of a batch
    of 2-D or 3-D images; inputs in fp32, fp64, fp16 or bf16 of any strides, computed in fp32."""
    if y.shape != y_pred.shape:
        raise ValueError(f"y_pred and y should have same shapes, got {y_pred.shape} and {y.shape}.")
    if spatial_dims not in (2, 3) or y_pred.dim() != spatial_dims + 2:
        raise ValueError(f"expected a batch of {spatial_dims}-D images [B, C, spatial...], got shape {tuple(y_pred.shape)}")
    taps, scale = separable_kernel(spatial_dims, kernel_type, kernel_size, kernel_sigma)
    require_cuda(y_pred, y)
    x5, y5 = as_5d(y_pred, spatial_dims), as_5d(y, spatial_dims)
    check_extent(x5.shape, taps)
    with device_of(y_pred):
        _, ssim_map, cs_map = ops.ssim_pass(x5, y5, taps, scale, (k1 * data_range) ** 2, (k2 * data_range) ** 2,
                                            maps=True)
    if spatial_dims == 2:
        ssim_map, cs_map = ssim_map.squeeze(2), cs_map.squeeze(2)
    return ssim_map, cs_map


def check_image_dims(spatial_dims: int, dims: int) -> None:
    if spatial_dims == 2 and dims != 4:
        raise ValueError(f"y_pred should have 4 dimensions (batch, channel, height, width) when using {spatial_dims} "
                         f"spatial dimensions, got {dims}.")
    if spatial_dims == 3 and dims != 5:
        raise ValueError(f"y_pred should have 4 dimensions (batch, channel, height, width, depth) when using "
                         f"{spatial_dims} spatial dimensions, got {dims}.")
    if spatial_dims not in (2, 3):
        raise ValueError(f"spatial_dims must be 2 or 3, got {spatial_dims}.")


class SSIMMetric(RegressionMetric):
    r"""Structural Similarity Index Measure per batch item:

    .. math::
        \operatorname{SSIM}(x, y) = \frac{(2 \mu_x \mu_y + c_1)(2 \sigma_{xy} + c_2)}
                                         {(\mu_x^2 + \mu_y^2 + c_1)(\sigma_x^2 + \sigma_y^2 + c_2)}

    averaged over the channels and the valid voxels of each item (Wang et al., IEEE TIP 13(4), 2004).

    Args:
        spatial_dims: 2 or 3.
        data_range: value range of the images (usually 1.0 or 255).
        kernel_type: "gaussian" or "uniform".
        kernel_size: window size, one int or one per spatial axis (any size up to 128 taps whose tile fits in
            shared memory: about 100 per axis in 3-D).
        kernel_sigma: standard deviation of the Gaussian window, one float or one per axis.
        k1, k2: stability constants of the luminance and contrast terms.
        reduction: how ``aggregate`` reduces the buffer: "none", "mean", "sum", "mean_batch", "sum_batch",
            "mean_channel" or "sum_channel", NaNs excluded.
        get_not_nans: ``aggregate`` also returns the count of non-NaN values.

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

    def _compute_metric(self, y_pred: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        check_image_dims(self.spatial_dims, y_pred.ndimension())
        taps, scale = separable_kernel(self.spatial_dims, self.kernel_type, self.kernel_size, self.kernel_sigma)
        require_cuda(y_pred, y)
        x5, y5 = as_5d(y_pred, self.spatial_dims), as_5d(y, self.spatial_dims)
        check_extent(x5.shape, taps)
        with device_of(y_pred):
            part, _, _ = ops.ssim_pass(x5, y5, taps, scale, (self.k1 * self.data_range) ** 2,
                                       (self.k2 * self.data_range) ** 2)
            ssim, _, _ = ops.ssim_combine([part], y_pred.shape[0])
        return ssim.view(-1, 1)

"""Sample-quality metrics of the reference's ``generative.metrics`` on the CUDA path: SSIM, MS-SSIM and MMD.

Every per-voxel operation runs in libb200gen.so (b200_ssim, b200_avgpool2_f32, b200_ssim_combine, b200_mmd); the
classes here restate MONAI's metric bookkeeping (a buffer of per-item values, ``aggregate`` / ``reset``) on the host.
FID is not provided: its cost is a dense matrix square root, which the reference itself computes with scipy."""
from .metric import Cumulative, CumulativeIterationMetric, IterationMetric, Metric, MetricReduction, RegressionMetric
from .metric import do_metric_reduction
from .mmd import MMDMetric
from .ms_ssim import MultiScaleSSIMMetric
from .ssim import KernelType, SSIMMetric, compute_ssim_and_cs

__all__ = ["KernelType", "SSIMMetric", "compute_ssim_and_cs", "MultiScaleSSIMMetric", "MMDMetric", "Metric",
           "IterationMetric", "Cumulative", "CumulativeIterationMetric", "RegressionMetric", "MetricReduction",
           "do_metric_reduction"]

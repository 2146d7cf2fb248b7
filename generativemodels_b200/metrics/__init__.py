"""Sample-quality metrics of the reference's ``generative.metrics`` on the CUDA path: SSIM, MS-SSIM, MMD and FID.

Every per-voxel operation runs in libb200gen.so (b200_ssim, b200_interpolate, b200_ssim_combine, b200_mmd); the
classes here restate MONAI's metric bookkeeping (a buffer of per-item values, ``aggregate`` / ``reset``) on the host.
FID runs whole on the GPU in fp64 (b200_fid_moments, b200_frechet): the trace of the matrix square root, which the
reference takes with scipy on the host, comes from the eigenvalues of a symmetric matrix of the same nonzero spectrum."""
from .fid import FIDMetric, compute_frechet_distance, get_fid_score
from .metric import Cumulative, CumulativeIterationMetric, IterationMetric, Metric, MetricReduction, RegressionMetric
from .metric import do_metric_reduction
from .mmd import MMDMetric
from .ms_ssim import MultiScaleSSIMMetric
from .ssim import KernelType, SSIMMetric, compute_ssim_and_cs

__all__ = ["KernelType", "SSIMMetric", "compute_ssim_and_cs", "MultiScaleSSIMMetric", "MMDMetric", "FIDMetric",
           "get_fid_score", "compute_frechet_distance", "Metric", "IterationMetric", "Cumulative",
           "CumulativeIterationMetric", "RegressionMetric", "MetricReduction", "do_metric_reduction"]

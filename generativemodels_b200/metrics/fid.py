"""FIDMetric (reference: generative/metrics/fid.py) on b200_fid_moments and b200_frechet."""
from __future__ import annotations

import torch

from .. import ops
from .metric import Metric, require_cuda
from .ssim import device_of


class FIDMetric(Metric):
    """Frechet Inception Distance (Heusel et al., "GANs trained by a two time-scale update rule converge to a local
    Nash equilibrium", NeurIPS 2017) between two sets of feature vectors, [number of images, number of features] each,
    from a pretrained network (Inception v3 pool_3 features, or RadImageNet / MedicalNet ones for medical images):

        FID = |mu_p - mu_y|^2 + tr Sigma_p + tr Sigma_y - 2 tr sqrt(Sigma_p Sigma_y)

    ``metric(y_pred, y)`` returns a 0-dim float64 tensor on the inputs' device; see :func:`get_fid_score`.
    """

    def __init__(self) -> None:
        super().__init__()

    def __call__(self, y_pred: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        return get_fid_score(y_pred, y)


def get_fid_score(y_pred: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """FID between the rows of ``y_pred`` [n_p, F] and ``y`` [n_y, F] (n_p and n_y may differ, both >= 2), fp32, fp64,
    fp16 or bf16 CUDA tensors of any strides, read in place.  Everything is computed in fp64 on the GPU without a host
    synchronisation, so a call can be captured in a CUDA graph.

    The moments are the reference's (column means; covariances with 1 / (n - 1) from the centred values).  The trace of
    the square root is that of the symmetric M = L^T Sigma_p L, Sigma_y = L L^T by pivoted Cholesky, from M's
    eigenvalues; eigenvalues at or below F * 2^-52 * max(eigenvalue) count as zero.  Where the reference differs:

    * It takes scipy's sqrtm of the non-symmetric Sigma_p Sigma_y; on rank-deficient covariances (fewer images than
      features) that trace carries noise of about 1e-8 relative, and on some inputs a rounding-level imaginary part
      makes it raise ``ValueError``.  Here the value is exact to rounding and never raises for it.
    * Non-finite features give NaN (scipy raises ``LinAlgError``; raising would need a host synchronisation).

    Raises ValueError when ``y`` has more than 2 dimensions (the reference's message), RuntimeError for other shapes the
    reference cannot compute (``y_pred`` not 2-D, one row, different feature counts) and for CPU tensors.
    """
    if y.ndim > 2:
        raise ValueError("Inputs should have (number images, number of features) shape.")
    require_cuda(y_pred, y)
    if y_pred.ndim != 2 or y.ndim != 2:
        raise RuntimeError(f"features must be [number of images, number of features], got y_pred "
                           f"{tuple(y_pred.shape)} and y {tuple(y.shape)}")
    if y_pred.shape[0] < 2 or y.shape[0] < 2:
        raise RuntimeError(f"a covariance needs at least 2 images, got {y_pred.shape[0]} and {y.shape[0]}")
    if y_pred.shape[1] != y.shape[1]:
        raise RuntimeError(f"y_pred has {y_pred.shape[1]} features but y has {y.shape[1]}")
    with device_of(y):
        mu_p, sigma_p = ops.fid_moments(y_pred)
        mu_y, sigma_y = ops.fid_moments(y)
        return ops.frechet(mu_p, sigma_p, mu_y, sigma_y)


def compute_frechet_distance(mu_x: torch.Tensor, sigma_x: torch.Tensor, mu_y: torch.Tensor, sigma_y: torch.Tensor,
                             epsilon: float = 1e-6) -> torch.Tensor:
    """The Frechet distance between N(mu_x, sigma_x) and N(mu_y, sigma_y): mu [F] and sigma [F, F] CUDA tensors, e.g.
    cached statistics of a real data set.  The sigmas must be symmetric positive semidefinite, as covariances are; they
    are read as fp64.  ``epsilon`` is accepted for the reference's signature: it is used there only to retry a
    non-finite matrix square root, which this formulation never produces.  Returns a 0-dim float64 tensor."""
    del epsilon
    require_cuda(mu_x, sigma_x, mu_y, sigma_y)
    F = mu_x.shape[0] if mu_x.ndim == 1 else -1
    if F < 1 or any(t.shape != (F,) for t in (mu_x, mu_y)) or any(t.shape != (F, F) for t in (sigma_x, sigma_y)):
        raise RuntimeError(f"expected mu [F] and sigma [F, F] of one F, got {tuple(mu_x.shape)}, "
                           f"{tuple(sigma_x.shape)}, {tuple(mu_y.shape)}, {tuple(sigma_y.shape)}")
    with device_of(mu_x):
        args = [t.to(torch.float64).contiguous() for t in (mu_x, sigma_x, mu_y, sigma_y)]
        return ops.frechet(*args)

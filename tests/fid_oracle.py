"""Torch / scipy restatement of the reference's FID arithmetic (generative/metrics/fid.py) that runs on NumPy 2 and
SciPy 1.18: fp64 moments, scipy's sqrtm of Sigma_p Sigma_y on the host, the finite check with its epsilon retry and the
imaginary-part check.  Pinned against the unmodified reference by tests/test_fid_oracle_vs_reference.py; the baseline
tools/metrics_probe.py times on the GPU (moments there, sqrtm on the host)."""
import numpy as np
import scipy.linalg
import torch


def cov(x):
    """fid.py's _cov(x, rowvar=False)."""
    if x.dim() < 2:
        x = x.view(1, -1)
    if x.size(0) != 1:
        x = x.t()
    factor = 1.0 / (x.size(1) - 1)
    x = x - torch.mean(x, dim=1, keepdim=True)
    return factor * x.matmul(x.t()).squeeze()


_SQRTM = scipy.linalg.sqrtm     # bound at import: tests patch scipy.linalg.sqrtm for the reference's own calls


def sqrtm(a):
    """scipy's sqrtm on the host in float64 (the reference's _sqrtm without the `disp` argument SciPy 1.18 dropped)."""
    return torch.from_numpy(_SQRTM(a.detach().cpu().numpy().astype(np.float64)))


def frechet_distance(mu_x, sigma_x, mu_y, sigma_y, epsilon=1e-6):
    diff = mu_x - mu_y
    covmean = sqrtm(sigma_x.mm(sigma_y))
    if not torch.isfinite(covmean).all():
        offset = torch.eye(sigma_x.size(0), device=mu_x.device, dtype=mu_x.dtype) * epsilon
        covmean = sqrtm((sigma_x + offset).mm(sigma_y + offset))
    if torch.is_complex(covmean):
        if not torch.allclose(torch.diagonal(covmean).imag, torch.tensor(0, dtype=torch.double), atol=1e-3):
            raise ValueError(f"Imaginary component {torch.max(torch.abs(covmean.imag))} too high.")
        covmean = covmean.real
    return diff.dot(diff) + torch.trace(sigma_x).cpu() + torch.trace(sigma_y).cpu() - 2 * torch.trace(covmean)


def fid(y_pred, y):
    """get_fid_score: fp64 moments (on the inputs' device), then frechet_distance."""
    y, y_pred = y.double(), y_pred.double()
    if y.ndimension() > 2:
        raise ValueError("Inputs should have (number images, number of features) shape.")
    return frechet_distance(torch.mean(y_pred, dim=0), cov(y_pred), torch.mean(y, dim=0), cov(y))

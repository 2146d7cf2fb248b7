"""Float64 reading of the FID entry points of include/b200gen_fid.h (b200_fid_moments, b200_frechet), the contract the
GPU tests hold the kernels to and the CPU stand-in (tests/fid_backend.py) computes with.  Inputs are converted to fp64
exactly, as the kernels load them; the factor follows the header's pivot and stop rule, the eigenvalues come from
numpy's eigvalsh and the header's cutoff drops the rounding-level ones.

Bounds (e = 2^-53, the fp64 unit roundoff), which the f64 tolerance adds one ulp to:
  mu (``moments_bound``): n values summed in fp64 in any order, then one division: (n + 2) e sum |x| / n.
  sigma: each centred value c = x - mu' (mu' the device's mean) rounds once, the Gram's n fp64 fmas round once each,
  and the scaling by fp64(1 / (n - 1)) twice: (n + 4) e sum_k |c_ki c_kj| / (n - 1).  The device's mean error
  d = mu' - mu enters as d_j sum_k c_ki + d_i sum_k c_kj + n d_i d_j; the exact centred columns sum to 0, so only
  n d_i d_j / (n - 1) is left, with |d| bounded as above.
  b200_frechet (``frechet_bounds``): the distance within 1e-8 S, S = tr Sigma_x + tr Sigma_y + |mu_x - mu_y|^2 (the
  scale of every term; tests/test_fid_gpu.py holds its sweep to the same bound), the eigenvalues within
  max(F, 4) 2^-52 max(mu_max, 0) (the backward error of the factor, the two GEMMs and the bisection, relative to the
  largest eigenvalue; at least the few roundings that form a 1 x 1 or 2 x 2 M) and the rank exactly.
"""
import numpy as np
import torch

F64 = torch.float64
E53 = 2.0 ** -53


def fid_moments(x):
    """b200_fid_moments of a 2-D [n, F] view: float64 column means and (X - mu)^T (X - mu) / (n - 1)."""
    x = x.to(F64)      # exact for every input format
    mu = x.mean(0)
    c = x - mu
    return mu, c.T @ c / (x.shape[0] - 1)


def moments_bound(x):
    """(mu_err [F], sigma_err [F, F]) of ``moments_bound`` in the module docstring, for a 2-D [n, F] view."""
    x = x.to(F64)
    n = x.shape[0]
    ax = x.abs()
    mu_err = (n + 2) * E53 * ax.sum(0) / n
    c = (x - x.mean(0)).abs()
    return mu_err, ((n + 4) * E53 * (c.T @ c) + n * torch.outer(mu_err, mu_err)) / (n - 1)


def frechet_bounds(mu_x, sx, mu_y, sy, eig):
    """(distance bound, eigenvalue bound) of ``frechet_bounds`` in the module docstring, float64."""
    mu_x, sx, mu_y, sy = (np.asarray(t, dtype=np.float64) for t in (mu_x, sx, mu_y, sy))
    d = mu_x - mu_y
    S = abs(float(np.trace(sx) + np.trace(sy) + d @ d))
    top = float(eig[-1]) if np.isfinite(eig[-1]) else 0.0
    return 1e-8 * S, max(mu_x.shape[0], 4) * 2.0 ** -52 * max(top, 0.0)


def pivoted_cholesky(s):
    """b200_frechet's factor of a symmetric PSD numpy [F, F]: (G = P L [F, F] in feature order, rank r).  The pivot is
    the largest remaining diagonal entry among features not yet chosen, the lowest feature index on a tie; the factor
    stops at the first step whose maximum is <= F * 2^-52 * max(diag) or not a number.  Rows and columns are swapped
    physically here (LAPACK's way), with `piv` mapping positions to features."""
    a = np.array(s, dtype=np.float64)
    n = a.shape[0]
    piv = np.arange(n)
    dg = np.diag(a)
    tol = n * 2.0 ** -52 * max(0.0, np.nanmax(np.where(dg > 0, dg, 0.0)))
    r = 0
    for j in range(n):
        rest = np.diag(a)[j:]
        rest = np.where(np.isnan(rest), -np.inf, rest)
        best = rest.max()
        if not best > tol:
            break
        ties = np.flatnonzero(rest == best)
        q = j + ties[np.argmin(piv[j + ties])]
        a[[j, q]] = a[[q, j]]
        a[:, [j, q]] = a[:, [q, j]]
        piv[[j, q]] = piv[[q, j]]
        d = np.sqrt(a[j, j])
        a[j, j] = d
        a[j + 1:, j] /= d
        a[j + 1:, j + 1:] -= np.outer(a[j + 1:, j], a[j + 1:, j])
        r = j + 1
    L = np.tril(a)[:, :r]
    G = np.zeros((n, n))
    G[piv, :r] = L
    return G, r


def frechet(mu_x, sx, mu_y, sy):
    """b200_frechet: (distance, the F eigenvalues of M = G^T sx G ascending, rank of G), float64 numpy."""
    mu_x, sx, mu_y, sy = (np.asarray(t, dtype=np.float64) for t in (mu_x, sx, mu_y, sy))
    n = mu_x.shape[0]
    G, r = pivoted_cholesky(sy)
    m = G.T @ (sx @ G)
    m = (m + m.T) / 2
    eig = np.linalg.eigvalsh(m) if np.isfinite(m).all() else np.full(n, np.nan)
    cutoff = n * 2.0 ** -52 * eig[-1]
    tr = np.sqrt(eig[~(eig <= cutoff)]).sum()
    d = mu_x - mu_y
    return float(d @ d + np.trace(sx) + np.trace(sy) - 2 * tr), eig, r

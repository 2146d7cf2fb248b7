"""Float64 reading of the FID entry points of include/b200gen_fid.h (b200_fid_moments, b200_frechet), the contract the
GPU tests hold the kernels to and the CPU stand-in (tests/fid_backend.py) computes with.  Inputs are converted to fp64
exactly, as the kernels load them; the factor follows the header's pivot and stop rule, the eigenvalues come from
numpy's eigvalsh and the header's cutoff drops the rounding-level ones."""
import numpy as np
import torch

F64 = torch.float64


def fid_moments(x):
    """b200_fid_moments of a 2-D [n, F] view: float64 column means and (X - mu)^T (X - mu) / (n - 1)."""
    x = x.to(F64)      # exact for every input format
    mu = x.mean(0)
    c = x - mu
    return mu, c.T @ c / (x.shape[0] - 1)


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

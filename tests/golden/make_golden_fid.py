"""Generate the FID fixture (tests/golden/g_fid.pt) by running the UNMODIFIED reference FIDMetric (the reference
checkout named by REFERENCE_DIR, CPU float64, MONAI shim):   python -m tests.golden.make_golden_fid

The reference's fid.py needs two shims on NumPy 2 / SciPy 1.18, applied around its calls only: numpy.float_ (removed in
NumPy 2) is numpy.float64, and scipy.linalg.sqrtm accepts `disp` again and returns (sqrtm(A), 0.0).

Inputs are regenerated from each case's seed by `inputs` below, so the fixture stores the seeds, the arguments, a
float64 checksum of the inputs, the reference's output (or the exception it raised) and an exact value.  "relu"
features are relu of correlated Gaussians with per-feature scales and offsets: a stand-in for the pooled activations of
a CNN.  Cases:
  ref_test_results          the reference's tests/test_compute_fid_metric.py (0.4444; Sigma_pred = 0)
  relu_100x64_vs_80x64      full rank, unequal counts
  singular_30x256_vs_40x256 fewer images than features in both sets
  two_rows                  2 x 16 vs 2 x 16
  identical                 one 50 x 32 set against itself
  dead_features             200 x 64 vs 150 x 64 with 8 features zero in both (singular with n > F)
  fp16                      150 x 96 vs 120 x 96 fp16 features
  tutorial_1000x2048        1000 x 2048 vs 1000 x 2048 (the realism-diversity tutorial's shape; RadImageNet ResNet-50
                            gives 2048 features)
  large_4000x2048           4000 x 2048 vs 3000 x 2048
  scaled_1e4                20 x 256 vs 20 x 256 features times 1e4, where the reference raises ValueError (a
                            rounding-level imaginary part of its sqrtm)
The exact value: with A the smaller set's centred data / sqrt(n - 1) and Sigma_o the other set's covariance, the
eigenvalues of A Sigma_o A^T when that set has at most F rows; otherwise those of W^T Sigma_p W with W = V Lambda^(1/2)
from eigh(Sigma_y).  Eigenvalues at or below F * 2^-52 * max(eigenvalue) count as zero, as b200_frechet counts them.
S = tr Sigma_p + tr Sigma_y + |mu_p - mu_y|^2, the scale of every tolerance, is recorded too.
"""
import numpy as np
import scipy.linalg
import torch

from tests.golden import save
from oracle import ref_import

F64 = torch.float64

CASES = {
    "ref_test_results": dict(gen="ref_test", singular=True),
    "relu_100x64_vs_80x64": dict(gen="relu", n=(100, 80), F=64, seed=1, singular=False),
    "singular_30x256_vs_40x256": dict(gen="relu", n=(30, 40), F=256, seed=2, singular=True),
    "two_rows": dict(gen="relu", n=(2, 2), F=16, seed=3, singular=True),
    "identical": dict(gen="identical", n=(50, 50), F=32, seed=4, singular=False),
    "dead_features": dict(gen="relu", n=(200, 150), F=64, seed=5, dead=8, singular=True),
    "fp16": dict(gen="relu", n=(150, 120), F=96, seed=6, dtype="fp16", singular=False),
    "tutorial_1000x2048": dict(gen="relu", n=(1000, 1000), F=2048, seed=7, singular=True),
    "large_4000x2048": dict(gen="relu", n=(4000, 3000), F=2048, seed=8, singular=False),
    "scaled_1e4": dict(gen="relu", n=(20, 20), F=256, seed=9, scale=1e4, singular=True),
}


def features(n, F, seed, shift=0.0, dead=0, scale=1.0):
    """relu of Gaussians correlated across neighbouring features, formed in float64 and rounded to fp32 once."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(n, F + 2, generator=g, dtype=F64)
    c = z[:, 2:] + 0.7 * z[:, 1:-1] + 0.3 * z[:, :-2]
    f = torch.arange(F, dtype=F64)
    x = torch.relu(c * (1 + (f % 7) / 3) + ((f % 5) - 2) * 0.25 + shift)
    if dead:
        x[:, :dead] = 0
    return (x * scale).float()


def inputs(case):
    """(y_pred, y) on the CPU."""
    if case["gen"] == "ref_test":
        return torch.Tensor([[1, 2], [1, 2], [1, 2]]), torch.Tensor([[2, 2], [1, 2], [1, 2]])
    (n_p, n_y), F, seed = case["n"], case["F"], case["seed"]
    kw = dict(dead=case.get("dead", 0), scale=case.get("scale", 1.0))
    y = features(n_y, F, 1000 + seed, **kw)
    p = y.clone() if case["gen"] == "identical" else features(n_p, F, seed, shift=0.1, **kw)
    if case.get("dtype") == "fp16":
        p, y = p.half(), y.half()
    return p, y


def checksum(t):
    return t.double().sum(0)


def exact(y_pred, y):
    """(FID, S) in float64 numpy through a symmetric eigenvalue problem (see the module docstring)."""
    p, q = y_pred.double().numpy(), y.double().numpy()
    F = p.shape[1]
    mp, mq = p.mean(0), q.mean(0)
    cp, cq = p - mp, q - mq
    sp, sq = cp.T @ cp / (len(p) - 1), cq.T @ cq / (len(q) - 1)
    a, other = (cp / np.sqrt(len(p) - 1), sq) if len(p) <= len(q) else (cq / np.sqrt(len(q) - 1), sp)
    if a.shape[0] <= F:
        m = a @ other @ a.T
    else:
        lam, v = np.linalg.eigh(sq)
        w = v * np.sqrt(np.clip(lam, 0, None))
        m = w.T @ sp @ w
    eig = np.linalg.eigvalsh((m + m.T) / 2)
    tr = np.sqrt(eig[eig > F * 2.0 ** -52 * eig[-1]]).sum()
    d = mp - mq
    s = float(np.trace(sp) + np.trace(sq) + d @ d)
    return float(d @ d + np.trace(sp) + np.trace(sq) - 2 * tr), s


class shims:
    """numpy.float_ and sqrtm(..., disp) for the reference's fid.py, restored on exit."""

    def __enter__(self):
        self.had_float_ = hasattr(np, "float_")
        self.sqrtm = scipy.linalg.sqrtm
        np.float_ = np.float64
        scipy.linalg.sqrtm = lambda a, disp=True: (self.sqrtm(a), 0.0)
        return self

    def __exit__(self, *exc):
        scipy.linalg.sqrtm = self.sqrtm
        if not self.had_float_:
            del np.float_
        return False


def main():
    ref_import.import_reference()
    from generative.metrics import FIDMetric
    out = {}
    for name, case in CASES.items():
        rec = dict(case)
        p, y = inputs(case)
        rec["checksum"] = [checksum(p), checksum(y)]
        rec["exact"], rec["S"] = exact(p, y)
        try:
            with shims():
                rec["out"] = torch.as_tensor(FIDMetric()(p, y), dtype=F64)
            rec["error"] = None
        except ValueError as e:
            rec["out"], rec["error"] = None, f"ValueError: {e}"
        out[name] = rec
        ref = "raised " + rec["error"] if rec["error"] else f"{float(rec['out']):.10e}"
        print(f"{name}: reference {ref}, exact {rec['exact']:.10e}, S {rec['S']:.4e}", flush=True)
    save(out, "g_fid")


if __name__ == "__main__":
    main()

"""TEST-ONLY CPU stand-in for the FID entry points of libb200gen.so (include/b200gen_fid.h), on HOST pointers:
tests/metrics_backend.MetricsFakeLib extended by b200_fid_moments, b200_frechet_workspace_bytes and b200_frechet, each
viewing its pointers as host arrays and storing what the float64 reading of the contract (tests/fid_emulator.py)
computes.  install() routes the product's C-ABI calls, the other metrics' and the sampling path's included, to it."""
import ctypes as C

from generativemodels_b200 import _lib
from tests import cpu_backend
from tests import fid_emulator as E
from tests import metrics_backend
from tests.cpu_backend import _np, _obj
from tests.cpu_backend import _strided as view


class FidFakeLib(metrics_backend.MetricsFakeLib):
    def b200_fid_moments(self, p, stream):
        p = _obj(p)
        x = view(p.x, p.x_dtype, list(p.x_strides), [p.n, p.F])
        mu, sigma = E.fid_moments(x)
        _np(p.mu, p.F, C.c_double)[:] = mu.numpy()
        _np(p.sigma, p.F * p.F, C.c_double)[:] = sigma.reshape(-1).numpy()
        return 0

    def b200_frechet_workspace_bytes(self, F):
        return 8

    def b200_frechet(self, p, stream):
        p = _obj(p)
        F_ = p.F
        mx, my = (_np(q, F_, C.c_double) for q in (p.mu_x, p.mu_y))
        sx, sy = (_np(q, F_ * F_, C.c_double).reshape(F_, F_) for q in (p.sigma_x, p.sigma_y))
        fid, eig, r = E.frechet(mx, sx, my, sy)
        _np(p.out, 1, C.c_double)[0] = fid
        if p.eigvals:
            _np(p.eigvals, F_, C.c_double)[:] = eig
        if p.rank:
            _np(p.rank, 1, C.c_int32)[0] = r
        return 0


def install(monkeypatch):
    """cpu_backend.install, with the stand-in that also serves the metric and FID entry points (tests only)."""
    cpu_backend.install(monkeypatch)
    fake = FidFakeLib()
    monkeypatch.setattr(_lib, "require_device", lambda: fake)
    return fake

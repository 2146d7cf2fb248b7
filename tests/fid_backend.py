"""TEST-ONLY CPU stand-in for the FID entry points of libb200gen.so (include/b200gen_fid.h), on HOST pointers:
tests/metrics_backend.MetricsFakeLib extended by b200_fid_moments, b200_frechet_workspace_bytes and b200_frechet, each
viewing its pointers as host arrays and storing what the float64 reading of the contract (tests/fid_emulator.py)
computes, with its bound, through cpu_backend's reporting store.  install() routes the product's C-ABI calls, the other
metrics' and the sampling path's included, to it."""
import ctypes as C

import numpy as np
import torch

from generativemodels_b200 import _lib
from tests import cpu_backend
from tests import elementwise_emulator as W
from tests import fid_emulator as E
from tests import metrics_backend
from tests.cpu_backend import _np, _obj, put
from tests.cpu_backend import _strided as view


def _f64(ptr, count):
    return torch.from_numpy(_np(ptr, count, C.c_double))


class FidFakeLib(metrics_backend.MetricsFakeLib):
    def b200_fid_moments(self, p, stream):
        p = _obj(p)
        x = view(p.x, p.x_dtype, list(p.x_strides), [p.n, p.F])
        mu, sigma = E.fid_moments(x)
        if cpu_backend.RECORDER is None:        # the bound costs a second Gram; only a recorder reads it
            emu, esig = torch.zeros_like(mu), torch.zeros_like(sigma)
        else:
            emu, esig = E.moments_bound(x)
        put(_f64(p.mu, p.F), W.Result(mu, mu, emu, "f64"))
        put(_f64(p.sigma, p.F * p.F).view(p.F, p.F), W.Result(sigma, sigma, esig, "f64"))
        return 0

    def b200_frechet_workspace_bytes(self, F):
        return 8

    def b200_frechet(self, p, stream):
        p = _obj(p)
        F_ = p.F
        mx, my = (_np(q, F_, C.c_double) for q in (p.mu_x, p.mu_y))
        sx, sy = (_np(q, F_ * F_, C.c_double).reshape(F_, F_) for q in (p.sigma_x, p.sigma_y))
        fid, eig, r = E.frechet(mx, sx, my, sy)
        efid, eeig = E.frechet_bounds(mx, sx, my, sy, eig)
        v = torch.tensor([fid], dtype=torch.float64)
        put(_f64(p.out, 1), W.Result(v, v, torch.tensor([efid], dtype=torch.float64), "f64"))
        if p.eigvals:
            ev = torch.from_numpy(np.ascontiguousarray(eig, dtype=np.float64))
            put(_f64(p.eigvals, F_), W.Result(ev, ev, torch.full_like(ev, eeig), "f64"))
        if p.rank:
            put(torch.from_numpy(_np(p.rank, 1, C.c_int32)), W.copy(torch.tensor([float(r)], dtype=torch.float64)))
        return 0


def install(monkeypatch):
    """cpu_backend.install, with the stand-in that also serves the metric and FID entry points (tests only)."""
    cpu_backend.install(monkeypatch)
    fake = FidFakeLib()
    monkeypatch.setattr(_lib, "require_device", lambda: fake)
    return fake

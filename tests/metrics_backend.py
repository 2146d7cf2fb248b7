"""TEST-ONLY CPU stand-in for the metric entry points of libb200gen.so (include/b200gen_metrics.h), on HOST pointers:
tests/cpu_backend.FakeLib extended by one method per metric symbol, each viewing its pointers as host tensors and
storing what the float64 reading of the contract (tests/metrics_emulator.py) computes; the pooling between MS-SSIM
scales is cpu_backend's b200_interpolate.  install() routes the product's
C-ABI calls, the sampling path's included, to it."""
import ctypes as C

import torch

from generativemodels_b200 import _lib
from tests import cpu_backend
from tests import metrics_emulator as M
from tests.cpu_backend import _np, _obj, store32
from tests.cpu_backend import _strided as view


class MetricsFakeLib(cpu_backend.FakeLib):
    def b200_ssim_workspace_bytes(self, p):
        return _obj(p).N * 16           # one slot per item: the reading's sums

    def b200_ssim(self, p, stream):
        p = _obj(p)
        shape = (p.N, p.C, p.D, p.H, p.W)
        x = view(p.x, p.x_dtype, list(p.x_strides), shape)
        y = view(p.y, p.y_dtype, list(p.y_strides), shape)
        taps = [list(t[:k]) for t, k in ((p.taps_d, p.kd), (p.taps_h, p.kh), (p.taps_w, p.kw))]
        s, cs = M.ssim(x, y, taps, p.scale, p.c1, p.c2)
        if p.ssim_map:
            store32(p.ssim_map, s)
        if p.cs_map:
            store32(p.cs_map, cs)
        sums = torch.stack([s.reshape(p.N, -1).sum(1), cs.reshape(p.N, -1).sum(1)], 1)
        _np(p.partials, p.N * 2, C.c_double)[:] = sums.reshape(-1).numpy()
        return 0

    def b200_ssim_combine(self, p, stream):
        p = _obj(p)
        S, N_ = p.n_scales, p.N
        sums = [torch.from_numpy(_np(p.partials[s], N_ * p.slots[s] * 2, C.c_double).copy()).view(N_, -1, 2).sum(1)
                for s in range(S)]
        ssim = torch.stack([v[:, 0] / p.count[s] for s, v in enumerate(sums)]).float()
        cs = torch.stack([v[:, 1] / p.count[s] for s, v in enumerate(sums)]).float()
        if p.ssim_mean:
            store32(p.ssim_mean, ssim)
        if p.cs_mean:
            store32(p.cs_mean, cs)
        if p.ms_ssim:
            store32(p.ms_ssim, M.combine(ssim, cs, list(p.weights[:S])))
        return 0

    def b200_mmd_workspace_bytes(self, shape):
        return 8

    def b200_mmd(self, y, ydt, ys, p, pdt, ps, shape, ws, out, stream):
        shp = [int(v) for v in shape[:5]]
        a = view(y, ydt, [int(v) for v in ys[:5]], shp)
        b = view(p, pdt, [int(v) for v in ps[:5]], shp)
        store32(out, M.mmd(a, b).reshape(1))
        return 0


def install(monkeypatch):
    """cpu_backend.install, with the stand-in that also serves the metric entry points (tests only)."""
    cpu_backend.install(monkeypatch)
    fake = MetricsFakeLib()
    monkeypatch.setattr(_lib, "require_device", lambda: fake)
    return fake

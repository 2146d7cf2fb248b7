"""TEST-ONLY CPU stand-in for the metric entry points of libb200gen.so (include/b200gen_metrics.h), on HOST pointers:
tests/cpu_backend.FakeLib extended by one method per metric symbol, each viewing its pointers as host tensors and
storing what the float64 reading of the contract (tests/metrics_emulator.py) computes.  install() routes the product's
C-ABI calls, the sampling path's included, to it."""
import ctypes as C

import numpy as np
import torch

from generativemodels_b200 import _lib
from tests import cpu_backend
from tests import metrics_emulator as M
from tests.cpu_backend import _np, _obj, store32

_CTYPES = {_lib.DT_F32: (C.c_float, np.float32, None), _lib.DT_F64: (C.c_double, np.float64, None),
           _lib.DT_FP16: (C.c_uint16, np.int16, torch.float16), _lib.DT_BF16: (C.c_uint16, np.int16, torch.bfloat16)}


def view(ptr, dt, strides, shape):
    """A strided host view of a metric input in any of its four formats."""
    ctype, npt, as_dtype = _CTYPES[dt]
    count = 1 + sum((s - 1) * st for s, st in zip(shape, strides))
    flat = torch.from_numpy(_np(ptr, count, ctype).view(npt))
    return torch.as_strided(flat.view(as_dtype) if as_dtype else flat, tuple(shape), tuple(strides))


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

    def b200_avgpool2_f32(self, x, dt, xs, N_, C_, D, H, W_, dims, y, stream):
        store32(y, M.avgpool2(view(x, dt, [int(v) for v in xs[:5]], (N_, C_, D, H, W_)), dims))
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

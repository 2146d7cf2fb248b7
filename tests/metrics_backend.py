"""TEST-ONLY CPU stand-in for the metric entry points of libb200gen.so (include/b200gen_metrics.h), on HOST pointers:
tests/cpu_backend.FakeLib extended by one method per metric symbol, each viewing its pointers as host tensors and
storing what the float64 reading of the contract (tests/metrics_emulator.py) computes, with its bound, through
cpu_backend's reporting stores; the pooling between MS-SSIM scales is cpu_backend's b200_interpolate.  install() routes
the product's C-ABI calls, the sampling path's included, to it."""
import ctypes as C

import torch

from generativemodels_b200 import _lib
from tests import cpu_backend
from tests import elementwise_emulator as W
from tests import metrics_emulator as M
from tests.cpu_backend import _np, _obj, report, store32
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
        if cpu_backend.RECORDER is None:        # the bound costs as much again; only a recorder reads it
            s, cs = M.ssim(x, y, taps, p.scale, p.c1, p.c2)
            es = ecs = torch.zeros_like(s)
        else:
            s, cs, es, ecs = M.ssim_bound(x, y, taps, p.scale, p.c1, p.c2)
        if p.ssim_map:
            store32(p.ssim_map, W.Result(s, W.f32(s), es, "f32"))
        if p.cs_map:
            store32(p.cs_map, W.Result(cs, W.f32(cs), ecs, "f32"))
        slots = max(1, self.b200_ssim_workspace_bytes(p) // (16 * p.N))
        part = torch.from_numpy(_np(p.partials, p.N * slots * 2, C.c_double)).view(p.N, slots, 2)
        part.zero_()
        part[:, 0] = torch.stack([s.reshape(p.N, -1).sum(1), cs.reshape(p.N, -1).sum(1)], 1)
        report(part, M.slot_sums(s, cs, es, ecs, slots))
        return 0

    def b200_ssim_combine(self, p, stream):
        p = _obj(p)
        S, N_ = p.n_scales, p.N
        parts = [torch.from_numpy(_np(p.partials[s], N_ * p.slots[s] * 2, C.c_double).copy()).view(N_, -1, 2)
                 for s in range(S)]
        sums = [v.sum(1) for v in parts]
        ssim64 = torch.stack([v[:, 0] / p.count[s] for s, v in enumerate(sums)])
        cs64 = torch.stack([v[:, 1] / p.count[s] for s, v in enumerate(sums)])
        ssim, cs = ssim64.float(), cs64.float()
        mean_err, ms_err = M.combine_bound(sums, [v.abs().sum(1) for v in parts], list(p.slots[:S]),
                                           list(p.count[:S]), ssim, cs, list(p.weights[:S]))
        if p.ssim_mean:
            store32(p.ssim_mean, W.Result(ssim64, ssim.double(), torch.stack([e[:, 0] for e in mean_err]), "f32"))
        if p.cs_mean:
            store32(p.cs_mean, W.Result(cs64, cs.double(), torch.stack([e[:, 1] for e in mean_err]), "f32"))
        if p.ms_ssim:
            ms = M.combine(ssim, cs, list(p.weights[:S]))
            store32(p.ms_ssim, W.Result(ms, W.f32(ms), ms_err, "f32"))
        return 0

    def b200_mmd_workspace_bytes(self, shape):
        return 8

    def b200_mmd(self, y, ydt, ys, p, pdt, ps, shape, ws, out, stream):
        shp = [int(v) for v in shape[:5]]
        a = view(y, ydt, [int(v) for v in ys[:5]], shp)
        b = view(p, pdt, [int(v) for v in ps[:5]], shp)
        v = M.mmd(a, b).reshape(1)
        store32(out, W.Result(v, W.f32(v), M.mmd_bound(a, b).reshape(1), "f32"))
        return 0


def install(monkeypatch):
    """cpu_backend.install, with the stand-in that also serves the metric entry points (tests only)."""
    cpu_backend.install(monkeypatch)
    fake = MetricsFakeLib()
    monkeypatch.setattr(_lib, "require_device", lambda: fake)
    return fake

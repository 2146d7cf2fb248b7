"""TEST-ONLY CPU stand-in for the loss entry points of libb200gen.so (include/b200gen_losses.h), on HOST pointers:
tests/perceptual_backend.PerceptualFakeLib extended by b200_spectral_fft, b200_spectral_distance and b200_adversarial,
each viewing its pointers as host tensors and storing what the float64 reading of the contract
(tests/losses_emulator.py) computes, with its bound, through cpu_backend's reporting stores.  install() routes the
product's C-ABI calls to it."""
import ctypes as C

import numpy as np
import torch

from generativemodels_b200 import _lib
from tests import elementwise_emulator as W
from tests import losses_emulator as E
from tests import perceptual_backend
from tests.cpu_backend import _np, _strided, put, store32


def _f64(ptr, count):
    return torch.from_numpy(_np(ptr, count, C.c_double))


def _complex(ptr, count):
    return torch.from_numpy(_np(ptr, 2 * count, C.c_float)).view(torch.complex64)


class LossesFakeLib(perceptual_backend.PerceptualFakeLib):
    def b200_spectral_fft(self, x, xdt, xs, y, ydt, ys, B, ext, sig, spec, stream):
        ext, sig = [ext[i] for i in range(4)], [sig[i] for i in range(4)]
        shape = [B, *ext]
        src = [_strided(p, dt, [st[i] for i in range(5)], shape).float() for p, dt, st in ((x, xdt, xs), (y, ydt, ys))]
        s = E.spectra(src[0], src[1], sig)
        put(_complex(spec, s.exact.numel()).view(s.exact.shape), s)
        return 0

    def b200_spectral_distance(self, spec, B, sig, scale, reduction, out, partials, result, stream):
        sig = [sig[i] for i in range(4)]
        h = sig[3] // 2 + 1
        s = _complex(spec, 2 * B * sig[0] * sig[1] * sig[2] * h).view(2, B, *sig[:3], h)
        scale = float(np.float32(scale))
        if reduction == _lib.REDUCTION_NONE:
            v = E.spectral_distance(s, sig, scale, 0)
            store32(out, W.Result(v, W.f32(v), E.distance_bound(s, sig, scale, 0), "f32"))
            return 0
        total, mean = E.spectral_distance(s, sig, scale, reduction)
        ts, tm = E.distance_bound(s, sig, scale, reduction)
        r = torch.stack([total, mean])
        if result:
            put(_f64(result, 2), W.Result(r, r, torch.stack([ts, tm]), "f64"))
        k = 0 if reduction == _lib.REDUCTION_SUM else 1
        store32(out, W.Result(r[k:k + 1], W.f32(r[k:k + 1]), torch.stack([ts, tm])[k:k + 1], "f32"))
        return 0

    def b200_adversarial(self, x, dtypes, shapes, strides, n_out, criterion, real, reduction, elem, partials, losses,
                         losses32, stream):
        xs = []
        for i in range(n_out):
            sz, st = [shapes[5 * i + d] for d in range(5)], [strides[5 * i + d] for d in range(5)]
            xs.append(_strided(x[i], dtypes[i], st, sz).float())
        per, vals = E.adversarial(xs, criterion, bool(real), reduction)
        errs = [E.adversarial_bound(t, criterion, bool(real)) for t in xs]
        eper = E.adversarial_losses_bound(vals, errs, criterion, reduction)
        put(_f64(losses, n_out + 1), W.Result(per, per, eper, "f64"))
        store32(losses32, W.Result(per, W.f32(per), eper, "f32"))
        if reduction == _lib.REDUCTION_NONE and criterion != _lib.ADV_HINGE:
            for i in range(n_out):
                store32(elem[i], W.Result(vals[i], W.f32(vals[i]), errs[i], "f32"))
        return 0


def install(monkeypatch):
    """perceptual_backend.install with the stand-in that also serves the loss entry points (tests only)."""
    perceptual_backend.install(monkeypatch)
    fake = LossesFakeLib()
    monkeypatch.setattr(_lib, "require_device", lambda: fake)
    import generativemodels_b200.losses.adversarial_loss as AL
    import generativemodels_b200.losses.spectral_loss as SL
    monkeypatch.setattr(AL, "require_cuda", lambda name, *t: None)
    monkeypatch.setattr(SL, "require_cuda", lambda name, *t: None)
    return fake

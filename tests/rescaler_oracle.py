"""Plain restatements for SpatialRescaler (generative/networks/blocks/encoder_modules.py) and b200_interpolate.

``header_interpolate`` evaluates include/b200gen.h's b200_interpolate rules literally (per-axis fp32 coordinates, then
one dense weight matrix per resampled axis, applied in float64; AREA as the header's fp32 sequence, exactly):
tests/test_spatial_rescaler_cpu.py pins it against F.interpolate, which pins the documented rules to ATen's;
tests/cpu_backend.py stands it in for the entry point, so the module's host code runs end to end without a GPU.
``resample_cl`` is the channels-last call ops makes for nearest x2, nearest resizing and the 2x average pool.  ``rescaler`` is the module
itself in plain PyTorch, from a ``state_dict`` and the constructor arguments.  Test infrastructure only."""
from __future__ import annotations

import itertools
import math
import zlib

import numpy as np
import torch
import torch.nn.functional as F

from generativemodels_b200 import _lib

NEAREST, LINEAR, BILINEAR, BICUBIC, TRILINEAR, AREA = (_lib.INTERPOLATE_NEAREST, _lib.INTERPOLATE_LINEAR,
                                                       _lib.INTERPOLATE_BILINEAR, _lib.INTERPOLATE_BICUBIC,
                                                       _lib.INTERPOLATE_TRILINEAR, _lib.INTERPOLATE_AREA)
MODES = {"nearest": NEAREST, "linear": LINEAR, "bilinear": BILINEAR, "bicubic": BICUBIC, "trilinear": TRILINEAR,
         "area": AREA}
_f = np.float32


def _fma(a, b, c):
    """fp32 fused multiply-add: the product of two fp32 values is exact in float64, the sum rounds once."""
    return _f(np.float64(a) * np.float64(b) + np.float64(c))


def _cc1(x):
    return _fma(_fma(_f(1.25), x, _f(-2.25)) * x, x, _f(1))


def _cc2(x):
    return _fma(_fma(_fma(_f(-0.75), x, _f(3.75)), x, _f(-6)), x, _f(3))


def axis_weights(mode: int, n_in: int, n_out: int, ratio: float) -> np.ndarray:
    """[n_out, n_in] float64 weights of one resampled axis, following the header's rules step by step in fp32."""
    w = np.zeros((n_out, n_in))
    r = _f(ratio)
    for o in range(n_out):
        if mode == NEAREST:
            w[o, min(int(np.floor(_f(o) * r)), n_in - 1)] = 1.0
        elif mode == AREA:
            s, e = o * n_in // n_out, -(-(o + 1) * n_in // n_out)
            w[o, s:e] = 1.0 / (e - s)
        elif mode == BICUBIC:
            s = _fma(r, _f(o) + _f(0.5), _f(-0.5))
            f0 = min(int(np.floor(s)), n_in - 1)
            t = min(max(s - _f(f0), _f(0)), _f(1))
            u = _f(1) - t
            for k, c in enumerate((_cc2(t + _f(1)), _cc1(t), _cc1(u), _cc2(u + _f(1)))):
                w[o, min(max(f0 - 1 + k, 0), n_in - 1)] += float(c)
        elif n_in == n_out:
            w[o, o] = 1.0
        else:
            s = max(_fma(r, _f(o) + _f(0.5), _f(-0.5)), _f(0))
            i0 = min(int(np.floor(s)), n_in - 1)
            lam = min(max(s - _f(i0), _f(0)), _f(1))
            w[o, i0] += float(_f(1) - lam)
            w[o, i0 + (1 if i0 < n_in - 1 else 0)] += float(lam)
    return w


def header_interpolate(x: torch.Tensor, out_sizes, ratios, mode: int) -> torch.Tensor:
    """b200_interpolate of a planar [N, C, *spatial] tensor (1 to 3 resampled axes, any input dtype: values are
    converted to fp32 on load), as float32."""
    x = x.float()
    if mode == AREA:
        return _area(x, out_sizes)
    y = x.double()
    dims = x.dim() - 2
    for a in range(dims):
        m = torch.from_numpy(axis_weights(mode, x.shape[2 + a], out_sizes[a], ratios[a]))
        y = torch.movedim(torch.tensordot(y, m, dims=([2 + a], [1])), -1, 2 + a)
    return y.float()


def _area(x: torch.Tensor, out_sizes) -> torch.Tensor:
    """AREA in fp32: each window summed from 0 in d, h, w order (the last axis innermost), then divided by the
    window's extent along each axis in turn."""
    wins = [[(o * n // m, -(-(o + 1) * n // m)) for o in range(m)] for n, m in zip(x.shape[2:], out_sizes)]
    starts = [torch.tensor([s for s, _ in w]) for w in wins]
    ext = [torch.tensor([e - s for s, e in w]) for w in wins]
    shape = lambda a: [-1 if b == a else 1 for b in range(len(wins))]
    acc = torch.zeros(*x.shape[:2], *out_sizes)
    for taps in itertools.product(*(range(int(e.max())) for e in ext)):
        idx = [(s + t).clamp_max(n - 1).view(shape(a)) for a, (s, t, n) in enumerate(zip(starts, taps, x.shape[2:]))]
        ok = math.prod((t < e).view(shape(a)) for a, (t, e) in enumerate(zip(taps, ext)))
        acc = acc + torch.where(ok.bool(), x[(slice(None), slice(None), *idx)], 0.0)
    for a, e in enumerate(ext):
        acc = acc / e.float().view(shape(a))
    return acc


def resample_cl(x: torch.Tensor, dims, mode: int, src=None) -> torch.Tensor:
    """ops' channels-last resampling: [N, D, H, W, pitch] (its first ``src`` voxels per axis) -> [N, *dims, pitch]
    float32, every channel, all three axes resampled with ratios fp32(in / out)."""
    src = tuple(src or x.shape[1:4])
    planar = x[:, :src[0], :src[1], :src[2]].permute(0, 4, 1, 2, 3)
    ratios = [float(np.float32(i) / np.float32(o)) for i, o in zip(src, dims)]
    return header_interpolate(planar, dims, ratios, mode).permute(0, 2, 3, 4, 1)


def rescaler(sd: dict, x: torch.Tensor, n_stages: int = 1, size=None, method: str = "bilinear",
             multiplier=None) -> torch.Tensor:
    """SpatialRescaler.forward: the 1x1 channel mapper (when ``sd`` holds it), then ``n_stages`` interpolations."""
    if "channel_mapper.conv.weight" in sd:
        conv = (None, F.conv1d, F.conv2d, F.conv3d)[x.dim() - 2]
        x = conv(x, sd["channel_mapper.conv.weight"], sd.get("channel_mapper.conv.bias"))
    for _ in range(n_stages):
        x = F.interpolate(x, size=size, scale_factor=multiplier, mode=method)
    return x


def seeded_weights(module, seed=0):
    """Deterministic parameters keyed by name (the reference and this package get the same values): N(0, 1/fan_in)
    for weights, N(0, 0.1^2) for biases."""
    with torch.no_grad():
        for name, p in module.named_parameters():
            g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
            std = 0.1 if p.dim() == 1 else (p[0].numel()) ** -0.5
            p.copy_(torch.randn(p.shape, generator=g) * std)
    return module


def input_of(case: dict) -> torch.Tensor:
    """The case's input: seeded normal values, rounded to fp16 so that every storage flavour reads them exactly."""
    g = torch.Generator().manual_seed(case["seed"])
    return torch.randn(case["shape"], generator=g).half().float()


def ulps_of(x: torch.Tensor, n: float) -> float:
    """n fp32 ulps of max|x|."""
    return n * math.ldexp(1.0, math.frexp(float(x.abs().max()))[1] - 24)

"""Plain restatements for SpatialRescaler (generative/networks/blocks/encoder_modules.py) and b200_interpolate.

``header_interpolate`` is tests/resample_emulator.py's reading of b200_interpolate on a planar tensor:
tests/test_spatial_rescaler_cpu.py pins it against F.interpolate, which pins the documented rules to ATen's.
``resample_cl`` is the channels-last call ops makes for nearest x2, nearest resizing and the 2x average pool.  ``rescaler`` is the module
itself in plain PyTorch, from a ``state_dict`` and the constructor arguments.  Test infrastructure only."""
from __future__ import annotations

import math
import zlib

import numpy as np
import torch
import torch.nn.functional as F

from generativemodels_b200 import _lib
from tests import resample_emulator as RE

NEAREST, LINEAR, BILINEAR, BICUBIC, TRILINEAR, AREA = (_lib.INTERPOLATE_NEAREST, _lib.INTERPOLATE_LINEAR,
                                                       _lib.INTERPOLATE_BILINEAR, _lib.INTERPOLATE_BICUBIC,
                                                       _lib.INTERPOLATE_TRILINEAR, _lib.INTERPOLATE_AREA)
MODES = {"nearest": NEAREST, "linear": LINEAR, "bilinear": BILINEAR, "bicubic": BICUBIC, "trilinear": TRILINEAR,
         "area": AREA}


def axis_weights(mode: int, n_in: int, n_out: int, ratio: float) -> np.ndarray:
    """[n_out, n_in] float64 weights of one resampled axis (AREA excluded): the reading's taps as a dense matrix."""
    idx, w = RE.axis_taps(mode, n_in, n_out, ratio)
    m = np.zeros((n_out, n_in))
    for k in range(idx.shape[1]):
        np.add.at(m, (np.arange(n_out), idx[:, k]), 1.0 if w is None else w[:, k].astype(np.float64))
    return m


def header_interpolate(x: torch.Tensor, out_sizes, ratios, mode: int) -> torch.Tensor:
    """b200_interpolate of a planar [N, C, *spatial] tensor (1 to 3 resampled axes, any input dtype: values are
    converted to fp32 on load), as float32 before the store (tests/resample_emulator.py)."""
    return RE.interpolate_f32(x, tuple(out_sizes), tuple(ratios), mode)


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

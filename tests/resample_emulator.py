"""Reading of the resampling and pooling entry points of include/b200gen.h: b200_interpolate, b200_upsample2x_interp
and b200_pool_s2 (CPU only; test infrastructure).

All three kernels spell out their fp32 sequence, so this module reproduces it bit for bit instead of bounding it:

  interpolate       per resampled axis the fp32 coordinate s = fma(r, dst + 0.5, -0.5), then the taps and weights of
                    the mode (nearest, linear family, Keys cubic); values are separable sums of separately rounded
                    products and sums, W first, then H, then D.  A linear-family axis with out == in is a copy.  AREA
                    sums each window from 0 in d, h, w order and divides by the window's D, H and W extents in turn.
  upsample2x_interp the weights are dyadic (0.25 / 0.75, and Keys weights at t = 0.25 / 0.75 with at most 9
                    significant bits), so the W step's products are exact and its fmas are fp32 adds; the H step is an
                    fma chain over the fp32 rows and needs a correctly rounded fma.
  pool_s2           avg: the in-bounds taps summed in fp32 in d, h, w order, one IEEE division by kernel^dims; max:
                    padding is -inf, a tap replaces the running value when it is larger or NaN.

numpy float32 arithmetic is IEEE single with round-to-nearest-even, so the separately rounded steps are numpy float32
operations; ``fma32`` gives a correctly rounded fp32 fma (the float64 product of two fp32 values is exact, the sum is
made round-to-odd with TwoSum before the one rounding to fp32).  16-bit stores are RN, and fp16 saturates at +-65504
as the kernels' cvt.rn.satfinite does.  Every function returns an elementwise_emulator Result of kind "copy": the
GPU test compares values bit for bit (NaN equal to NaN).
"""
from __future__ import annotations

import itertools
import math

import numpy as np
import torch

from generativemodels_b200 import _lib
from tests.elementwise_emulator import Result, copy
from tests.norm_emulator import F64, h16  # noqa: F401

NEAREST, LINEAR, BILINEAR, BICUBIC, TRILINEAR, AREA = (_lib.INTERPOLATE_NEAREST, _lib.INTERPOLATE_LINEAR,
                                                       _lib.INTERPOLATE_BILINEAR, _lib.INTERPOLATE_BICUBIC,
                                                       _lib.INTERPOLATE_TRILINEAR, _lib.INTERPOLATE_AREA)
LINEAR_FAMILY = (LINEAR, BILINEAR, TRILINEAR)
_f = np.float32


def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c) elementwise (numpy, broadcasting).  a b is exact in float64; the float64
    sum is made round-to-odd (TwoSum gives its error; an inexact sum with an even last bit moves one float64 step
    toward the exact value), and a round-to-odd value with 29 bits to spare rounds to fp32 as the exact sum would."""
    a, b, c = (np.asarray(v, dtype=_f).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    with np.errstate(invalid="ignore"):
        fix = np.isfinite(s) & (err != 0) & ((np.asarray(s).view(np.int64) & 1) == 0)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    with np.errstate(over="ignore"):
        return s.astype(_f)


def _cc1(x):
    return fma32(_f(fma32(_f(1.25), x, _f(-2.25)) * x), x, _f(1))


def _cc2(x):
    return fma32(fma32(fma32(_f(-0.75), x, _f(3.75)), x, _f(-6)), x, _f(3))


def axis_taps(mode: int, n_in: int, n_out: int, ratio: float):
    """Taps [n_out, T] (int64) and fp32 weights [n_out, T] of one resampled axis of b200_interpolate, from the header's
    rules in fp32; weights None for nearest and for a linear-family axis with n_out == n_in (a copy)."""
    o = np.arange(n_out, dtype=np.int64)
    r = _f(ratio)
    if mode == NEAREST:
        return np.minimum(np.floor(o.astype(_f) * r).astype(np.int64), n_in - 1)[:, None], None
    if mode in LINEAR_FAMILY and n_in == n_out:
        return o[:, None], None
    s = fma32(r, o.astype(_f) + _f(0.5), _f(-0.5))
    if mode == BICUBIC:
        f = np.minimum(np.floor(s).astype(np.int64), n_in - 1)
        t = np.clip(s - f.astype(_f), _f(0), _f(1))
        u = _f(1) - t
        w = np.stack([_cc2(t + _f(1)), _cc1(t), _cc1(u), _cc2(u + _f(1))], 1)
        return np.clip(f[:, None] - 1 + np.arange(4), 0, n_in - 1), w
    s = np.maximum(s, _f(0))
    i0 = np.minimum(np.floor(s).astype(np.int64), n_in - 1)
    i1 = i0 + (i0 < n_in - 1)
    lam = np.clip(s - i0.astype(_f), _f(0), _f(1))
    return np.stack([i0, i1], 1), np.stack([_f(1) - lam, lam], 1)


def _axis_step(x: np.ndarray, axis: int, idx, w) -> np.ndarray:
    """One 1-D step along `axis`: sum_k x[idx_k] w_k with products and sums rounded separately (a copy: x[idx])."""
    take = lambda k: np.take(x, idx[:, k], axis=axis)
    if w is None:
        return take(0)
    shape = [1] * x.ndim
    shape[axis] = -1
    acc = take(0) * w[:, 0].reshape(shape)
    for k in range(1, idx.shape[1]):
        acc = acc + take(k) * w[:, k].reshape(shape)
    return acc


def area_windows(n_in: int, n_out: int):
    """[floor(o in / out), ceil((o + 1) in / out)) for every o, in integer arithmetic."""
    return [(o * n_in // n_out, -(-(o + 1) * n_in // n_out)) for o in range(n_out)]


def _area(x: np.ndarray, out_sizes) -> np.ndarray:
    """AREA on the last len(out_sizes) axes of x (fp32): each window summed from 0 with the last axis innermost, then
    divided by the window's extent along each axis in turn."""
    dims = len(out_sizes)
    wins = [area_windows(n, m) for n, m in zip(x.shape[-dims:], out_sizes)]
    starts = [np.array([s for s, _ in w]) for w in wins]
    ext = [np.array([e - s for s, e in w]) for w in wins]
    shape = lambda a: [-1 if b == a else 1 for b in range(dims)]
    acc = np.zeros((*x.shape[:-dims], *out_sizes), dtype=_f)
    lead = (slice(None),) * (x.ndim - dims)
    for taps in itertools.product(*(range(int(e.max())) for e in ext)):
        idx = [np.minimum(s + t, n - 1) for s, t, n in zip(starts, taps, x.shape[-dims:])]
        ok = np.ones([1] * dims, dtype=bool)
        for a, (t, e) in enumerate(zip(taps, ext)):
            ok = ok & (t < e).reshape(shape(a))
        acc = np.where(ok, acc + x[(*lead, *np.ix_(*idx))], acc)
    for a, e in enumerate(ext):
        acc = acc / e.astype(_f).reshape([1] * (x.ndim - dims) + shape(a))
    return acc


def interpolate_f32(x: torch.Tensor, out_sizes, ratios, mode: int) -> torch.Tensor:
    """b200_interpolate of [..., *spatial] (the last len(out_sizes) axes resampled; any dtype, converted to fp32 on
    load as the kernel does) before the store, as float32."""
    xf = x.float().numpy() if x.dtype != torch.float32 else x.numpy()
    dims = len(out_sizes)
    if mode == AREA:
        return torch.from_numpy(_area(xf, out_sizes))
    y = xf
    for a in reversed(range(dims)):                      # W, then H, then D
        axis = xf.ndim - dims + a
        idx, w = axis_taps(mode, xf.shape[axis], out_sizes[a], ratios[a])
        y = _axis_step(y, axis, idx, w)
    return torch.from_numpy(np.ascontiguousarray(y, dtype=_f))


def store(v: torch.Tensor, y_h16: bool) -> torch.Tensor:
    """The stored value as float64: h16 RN (fp16 saturating) or the fp32 value itself."""
    return h16(v.to(F64)) if y_h16 else v.to(F64)


def vector_path(C: int, x_dtype: int, xs, ys, x_addr: int, y_addr: int) -> bool:
    """Whether b200_interpolate takes its 8-channel path: an h16 or fp32 input, channel stride 1 on both sides, every
    other stride a multiple of 8, 16-byte aligned pointers and voxel strides >= round_up(C, 8).  That path reads and
    writes channels [0, round_up(C, 8)); the other one channels [0, C)."""
    c8 = (C + 7) // 8 * 8
    return (x_dtype in (_lib.DT_H16, _lib.DT_F32) and xs[1] == 1 and ys[1] == 1 and x_addr % 16 == 0 and
            y_addr % 16 == 0 and xs[4] >= c8 and ys[4] >= c8 and all(xs[i] % 8 == 0 and ys[i] % 8 == 0 for i in (0, 2, 3, 4)))


def interpolate(x: torch.Tensor, out_sizes, ratios, mode: int, y_h16: bool) -> Result:
    """b200_interpolate of a (strided) host view [N, C, D, H, W] of the input: Result [N, C, OD, OH, OW] as stored."""
    return copy(store(interpolate_f32(x, tuple(out_sizes), ratios, mode), y_h16))


# ----------------------------------------------------------------------------------------------------------------
# fixed x2 upsampling of SPADENet (channels-last h16)
# ----------------------------------------------------------------------------------------------------------------
def up2_taps(mode: int, n: int):
    """Taps [2n, T] and weights [2n, T] (exact dyadic values, as float32) of b200_upsample2x_interp along one axis."""
    o = np.arange(2 * n)
    i, odd = o >> 1, (o & 1) == 1
    if mode == _lib.INTERP_BILINEAR:
        idx = np.where(odd[:, None], np.stack([i, np.minimum(i + 1, n - 1)], 1),
                       np.stack([np.maximum(i - 1, 0), np.where(i == 0, min(1, n - 1), i)], 1))
        w = np.where(odd[:, None], [0.75, 0.25], np.where((i == 0)[:, None], [1.0, 0.0], [0.25, 0.75]))
        return idx, w.astype(_f)
    f = np.where(odd, i, i - 1)
    t = np.where(odd, 0.25, 0.75)
    A = -0.75
    cc1 = lambda v: ((A + 2) * v - (A + 3)) * v * v + 1
    cc2 = lambda v: ((A * v - 5 * A) * v + 8 * A) * v - 4 * A
    w = np.stack([cc2(t + 1), cc1(t), cc1(1 - t), cc2(2 - t)], 1)
    assert (w.astype(_f) == w).all()
    return np.clip(f[:, None] - 1 + np.arange(4), 0, n - 1), w.astype(_f)


def upsample2x_interp(x: torch.Tensor, N: int, H: int, W: int, pitch: int, mode: int) -> Result:
    """[N][H][W][pitch] h16 -> [N][2H][2W][pitch] as stored: along W within each source row (fp32 adds of exact
    products from 0), then an fma chain along H over those rows from 0; every channel, pad channels included."""
    X = x[:N * H * W * pitch].float().numpy().reshape(N, H, W, pitch)
    hi, hw = up2_taps(mode, H)
    wi, ww = up2_taps(mode, W)
    rows = np.zeros((N, H, 2 * W, pitch), dtype=_f)
    for b in range(wi.shape[1]):
        rows = rows + X[:, :, wi[:, b], :] * ww[:, b][None, None, :, None]
    out = np.zeros((N, 2 * H, 2 * W, pitch), dtype=_f)
    for a in range(hi.shape[1]):
        out = fma32(rows[:, hi[:, a]], hw[:, a][None, :, None, None], out)
    return copy(store(torch.from_numpy(out), True))


# ----------------------------------------------------------------------------------------------------------------
# stride-2 pooling of the PatchGAN pyramid (channels-last h16)
# ----------------------------------------------------------------------------------------------------------------
def pool_extent(n: int, k: int, pad: int) -> int:
    return (n + 2 * pad - k) // 2 + 1


def pool_s2(x: torch.Tensor, N: int, D: int, H: int, W: int, pitch: int, dims: int, k: int, pad: int,
            mode: int) -> Result:
    """[N][D][H][W][pitch] h16 -> [N][OD][OH][OW][pitch] as stored (dims == 2 pools H and W of every D slice)."""
    X = x[:N * D * H * W * pitch].float().reshape(N, D, H, W, pitch)
    kd, pd = (k, pad) if dims == 3 else (1, 0)
    OD = pool_extent(D, kd, pd) if dims == 3 else D
    OH, OW = pool_extent(H, k, pad), pool_extent(W, k, pad)
    od, oh, ow = (torch.arange(n) * (2 if s else 1) for n, s in ((OD, dims == 3), (OH, True), (OW, True)))
    mx = mode == _lib.POOL_MAX
    acc = torch.full((N, OD, OH, OW, pitch), -math.inf if mx else 0.0, dtype=torch.float32)
    for a, b, c in itertools.product(range(kd), range(k), range(k)):
        i_d, i_h, i_w = od + a - pd, oh + b - pad, ow + c - pad
        ok = ((i_d >= 0) & (i_d < D))[:, None, None] & ((i_h >= 0) & (i_h < H))[None, :, None] & \
            ((i_w >= 0) & (i_w < W))[None, None, :]
        v = X[:, i_d.clamp(0, D - 1)][:, :, i_h.clamp(0, H - 1)][:, :, :, i_w.clamp(0, W - 1)]
        ok = ok[None, :, :, :, None]
        if mx:
            acc = torch.where(ok & ((v > acc) | torch.isnan(v)), v, acc)
        else:
            acc = torch.where(ok, acc + v, acc)
    if not mx:
        acc = acc / float(kd * k * k)
    return copy(store(acc, True))

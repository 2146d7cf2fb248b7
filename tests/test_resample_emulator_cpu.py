"""tests/resample_emulator.py against plain float64 PyTorch, and its bit-exact comparison rejecting kernel-shaped
mutants (CPU only).

The reading reproduces fp32 sequences, so a mutant is rejected when it stores a different value anywhere; each test
reports by how much, in 16-bit (or fp32) ulps of the value it should have stored.  The float64 comparisons pin the
reading to F.interpolate, F.avg_pool*, F.max_pool* and F.linear within the fp32 rounding of the kernel's arithmetic.
"""
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from generativemodels_b200 import _lib
from tests import elementwise_emulator as E
from tests import resample_emulator as R
from tests.norm_emulator import storage

F64 = torch.float64
FLAVOURS = [torch.float16, torch.bfloat16]


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def ulps(ref, got, ulp):
    """Largest |got - ref| in ulps of ref (NaN against a number, or the reverse, is inf)."""
    d = (got - ref).abs() / ulp(ref)
    nan_mismatch = torch.isnan(got) != torch.isnan(ref)
    d = torch.where(torch.isnan(got) & torch.isnan(ref), torch.zeros_like(d), d)
    return math.inf if bool(nan_mismatch.any()) else float(d.nan_to_num(math.inf).max())


def rejected(name, want, got, ulp=E.ulp16):
    factor = ulps(want.out, got, ulp)
    print(f"\nMUTANT {name} rejected: {factor:.3g} ulps off")
    assert factor > 0, f"mutant {name} stores the same values"


def r32(i, o):
    return float(np.float32(i) / np.float32(o))


# ------------------------------------------------------------------------------------------------------------------
# fma32
# ------------------------------------------------------------------------------------------------------------------
def test_fma32_is_correctly_rounded():
    """Against exact rational arithmetic, including sums whose float64 rounding lands on an fp32 midpoint (where a
    plain float64 sum rounds twice)."""
    from fractions import Fraction
    rng = np.random.default_rng(0)
    a = rng.standard_normal(4000).astype(np.float32)
    b = rng.standard_normal(4000).astype(np.float32)
    c = (rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 30, 4000)).astype(np.float32)
    # midpoint cases: c = 2^e (1 + 2^-23) has an odd last bit, a b = 2^(e-24) (1 - 2^-46) puts the exact sum just
    # below the midpoint above c; the float64 sum rounds onto that midpoint and then to the even neighbour
    e = np.arange(-20, 30, dtype=np.float64)
    a = np.concatenate([a, (2.0 ** (e - 24) * (1 + 2.0 ** -23)).astype(np.float32)])
    b = np.concatenate([b, np.full(e.size, 1 - 2.0 ** -23, np.float32)])
    c = np.concatenate([c, (2.0 ** e * (1 + 2.0 ** -23)).astype(np.float32)])
    got = R.fma32(a, b, c)
    for x, y, z, g in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        lo = np.float32(float(exact))
        cands = [lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.asarray(v).view(np.int32)) & 1))
        assert g == best, (x, y, z, g, best)
    twice = (a.astype(np.float64) * b + c).astype(np.float32)
    assert (twice != got).any(), "the midpoint cases must separate one rounding from two"


# ------------------------------------------------------------------------------------------------------------------
# interpolate against float64 F.interpolate
# ------------------------------------------------------------------------------------------------------------------
TORCH_MODE = {R.NEAREST: "nearest", R.LINEAR: "linear", R.BILINEAR: "bilinear", R.BICUBIC: "bicubic",
              R.TRILINEAR: "trilinear", R.AREA: "area"}
CASES = [(m, d) for m, dd in ((R.NEAREST, (1, 2, 3)), (R.LINEAR, (1,)), (R.BILINEAR, (2,)), (R.BICUBIC, (2,)),
                              (R.TRILINEAR, (3,)), (R.AREA, (1, 2, 3))) for d in dd]


@pytest.mark.parametrize("mode,dims", CASES, ids=[f"{TORCH_MODE[m]}_{d}d" for m, d in CASES])
@pytest.mark.parametrize("spec", ["size_odd", "scale_half", "scale_2", "scale_1.5"])
def test_interpolate_reading_against_float64_torch(mode, dims, spec):
    g = gen(f"{mode}{dims}{spec}")
    shape = (2, 3, *(9, 7, 11)[3 - dims:])
    x = torch.randn(*shape, generator=g).float()
    ins = shape[2:]
    if spec == "size_odd":
        outs = tuple((5, 12, 4)[3 - dims:])
        kw = dict(size=outs)
        ratios = [r32(i, o) for i, o in zip(ins, outs)]
    else:
        f = {"scale_half": 0.5, "scale_2": 2.0, "scale_1.5": 1.5}[spec]
        outs = tuple(int(math.floor(i * f)) for i in ins)
        kw = dict(scale_factor=f)
        ratios = [float(np.float32(1.0 / f))] * dims
    if mode == R.AREA:
        want = F.adaptive_avg_pool3d(x.double().reshape(shape[0], shape[1], *(1,) * (3 - dims), *ins),
                                     (1,) * (3 - dims) + outs).reshape(shape[0], shape[1], *outs)
    else:
        want = F.interpolate(x.double(), mode=TORCH_MODE[mode], **kw)
    got = R.interpolate_f32(x, outs, ratios, mode).double()
    tol = 2.0 ** -18 * float(x.abs().max()) * (1 if mode in (R.NEAREST, R.AREA) else 8)
    if mode == R.NEAREST and spec in ("size_odd", "scale_1.5"):
        # for float64 inputs ATen forms the scale in double: compare with the float32 call, which uses fp32 scales
        want = F.interpolate(x, mode="nearest", **kw).double()
        tol = 0.0
    assert (got - want).abs().max() <= tol, float((got - want).abs().max())


def test_interpolate_reading_copies_identity_axes():
    x = torch.randn(1, 2, 4, 5)
    x[0, 0, 1, 2], x[0, 1, 3, 0], x[0, 0, 0, 4] = math.inf, -math.inf, math.nan
    for mode in (R.BILINEAR, R.NEAREST):
        y = R.interpolate_f32(x, (4, 5), (1.0, 1.0), mode)
        assert torch.equal(torch.nan_to_num(y, 7.0), torch.nan_to_num(x, 7.0)) and torch.isnan(y).sum() == 1
    y = R.interpolate_f32(x, (4, 9), (1.0, r32(5, 9)), R.BILINEAR)
    assert torch.isfinite(y[0, 0, 2]).all() and not torch.isfinite(y[0, 0, 1]).all()


# ------------------------------------------------------------------------------------------------------------------
# upsample2x_interp and pool_s2 against float64 torch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", FLAVOURS, ids=["fp16", "bf16"])
@pytest.mark.parametrize("mode", [_lib.INTERP_BILINEAR, _lib.INTERP_BICUBIC], ids=["bilinear", "bicubic"])
@pytest.mark.parametrize("HW", [(1, 1), (2, 3), (7, 5), (16, 16)])
def test_upsample2x_reading_against_float64_torch(flavour, mode, HW):
    H, W = HW
    with storage(flavour):
        x = torch.randn(2, H, W, 8, generator=gen(f"up{mode}{HW}")).to(flavour)
        got = R.upsample2x_interp(x.reshape(-1), 2, H, W, 8, mode).out
        ref = F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=2,
                            mode="bilinear" if mode == _lib.INTERP_BILINEAR else "bicubic").permute(0, 2, 3, 1)
        tol = E.ulp16(torch.maximum(ref.abs(), got.abs())) + 2.0 ** -21 * float(x.double().abs().max())
        assert ((got - ref).abs() <= tol).all()


POOL = [(k, p, d) for k in range(1, 6) for p in range(k // 2 + 1) for d in (2, 3)]


@pytest.mark.parametrize("flavour", FLAVOURS, ids=["fp16", "bf16"])
@pytest.mark.parametrize("k,pad,dims", POOL, ids=[f"k{k}p{p}_{d}d" for k, p, d in POOL])
def test_pool_s2_reading_against_float64_torch(flavour, k, pad, dims):
    N, D, H, W, P = 2, 5, 7, 6, 8
    with storage(flavour):
        x = torch.randn(N, D, H, W, P, generator=gen(f"pool{k}{pad}{dims}")).to(flavour)
        X = x.double().permute(0, 4, 1, 2, 3)
        kk, pp, ss = ((k,) * 3, (pad,) * 3, 2) if dims == 3 else ((1, k, k), (0, pad, pad), (1, 2, 2))
        for mode, ref in ((_lib.POOL_AVG, F.avg_pool3d(X, kk, ss, pp, count_include_pad=True)),
                          (_lib.POOL_MAX, F.max_pool3d(X, kk, ss, pp))):
            got = R.pool_s2(x.reshape(-1), N, D, H, W, P, dims, k, pad, mode).out
            ref = E.h16(ref.permute(0, 2, 3, 4, 1))
            tol = 0 if mode == _lib.POOL_MAX else E.ulp16(ref)
            assert ((got - ref).abs() <= tol).all()


def test_pool_max_reading_propagates_nan():
    x = torch.zeros(1, 1, 4, 4, 8)
    x[0, 0, 1, 1, 0] = math.nan
    y = R.pool_s2(x.reshape(-1), 1, 1, 4, 4, 8, 2, 2, 0, _lib.POOL_MAX).out
    assert torch.isnan(y[0, 0, 0, 0, 0]) and torch.isnan(y).sum() == 1


# ------------------------------------------------------------------------------------------------------------------
# mutants of the resampling kernels
# ------------------------------------------------------------------------------------------------------------------
def _interp_case(mode, shape=(1, 2, 1, 9, 13), out=(1, 6, 20)):
    x = torch.randn(*shape, generator=gen(f"mut{mode}{shape}")).float()
    dims = 2
    ratios = [r32(i, o) for i, o in zip(shape[2:], out)][3 - dims:]
    return x, out[3 - dims:], ratios


def _mutant_interp(monkeypatch, mode, patch, shape=(1, 2, 1, 9, 13), out=(1, 6, 20)):
    x, outs, ratios = _interp_case(mode, shape, out)
    want = R.interpolate(x, outs, ratios, mode, False)
    with monkeypatch.context() as m:
        patch(m)
        got = R.interpolate(x, outs, ratios, mode, False).out
    return want, got


def _wrap_taps(transform):
    real = R.axis_taps

    def taps(mode, n_in, n_out, ratio):
        return transform(mode, n_in, n_out, ratio, *real(mode, n_in, n_out, ratio))
    return taps


def test_mutant_coordinate_rounded_twice(monkeypatch):
    twice = lambda a, b, c: (np.asarray(a, np.float32) * np.asarray(b, np.float32) + np.asarray(c, np.float32))
    want, got = _mutant_interp(monkeypatch, R.BILINEAR, lambda m: m.setattr(R, "fma32", twice),
                               shape=(1, 2, 1, 17, 23), out=(1, 10, 31))
    rejected("coordinate rounded twice", want, got, E.ulp32)


def test_mutant_nearest_rounds_instead_of_flooring(monkeypatch):
    def rint(mode, n_in, n_out, ratio, idx, w):
        if mode != R.NEAREST:
            return idx, w
        o = np.arange(n_out, dtype=np.float32)
        return np.minimum(np.rint(o * np.float32(ratio)).astype(np.int64), n_in - 1)[:, None], None
    want, got = _mutant_interp(monkeypatch, R.NEAREST, lambda m: m.setattr(R, "axis_taps", _wrap_taps(rint)))
    rejected("nearest round instead of floor", want, got, E.ulp32)


def test_mutant_linear_i1_not_clamped(monkeypatch):
    def unclamped(mode, n_in, n_out, ratio, idx, w):
        if w is None:
            return idx, w
        idx = idx.copy()
        idx[:, 1] = (idx[:, 0] + 1) % n_in          # past the last sample: the next row's first
        return idx, w
    want, got = _mutant_interp(monkeypatch, R.BILINEAR, lambda m: m.setattr(R, "axis_taps", _wrap_taps(unclamped)),
                               out=(1, 18, 26))
    rejected("linear i1 not clamped", want, got, E.ulp32)


def test_mutant_cubic_taps_not_clamped(monkeypatch):
    def unclamped(mode, n_in, n_out, ratio, idx, w):
        o = np.arange(n_out, dtype=np.float32)
        s = R.fma32(np.float32(ratio), o + np.float32(0.5), np.float32(-0.5))
        f = np.minimum(np.floor(s).astype(np.int64), n_in - 1)
        return (f[:, None] - 1 + np.arange(4)) % n_in, w
    want, got = _mutant_interp(monkeypatch, R.BICUBIC, lambda m: m.setattr(R, "axis_taps", _wrap_taps(unclamped)))
    rejected("cubic taps not clamped", want, got, E.ulp32)


def test_mutant_area_end_floored(monkeypatch):
    floored = lambda n_in, n_out: [(o * n_in // n_out, max((o + 1) * n_in // n_out, o * n_in // n_out + 1))
                                   for o in range(n_out)]
    want, got = _mutant_interp(monkeypatch, R.AREA, lambda m: m.setattr(R, "area_windows", floored))
    rejected("AREA end index floored", want, got, E.ulp32)


def test_mutant_area_divided_once_by_the_product():
    x, outs, _ = _interp_case(R.AREA, shape=(1, 64, 1, 9, 13), out=(1, 3, 3))
    want = R.interpolate(x, outs, [1.0, 1.0], R.AREA, False)
    X = x.numpy()[:, :, 0]
    wh, ww = R.area_windows(9, 3), R.area_windows(13, 3)
    got = np.zeros((1, 64, 3, 3), np.float32)
    for i, (h0, h1) in enumerate(wh):
        for j, (w0, w1) in enumerate(ww):
            acc = np.zeros((1, 64), np.float32)
            for h in range(h0, h1):
                for w in range(w0, w1):
                    acc = acc + X[:, :, h, w]
            got[:, :, i, j] = acc / np.float32((h1 - h0) * (w1 - w0))
    rejected("AREA divided once by the product", want, torch.from_numpy(got).double()[:, :, None], E.ulp32)


@pytest.mark.parametrize("flavour", FLAVOURS, ids=["fp16", "bf16"])
def test_mutant_pool_divisor_counts_in_bounds_taps(flavour):
    with storage(flavour):
        x = torch.randn(1, 1, 7, 6, 8, generator=gen("poolmut")).to(flavour)
        want = R.pool_s2(x.reshape(-1), 1, 1, 7, 6, 8, 2, 3, 1, _lib.POOL_AVG)
        got = F.avg_pool3d(x.double().permute(0, 4, 1, 2, 3), (1, 3, 3), (1, 2, 2), (0, 1, 1), count_include_pad=False)
        rejected("pool divisor counting in-bounds taps", want, E.h16(got.permute(0, 2, 3, 4, 1)))


def test_mutant_max_ignoring_nan():
    x = torch.randn(1, 1, 6, 6, 8, generator=gen("maxnan"))
    x[0, 0, 2, 3, 1] = math.nan
    want = R.pool_s2(x.reshape(-1), 1, 1, 6, 6, 8, 2, 3, 1, _lib.POOL_MAX)
    got = F.max_pool3d(torch.nan_to_num(x, nan=-math.inf).permute(0, 4, 1, 2, 3), (1, 3, 3), (1, 2, 2), (0, 1, 1))
    rejected("max ignoring NaN", want, E.h16(got.permute(0, 2, 3, 4, 1).double()))


@pytest.mark.parametrize("mode", [_lib.INTERP_BILINEAR, _lib.INTERP_BICUBIC], ids=["bilinear", "bicubic"])
def test_mutant_upsample_parities_swapped(monkeypatch, mode):
    x = torch.randn(1, 5, 6, 8, generator=gen("par")).half()
    want = R.upsample2x_interp(x.reshape(-1), 1, 5, 6, 8, mode)
    real = R.up2_taps

    def swapped(m, n):
        idx, w = real(m, n)
        flip = lambda a: a.reshape(n, 2, -1)[:, ::-1].reshape(2 * n, -1)
        return flip(idx), flip(w)
    monkeypatch.setattr(R, "up2_taps", swapped)
    rejected("upsample parities swapped", want, R.upsample2x_interp(x.reshape(-1), 1, 5, 6, 8, mode).out)


def test_mutant_bicubic_a_minus_half(monkeypatch):
    f = np.float32
    cc1 = lambda v: R.fma32(f(R.fma32(f(1.5), v, f(-2.5)) * v), v, f(1))
    cc2 = lambda v: R.fma32(R.fma32(R.fma32(f(-0.5), v, f(2.5)), v, f(-4)), v, f(2))
    want, got = _mutant_interp(monkeypatch, R.BICUBIC, lambda m: (m.setattr(R, "_cc1", cc1), m.setattr(R, "_cc2", cc2)))
    rejected("bicubic A = -0.5", want, got, E.ulp32)

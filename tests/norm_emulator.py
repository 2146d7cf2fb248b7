"""Float64 reading of the normalisation entry points of include/b200gen.h (CPU only; test infrastructure).

One function per entry point.  Each takes flat host tensors laid out as the C ABI describes them (up to two channels-
last sources with their own channel pitches, N samples of `spatial` voxels, an output pitch with pad channels) and
returns a Result: the float64 value before the final 16-bit rounding (`exact`), the rounded value (`out`) and the
accuracy term of the bound (`err`), one per element of the output rows [N * spatial, y_pitch].  Each function mirrors
the arithmetic its kernel documents:

  statistics      the biased mean and variance of the group (GroupNorm) or row (LayerNorm) of the 16-bit inputs,
                  rstd = 1 / sqrt(var + eps).  The header states their accuracy (see STAT_GN below).
  affine pair     a = fp32(fp32(rstd) gamma), b = fp32(beta - fp32(mean) a), per (sample, channel): the table
                  b200_groupnorm_stats and _from_partials write, and what apply / fused use.
  GroupNorm out   h16(act(fma(x, a, b))); SiLU as x / (1 + e^-x) within the error of __expf / __fdividef.
  SPADE out       h16(act(fma(nx, 1 + gg, tt))), nx = fma(x, ax, bx), gg = fma(g, ag, bg), tt = fma(t, at, bt).
  LayerNorm out   h16((x - mean) rstd gamma + beta); the rows_linear prologue stages the same h16 row.
  pads            output channels [C, y_pitch) are +0.

16-bit rounding goes through fp32 (the kernels round their fp32 values with RN); fp16 stores saturate at +-65504.

Value bound, per output element (tolerance()):

    |got - want| <= ulp16(max(|got|, |want|)) + err

err of a normalised value t = x a + b (before the activation) is

    |x - mean| |gamma| d_rstd + |a| d_mean + 2^-22 (|x a| + |b|)

the statistics term from the header's accuracy of mean and rstd (d_mean, d_rstd) and the fp32 term covering the
rounding of a, b, fp32(mean) and the fma.  The activation carries it through its slope (at most 1.1) and adds its
own error.  A constant offset k std on a group makes |x a| and |b| about k |gamma|, so the fp32 term grows with k
while the statistics term stays at the spread's scale: a kernel that forms E[x^2] - mean^2 from fp32 sums loses
about k^2 2^-24 of rstd and falls outside the bound from k ~ 100 (tests/test_norm_emulator_cpu.py shows the mutants
it rejects).
"""
from __future__ import annotations

import contextlib
import math
from dataclasses import dataclass

import torch

from generativemodels_b200._lib import ACT_DTYPE

F64 = torch.float64
H16 = torch.float16 if ACT_DTYPE == "fp16" else torch.bfloat16

# the header's accuracy of the statistics (see b200_groupnorm_stats, b200_layernorm): with p the group's pivot (its
# first channel at voxel 0) and s = sqrt(var + eps),
#   GroupNorm (stats, fused)  |d mean| <= STAT_GN (s + |mean - p|),  |d rstd| <= STAT_GN rstd (1 + (mean - p)^2 / s^2)
#   LayerNorm (both kernels, rows_linear)  with u = 2^-24 (C / 32 + 8), the fp32 error of a lane's chain and the
#                             warp tree:  |d mean| <= u (|mean| + s),  |d rstd| <= rstd (u + 2^-21 + (d mean / s)^2)
#   from_partials             exact to its fp32 partials up to fp64 rounding
STAT_GN = 2.0 ** -12
STAT_PARTIALS = 2.0 ** -40
FP32 = 2.0 ** -22

ACT_NONE, ACT_RELU, ACT_SILU, ACT_LEAKYRELU, ACT_GELU, ACT_LEAKYRELU02 = 0, 1, 2, 3, 4, 8
SLOPE = {ACT_LEAKYRELU: 0.01, ACT_LEAKYRELU02: 0.2}


@contextlib.contextmanager
def storage(dtype):
    """Emulate the library flavour whose 16-bit type is `dtype` (torch.float16 or torch.bfloat16) inside the block."""
    global H16
    old, H16 = H16, dtype
    try:
        yield
    finally:
        H16 = old


def f32(x):
    return x.to(torch.float32).to(F64)


def h16(x):
    """fp32 -> 16-bit with round-to-nearest-even, as the kernels store; fp16 saturates at +-65504."""
    x = x.to(torch.float32)
    if H16 is torch.float16:
        x = x.clamp(-65504.0, 65504.0)
    return x.to(H16).to(F64)


def ulp16(x):
    emin, mant = (-14, 10) if H16 is torch.float16 else (-126, 7)
    m = x.abs().clamp_min(2.0 ** emin)
    return torch.exp2(torch.floor(torch.log2(m)) - mant)


@dataclass
class Result:
    exact: torch.Tensor       # float64 before the final 16-bit rounding
    out: torch.Tensor         # the rounded result, as float64
    err: torch.Tensor         # accuracy term of the bound (see the module docstring)


@dataclass
class Affine:
    """The [N, C] affine table (a, b) with its accuracy, and the statistics behind it ([N, groups])."""
    a: torch.Tensor
    b: torch.Tensor
    a_err: torch.Tensor
    b_err: torch.Tensor
    mean: torch.Tensor
    rstd: torch.Tensor
    d_mean: torch.Tensor
    d_rstd: torch.Tensor
    gamma: torch.Tensor       # [1, C]


def tolerance(r: Result, got: torch.Tensor) -> torch.Tensor:
    return ulp16(torch.maximum(got.abs(), r.out.abs())) + r.err


def excess(r: Result, got: torch.Tensor) -> torch.Tensor:
    """|got - out| / tolerance per element (> 1 is outside the bound; a NaN or inf the emulator does not have is inf)."""
    got = got.to(F64)
    ratio = (got - r.out).abs() / tolerance(r, got)
    bad = ~torch.isfinite(got) & torch.isfinite(r.out)
    return torch.where(bad, torch.full_like(ratio, math.inf), ratio.nan_to_num(0.0))


def affine_excess(t: Affine, got: torch.Tensor) -> torch.Tensor:
    """got: [N, C, 2] fp32 as the kernels write it; the larger of the two per-entry ratios."""
    got = got.to(F64)
    ra = (got[..., 0] - t.a).abs() / t.a_err
    rb = (got[..., 1] - t.b).abs() / t.b_err
    r = torch.maximum(ra, rb)
    return torch.where(torch.isfinite(got).all(-1), r, torch.full_like(r, math.inf))


# ----------------------------------------------------------------------------------------------------------------
# layout
# ----------------------------------------------------------------------------------------------------------------
def rows_of(buf, n, pitch, c=None):
    """The first n rows of a flat buffer of `pitch`-element rows, columns [0, c), as float64."""
    v = buf[:n * pitch].view(n, pitch)
    return (v if c is None else v[:, :c]).to(F64)


def concat(x0, x1, C0, C1, pitch0, pitch1, N, spatial):
    """The virtual concat of the two sources: [N, spatial, C0 + C1] float64."""
    parts = [rows_of(x0, N * spatial, pitch0, C0)]
    if C1:
        parts.append(rows_of(x1, N * spatial, pitch1, C1))
    return torch.cat(parts, 1).view(N, spatial, C0 + C1)


# ----------------------------------------------------------------------------------------------------------------
# statistics and the affine table
# ----------------------------------------------------------------------------------------------------------------
def group_moments(X, groups):
    """X [N, spatial, C] -> mean, var, pivot [N, groups] (biased variance, pivot = the group's first element)."""
    N, S, C = X.shape
    Xg = X.view(N, S, groups, C // groups)
    mean = Xg.mean((1, 3))
    var = ((Xg - mean[:, None, :, None]) ** 2).mean((1, 3))
    return mean, var, Xg[:, 0, :, 0]


def affine_table(mean, rstd, d_mean, d_rstd, gamma, beta, groups):
    """a = fp32(fp32(rstd) gamma), b = fp32(beta - fp32(mean) a) per channel, with the accuracy of each."""
    cpg = gamma.numel() // groups
    g, bt = gamma.to(F64)[None], beta.to(F64)[None]
    ex = lambda t: t.repeat_interleave(cpg, 1)
    m, r, dm, dr = ex(mean), ex(rstd), ex(d_mean), ex(d_rstd)
    a = f32(f32(r) * g)
    b = f32(bt - f32(m) * a)
    a_err = g.abs() * dr + 2.0 ** -23 * a.abs() + 1e-300
    b_err = m.abs() * a_err + a.abs() * dm + 2.0 ** -23 * (b.abs() + (m * a).abs()) + 1e-300
    return Affine(a, b, a_err, b_err, mean, rstd, d_mean, d_rstd, g)


def gn_affine(X, groups, eps, gamma, beta, stat=STAT_GN):
    """The affine table b200_groupnorm_stats / _fused compute from the inputs X [N, spatial, C]."""
    return stats_affine(*group_moments(X, groups), eps, gamma, beta, groups, stat)


def stats_affine(mean, var, piv, eps, gamma, beta, groups, stat=STAT_GN):
    """gn_affine from the float64 moments and pivots [N, groups] of the inputs."""
    s2 = var + eps
    rstd = 1.0 / torch.sqrt(s2)
    off = (mean - piv).abs()
    d_mean = stat * (torch.sqrt(s2) + off)
    d_rstd = stat * rstd * (1.0 + off ** 2 / s2)
    return affine_table(mean, rstd, d_mean, d_rstd, gamma, beta, groups)


def gn_stats(x0, x1, C0, C1, pitch0, pitch1, N, spatial, groups, eps, gamma, beta):
    """b200_groupnorm_stats: the [N, C] affine table."""
    return gn_affine(concat(x0, x1, C0, C1, pitch0, pitch1, N, spatial), groups, eps, gamma, beta)


def gn_from_partials(parts, slots, widths, C0, C1, N, spatial, groups, eps, gamma, beta):
    """b200_groupnorm_from_partials_ex: parts[i] = fp32 [N][slots[i]][C_i / widths[i]][2] of (sum, sum of squares)
    per producer group; each consumer group adds the slots of the producer groups it spans in fp64."""
    C = C0 + C1
    cpg = C // groups
    S = torch.zeros(N, groups, dtype=F64)
    Q = torch.zeros_like(S)
    for g in range(groups):
        c = g * cpg
        i, cc = (0, c) if c < C0 else (1, c - C0)
        w, Ci = widths[i], (C0, C1)[i]
        P = parts[i][:N * slots[i] * (Ci // w) * 2].view(N, slots[i], Ci // w, 2).to(F64)
        sel = P[:, :, cc // w:(cc + cpg) // w]
        S[:, g], Q[:, g] = sel[..., 0].sum((1, 2)), sel[..., 1].sum((1, 2))
    cnt = float(spatial * cpg)
    mean = S / cnt
    var = (Q / cnt - mean ** 2).clamp_min(0.0)
    s2 = var + eps
    rstd = 1.0 / torch.sqrt(s2)
    d_mean = STAT_PARTIALS * (mean.abs() + torch.sqrt(s2))
    d_rstd = STAT_PARTIALS * rstd * (Q / cnt + mean ** 2) / s2
    return affine_table(mean, rstd, d_mean, d_rstd, gamma, beta, groups)


def partials_from(X, slots, width):
    """Synthetic producer partials: fp32 (sum, sum of squares) of X [N, spatial, C] per producer group of `width`
    channels and per slot (a contiguous run of voxels), laid out [N][slots][C / width][2] as b200_igemm leaves them."""
    N, S, C = X.shape
    P = torch.zeros(N, slots, C // width, 2, dtype=torch.float32)
    edges = torch.linspace(0, S, slots + 1).long()
    for s in range(slots):
        seg = X[:, edges[s]:edges[s + 1]].reshape(N, -1, C // width, width)
        P[:, s, :, 0], P[:, s, :, 1] = seg.sum((1, 3)).float(), (seg ** 2).sum((1, 3)).float()
    return P


# ----------------------------------------------------------------------------------------------------------------
# activations and outputs
# ----------------------------------------------------------------------------------------------------------------
def act(t, t_err, code):
    """act(t) and its error given |d t| <= t_err: the slope carries t_err, SiLU adds the __expf / __fdividef error."""
    if code == ACT_NONE:
        return t, t_err
    if code == ACT_SILU:
        y = t * torch.sigmoid(t)
        return y, 1.1 * t_err + (8 + 1.2 * t.abs()) * 2.0 ** -24 * y.abs()
    if code in SLOPE:
        y = torch.where(t > 0, t, SLOPE[code] * t)
        return y, t_err
    raise ValueError(f"activation {code} is not one the normalisation kernels take")


def _store(y, y_err, N, spatial, C, y_pitch):
    """[N, spatial, C] values -> Result over the output rows [N * spatial, y_pitch] (pad channels +0)."""
    exact = torch.zeros(N * spatial, y_pitch, dtype=F64)
    err = torch.zeros_like(exact)
    exact[:, :C] = y.reshape(-1, C)
    err[:, :C] = y_err.reshape(-1, C)
    return Result(exact, h16(exact), err)


def gn_output(X, t: Affine, code, y_pitch):
    """h16(act(fma(x, a, b))) over X [N, spatial, C] with the affine table t."""
    N, S, C = X.shape
    a, b = t.a[:, None], t.b[:, None]
    ex = lambda v: v.repeat_interleave(C // t.mean.shape[1], 1)[:, None]
    m, dr, dm = ex(t.mean), ex(t.d_rstd), ex(t.d_mean)
    tt = X * a + b
    t_err = (X - m).abs() * t.gamma.abs()[:, None] * dr + a.abs() * dm + FP32 * ((X * a).abs() + b.abs())
    y, y_err = act(tt, t_err, code)
    return _store(y, y_err, N, S, C, y_pitch)


def groupnorm(x0, x1, C0, C1, pitch0, pitch1, N, spatial, groups, eps, gamma, beta, code, y_pitch):
    """b200_groupnorm_stats + b200_groupnorm_apply, and b200_groupnorm_fused: (Result, Affine)."""
    X = concat(x0, x1, C0, C1, pitch0, pitch1, N, spatial)
    t = gn_affine(X, groups, eps, gamma, beta)
    return gn_output(X, t, code, y_pitch), t


def spade(x0, x1, C0, C1, pitch0, pitch1, N, spatial, ax, gb, gb_pitch, gba, code, y_pitch):
    """b200_spade_apply: ax [N, C, 2] the affine table of x, gba [N, 2C, 2] that of gb's gamma / beta halves."""
    C = C0 + C1
    X = concat(x0, x1, C0, C1, pitch0, pitch1, N, spatial)
    G = rows_of(gb, N * spatial, gb_pitch, 2 * C).view(N, spatial, 2 * C)
    ax, gba = ax.to(F64), gba.to(F64)
    g, t = G[..., :C], G[..., C:]
    fa = lambda v, tab: (v * tab[:, None, :, 0] + tab[:, None, :, 1],
                         2.0 ** -23 * ((v * tab[:, None, :, 0]).abs() + tab[:, None, :, 1].abs()))
    nx, e_nx = fa(X, ax)
    gg, e_gg = fa(g, gba[:, :C])
    tb, e_tt = fa(t, gba[:, C:])
    one = 1.0 + gg
    v = nx * one + tb
    v_err = (e_nx * one.abs() + nx.abs() * (e_gg + 2.0 ** -24 * one.abs()) + e_tt
             + 2.0 ** -23 * ((nx * one).abs() + tb.abs()))
    y, y_err = act(v, v_err, code)
    return _store(y, y_err, N, spatial, C, y_pitch)


def ln_rows(X, gamma, beta, eps):
    """LayerNorm of the rows X [M, C] float64: (value, err)."""
    mean = X.mean(1, keepdim=True)
    var = ((X - mean) ** 2).mean(1, keepdim=True)
    s2 = var + eps
    rstd = 1.0 / torch.sqrt(s2)
    g, b = gamma.to(F64)[None], beta.to(F64)[None]
    u = 2.0 ** -24 * (X.shape[1] / 32 + 8)
    d_mean = u * (mean.abs() + torch.sqrt(s2))
    d_rstd = rstd * (u + 2.0 ** -21 + d_mean ** 2 / s2)
    y = (X - mean) * rstd * g + b
    err = ((X - mean).abs() * g.abs() * d_rstd + rstd * g.abs() * d_mean
           + FP32 * ((X - mean).abs() * rstd * g.abs() + b.abs() + X.abs() * rstd * g.abs()))
    return y, err


def layernorm(x, M, C, x_pitch, gamma, beta, eps, y_pitch):
    """b200_layernorm: Result over [M, y_pitch]."""
    y, err = ln_rows(rows_of(x, M, x_pitch, C), gamma, beta, eps)
    return _store(y, err, 1, M, C, y_pitch)


def rows_linear_ln(x, M, K, x_pitch, gamma, beta, eps):
    """The LayerNorm prologue of b200_rows_linear: the staged h16 row [M, K] (what an identity weight returns)."""
    return layernorm(x, M, K, x_pitch, gamma, beta, eps, K)

"""Float64 reading of include/b200gen_losses.h: what b200_spectral_fft, b200_spectral_distance and b200_adversarial
compute, with torch.fft in fp64 as the transform, and the bounds their device results are held to (u = 2^-24,
e = 2^-53).

  b200_spectral_fft (``Spectra``): per (side, image) spectrum, |X_device - X|_2 <= FFT_C sum_axes log2(n) u |X|_2.
  Norm-wise, not per coefficient: an FFT's rounding errors spread over all coefficients of a transform, so a small
  coefficient next to large ones carries an error of the size of the large ones' (FFT_C below bounds it by the RMS of
  its 1-D transform, which an N-D spectrum does not keep per coefficient); the 2-norm of the whole spectrum is what
  the per-level analysis bounds.
  b200_spectral_distance, per bin of the device's own spectrum (``distance_bound``): the scale, the two squares, the
  sum and the sqrt each round correctly, so a = |scale X| errs by 3 u a (plus 2^-74 where the squares are subnormal);
  d = a_0 - a_1 rounds once, v = d^2 once: e_v = 2 |d| (e_a0 + e_a1 + u |d|) + u v.  The reductions sum m e_v over the
  half spectrum, in fp64 (n e sum m v) with one more e for the division; out is one fp32 rounding of them.
  b200_adversarial, per element (``adversarial_bound``): BCE's p = 1 / (1 + exp(-z)) with CUDA's expf (2 ulp) against
  the reading's fp32 sigmoid (at most 2 ulp more), the add and the division: e_p = p ((1 - p) 2 LIBM + 2 u) + 2^-149;
  log p then errs by e_p / p and log1p(-p) by e_p / (1 - p), each plus its 1 ulp, and the -100 clamp only shrinks the
  difference.  Hinge: tanhf's 2 ulp.  Least squares: the 0.05f product and constant 2 u |a|, the difference and the
  square one u each, through v = (a - t)^2.  losses[i] are fp64 sums of the fp32 values: sum (e_v + u v) + n e sum v,
  then a division (one e) and the stacked sum or mean; losses32 one fp32 rounding more.
"""
import math
from dataclasses import dataclass

import torch

F64 = torch.float64
U = 2.0 ** -24
E53 = 2.0 ** -53
LIBM = 2.0 ** -22          # 2 ulp: expf, tanhf
LOG1 = 2.0 ** -23          # 1 ulp: logf, log1pf
# Per coefficient, |X_device - X| <= FFT_C * log2(n) * U * RMS(X) for a 1-D transform of length n (log2(n) taken as 1
# for n < 2).  Each radix-2 level of an fp32 FFT adds a relative error of about sqrt(2) U to the coefficients' RMS
# (one add and, on half of them, a complex multiply by a twiddle rounded once); radix 4 / 8 butterflies spend fewer
# roundings per level.  A Bluestein transform of length n runs three power-of-two transforms of M <= 4n, whose errors
# add, so its RMS error is about sqrt(3) (log2(n) + 2) sqrt(2) U.  The largest of the n coefficients' errors stays
# within three RMS errors in the measured cases, which gives 3 * sqrt(2) * sqrt(3) ~ 7.3; FFT_C = 8 leaves headroom.
# The FFT's measured worst is about 1.5 (lengths 1 .. 4096, powers of two and primes).
FFT_C = 8.0


def sig4(sig):
    return [sig[0]] + [1] * (4 - len(sig)) + list(sig[1:])


def spectral_fft(x: torch.Tensor, y: torch.Tensor, sig) -> torch.Tensor:
    """The complex128 half spectra [2, B, nC, n1, n2, n3 // 2 + 1] (leading spatial sizes 1 for fewer dims)."""
    dims = tuple(range(1, x.dim()))
    out = []
    for t in (x, y):
        s = torch.fft.rfftn(t.to(F64), s=list(sig), dim=dims)
        out.append(s.reshape(t.shape[0], *sig4(sig)[:3], -1))
    return torch.stack(out)


@dataclass
class Spectra:
    """b200_spectral_fft's result: the exact spectra [2, B, ...] (complex128), the complex64 values the reading stores
    (`out`) and the norm bound per (side, image) spectrum (`err`, [2, B])."""
    exact: torch.Tensor
    out: torch.Tensor
    err: torch.Tensor
    kind: str = "norm"


def spectra(x: torch.Tensor, y: torch.Tensor, sig) -> Spectra:
    s = spectral_fft(x, y, sig)
    tol = FFT_C * sum(max(1.0, math.log2(n)) for n in sig) * U
    return Spectra(s, s.to(torch.complex64).to(torch.complex128), tol * s.abs().flatten(2).norm(dim=2), "norm")


def norm_excess(r: Spectra, got: torch.Tensor) -> torch.Tensor:
    """|got - exact|_2 / err per (side, image) spectrum: > 1 is outside the bound; non-finite values are inf."""
    d = (got.to(torch.complex128) - r.exact).abs().flatten(2).norm(dim=2)
    ratio = torch.where(d == 0, torch.zeros_like(d), d / r.err)
    return torch.where(torch.isfinite(ratio), ratio, torch.full_like(ratio, math.inf))


def weights(sig) -> torch.Tensor:
    """Hermitian multiplicity of each last-axis bin: 1 for k = 0 and (even n) k = n / 2, else 2."""
    n3 = sig4(sig)[3]
    w = torch.full((n3 // 2 + 1,), 2.0, dtype=F64)
    w[0] = 1.0
    if n3 % 2 == 0:
        w[-1] = 1.0
    return w


def spectral_distance(spec: torch.Tensor, sig, scale: float, reduction: int):
    """REDUCTION_NONE (0): the full fp64 [B, nC, *sig[1:]] tensor; MEAN (1) / SUM (2): (sum, mean) in fp64."""
    a = (spec.to(torch.complex128) * scale).abs()
    v = (a[0] - a[1]) ** 2
    B = spec.shape[1]
    if reduction == 0:
        return full_spectrum(v, sig)
    s = (v * weights(sig)).sum()
    return s, s / (B * math.prod(sig))


def full_spectrum(v: torch.Tensor, sig) -> torch.Tensor:
    """The half-spectrum values v [B, nC, n1, n2, h] on the full spectrum [B, *sig], mirrored bins read from their
    partners ((-k0) mod nC, (-k1) mod n1, (-k2) mod n2, n3 - k3)."""
    B = v.shape[0]
    n3 = sig4(sig)[3]
    h = n3 // 2 + 1
    out = torch.empty((B, *sig4(sig)), dtype=F64)
    out[..., :h] = v
    if n3 > h:
        k3 = torch.arange(h, n3)
        mirror = v[..., n3 - k3]
        for ax in (1, 2, 3):
            mirror = torch.roll(torch.flip(mirror, dims=(ax,)), shifts=1, dims=ax)
        out[..., h:] = mirror
    return out.reshape(B, *sig)


def distance_bound(spec: torch.Tensor, sig, scale: float, reduction: int):
    """The module docstring's bound on b200_spectral_distance: per half-spectrum bin [B, nC, n1, n2, h] mirrored to the
    full spectrum for REDUCTION_NONE (0), else (sum bound, mean bound) of the fp64 results."""
    a = (spec.to(torch.complex128) * scale).abs()
    ea = 3 * U * a + 2.0 ** -74
    d = a[0] - a[1]
    v = d * d
    ev = 2 * d.abs() * (ea[0] + ea[1] + U * d.abs()) + U * v
    if reduction == 0:
        return full_spectrum(ev, sig)
    m = weights(sig)
    s = (m * (ev + U * v)).sum() + v.numel() * E53 * (m * v).sum()
    count = spec.shape[1] * math.prod(sig)
    return s, s / count + E53 * (m * v).sum() / count


ADV_BCE, ADV_HINGE, ADV_LSQ, ADV_LSQ_RAW = 0, 1, 2, 3


def adversarial_values(x: torch.Tensor, criterion: int, real: bool) -> torch.Tensor:
    """Per-element values of one output, in float64; BCE's probability is the contract's fp32 one, so a logit of 40
    gives p = 1 and the clamped -100 log, as in the fp32 reference (in fp64 it would give 40)."""
    z = x.to(F64)
    t = 1.0 if real else 0.0
    if criterion == ADV_BCE:
        p = (1.0 / (1.0 + torch.exp(-x.float()))).to(F64)
        return -(t * torch.log(p).clamp(min=-100) + (1 - t) * torch.log1p(-p).clamp(min=-100))
    if criterion == ADV_HINGE:
        a = torch.tanh(z) if real else -torch.tanh(z)
        return torch.clamp(a - 1, max=0)
    a = torch.where(z < 0, 0.05 * z, z) if criterion == ADV_LSQ else z
    return (a - t) ** 2


def adversarial_bound(x: torch.Tensor, criterion: int, real: bool) -> torch.Tensor:
    """Per-element bound of the module docstring on a device's fp32 value before its own rounding, float64."""
    z = x.to(F64)
    t = 1.0 if real else 0.0
    if criterion == ADV_BCE:
        p = (1.0 / (1.0 + torch.exp(-x.float()))).to(F64)
        ep = p * ((1 - p) * 2 * LIBM + 2 * U) + 2.0 ** -149
        if real:
            lg = torch.log(p)
            e = torch.where(p > 0, ep / p, torch.zeros_like(p)) + LOG1 * lg.abs().clamp(max=100)
        else:
            lg = torch.log1p(-p)
            e = torch.where(p < 1, ep / (1 - p), torch.zeros_like(p)) + LOG1 * lg.abs().clamp(max=100)
        return torch.nan_to_num(e, nan=math.inf)
    if criterion == ADV_HINGE:
        a = torch.tanh(z).abs()
        return LIBM * a + U * (a + 1)
    a = torch.where(z < 0, 0.05 * z, z) if criterion == ADV_LSQ else z
    ea = torch.where(z < 0, 2 * U * a.abs(), torch.zeros_like(a)) if criterion == ADV_LSQ else torch.zeros_like(a)
    d = (a - t).abs()
    return 2 * d * (ea + U * d) + U * d * d


def adversarial_losses_bound(vals, errs, criterion: int, reduction: int) -> torch.Tensor:
    """[n + 1] bound of the module docstring on the fp64 losses from per-element values and bounds."""
    per = []
    for v, e in zip(vals, errs):
        s = (e + U * v.abs()).sum() + v.numel() * E53 * v.abs().sum()
        mean = s / v.numel() + E53 * v.abs().sum() / v.numel()
        per.append(s if (reduction == 2 and criterion != ADV_HINGE) else mean)
    per = torch.stack(per)
    total = per.sum() + len(vals) * E53 * per.abs().sum()
    return torch.cat([per, (total if reduction == 2 else total / len(vals))[None]])


def adversarial(xs, criterion: int, real: bool, reduction: int):
    """(fp64 [n + 1] per-output losses then the stacked reduction, per-element fp64 values per output)."""
    vals = [adversarial_values(x, criterion, real) for x in xs]
    per = []
    for v in vals:
        s = v.sum()
        if criterion == ADV_HINGE:
            per.append(-s / v.numel())
        else:
            per.append(s if reduction == 2 else s / v.numel())
    per = torch.stack(per)
    total = per.sum() if reduction == 2 else per.sum() / len(xs)
    return torch.cat([per, total[None]]), vals

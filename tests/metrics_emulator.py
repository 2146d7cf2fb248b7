"""Float64 reading of the metric entry points of include/b200gen_metrics.h (b200_ssim, b200_ssim_combine, b200_mmd),
the contract the GPU tests hold the kernels to and the CPU stand-in computes with.  Inputs are converted to fp32 first,
as the kernels load them; the filters, moments and sums are then float64, so a kernel's fp32 arithmetic shows up as its
difference from this reading.  The pooling between MS-SSIM scales is b200_interpolate's: ``pool`` reads it with
tests/rescaler_oracle.py, exactly.

Bounds (u = 2^-24, the fp32 unit roundoff; e = 2^-53, fp64's), each the first-order error of the header's arithmetic:

  b200_ssim, per voxel (``ssim_bound``).  A filtered moment is an fma chain over W, then over H of the stored
  W-results, then over D: each of the kw + kh + kd fmas rounds once, by at most u times the filter of |values| so
  far, and the product a * b (or a * a) under the W chain once more, so mu_t is off by
      e_t <= (kw + kh + kd + 2) u scale F(|t|),   F the same separable filter with |taps|
  (the second 1: the multiplication by `scale`).  The cancellations carry those errors plus one rounding of the
  product and one of the difference:  e_sx <= e_xx + 2 |mu_x| e_x + u mu_x^2 + u |sx|  (sy alike),
      e_sxy <= e_xy + |mu_y| e_x + |mu_x| e_y + u |mu_x mu_y| + u |sxy|.
  A quotient n / d with |n| errs by e_n and d by e_d is off by (e_n + |n / d| e_d) / |d| plus its own rounding
  u |n / d|; c2 > 0 (c1 > 0) keeps d away from 0 because the exact sx + sy and mu_x^2 + mu_y^2 are >= 0.  cs takes
  e_n = 2 e_sxy + u |n|, e_d = e_sx + e_sy + 2 u (|sx| + |sy| + c2); the luminance l takes e_n = 2 (|mu_y| e_x +
  |mu_x| e_y) + 2 u |mu_x mu_y| + u |n|, e_d = 2 (|mu_x| e_x + |mu_y| e_y) + 2 u (mu_x^2 + mu_y^2 + d); ssim = l cs
  errs by |l| e_cs + |cs| e_l + u |ssim|.  Terms of order (k u)^2 (below 1e-5 relative for k <= 3 * 128) are dropped.
  The per-item sums a call leaves in its partial slots (``SlotSums``) are held to the sum of these bounds plus the
  fp64 summation's n e sum |v|: the device's slot layout is its own, so the slots are compared summed per item.
  b200_ssim_combine (``combine_bound``): a mean is the fp64 sum over `slots` partials (slots e sum |p|), one fp64
  division and one fp32 rounding, which the f32 tolerance's ulp holds; ms_ssim is a product of powf factors of fp32
  means that may differ from the reading's by an ulp: per factor w_s (ulp32(v_s) + e_v) / v_s relative for the
  mean, CUDA's 4 ulp for powf (2^-21 relative) and u for the product.
  b200_mmd (``mmd_bound``): d_v = sum_b (y - p) of fp32 values in fp64 errs by 2 B e sum_b (|y| + |p|); its square
  by 2 |d_v| e_d + e d_v^2; the fp64 sum over V by V e sum d_v^2; the division by one e.  One fp32 rounding on
  top (the f32 tolerance's ulp).
"""
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from tests import rescaler_oracle as R
from tests.elementwise_emulator import ulp32

F64 = torch.float64
U = 2.0 ** -24
E53 = 2.0 ** -53
POWF = 2.0 ** -21          # CUDA's powf: 4 ulp


@dataclass
class SlotSums:
    """The per-item sums of ssim and cs [N, 2] a b200_ssim call spreads over its partial slots: the reading's values
    (`exact`) and the bound on a device's slot total (`err`)."""
    exact: torch.Tensor
    err: torch.Tensor
    kind: str = "slots"


def filter3(t, taps):
    """Valid separable filtering of [N, C, D, H, W] with (taps_d, taps_h, taps_w), float64."""
    N, C = t.shape[:2]
    t = t.reshape(N * C, 1, *t.shape[2:])
    for axis, k in zip((2, 3, 4), taps):
        w = torch.tensor(k, dtype=F64).view(1, 1, *[len(k) if a == axis else 1 for a in (2, 3, 4)])
        t = F.conv3d(t, w)
    return t.reshape(N, C, *t.shape[2:])


def ssim(x, y, taps, scale, c1, c2):
    """(ssim_map, cs_map) float64 [N, C, OD, OH, OW] of b200_ssim on 5-D views x (= y_pred), y."""
    x, y = x.float().to(F64), y.float().to(F64)
    mx, my, mxx, myy, mxy = (filter3(t, taps) * scale for t in (x, y, x * x, y * y, x * y))
    sx, sy, sxy = mxx - mx * mx, myy - my * my, mxy - mx * my
    cs = (2 * sxy + c2) / (sx + sy + c2)
    return ((2 * mx * my + c1) / (mx * mx + my * my + c1)) * cs, cs


def ssim_bound(x, y, taps, scale, c1, c2):
    """(ssim_map, cs_map, ssim_err, cs_err) float64 [N, C, OD, OH, OW]: the maps of ``ssim`` and the bound of the
    module docstring on a device's fp32 values (before the store's own rounding, which the f32 tolerance adds)."""
    x, y = x.float().to(F64), y.float().to(F64)
    k = sum(len(t) for t in taps)
    absf = lambda t: filter3(t, [[abs(v) for v in a] for a in taps]) * abs(scale)
    mx, my, mxx, myy, mxy = (filter3(t, taps) * scale for t in (x, y, x * x, y * y, x * y))
    ex, ey, exx, eyy, exy = ((k + 2) * U * absf(t) for t in (x.abs(), y.abs(), x * x, y * y, (x * y).abs()))
    sx, sy, sxy = mxx - mx * mx, myy - my * my, mxy - mx * my
    esx = exx + 2 * mx.abs() * ex + U * mx * mx + U * sx.abs()
    esy = eyy + 2 * my.abs() * ey + U * my * my + U * sy.abs()
    esxy = exy + my.abs() * ex + mx.abs() * ey + U * (mx * my).abs() + U * sxy.abs()
    nc, dc = 2 * sxy + c2, sx + sy + c2
    cs = nc / dc
    ecs = (2 * esxy + U * nc.abs() + cs.abs() * (esx + esy + 2 * U * (sx.abs() + sy.abs() + c2))) / dc.abs() \
        + U * cs.abs()
    nl, dl = 2 * mx * my + c1, mx * mx + my * my + c1
    lum = nl / dl
    enl = 2 * (my.abs() * ex + mx.abs() * ey) + 2 * U * (mx * my).abs() + U * nl.abs()
    edl = 2 * (mx.abs() * ex + my.abs() * ey) + 2 * U * (mx * mx + my * my + dl.abs())
    el = (enl + lum.abs() * edl) / dl.abs() + U * lum.abs()
    ss = lum * cs
    return ss, cs, lum.abs() * ecs + cs.abs() * el + U * ss.abs(), ecs


def slot_sums(ssim_map, cs_map, ssim_err, cs_err, slots):
    """SlotSums of one b200_ssim call with `slots` partial slots per item."""
    N = ssim_map.shape[0]
    cols = []
    for v, e in ((ssim_map, ssim_err), (cs_map, cs_err)):
        v, e = v.reshape(N, -1), e.reshape(N, -1)
        cols.append((v.sum(1), (e + ulp32(v)).sum(1) + (v.shape[1] + slots) * E53 * v.abs().sum(1)))
    return SlotSums(torch.stack([cols[0][0], cols[1][0]], 1), torch.stack([cols[0][1], cols[1][1]], 1))


def combine_bound(sums, sums_abs, slots, count, ssim_means, cs_means, weights):
    """Bounds of b200_ssim_combine from the device's partials: (mean_err [N] per scale for the ssim / cs means,
    ms_err [N]).  sums_abs[s]: sum over the item's slots of |partial| [N, 2]."""
    mean_err = [(slots[s] + 2) * E53 * sums_abs[s] / count[s] for s in range(len(sums))]
    v = cs_means.to(F64).clone()
    v[-1] = ssim_means[-1].to(F64)
    ve = torch.stack([mean_err[s][:, 1] for s in range(len(sums))])
    ve[-1] = mean_err[-1][:, 0]
    w = torch.tensor([float(a) for a in weights], dtype=F64).view(-1, 1)
    ms = combine(ssim_means, cs_means, weights)
    pos = v.clamp_min(0)
    rel = torch.where(pos > 0, w * (ulp32(pos) + ve) / pos.clamp_min(1e-300), torch.zeros_like(pos))
    return mean_err, ms.abs() * (rel + POWF + U).sum(0)


def per_item_means(m):
    return m.reshape(m.shape[0], -1).mean(1)


def combine(ssim_means, cs_means, weights):
    """b200_ssim_combine from per-scale fp32 means [S, N]: prod_s relu(v_s) ** w_s, v = cs, ssim at the last scale."""
    v = cs_means.clone()
    v[-1] = ssim_means[-1]
    w = torch.tensor([float(a) for a in weights], dtype=F64).view(-1, 1)
    return torch.prod(v.to(F64).clamp_min(0) ** w, dim=0)


def pool(x, dims):
    """ops.avgpool2_f32 of a 5-D [N, C, D, H, W] tensor (2-D: D == 1, not pooled): AREA over the even part of each
    pooled extent, fp32."""
    N, C, D, H, W = x.shape
    out = (D // 2 if dims == 3 else D, H // 2, W // 2)
    src = (2 * out[0] if dims == 3 else D, 2 * out[1], 2 * out[2])
    return R.header_interpolate(x[:, :, :src[0], :src[1], :src[2]], out, (1.0, 1.0, 1.0), R.AREA)


def mmd(y, y_pred):
    """b200_mmd: sum_v (ybar_v - pbar_v)^2 / V over the flattened rows, float64."""
    d = (y.float().to(F64) - y_pred.float().to(F64)).reshape(y.shape[0], -1).mean(0)
    return (d * d).mean()


def mmd_bound(y, y_pred):
    """The module docstring's bound on b200_mmd's value before its fp32 rounding, float64 0-dim."""
    a, b = (t.float().to(F64).reshape(t.shape[0], -1) for t in (y, y_pred))
    B, V = a.shape
    d = (a - b).sum(0)
    ed = 2 * B * E53 * (a.abs() + b.abs()).sum(0)
    return ((2 * d.abs() * ed).sum() + (V + 2) * E53 * (d * d).sum()) / (B * B * V)

"""Float64 reading of the metric entry points of include/b200gen_metrics.h (b200_ssim, b200_ssim_combine, b200_mmd),
the contract the GPU tests hold the kernels to and the CPU stand-in computes with.  Inputs are converted to fp32 first,
as the kernels load them; the filters, moments and sums are then float64, so a kernel's fp32 arithmetic shows up as its
difference from this reading.  The pooling between MS-SSIM scales is b200_interpolate's: ``pool`` reads it with
tests/rescaler_oracle.py, exactly."""
import torch
import torch.nn.functional as F

from tests import rescaler_oracle as R

F64 = torch.float64


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

"""Float64 reading of include/b200gen_perceptual.h: what b200_perceptual_prep, b200_perceptual_distance and
b200_perceptual_mean compute, and the bound a device result of the distance is held to."""
import numpy as np
import torch

F64 = torch.float64
MEAN32 = torch.tensor([0.485, 0.456, 0.406], dtype=torch.float32)
STD32 = torch.tensor([0.229, 0.224, 0.225], dtype=torch.float32)
EPS32 = float(np.float32(1e-10))
U = 2.0 ** -24


def gather(src: torch.Tensor, S: int, idx) -> torch.Tensor:
    """Images [n_out, C, OH, OW] of a 5-D view [N, C, S, OH, OW] (image q = n * S + slice) picked by idx (or all)."""
    N, C, _, OH, OW = src.shape
    flat = src.permute(0, 2, 1, 3, 4).reshape(N * S, C, OH, OW)
    return flat if idx is None else flat[torch.as_tensor(idx, dtype=torch.long)]


def prep(images: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """[n, C, OH, OW] source images (C = 1: repeated) -> the z-scored [n, 3, OH, OW] in `dtype` (fp32: the contract's
    arithmetic, correctly rounded subtraction then division; float64: the exact value)."""
    x = images.float().to(dtype)
    if x.shape[1] == 1:
        x = x.repeat(1, 3, 1, 1)
    m, s = MEAN32.to(dtype)[None, :, None, None], STD32.to(dtype)[None, :, None, None]
    return (x - m) / s


def pixel_distance(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """[B, HW, C] features -> [B, HW] sum_c (x / (|x| + eps) - y / (|y| + eps))^2, in float64."""
    x, y = x.to(F64), y.to(F64)
    nx = x.pow(2).sum(-1, keepdim=True).sqrt()
    ny = y.pow(2).sum(-1, keepdim=True).sqrt()
    return (x / (nx + EPS32) - y / (ny + EPS32)).pow(2).sum(-1)


def distance(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """Per-image spatial means [B] (float64)."""
    return pixel_distance(x, y).mean(1)


def distance_bound(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """Per image: the mean over pixels of 4 u sqrt(v) + 160 u v, v the pixel's exact value (u = 2^-24).  Rounding
    the quotients x_c / (n_x + eps) and y_c / (n_y + eps) moves each d_c by at most u (|x^_c| + |y^_c|), which changes
    sum d_c^2 by at most 2 u sum |d_c| (|x^_c| + |y^_c|) <= 4 u sqrt(v) (Cauchy-Schwarz, unit vectors).  A relative
    error e of a norm scales x^ by (1 + e) and changes the sum by 2 e sum d_c x^_c = e v (for unit vectors
    sum d_c x^_c = v / 2), and the sums of squares (32-lane fused multiply-adds over 64 terms, a 5-level butterfly)
    err by at most 69 u relatively: together below 160 u v.  The direct form's error vanishes with v; the expanded
    form's does not."""
    v = pixel_distance(x, y)
    return (4 * U * v.sqrt() + 160 * U * v).mean(1)


def mean(image: torch.Tensor, counts) -> torch.Tensor:
    """Group means then their sum, float64 [len(counts) + 1]."""
    out, o = [], 0
    for k in counts:
        out.append(image[o:o + k].to(F64).sum() / k)
        o += k
    out.append(sum(out[1:], out[0]))
    return torch.stack(out)

"""Torch restatements of the reference's metric arithmetic (generative/metrics/ssim.py, ms_ssim.py, mmd.py): full
depthwise kernels through F.conv{2,3}d for SSIM / CS, F.avg_pool between MS-SSIM scales and three Gram GEMMs for MMD,
in fp32 as the reference computes.  Pinned against the reference by tests/test_metrics_oracle_vs_reference.py; the
baseline tools/metrics_probe.py times on the GPU."""
import torch
import torch.nn.functional as F


def gaussian_1d(k, sigma):
    dist = torch.arange(start=(1 - k) / 2, end=(1 + k) / 2, step=1)
    g = torch.exp(-torch.pow(dist / sigma, 2) / 2)
    return g / g.sum()


def full_kernel(spatial_dims, channels, kernel_type, kernel_size, kernel_sigma):
    """The depthwise [C, 1, *k] window: the outer product of the per-axis Gaussians in fp32, or 1 / prod(k)."""
    ks = tuple(kernel_size)[:spatial_dims]
    if kernel_type == "gaussian":
        k = gaussian_1d(ks[0], kernel_sigma[0])
        for ax in range(1, spatial_dims):
            k = k.unsqueeze(-1) * gaussian_1d(ks[ax], kernel_sigma[ax])
    else:
        k = torch.ones(ks) / torch.prod(torch.tensor(ks))
    return k.expand(channels, 1, *ks)


def ssim_and_cs(y_pred, y, spatial_dims, data_range=1.0, kernel_type="gaussian", kernel_size=(11, 11, 11),
                kernel_sigma=(1.5, 1.5, 1.5), k1=0.01, k2=0.03):
    x, y = y_pred.float(), y.float()
    C = x.shape[1]
    w = full_kernel(spatial_dims, C, kernel_type, kernel_size, kernel_sigma).to(x.device)
    conv = getattr(F, f"conv{spatial_dims}d")
    mx, my, mxx, myy, mxy = (conv(t, w, groups=C) for t in (x, y, x * x, y * y, x * y))
    sx, sy, sxy = mxx - mx * mx, myy - my * my, mxy - mx * my
    cs = (2 * sxy + (k2 * data_range) ** 2) / (sx + sy + (k2 * data_range) ** 2)
    return ((2 * mx * my + (k1 * data_range) ** 2) / (mx ** 2 + my ** 2 + (k1 * data_range) ** 2)) * cs, cs


def ssim(y_pred, y, spatial_dims, **kw):
    s, _ = ssim_and_cs(y_pred, y, spatial_dims, **kw)
    return s.reshape(s.shape[0], -1).mean(1, keepdim=True)


def ms_ssim(y_pred, y, spatial_dims, weights=(0.0448, 0.2856, 0.3001, 0.2363, 0.1333), **kw):
    pool = getattr(F, f"avg_pool{spatial_dims}d")
    vals = []
    for _ in weights:
        s, cs = ssim_and_cs(y_pred, y, spatial_dims, **kw)
        vals.append(torch.relu(cs.reshape(cs.shape[0], -1).mean(1)))
        y_pred, y = pool(y_pred, kernel_size=2), pool(y, kernel_size=2)
    vals[-1] = torch.relu(s.reshape(s.shape[0], -1).mean(1))
    w = torch.tensor(list(weights), dtype=torch.float, device=s.device).view(-1, 1)
    return torch.prod(torch.stack(vals) ** w, dim=0).view(-1, 1)


def mmd(y, y_pred):
    y, y_pred = y.reshape(y.shape[0], -1), y_pred.reshape(y_pred.shape[0], -1)
    V = y.shape[1]
    return (torch.mm(y, y.t()) / V).mean() + (torch.mm(y_pred, y_pred.t()) / V).mean() - \
        2 * (torch.mm(y_pred, y.t()) / V).mean()

"""Plain-PyTorch restatement of PatchDiscriminator / MultiScalePatchDiscriminator
(generative/networks/nets/patchgan_discriminator.py) in eval mode, from a ``state_dict`` and the constructor arguments:
F.conv, F.batch_norm with the running statistics, F.instance_norm, F.avg_pool / F.max_pool and the activations.  Pinned
against the unmodified reference and the committed fixture (tests/golden/g_patchgan.pt) by tests/test_patchgan_cpu.py;
the CUDA path is checked against both.

Also the name-seeded weights the fixture uses (:func:`seeded_weights`) and a CPU stand-in for the two library entry
points the discriminators add (:func:`install`)."""
from __future__ import annotations

import zlib

import torch
import torch.nn.functional as F

from generativemodels_b200 import _lib

LEAKY02 = ("LEAKYRELU", {"negative_slope": 0.2})


def act_fn(activation):
    """monai's Act[...] (a name or a (name, kwargs) tuple) as a function."""
    if activation is None:
        return lambda x: x
    if isinstance(activation, str):
        name, kw = activation, {}
    else:
        name, kw = activation[0], dict(activation[1]) if len(activation) > 1 else {}
    fns = {"LEAKYRELU": lambda x: F.leaky_relu(x, kw.get("negative_slope", 0.01)), "RELU": F.relu, "SILU": F.silu,
           "SWISH": F.silu, "GELU": F.gelu, "TANH": torch.tanh, "SIGMOID": torch.sigmoid}
    return fns[str(name).upper()]


def _conv(sd, p, x, stride, padding):
    conv = F.conv2d if x.dim() == 4 else F.conv3d
    return conv(x, sd[p + ".conv.weight"], sd.get(p + ".conv.bias"), stride=stride, padding=padding)


def patch_discriminator(sd, x, num_layers_d=3, kernel_size=4, activation=LEAKY02, norm="BATCH", padding=1,
                        last_conv_kernel_size=None, prefix="", **_):
    """PatchDiscriminator.forward in eval mode: every layer's output, the patch scores last.  ``prefix`` is the
    module's key prefix in ``sd`` (empty for a bare PatchDiscriminator)."""
    act = act_fn(activation)
    pre = prefix + "." if prefix else ""
    h = act(_conv(sd, pre + "initial_conv", x, 2, padding))
    out = [h]
    for l_ in range(num_layers_d):
        h = _conv(sd, f"{pre}{l_}", h, 1 if l_ == num_layers_d - 1 else 2, padding)
        if norm.lower() == "batch":
            n = f"{pre}{l_}.adn.N."
            h = F.batch_norm(h, sd[n + "running_mean"], sd[n + "running_var"], sd[n + "weight"], sd[n + "bias"],
                             training=False, eps=1e-5)
        else:
            h = F.instance_norm(h, eps=1e-5)
        h = act(h)
        out.append(h)
    k = kernel_size if last_conv_kernel_size is None else last_conv_kernel_size
    out.append(_conv(sd, pre + "final_conv", h, 1, int((k - 1) / 2)))
    return out


def pool(x, method, kernel_size):
    pad = int((kernel_size - 1) / 2)
    fn = {("avg", 4): F.avg_pool2d, ("avg", 5): F.avg_pool3d, ("max", 4): F.max_pool2d, ("max", 5): F.max_pool3d}
    return fn[(method.lower(), x.dim())](x, kernel_size, 2, pad)


def layers_per_discriminator(num_d, num_layers_d, pooling_method):
    if isinstance(num_layers_d, int):
        return [num_layers_d * i for i in range(1, num_d + 1)] if pooling_method is None else [num_layers_d] * num_d
    return list(num_layers_d)


def multiscale(sd, x, num_d, num_layers_d, pooling_method=None, kernel_size=4, activation=LEAKY02, norm="BATCH",
               last_conv_kernel_size=1, **_):
    """MultiScalePatchDiscriminator.forward in eval mode: (outputs, features); discriminator i sees the input pooled
    i times when ``pooling_method`` is set."""
    layers = layers_per_discriminator(num_d, num_layers_d, pooling_method)
    outs, feats = [], []
    for i in range(num_d):
        xi, prefix = x, f"discriminator_{i}"
        if pooling_method is not None and i > 0:
            for _ in range(i):
                xi = pool(xi, pooling_method, kernel_size)
            prefix += f".{i}"
        o = patch_discriminator(sd, xi, layers[i], kernel_size, activation, norm, int((kernel_size - 1) / 2),
                                last_conv_kernel_size, prefix)
        outs.append(o[-1])
        feats.append(o[:-1])
    return outs, feats


def seeded_weights(module, seed=0):
    """Deterministic parameters AND BatchNorm statistics keyed by name (independent of construction order, so the
    reference and this package get the same values): convolution weights N(0, 1/fan_in), biases N(0, 0.1^2), BatchNorm
    gamma 1 + N(0, 0.25^2), beta N(0, 0.1^2), running mean N(0, 0.2^2), running var U(0.3, 1.5).  Nothing is left at
    its default, so the BatchNorm fold is exercised."""
    with torch.no_grad():
        named = list(module.named_parameters()) + [(n, b) for n, b in module.named_buffers() if b.is_floating_point()]
        for name, t in named:
            g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
            r = torch.randn(t.shape, generator=g)
            if name.endswith("adn.N.weight"):
                v = 1 + 0.25 * r
            elif name.endswith("running_mean"):
                v = 0.2 * r
            elif name.endswith("running_var"):
                v = 0.3 + 1.2 * torch.rand(t.shape, generator=g)
            elif t.dim() == 1:
                v = 0.1 * r
            else:
                v = r * t[0].numel() ** -0.5
            t.copy_(v)
    return module


def input_of(rec):
    """The fixture's fp32 input: the stored fp16 tensor, repeated ``repeat`` times along every spatial axis."""
    x = rec["x16"].float()
    for d in range(2, x.dim()):
        x = x.repeat_interleave(rec["repeat"], d)
    return x


# ---------------------------------------------------------------------------------------------------------------------
# CPU stand-in for the new entry points (tests only)
# ---------------------------------------------------------------------------------------------------------------------
def install(monkeypatch):
    """tests/cpu_backend.install plus b200_pool_s2 and b200_batchnorm_fold, restated from include/b200gen.h."""
    from tests import cpu_backend as CB
    import generativemodels_b200.networks.nets.patchgan_discriminator as PG
    from tests import spadenet_oracle as SO
    fake = SO.install(monkeypatch)                       # LeakyReLU(0.2) in the stand-in and the igemm emulator

    def pool_s2(x, N, D, H, W, pitch, dims, k, pad, mode, y, stream):
        src = CB.bf16(x, N * D * H * W * pitch).view(N, D, H, W, pitch).float().permute(0, 4, 1, 2, 3)
        kk, pp, ss = ((k, k, k), (pad, pad, pad), 2) if dims == 3 else ((1, k, k), (0, pad, pad), (1, 2, 2))
        if mode == _lib.POOL_AVG:
            o = F.avg_pool3d(src, kk, ss, pp, count_include_pad=True)
        else:
            o = F.max_pool3d(src, kk, ss, pp)
        o = o.permute(0, 2, 3, 4, 1).contiguous()
        CB.bf16(y, o.numel()).view(o.shape).copy_(o.to(CB.ops.H16))
        return 0

    def batchnorm_fold(w, b, gamma, beta, mean, var, eps, cout, per, w_out, b_out, stream):
        s = CB.f32(gamma, cout).double() / (CB.f32(var, cout).double() + eps).sqrt()
        ww = CB.f32(w, cout * per).view(cout, per).double()
        bb = CB.f32(b, cout).double() if b else torch.zeros(cout, dtype=torch.float64)
        CB.f32(w_out, cout * per).view(cout, per).copy_(ww * s[:, None])
        CB.f32(b_out, cout).copy_(CB.f32(beta, cout).double() + (bb - CB.f32(mean, cout).double()) * s)
        return 0
    fake.b200_pool_s2 = pool_s2
    fake.b200_batchnorm_fold = batchnorm_fold
    monkeypatch.setattr(PG, "require_cuda", lambda x, m: None)
    return fake

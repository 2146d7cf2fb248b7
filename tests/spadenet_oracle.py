"""Plain-PyTorch restatement of SPADENet (generative/networks/nets/spade_network.py) from a ``state_dict`` and the
constructor arguments, pinned against the unmodified reference by tests/test_spadenet_cpu.py.  Test infrastructure: the
CUDA path is checked against this and against the committed fixture tests/golden/g_spadenet.pt."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def _conv(sd, p, x, stride=1, padding=None):
    w = sd[p + ".weight"]
    k = w.shape[-1]
    conv = F.conv2d if x.dim() == 4 else F.conv3d
    return conv(x, w, sd.get(p + ".bias"), stride=stride, padding=(k - 1) // 2 if padding is None else padding)


def spade(sd, p, x, seg):
    """SPADE.forward with the INSTANCE base norm: instance_norm(x) * (1 + IN(gamma)) + IN(beta), mlp_shared with
    LeakyReLU(0.01) and no norm, mlp_gamma / mlp_beta with monai's default INSTANCE norm."""
    seg = F.interpolate(seg, size=x.shape[2:], mode="nearest")
    k = sd[p + ".mlp_shared.conv.weight"].shape[-1]
    actv = F.leaky_relu(_conv(sd, p + ".mlp_shared.conv", seg, padding=k // 2), 0.01)
    gamma = F.instance_norm(_conv(sd, p + ".mlp_gamma.conv", actv, padding=k // 2))
    beta = F.instance_norm(_conv(sd, p + ".mlp_beta.conv", actv, padding=k // 2))
    return F.instance_norm(x) * (1 + gamma) + beta


def resnet_block(sd, p, x, seg):
    if (p + ".conv_s.conv.weight") in sd:
        x_s = _conv(sd, p + ".conv_s.conv", spade(sd, p + ".norm_s", x, seg))
    else:
        x_s = x
    dx = _conv(sd, p + ".conv_0.conv", F.leaky_relu(spade(sd, p + ".norm_0", x, seg), 0.2))
    dx = _conv(sd, p + ".conv_1.conv", F.leaky_relu(spade(sd, p + ".norm_1", dx, seg), 0.2))
    return x_s + dx


def encoder(sd, x, depth):
    """(mu, logvar): ``depth`` stride-2 conv -> InstanceNorm -> LeakyReLU(0.2) blocks, then fc_mu / fc_var on the
    channels-first flattening."""
    for i in range(depth):
        x = F.leaky_relu(F.instance_norm(_conv(sd, f"encoder.blocks.{i}.conv", x, stride=2)), 0.2)
    x = x.reshape(x.shape[0], -1)
    return (F.linear(x, sd["encoder.fc_mu.weight"], sd["encoder.fc_mu.bias"]),
            F.linear(x, sd["encoder.fc_var.weight"], sd["encoder.fc_var.bias"]))


def kld(mu, logvar):
    return -0.5 * torch.sum(1 + logvar - mu.pow(2) - logvar.exp())


def _upsample(x, mode):
    return F.interpolate(x, scale_factor=2, mode=mode)


def decoder(sd, seg, z, c0, latent, n_blocks, is_gan, upsampling_mode="nearest", last_act=0.2, p="decoder"):
    """SPADEDecoder.forward.  ``c0`` channels at the latent grid ``latent``; ``last_act`` the LeakyReLU slope of the
    output convolution (None = no activation)."""
    if is_gan:
        x = F.linear(F.interpolate(seg, size=tuple(latent)), sd[p + ".fc.weight"], sd[p + ".fc.bias"])
    else:
        x = F.linear(z, sd[p + ".fc.weight"], sd[p + ".fc.bias"]).view(-1, c0, *latent)
    for i in range(n_blocks):
        x = _upsample(resnet_block(sd, f"{p}.blocks.{i}", x, seg), upsampling_mode)
    x = _conv(sd, p + ".last_conv.conv", x)
    return x if last_act is None else F.leaky_relu(x, last_act)


def spadenet_vae(sd, seg, x, eps, depth, upsampling_mode="nearest", last_act=0.2):
    """SPADENet.forward in VAE mode with the draw ``eps`` given: (image, kld, mu, logvar, z)."""
    mu, logvar = encoder(sd, x, depth)
    z = eps * torch.exp(0.5 * logvar) + mu
    c0 = sd["decoder.blocks.0.conv_0.conv.weight"].shape[1]
    latent = [s // 2 ** depth for s in x.shape[2:]]
    img = decoder(sd, seg, z, c0, latent, depth, False, upsampling_mode, last_act)
    return img, kld(mu, logvar), mu, logvar, z


def randomize(module, seed=0):
    """Re-draw zero-initialised parameters (as the other fixtures do) so every path contributes."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            if float(p.abs().max()) == 0.0:
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
    return module


def one_hot_seg(n, label_nc, shape, seed=0):
    g = np.random.default_rng(seed)
    lab = torch.from_numpy(g.integers(0, label_nc, size=(n, *[max(1, s // 8) for s in shape])))
    lab = F.interpolate(lab[:, None].float(), size=tuple(shape), mode="nearest")[:, 0].long()
    return F.one_hot(lab, label_nc).movedim(-1, 1).float()


def seeded_weights(module, seed=0):
    """Deterministic weights for every parameter, keyed by name (independent of construction order, so the reference
    and this package get the same values): N(0, 1/fan_in) for weights, N(0, 0.1^2) for biases.  No parameter is left
    at zero, so every path of the network contributes."""
    import zlib
    with torch.no_grad():
        for name, p in module.named_parameters():
            g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
            std = 0.1 if p.dim() == 1 else (p[0].numel()) ** -0.5
            p.copy_(torch.randn(p.shape, generator=g) * std)
    return module


def labels_to_onehot(labels, label_nc):
    return F.one_hot(labels.long(), label_nc).movedim(-1, 1).float()

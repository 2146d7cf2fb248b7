"""SPADENet — ``generative/networks/nets/spade_network.py`` on the H100 kernels: the semantic image synthesis VAE-GAN of
Park et al. 2019 (a one-hot segmentation map plus a style code in, an image out), for inference.

Same constructor signatures, attributes, module tree and ``state_dict`` keys as the reference, including its quirks:
the constructor reverses the caller's ``num_channels`` list in place and the decoder appends ``out_channels`` to it;
``decode(seg)`` without ``z`` raises ``AttributeError`` (the reference reads a missing ``self.opt``); in GAN mode the
decoder's ``fc`` runs along the LAST SPATIAL AXIS of the resized segmentation map.

Where the work goes:
- encoder blocks: stride-2 convolution (igemm) -> InstanceNorm + LeakyReLU(0.2) in one normalisation pass;
- ``fc_mu`` / ``fc_var`` read the channels-last encoder output directly: their weight columns are permuted once, when
  they are packed, from the reference's channels-first flattening; the decoder ``fc`` has its rows permuted so that it
  writes the channels-last ``[N, *latent, C0]`` tensor.  No activation is ever transposed;
- z = eps * exp(logvar / 2) + mu and the KL term in one kernel (b200_vae_reparam_kld), eps drawn with
  ``torch.randn_like`` as the reference does;
- residual blocks: SPADE (InstanceNorm base) with the block's LeakyReLU(0.2) fused into the modulation pass, k3
  convolutions on igemm, the residual add fused into ``conv_1``'s epilogue;
- x2 upsampling: nearest (2-D and 3-D) or bilinear / bicubic (2-D, b200_upsample2x_interp).
"""
from __future__ import annotations

from enum import Enum
from typing import Sequence

import numpy as np
import torch
import torch.nn as nn

from ... import _lib, ops
from ...ops import ACT_LEAKYRELU02, CL
from .._holders import Convolution, _Cached, on_input_device, require_cuda
from ..blocks.spade_norm import SPADE, SegPyramid

__all__ = ["KLDLoss", "UpsamplingModes", "SPADEResNetBlock", "SPADEEncoder", "SPADEDecoder", "SPADENet"]

_LEAKY02 = ("LEAKYRELU", {"negative_slope": 0.2})


class KLDLoss(nn.Module):
    """-0.5 * sum(1 + logvar - mu^2 - exp(logvar)) over every element (b200_vae_reparam_kld)."""

    def forward(self, mu: torch.Tensor, logvar: torch.Tensor) -> torch.Tensor:
        require_cuda(mu, self)
        return ops.vae_reparam_kld(mu, logvar, torch.zeros_like(mu, dtype=torch.float32))[1]


class UpsamplingModes(str, Enum):
    bicubic = "bicubic"
    nearest = "nearest"
    bilinear = "bilinear"

    def __str__(self) -> str:
        return self.value


def _check_shape(spatial_dims: int, input_shape: Sequence[int], depth: int) -> list[int]:
    if len(input_shape) != spatial_dims:
        raise ValueError("Length of parameter input shape must match spatial_dims; got %s" % (input_shape))
    for s_ind, s_ in enumerate(input_shape):
        if s_ / (2 ** depth) != s_ // (2 ** depth):
            raise ValueError(
                "Each dimension of your input must be divisible by 2 ** (autoencoder depth)."
                "The shape in position %d, %d is not divisible by %d. " % (s_ind, s_, depth))
    return [s_ // (2 ** depth) for s_ in input_shape]


class SPADEResNetBlock(nn.Module):
    """Residual block with SPADE normalisation (reference lines 44-129).  ``forward`` works on channels-last
    activations: ``x`` a :class:`ops.CL`, ``seg`` the :class:`SegPyramid` of the forward pass."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int, label_nc: int,
                 spade_intermediate_channels: int = 128, norm: str | tuple = "INSTANCE", kernel_size: int = 3):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.int_channels = min(self.in_channels, self.out_channels)
        self.learned_shortcut = self.in_channels != self.out_channels
        self.conv_0 = Convolution(spatial_dims, self.in_channels, self.int_channels)
        self.conv_1 = Convolution(spatial_dims, self.int_channels, self.out_channels)
        self.activation = nn.LeakyReLU(0.2, False)
        spade = dict(label_nc=label_nc, kernel_size=kernel_size, spatial_dims=spatial_dims,
                     hidden_channels=spade_intermediate_channels, norm=norm)
        self.norm_0 = SPADE(norm_nc=self.in_channels, **spade)
        self.norm_1 = SPADE(norm_nc=self.int_channels, **spade)
        if self.learned_shortcut:
            self.conv_s = Convolution(spatial_dims, self.in_channels, self.out_channels, kernel_size=1)
            self.norm_s = SPADE(norm_nc=self.in_channels, **spade)

    def forward(self, x: CL, seg: SegPyramid) -> CL:
        x_s = self.shortcut(x, seg)
        dx = self.conv_0(self.norm_0(x, seg, act=ACT_LEAKYRELU02))
        return self.conv_1(self.norm_1(dx, seg, act=ACT_LEAKYRELU02), residual=x_s)

    def shortcut(self, x: CL, seg: SegPyramid) -> CL:
        return self.conv_s(self.norm_s(x, seg)) if self.learned_shortcut else x


class SPADEEncoder(nn.Module, _Cached):
    """VAE encoding branch (reference lines 132-218): stride-2 conv -> InstanceNorm -> act blocks, then ``fc_mu`` and
    ``fc_var`` on the flattened feature map."""

    def __init__(self, spatial_dims: int, in_channels: int, z_dim: int, num_channels: Sequence[int],
                 input_shape: Sequence[int], kernel_size: int = 3, norm: str | tuple = "INSTANCE",
                 act: str | tuple = _LEAKY02):
        super().__init__()
        self.in_channels = in_channels
        self.z_dim = z_dim
        self.num_channels = num_channels
        self.latent_spatial_shape = _check_shape(spatial_dims, input_shape, len(num_channels))
        self.input_shape = input_shape
        blocks = []
        ch_init = self.in_channels
        for ch_value in num_channels:
            blocks.append(Convolution(spatial_dims, ch_init, ch_value, strides=2, kernel_size=kernel_size,
                                      conv_only=False, norm=norm, act=act))
            ch_init = ch_value
        self.blocks = nn.ModuleList(blocks)
        self.fc_mu = nn.Linear(in_features=np.prod(self.latent_spatial_shape) * self.num_channels[-1],
                               out_features=self.z_dim)
        self.fc_var = nn.Linear(in_features=np.prod(self.latent_spatial_shape) * self.num_channels[-1],
                                out_features=self.z_dim)

    def _packed_fc(self, name: str, C_: int, pitch: int, S: int) -> ops.PackedLinear:
        """``name`` with its input columns moved from channels-first (c * S + s) to channels-last (s * pitch + c)
        order; the columns of pad channels are zero."""
        lin = getattr(self, name)
        return self._cached((name, C_, pitch, S), (lin.weight, lin.bias),
                            lambda: ops.PackedLinear.channels_first_input(lin.weight, lin.bias, C_, pitch, S))

    def _features(self, x: torch.Tensor) -> CL:
        h = ops.to_cl(x)
        for block in self.blocks:
            h = block(h)
        return h

    def _mu_logvar(self, h: CL) -> tuple[torch.Tensor, torch.Tensor]:
        S = h.spatial
        if S * h.C != self.fc_mu.in_features:
            raise RuntimeError(f"encoder features {h.C} x {S} do not match fc_mu's {self.fc_mu.in_features} inputs")
        rows = ops.as_rows(h.t.reshape(h.N, S * h.pitch), S * h.pitch)
        out = []
        for name in ("fc_mu", "fc_var"):
            y = ops.linear(rows, self._packed_fc(name, h.C, h.pitch, S), out_f32=True)
            out.append(y.reshape(h.N, -1)[:, :self.z_dim].contiguous())
        return out[0], out[1]

    @on_input_device
    def forward(self, x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        require_cuda(x, self)
        return self._mu_logvar(self._features(x))

    @on_input_device
    def encode(self, x: torch.Tensor) -> torch.Tensor:
        return self.reparameterize(*self.forward(x))

    def reparameterize(self, mu: torch.Tensor, logvar: torch.Tensor) -> torch.Tensor:
        return ops.vae_reparam_kld(mu, logvar, torch.randn_like(mu))[0]


class SPADEDecoder(nn.Module, _Cached):
    """Generator branch (reference lines 221-320), used as a GAN (``is_gan``) or coupled to :class:`SPADEEncoder`."""

    def __init__(self, spatial_dims: int, out_channels: int, label_nc: int, input_shape: Sequence[int],
                 num_channels: Sequence[int], z_dim: int | None = None, is_gan: bool = False,
                 spade_intermediate_channels: int = 128, norm: str | tuple = "INSTANCE",
                 act: str | tuple | None = _LEAKY02, last_act: str | tuple | None = _LEAKY02, kernel_size: int = 3,
                 upsampling_mode: str = UpsamplingModes.nearest.value):
        super().__init__()
        self.is_gan = is_gan
        self.out_channels = out_channels
        self.label_nc = label_nc
        self.num_channels = num_channels
        self.spatial_dims = spatial_dims
        self.latent_spatial_shape = _check_shape(spatial_dims, input_shape, len(num_channels))
        if self.is_gan:
            self.fc = nn.Linear(label_nc, np.prod(self.latent_spatial_shape) * num_channels[0])
        else:
            self.fc = nn.Linear(z_dim, np.prod(self.latent_spatial_shape) * num_channels[0])
        num_channels.append(self.out_channels)
        self.upsampling_mode = str(upsampling_mode)
        self.upsampling = torch.nn.Upsample(scale_factor=2, mode=upsampling_mode)
        self.blocks = torch.nn.ModuleList([
            SPADEResNetBlock(spatial_dims, ch_value, num_channels[ch_ind + 1], label_nc, spade_intermediate_channels,
                             norm, kernel_size) for ch_ind, ch_value in enumerate(num_channels[:-1])])
        self.last_conv = Convolution(spatial_dims, num_channels[-1], out_channels, padding=(kernel_size - 1) // 2,
                                     kernel_size=kernel_size, conv_only=False, act=last_act)

    def _upsample(self, x: CL) -> CL:
        mode = self.upsampling_mode
        if mode == "nearest":
            return ops.upsample_nearest2x(x)
        if mode in ("bilinear", "bicubic"):
            if self.spatial_dims != 2:
                raise NotImplementedError(f"{mode} upsampling needs 4-D input, got {self.spatial_dims + 2}-D "
                                          "(torch.nn.Upsample has no 3-D form of it either)")
            return ops.upsample2x_interp(x, mode)
        raise NotImplementedError(f"upsampling_mode {mode!r} is not supported: nearest, bilinear or bicubic")

    def _packed_fc_cl(self, pitch: int) -> ops.PackedLinear:
        """``fc`` with its output rows moved from channels-first (c * S + s) to channels-last (s * pitch + c) order,
        so the GEMM writes the [N, *latent, C0] activation; rows (and bias) of pad channels are zero."""
        C0, S = self.num_channels[0], int(np.prod(self.latent_spatial_shape))

        def build():
            w, b = ops._src_f32(self.fc.weight), ops._src_f32(self.fc.bias)
            wp = torch.zeros((S, pitch, w.shape[1]), dtype=torch.float32, device=w.device)
            wp[:, :C0] = w.view(C0, S, w.shape[1]).transpose(0, 1)
            bp = torch.zeros((S, pitch), dtype=torch.float32, device=w.device)
            bp[:, :C0] = b.view(C0, S).t()
            return ops.PackedLinear(wp.view(S * pitch, w.shape[1]), bp.view(-1))
        return self._cached(("fc_cl", pitch), (self.fc.weight, self.fc.bias), build)

    def _from_z(self, z: torch.Tensor) -> CL:
        N, C0 = z.shape[0], self.num_channels[0]
        if z.dim() != 2 or z.shape[1] != self.fc.in_features:
            raise RuntimeError(f"z of shape {tuple(z.shape)} does not match fc's {self.fc.in_features} inputs")
        zc = ops.to_cl(z.reshape(N, -1, 1, 1))
        pitch = ops.round_up(C0, 8)
        y = ops.linear(zc, self._packed_fc_cl(pitch))
        lat = list(self.latent_spatial_shape)
        dims = (1, *lat) if self.spatial_dims == 2 else tuple(lat)
        return CL(y.t.reshape(N, *dims, pitch), C0, self.spatial_dims)

    def _from_seg_gan(self, seg: SegPyramid) -> CL:
        """The reference's GAN input: ``fc`` applied along the last spatial axis of the segmentation map resized to
        the latent shape, ``[N, label_nc, *latent[:-1], F]`` read as channels x spatial (F = fc.out_features)."""
        lib = _lib.require_device()
        lat = list(self.latent_spatial_shape)
        L = seg.base.C
        if lat[-1] != self.fc.in_features:
            raise RuntimeError(f"mat1 and mat2 shapes cannot be multiplied: the decoder's fc takes "
                               f"{self.fc.in_features} features along the last axis of the resized map, which has "
                               f"{lat[-1]}")
        if L != self.num_channels[0]:
            raise RuntimeError(f"the GAN input has {L} channels (label_nc) but the first block expects "
                               f"{self.num_channels[0]}")
        s = ops.from_cl(seg.at(lat))                                      # [N, L, *lat] fp32
        N, w, F_ = s.shape[0], lat[-1], self.fc.out_features
        M = s.numel() // w
        dev = s.device
        rows = torch.empty((M, ops.round_up(w, 8)), dtype=ops.H16, device=dev)
        pl = self._cached(("fc",), (self.fc.weight, self.fc.bias), lambda: ops.PackedLinear(self.fc.weight,
                                                                                            self.fc.bias))
        for r0 in range(0, M, 65535):                                    # rows of w values -> h16 GEMM rows
            r = min(65535, M - r0)
            ops.check(lib.b200_nchw_to_nhwc(s.data_ptr() + r0 * w * 4, r, w, 1, rows.data_ptr() + r0 * rows.shape[1] * 2,
                                            rows.shape[1], ops._stream()), "b200_nchw_to_nhwc")
        yp = ops.linear(ops.as_rows(rows, w), pl, out_f32=True).reshape(M, -1)
        y = yp
        if yp.shape[1] != F_:                                             # drop the fp32 row padding
            y = torch.empty((M, F_), dtype=torch.float32, device=dev)
            for r0 in range(0, M, 65535):
                r = min(65535, M - r0)
                ops.check(lib.b200_nhwc_to_nchw(yp.data_ptr() + r0 * yp.shape[1] * 4, _lib.DT_F32, r, F_, 1,
                                                yp.shape[1], y.data_ptr() + r0 * F_ * 4, ops._stream()),
                          "b200_nhwc_to_nchw")
        dims = (1, *lat[:-1], F_) if self.spatial_dims == 2 else (*lat[:-1], F_)
        out = ops.new_cl(N, dims, L, dev, self.spatial_dims)
        sp = int(np.prod(dims))
        ops.check(lib.b200_nchw_to_nhwc(y.data_ptr(), N, L, sp, out.t.data_ptr(), out.pitch, ops._stream()),
                  "b200_nchw_to_nhwc")
        return out

    def _decode_cl(self, seg: torch.Tensor, z: torch.Tensor | None) -> CL:
        pyr = SegPyramid(seg)
        if self.is_gan:
            x = self._from_seg_gan(pyr)
        else:
            if z is None:
                raise AttributeError(f"'{type(self).__name__}' object has no attribute 'opt' (the reference draws z "
                                     "from self.opt.z_dim, which it never sets: pass z)")
            x = self._from_z(z)
        for res_block in self.blocks:
            x = self._upsample(res_block(x, pyr))
        return self.last_conv(x)

    @on_input_device
    def forward(self, seg: torch.Tensor, z: torch.Tensor | None = None) -> torch.Tensor:
        require_cuda(seg, self)
        return ops.from_cl(self._decode_cl(seg, z))


class SPADENet(nn.Module):
    """SPADE network (reference lines 323-420): ``forward(seg, x)`` returns ``(image, kld)`` in VAE mode and
    ``(image,)`` in GAN mode; ``encode(x)`` draws z; ``decode(seg, z)`` generates."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int, label_nc: int,
                 input_shape: Sequence[int], num_channels: Sequence[int], z_dim: int | None = None,
                 is_vae: bool = True, spade_intermediate_channels: int = 128, norm: str | tuple = "INSTANCE",
                 act: str | tuple | None = _LEAKY02, last_act: str | tuple | None = _LEAKY02, kernel_size: int = 3,
                 upsampling_mode: str = UpsamplingModes.nearest.value):
        super().__init__()
        self.is_vae = is_vae
        # the reference builds this ValueError without raising it: z_dim=None fails later, in nn.Linear
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.num_channels = num_channels
        self.label_nc = label_nc
        self.input_shape = input_shape
        self.kld_loss = KLDLoss()
        if self.is_vae:
            self.encoder = SPADEEncoder(spatial_dims, in_channels, z_dim, num_channels, input_shape, kernel_size,
                                        norm, act)
        decoder_channels = num_channels
        decoder_channels.reverse()
        self.decoder = SPADEDecoder(spatial_dims, out_channels, label_nc, input_shape, decoder_channels, z_dim,
                                    not is_vae, spade_intermediate_channels, norm, act, last_act, kernel_size,
                                    upsampling_mode)

    @on_input_device
    def forward(self, seg: torch.Tensor, x: torch.Tensor | None = None):
        require_cuda(seg, self)
        if self.is_vae:
            mu, logvar = self.encoder(x)
            z, kld = ops.vae_reparam_kld(mu, logvar, torch.randn_like(mu))
            return self.decoder(seg, z), kld
        return (self.decoder(seg, None),)

    def encode(self, x: torch.Tensor) -> torch.Tensor:
        return self.encoder.encode(x)

    def decode(self, seg: torch.Tensor, z: torch.Tensor | None = None) -> torch.Tensor:
        return self.decoder(seg, z)

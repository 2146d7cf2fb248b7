"""AutoencoderKL on the H100 kernels — classes, arguments and state_dict keys of
generative/networks/nets/autoencoderkl.py (reference lines cited per class)."""
from __future__ import annotations

import math
from collections.abc import Sequence

import torch
import torch.nn as nn

from ... import ops
from ...ops import ACT_NONE, ACT_SILU, CL
from ..blocks.spade_norm import SPADE
from .._holders import Convolution, on_input_device, require_cuda
from .diffusion_model_unet import _sdp, ensure_tuple_rep

__all__ = ["AutoencoderKL"]


class Upsample(nn.Module):
    """autoencoderkl.py:41-93: ConvTranspose k3 s2 p1 (output_padding 1) or nearest x2 + k3 conv."""

    def __init__(self, spatial_dims: int, in_channels: int, use_convtranspose: bool) -> None:
        super().__init__()
        if use_convtranspose:
            self.conv = Convolution(spatial_dims, in_channels, in_channels, strides=2, kernel_size=3, padding=1,
                                    is_transposed=True)
        else:
            self.conv = Convolution(spatial_dims, in_channels, in_channels, strides=1, kernel_size=3, padding=1)
        self.use_convtranspose = use_convtranspose

    def forward(self, x: CL) -> CL:
        if self.use_convtranspose:
            return self.conv(x)
        return self.conv.forward_upsampled(x)


class Downsample(nn.Module):
    """autoencoderkl.py:96-122: F.pad (0, 1) per dim, then k3 s2 p0 — the asymmetric pad is folded into the TMA
    coordinates (out-of-range rows are zero-filled), no padded copy is made."""

    def __init__(self, spatial_dims: int, in_channels: int) -> None:
        super().__init__()
        self.pad = (0, 1) * spatial_dims
        self.spatial_dims = spatial_dims
        self.conv = Convolution(spatial_dims, in_channels, in_channels, strides=2, kernel_size=3, padding=0)

    def forward(self, x: CL) -> CL:
        pc = self.conv.packed([x.C], padding=[(0, 1)] * self.spatial_dims)
        return ops.conv(x, pc)


class ResBlock(nn.Module):
    """autoencoderkl.py:125-193 (GroupNorm+SiLU+conv twice, 1x1 nin_shortcut when channels change)."""

    def __init__(self, spatial_dims: int, in_channels: int, norm_num_groups: int, norm_eps: float,
                 out_channels: int, label_nc: int | None = None, spade_intermediate_channels: int = 128) -> None:
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = in_channels if out_channels is None else out_channels
        self.spade = label_nc is not None

        def make_norm(ch):
            if self.spade:     # SPADEResBlock (spade_autoencoderkl.py:72-107): GroupNorm without affine, default eps
                return SPADE(label_nc=label_nc, norm_nc=ch, norm="GROUP",
                             norm_params={"num_groups": norm_num_groups, "affine": False},
                             hidden_channels=spade_intermediate_channels, kernel_size=3, spatial_dims=spatial_dims)
            return nn.GroupNorm(num_groups=norm_num_groups, num_channels=ch, eps=norm_eps, affine=True)

        self.norm1 = make_norm(in_channels)
        self.conv1 = Convolution(spatial_dims, self.in_channels, self.out_channels, strides=1, kernel_size=3,
                                 padding=1)
        self.norm2 = make_norm(out_channels)
        self.conv2 = Convolution(spatial_dims, self.out_channels, self.out_channels, strides=1, kernel_size=3,
                                 padding=1)
        if self.in_channels != self.out_channels:
            self.nin_shortcut = Convolution(spatial_dims, self.in_channels, self.out_channels, strides=1,
                                            kernel_size=1, padding=0)
        else:
            self.nin_shortcut = nn.Identity()

    def _norm(self, norm, x, seg):
        if self.spade:
            if seg is None:
                raise ValueError("a SPADE ResBlock needs the segmentation map (seg)")
            return norm(x, seg, act=ACT_SILU)
        return ops.groupnorm(x, norm.num_groups, norm.eps, norm.weight, norm.bias, act=ACT_SILU)

    def forward(self, x: CL, seg=None) -> CL:
        h = self.conv1(self._norm(self.norm1, x, seg))
        h = self._norm(self.norm2, h, seg)
        skip = x if isinstance(self.nin_shortcut, nn.Identity) else self.nin_shortcut(x)
        return self.conv2(h, residual=skip)


class AttentionBlock(nn.Module):
    """autoencoderkl.py:196-312 (single head unless num_head_channels is given; proj_attn unused in forward)."""

    def __init__(self, spatial_dims: int, num_channels: int, num_head_channels: int | None = None,
                 norm_num_groups: int = 32, norm_eps: float = 1e-6, use_flash_attention: bool = False) -> None:
        super().__init__()
        self.use_flash_attention = use_flash_attention
        self.spatial_dims, self.num_channels = spatial_dims, num_channels
        self.num_heads = num_channels // num_head_channels if num_head_channels is not None else 1
        self.scale = 1 / math.sqrt(num_channels / self.num_heads)
        self.norm = nn.GroupNorm(num_groups=norm_num_groups, num_channels=num_channels, eps=norm_eps, affine=True)
        self.to_q = nn.Linear(num_channels, num_channels)
        self.to_k = nn.Linear(num_channels, num_channels)
        self.to_v = nn.Linear(num_channels, num_channels)
        self.proj_attn = nn.Linear(num_channels, num_channels)

    def forward(self, x: CL) -> CL:
        h = ops.groupnorm(x, self.norm.num_groups, self.norm.eps, self.norm.weight, self.norm.bias)
        return _sdp(self, h, h, self.num_heads, self.num_channels // self.num_heads, self.scale, x, True)


def _run_blocks(blocks: nn.ModuleList, x: CL, out_f32_last: bool, seg=None):
    n = len(blocks)
    for i, block in enumerate(blocks):
        if isinstance(block, nn.GroupNorm):      # bare GroupNorm before the last conv: no activation
            x = ops.groupnorm(x, block.num_groups, block.eps, block.weight, block.bias, act=ACT_NONE)
        elif isinstance(block, ResBlock) and block.spade:
            x = block(x, seg)
        elif i == n - 1 and out_f32_last:
            x = block(x, out_f32=True)
        else:
            x = block(x)
    return x


class Encoder(nn.Module):
    """autoencoderkl.py:315-452."""

    def __init__(self, spatial_dims: int, in_channels: int, num_channels: Sequence[int], out_channels: int,
                 num_res_blocks: Sequence[int], norm_num_groups: int, norm_eps: float,
                 attention_levels: Sequence[bool], with_nonlocal_attn: bool = True,
                 use_flash_attention: bool = False) -> None:
        super().__init__()
        self.spatial_dims, self.in_channels, self.num_channels = spatial_dims, in_channels, num_channels
        self.out_channels, self.num_res_blocks = out_channels, num_res_blocks
        self.norm_num_groups, self.norm_eps, self.attention_levels = norm_num_groups, norm_eps, attention_levels
        blocks: list[nn.Module] = [Convolution(spatial_dims, in_channels, num_channels[0], strides=1, kernel_size=3,
                                               padding=1)]
        output_channel = num_channels[0]
        for i in range(len(num_channels)):
            input_channel = output_channel
            output_channel = num_channels[i]
            is_final_block = i == len(num_channels) - 1
            for _ in range(self.num_res_blocks[i]):
                blocks.append(ResBlock(spatial_dims, input_channel, norm_num_groups, norm_eps, output_channel))
                input_channel = output_channel
                if attention_levels[i]:
                    blocks.append(AttentionBlock(spatial_dims, input_channel, norm_num_groups=norm_num_groups,
                                                 norm_eps=norm_eps, use_flash_attention=use_flash_attention))
            if not is_final_block:
                blocks.append(Downsample(spatial_dims, input_channel))
        if with_nonlocal_attn is True:
            blocks.append(ResBlock(spatial_dims, num_channels[-1], norm_num_groups, norm_eps, num_channels[-1]))
            blocks.append(AttentionBlock(spatial_dims, num_channels[-1], norm_num_groups=norm_num_groups,
                                         norm_eps=norm_eps, use_flash_attention=use_flash_attention))
            blocks.append(ResBlock(spatial_dims, num_channels[-1], norm_num_groups, norm_eps, num_channels[-1]))
        blocks.append(nn.GroupNorm(num_groups=norm_num_groups, num_channels=num_channels[-1], eps=norm_eps,
                                   affine=True))
        blocks.append(Convolution(spatial_dims, num_channels[-1], out_channels, strides=1, kernel_size=3, padding=1))
        self.blocks = nn.ModuleList(blocks)

    def forward(self, x: CL) -> CL:
        return _run_blocks(self.blocks, x, out_f32_last=False)


class Decoder(nn.Module):
    """autoencoderkl.py:455-597."""

    def __init__(self, spatial_dims: int, num_channels: Sequence[int], in_channels: int, out_channels: int,
                 num_res_blocks: Sequence[int], norm_num_groups: int, norm_eps: float,
                 attention_levels: Sequence[bool], with_nonlocal_attn: bool = True,
                 use_flash_attention: bool = False, use_convtranspose: bool = False, label_nc: int | None = None,
                 spade_intermediate_channels: int = 128) -> None:
        super().__init__()
        spade = dict(label_nc=label_nc, spade_intermediate_channels=spade_intermediate_channels)
        self.label_nc = label_nc
        self.spatial_dims, self.num_channels, self.in_channels = spatial_dims, num_channels, in_channels
        self.out_channels, self.num_res_blocks = out_channels, num_res_blocks
        self.norm_num_groups, self.norm_eps, self.attention_levels = norm_num_groups, norm_eps, attention_levels
        rev_ch = list(reversed(num_channels))
        blocks: list[nn.Module] = [Convolution(spatial_dims, in_channels, rev_ch[0], strides=1, kernel_size=3,
                                               padding=1)]
        if with_nonlocal_attn is True:
            blocks.append(ResBlock(spatial_dims, rev_ch[0], norm_num_groups, norm_eps, rev_ch[0], **spade))
            blocks.append(AttentionBlock(spatial_dims, rev_ch[0], norm_num_groups=norm_num_groups, norm_eps=norm_eps,
                                         use_flash_attention=use_flash_attention))
            blocks.append(ResBlock(spatial_dims, rev_ch[0], norm_num_groups, norm_eps, rev_ch[0], **spade))
        rev_attn = list(reversed(attention_levels))
        rev_res = list(reversed(num_res_blocks))
        block_out_ch = rev_ch[0]
        for i in range(len(rev_ch)):
            block_in_ch = block_out_ch
            block_out_ch = rev_ch[i]
            is_final_block = i == len(num_channels) - 1
            for _ in range(rev_res[i]):
                blocks.append(ResBlock(spatial_dims, block_in_ch, norm_num_groups, norm_eps, block_out_ch, **spade))
                block_in_ch = block_out_ch
                if rev_attn[i]:
                    blocks.append(AttentionBlock(spatial_dims, block_in_ch, norm_num_groups=norm_num_groups,
                                                 norm_eps=norm_eps, use_flash_attention=use_flash_attention))
            if not is_final_block:
                blocks.append(Upsample(spatial_dims, block_in_ch, use_convtranspose))
        blocks.append(nn.GroupNorm(num_groups=norm_num_groups, num_channels=block_in_ch, eps=norm_eps, affine=True))
        blocks.append(Convolution(spatial_dims, block_in_ch, out_channels, strides=1, kernel_size=3, padding=1))
        self.blocks = nn.ModuleList(blocks)

    def forward(self, x: CL, seg=None):
        return _run_blocks(self.blocks, x, out_f32_last=True, seg=seg)


class AutoencoderKL(nn.Module):
    """autoencoderkl.py:600-799."""

    def __init__(self, spatial_dims: int, in_channels: int = 1, out_channels: int = 1,
                 num_res_blocks: Sequence[int] | int = (2, 2, 2, 2), num_channels: Sequence[int] = (32, 64, 64, 64),
                 attention_levels: Sequence[bool] = (False, False, True, True), latent_channels: int = 3,
                 norm_num_groups: int = 32, norm_eps: float = 1e-6, with_encoder_nonlocal_attn: bool = True,
                 with_decoder_nonlocal_attn: bool = True, use_flash_attention: bool = False,
                 use_checkpointing: bool = False, use_convtranspose: bool = False, _label_nc: int | None = None,
                 _spade_intermediate_channels: int = 128) -> None:
        super().__init__()
        if any((out_channel % norm_num_groups) != 0 for out_channel in num_channels):
            raise ValueError("AutoencoderKL expects all num_channels being multiple of norm_num_groups")
        if len(num_channels) != len(attention_levels):
            raise ValueError("AutoencoderKL expects num_channels being same size of attention_levels")
        if isinstance(num_res_blocks, int):
            num_res_blocks = ensure_tuple_rep(num_res_blocks, len(num_channels))
        if len(num_res_blocks) != len(num_channels):
            raise ValueError("`num_res_blocks` should be a single integer or a tuple of integers with the same "
                             "length as `num_channels`.")
        self.spatial_dims = spatial_dims
        self.encoder = Encoder(spatial_dims, in_channels, num_channels, latent_channels, num_res_blocks,
                               norm_num_groups, norm_eps, attention_levels, with_encoder_nonlocal_attn,
                               use_flash_attention)
        self.decoder = Decoder(spatial_dims, num_channels, latent_channels, out_channels, num_res_blocks,
                               norm_num_groups, norm_eps, attention_levels, with_decoder_nonlocal_attn,
                               use_flash_attention, use_convtranspose, _label_nc, _spade_intermediate_channels)
        self.quant_conv_mu = Convolution(spatial_dims, latent_channels, latent_channels, strides=1, kernel_size=1,
                                         padding=0)
        self.quant_conv_log_sigma = Convolution(spatial_dims, latent_channels, latent_channels, strides=1,
                                                kernel_size=1, padding=0)
        self.post_quant_conv = Convolution(spatial_dims, latent_channels, latent_channels, strides=1, kernel_size=1,
                                           padding=0)
        self.latent_channels = latent_channels
        self.out_channels = out_channels
        self.use_checkpointing = use_checkpointing     # activation checkpointing is a training feature: ignored

    @on_input_device
    @torch.no_grad()
    def encode(self, x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        require_cuda(x, self)
        h = self.encoder(ops.to_cl(x))
        mu = ops.from_cl_f32(self.quant_conv_mu(h, out_f32=True), self.latent_channels, self.spatial_dims)
        log_var = ops.from_cl_f32(self.quant_conv_log_sigma(h, out_f32=True), self.latent_channels,
                                  self.spatial_dims)
        return mu, ops.exp_half_clamped(log_var, -30.0, 20.0)

    def sampling(self, z_mu: torch.Tensor, z_sigma: torch.Tensor) -> torch.Tensor:
        eps = torch.randn_like(z_sigma)       # RNG stays with PyTorch so seeds behave like the reference's
        return ops.fma_f32(z_mu, eps, z_sigma)

    @on_input_device
    def reconstruct(self, x: torch.Tensor) -> torch.Tensor:
        z_mu, _ = self.encode(x)
        return self.decode(z_mu)

    @on_input_device
    @torch.no_grad()
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        return self._decode(z, None)

    def _decode(self, z: torch.Tensor, seg) -> torch.Tensor:
        require_cuda(z, self)
        y = self.decoder(self.post_quant_conv(ops.to_cl(z)), seg)
        out = ops.from_cl_f32(y, self.out_channels, self.spatial_dims)
        return out if z.dtype == torch.float32 else out.to(z.dtype)

    @on_input_device
    def forward(self, x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        z_mu, z_sigma = self.encode(x)
        z = self.sampling(z_mu, z_sigma)
        return self.decode(z), z_mu, z_sigma

    @on_input_device
    def encode_stage_2_inputs(self, x: torch.Tensor) -> torch.Tensor:
        z_mu, z_sigma = self.encode(x)
        return self.sampling(z_mu, z_sigma)

    @on_input_device
    def decode_stage_2_outputs(self, z: torch.Tensor) -> torch.Tensor:
        return self.decode(z)

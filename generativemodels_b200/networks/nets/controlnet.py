"""ControlNet on the H100 kernels — classes, arguments and state_dict keys of
generative/networks/nets/controlnet.py (reference lines cited per class)."""
from __future__ import annotations

from collections.abc import Sequence

import torch
import torch.nn as nn

from ... import ops
from ...ops import ACT_SILU, CL
from .._holders import Convolution, on_input_device, require_cuda
from .diffusion_model_unet import (_context_cl, ensure_tuple_rep, get_down_block, get_mid_block, project_time_embedding,
                                   time_embedding,
                                   zero_module)

__all__ = ["ControlNet"]


class ControlNetConditioningEmbedding(nn.Module):
    """controlnet.py:45-116: conv_in, SiLU, [conv s1, SiLU, conv s2, SiLU]*, zero-init conv_out.  The SiLUs run in
    the conv epilogues; ``forward`` takes the tensor the embedding is added to (``h += embedding``, 405-407) as the
    residual of the last conv."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int,
                 num_channels: Sequence[int] = (16, 32, 96, 256)):
        super().__init__()
        self.conv_in = Convolution(spatial_dims, in_channels, num_channels[0], strides=1, kernel_size=3, padding=1)
        self.blocks = nn.ModuleList([])
        for i in range(len(num_channels) - 1):
            self.blocks.append(Convolution(spatial_dims, num_channels[i], num_channels[i], strides=1, kernel_size=3,
                                           padding=1))
            self.blocks.append(Convolution(spatial_dims, num_channels[i], num_channels[i + 1], strides=2,
                                           kernel_size=3, padding=1))
        self.conv_out = zero_module(Convolution(spatial_dims, num_channels[-1], out_channels, strides=1,
                                                kernel_size=3, padding=1))

    def forward(self, conditioning: CL, add_to: CL | None = None) -> CL:
        e = self.conv_in(conditioning, act1=ACT_SILU)
        for block in self.blocks:
            e = block(e, act1=ACT_SILU)
        return self.conv_out(e, residual=add_to)


class _BareConv(nn.Module):
    """``controlnet_down_blocks[0]`` is the bare nn.Conv (controlnet.py:283-284), i.e. keys ``...0.weight``."""


class ControlNet(nn.Module):
    """controlnet.py:119-436."""

    def __init__(self, spatial_dims: int, in_channels: int, num_res_blocks: Sequence[int] | int = (2, 2, 2, 2),
                 num_channels: Sequence[int] = (32, 64, 64, 64),
                 attention_levels: Sequence[bool] = (False, False, True, True), norm_num_groups: int = 32,
                 norm_eps: float = 1e-6, resblock_updown: bool = False, num_head_channels: int | Sequence[int] = 8,
                 with_conditioning: bool = False, transformer_num_layers: int = 1,
                 cross_attention_dim: int | None = None, num_class_embeds: int | None = None,
                 upcast_attention: bool = False, use_flash_attention: bool = False,
                 conditioning_embedding_in_channels: int = 1,
                 conditioning_embedding_num_channels: Sequence[int] | None = (16, 32, 96, 256)) -> None:
        super().__init__()
        if with_conditioning is True and cross_attention_dim is None:
            raise ValueError("ControlNet expects dimension of the cross-attention conditioning (cross_attention_dim) "
                             "when using with_conditioning.")
        if cross_attention_dim is not None and with_conditioning is False:
            raise ValueError("ControlNet expects with_conditioning=True when specifying the cross_attention_dim.")
        if any((out_channel % norm_num_groups) != 0 for out_channel in num_channels):
            raise ValueError("ControlNet expects all num_channels being multiple of norm_num_groups")
        if len(num_channels) != len(attention_levels):
            raise ValueError("ControlNet expects num_channels being same size of attention_levels")
        if isinstance(num_head_channels, int):
            num_head_channels = ensure_tuple_rep(num_head_channels, len(attention_levels))
        if len(num_head_channels) != len(attention_levels):
            raise ValueError("num_head_channels should have the same length as attention_levels. For the i levels "
                             "without attention, i.e. `attention_level[i]=False`, the num_head_channels[i] will be "
                             "ignored.")
        if isinstance(num_res_blocks, int):
            num_res_blocks = ensure_tuple_rep(num_res_blocks, len(num_channels))
        if len(num_res_blocks) != len(num_channels):
            raise ValueError("`num_res_blocks` should be a single integer or a tuple of integers with the same "
                             "length as `num_channels`.")
        self.spatial_dims = spatial_dims
        self.in_channels = in_channels
        self.block_out_channels = num_channels
        self.num_res_blocks = num_res_blocks
        self.attention_levels = attention_levels
        self.num_head_channels = num_head_channels
        self.with_conditioning = with_conditioning

        self.conv_in = Convolution(spatial_dims, in_channels, num_channels[0], strides=1, kernel_size=3, padding=1)
        time_embed_dim = num_channels[0] * 4
        self.time_embed = nn.Sequential(nn.Linear(num_channels[0], time_embed_dim), nn.SiLU(),
                                        nn.Linear(time_embed_dim, time_embed_dim))
        self.num_class_embeds = num_class_embeds
        if num_class_embeds is not None:
            self.class_embedding = nn.Embedding(num_class_embeds, time_embed_dim)
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(
            spatial_dims, conditioning_embedding_in_channels, num_channels[0], conditioning_embedding_num_channels)

        def zero_conv(ch):
            return zero_module(Convolution(spatial_dims, ch, ch, strides=1, kernel_size=1, padding=0))

        self.down_blocks = nn.ModuleList([])
        self.controlnet_down_blocks = nn.ModuleList([])
        output_channel = num_channels[0]
        self.controlnet_down_blocks.append(zero_conv(output_channel).conv)      # bare conv: keys "...0.weight"
        for i in range(len(num_channels)):
            input_channel = output_channel
            output_channel = num_channels[i]
            is_final_block = i == len(num_channels) - 1
            self.down_blocks.append(get_down_block(
                spatial_dims, input_channel, output_channel, time_embed_dim, num_res_blocks[i], norm_num_groups,
                norm_eps, not is_final_block, resblock_updown, attention_levels[i] and not with_conditioning,
                attention_levels[i] and with_conditioning, num_head_channels[i], transformer_num_layers,
                cross_attention_dim, upcast_attention, use_flash_attention))
            for _ in range(num_res_blocks[i]):
                self.controlnet_down_blocks.append(zero_conv(output_channel))
            if not is_final_block:
                self.controlnet_down_blocks.append(zero_conv(output_channel))
        self.middle_block = get_mid_block(spatial_dims, num_channels[-1], time_embed_dim, norm_num_groups, norm_eps,
                                          with_conditioning, num_head_channels[-1], transformer_num_layers,
                                          cross_attention_dim, upcast_attention, use_flash_attention)
        self.controlnet_mid_block = zero_conv(output_channel)

    def _zero_conv(self, block: nn.Module, x: CL, scale: float) -> CL:
        if isinstance(block, Convolution):
            return block(x, scale=scale)
        cache = self.__dict__.setdefault("_bare_cache", {})
        key = (block.weight.data_ptr(), block.weight._version)
        if cache.get("key") != key:
            cache["key"], cache["pc"] = key, ops.PackedConv(block.weight, block.bias, 1, 0)
        return ops.conv(x, cache["pc"], scale=scale)

    @on_input_device
    @torch.no_grad()
    def forward(self, x: torch.Tensor, timesteps: torch.Tensor, controlnet_cond: torch.Tensor,
                conditioning_scale: float = 1.0, context: torch.Tensor | None = None,
                class_labels: torch.Tensor | None = None, _internal: bool = False):
        """-> (down residuals, mid residual) as NC[D]HW tensors (controlnet.py:367-436); with ``_internal`` the
        inferers get the channels-last handles and skip two layout passes per residual."""
        require_cuda(x, self)
        emb = project_time_embedding(self, time_embedding(self, x, timesteps, class_labels))
        if context is not None and self.with_conditioning is False:
            raise ValueError("model should have with_conditioning = True if context is provided")
        ctx = _context_cl(context) if context is not None else None
        h = self.conv_in(ops.to_cl(x))
        h = self.controlnet_cond_embedding(ops.to_cl(controlnet_cond.to(x.device)), add_to=h)
        res: list[CL] = [h]
        for block in self.down_blocks:
            h, samples = block(hidden_states=h, temb=emb, context=ctx)
            res.extend(samples)
        h = self.middle_block(hidden_states=h, temb=emb, context=ctx)
        s = float(conditioning_scale)
        down = [self._zero_conv(b, r, s) for r, b in zip(res, self.controlnet_down_blocks)]
        mid = self._zero_conv(self.controlnet_mid_block, h, s)
        if _internal:
            return down, mid
        return [ops.from_cl(d, x.dtype) for d in down], ops.from_cl(mid, x.dtype)

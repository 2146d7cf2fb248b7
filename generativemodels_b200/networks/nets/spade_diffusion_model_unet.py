"""SPADEDiffusionModelUNet — ``generative/networks/nets/spade_diffusion_model_unet.py:612-912`` on the H100 kernels.

The reference class is DiffusionModelUNet whose up path uses ResnetBlocks with SPADE norms (semantic conditioning
by a segmentation map, Park et al. 2019); encoder, middle block, attention and heads are identical and so are the
state_dict keys (``up_blocks.i.resnets.j.norm{1,2}.{param_free_norm.N,mlp_shared.conv,mlp_gamma.conv,mlp_beta.conv}``).
It is reached from the same inferers through ``seg=`` (inferer.py:121-125, 445-446).
"""
from __future__ import annotations

from collections.abc import Sequence

import torch

from ..blocks.spade_norm import SegPyramid
from .diffusion_model_unet import DiffusionModelUNet, ResnetBlock

__all__ = ["SPADEDiffusionModelUNet", "SPADEResnetBlock"]


class SPADEResnetBlock(ResnetBlock):
    """spade_diffusion_model_unet.py:72-200 (ResnetBlock with SPADE norms; ``forward(x, emb, seg)``)."""

    def __init__(self, spatial_dims: int, in_channels: int, temb_channels: int, label_nc: int,
                 out_channels: int | None = None, up: bool = False, down: bool = False, norm_num_groups: int = 32,
                 norm_eps: float = 1e-6, spade_intermediate_channels: int = 128) -> None:
        super().__init__(spatial_dims, in_channels, temb_channels, out_channels, up, down, norm_num_groups, norm_eps,
                         label_nc=label_nc, spade_intermediate_channels=spade_intermediate_channels)


class SPADEDiffusionModelUNet(DiffusionModelUNet):
    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int, label_nc: int,
                 num_res_blocks: Sequence[int] | int = (2, 2, 2, 2), num_channels: Sequence[int] = (32, 64, 64, 64),
                 attention_levels: Sequence[bool] = (False, False, True, True), norm_num_groups: int = 32,
                 norm_eps: float = 1e-6, resblock_updown: bool = False, num_head_channels: int | Sequence[int] = 8,
                 with_conditioning: bool = False, transformer_num_layers: int = 1,
                 cross_attention_dim: int | None = None, num_class_embeds: int | None = None,
                 upcast_attention: bool = False, use_flash_attention: bool = False,
                 spade_intermediate_channels: int = 128) -> None:
        try:
            super().__init__(spatial_dims, in_channels, out_channels, num_res_blocks, num_channels, attention_levels,
                             norm_num_groups, norm_eps, resblock_updown, num_head_channels, with_conditioning,
                             transformer_num_layers, cross_attention_dim, num_class_embeds, upcast_attention,
                             use_flash_attention, 0.0, _label_nc=label_nc,
                             _spade_intermediate_channels=spade_intermediate_channels)
        except ValueError as e:      # the reference raises the same conditions under its own class name
            raise ValueError(str(e).replace("DiffusionModelUNet", "SPADEDiffusionModelUNet", 1)) from None
        self.label_nc = label_nc

    @torch.no_grad()
    def forward(self, x: torch.Tensor, timesteps: torch.Tensor, seg: torch.Tensor,
                context: torch.Tensor | None = None, class_labels: torch.Tensor | None = None,
                down_block_additional_residuals: tuple[torch.Tensor] | None = None,
                mid_block_additional_residual: torch.Tensor | None = None) -> torch.Tensor:
        """spade_diffusion_model_unet.py:836-912 (``seg``: B x label_nc x spatial, any resolution)."""
        return self._forward(x, timesteps, context, class_labels, down_block_additional_residuals,
                             mid_block_additional_residual, SegPyramid(seg))

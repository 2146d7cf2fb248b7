"""SPADEAutoencoderKL — ``generative/networks/nets/spade_autoencoderkl.py:292-484`` on the H100 kernels: AutoencoderKL
whose decoder ResBlocks use SPADE norms (GroupNorm without affine at PyTorch's default eps, modulated by the
segmentation map); the encoder is the plain one.  Same state_dict keys, ``decode(z, seg)`` / ``forward(x, seg)``."""
from __future__ import annotations

from collections.abc import Sequence

import torch

from ..blocks.spade_norm import SegPyramid
from .autoencoderkl import AutoencoderKL

__all__ = ["SPADEAutoencoderKL"]


class SPADEAutoencoderKL(AutoencoderKL):
    def __init__(self, spatial_dims: int, label_nc: int, in_channels: int = 1, out_channels: int = 1,
                 num_res_blocks: Sequence[int] | int = (2, 2, 2, 2), num_channels: Sequence[int] = (32, 64, 64, 64),
                 attention_levels: Sequence[bool] = (False, False, True, True), latent_channels: int = 3,
                 norm_num_groups: int = 32, norm_eps: float = 1e-6, with_encoder_nonlocal_attn: bool = True,
                 with_decoder_nonlocal_attn: bool = True, use_flash_attention: bool = False,
                 spade_intermediate_channels: int = 128) -> None:
        try:
            super().__init__(spatial_dims, in_channels, out_channels, num_res_blocks, num_channels, attention_levels,
                             latent_channels, norm_num_groups, norm_eps, with_encoder_nonlocal_attn,
                             with_decoder_nonlocal_attn, use_flash_attention, False, False, _label_nc=label_nc,
                             _spade_intermediate_channels=spade_intermediate_channels)
        except ValueError as e:
            raise ValueError(str(e).replace("AutoencoderKL", "SPADEAutoencoderKL", 1)) from None
        self.label_nc = label_nc

    def reconstruct(self, x: torch.Tensor, seg: torch.Tensor) -> torch.Tensor:
        z_mu, _ = self.encode(x)
        return self.decode(z_mu, seg)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, seg: torch.Tensor) -> torch.Tensor:
        """spade_autoencoderkl.py:457-469."""
        return self._decode(z, SegPyramid(seg))

    def forward(self, x: torch.Tensor, seg: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        z_mu, z_sigma = self.encode(x)
        z = self.sampling(z_mu, z_sigma)
        return self.decode(z, seg), z_mu, z_sigma

    def decode_stage_2_outputs(self, z: torch.Tensor, seg: torch.Tensor) -> torch.Tensor:
        return self.decode(z, seg)

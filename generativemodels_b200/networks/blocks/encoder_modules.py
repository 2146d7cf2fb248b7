"""SpatialRescaler — ``generative/networks/blocks/encoder_modules.py``, the latent-diffusion conditioning resizer, on the
H100 kernels, forward only: an optional 1x1 channel mapper, then ``n_stages`` rounds of ``F.interpolate``.

Same constructor signature, defaults, attributes (``n_stages``, ``multiplier``, ``remap_output``, ``interpolator``),
``encode`` and ``state_dict`` keys (``channel_mapper.conv.weight``, plus ``.bias`` with ``bias=True``) as the reference.
Its quirks are kept: ``AssertionError`` for an unknown ``method`` or ``n_stages < 0``; the two constructor
``ValueError``s; the message printed when remapping channels; ``size=None, multiplier=None`` is only an error once
``forward`` interpolates (F.interpolate's ``ValueError``); a mode the input's rank does not take raises
F.interpolate's ``NotImplementedError`` and a multiplier sequence of the wrong length its ``ValueError``;
``n_stages=0`` returns the input (after the mapper, if any).  Each stage's output extent is int(in * multiplier) in
double precision, F.interpolate's rule, and stages chain.

Where the work goes (b200_interpolate, ATen's coordinate rules at any size or scale):
- without a mapper every stage is one launch, planar fp32 -> planar fp32, with no layout pass;
- with a mapper the input goes channels-last (to_cl), the 1x1 convolution runs on igemm as a linear over the voxel
  rows and stores fp32 channels-last, the stages resample that fp32 tensor, and the last one writes NC[D]HW directly
  through its output strides.
Inputs and outputs are in the caller's dtype; the arithmetic is fp32.
"""
from __future__ import annotations

from collections.abc import Sequence
from functools import partial

import torch
import torch.nn as nn

from ... import ops
from ...ops import CL
from .._holders import Convolution, on_input_device, require_cuda

__all__ = ["SpatialRescaler"]

_METHODS = ["nearest", "linear", "bilinear", "trilinear", "bicubic", "area"]


def interpolate(x: torch.Tensor, size=None, scale_factor=None, mode: str = "nearest") -> torch.Tensor:
    """F.interpolate(x, size | scale_factor, mode, align_corners=False) of a planar NC[D]HW CUDA tensor, in its
    dtype (computed in fp32 by one b200_interpolate launch)."""
    require_cuda(x, interpolate)
    y = ops.interpolate(x.float(), size, scale_factor, mode)
    return y if x.dtype == torch.float32 else y.to(x.dtype)


class SpatialRescaler(nn.Module):
    """SpatialRescaler based on https://github.com/CompVis/latent-diffusion/blob/main/ldm/modules/encoders/modules.py

    Args:
        spatial_dims: number of spatial dimensions.
        n_stages: number of interpolation stages.
        size: output spatial size (int or Tuple[int] or Tuple[int, int] or Tuple[int, int, int]).
        method: algorithm used for sampling.
        multiplier: multiplier for spatial size. If `multiplier` is a sequence,
            its length has to match the number of spatial dimensions; `input.dim() - 2`.
        in_channels: number of input channels.
        out_channels: number of output channels.
        bias: whether to have a bias term.
    """

    def __init__(
        self,
        spatial_dims: int = 2,
        n_stages: int = 1,
        size: Sequence[int] | int | None = None,
        method: str = "bilinear",
        multiplier: Sequence[float] | float | None = None,
        in_channels: int = 3,
        out_channels: int = None,
        bias: bool = False,
    ):
        super().__init__()
        self.n_stages = n_stages
        assert self.n_stages >= 0
        assert method in _METHODS
        if size is not None and n_stages != 1:
            raise ValueError("when size is not None, n_stages should be 1.")
        if size is not None and multiplier is not None:
            raise ValueError("only one of size or multiplier should be defined.")
        self.multiplier = multiplier
        self.interpolator = partial(interpolate, mode=method, size=size)
        self.remap_output = out_channels is not None
        if self.remap_output:
            print(f"Spatial Rescaler mapping from {in_channels} to {out_channels} channels before resizing.")
            self.channel_mapper = Convolution(
                spatial_dims=spatial_dims,
                in_channels=in_channels,
                out_channels=out_channels,
                kernel_size=1,
                conv_only=True,
                bias=bias,
            )

    def _packed_mapper(self) -> ops.PackedLinear:
        """The 1x1 convolution's weight [out, in, 1...] as a linear over the channels, cached like the holder's own."""
        conv = self.channel_mapper.conv
        return self.channel_mapper._cached(("rows",), (conv.weight, conv.bias), lambda: ops.PackedLinear(
            conv.weight.reshape(conv.out_channels, -1), conv.bias))

    def _remap(self, x: torch.Tensor) -> tuple[torch.Tensor, int]:
        """channel_mapper(x) as fp32 channels-last [N, D, H, W, round_up(out, 4)] (a 1-D input has D == H == 1)."""
        conv = self.channel_mapper.conv
        sd = conv.weight.dim() - 2
        if x.dim() != sd + 2 or x.shape[1] != conv.in_channels:
            raise RuntimeError(f"channel_mapper ({type(conv).__name__}, {conv.in_channels} input channels) cannot "
                               f"take an input of shape {tuple(x.shape)}")
        cl = ops.to_cl(x.unsqueeze(2) if sd == 1 else x)
        return ops.linear(cl, self._packed_mapper(), out_f32=True), sd

    @on_input_device
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        require_cuda(x, self)
        mode, size = self.interpolator.keywords["mode"], self.interpolator.keywords["size"]
        with torch.no_grad():
            if not self.remap_output:
                if self.n_stages == 0:
                    return x
                y = x.float()
                for _ in range(self.n_stages):
                    y = ops.interpolate(y, size, self.multiplier, mode)
            else:
                t, sd = self._remap(x)
                cout = self.channel_mapper.conv.out_channels
                if self.n_stages == 0:
                    y = ops.from_cl_f32(t, cout, 2 if sd == 1 else sd)
                    y = y.reshape(y.shape[0], cout, -1) if sd == 1 else y
                else:
                    h = CL(t, cout, sd)
                    for i in range(self.n_stages):
                        h = ops.interpolate(h, size, self.multiplier, mode, planar_out=i == self.n_stages - 1)
                    y = h
        return y if x.dtype == torch.float32 else y.to(x.dtype)

    def encode(self, x: torch.Tensor) -> torch.Tensor:
        return self(x)

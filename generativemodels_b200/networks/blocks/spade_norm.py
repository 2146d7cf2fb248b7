"""SPADE normalisation (Park et al. 2019) with the module tree of ``generative/networks/blocks/spade_norm.py``:
``param_free_norm.N`` (GroupNorm for the diffusion / autoencoder blocks, parameter-free InstanceNorm for SPADENet),
``mlp_shared.conv`` (+LeakyReLU),
``mlp_gamma.conv`` and ``mlp_beta.conv``.

Reference forward (spade_norm.py:78-96):  ``norm(x) * (1 + gamma(seg)) + beta(seg)`` with the segmentation map resized
(nearest) to x.  ``mlp_gamma`` / ``mlp_beta`` are monai ``Convolution`` blocks built with ``act=None`` and the default
``norm="INSTANCE"``, so each is conv -> InstanceNorm (no affine) — restated in oracle/torch_oracle.py::spade_norm and
pinned against the unmodified reference there.

Here: the two convolutions run as ONE implicit GEMM with 2C output columns, their InstanceNorm statistics and the
GroupNorm statistics of x reduce to per-(sample, channel) affine tables, and a single kernel (b200_spade_apply) reads
x and gamma|beta once and writes act(modulated) — the normalised tensor, gamma and beta never exist on their own.
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn as nn

from ... import ops
from ...ops import ACT_LEAKYRELU, ACT_NONE, CL
from .._holders import Convolution, _Cached


class SegPyramid:
    """The segmentation map of one forward pass, channels-last, resized (nearest) once per spatial extent that asks."""

    def __init__(self, seg: torch.Tensor):
        self.base = ops.to_cl(seg)
        self._levels: dict = {}

    def at(self, dims: Sequence[int]) -> CL:
        d = tuple(int(v) for v in dims)
        if d not in self._levels:
            self._levels[d] = ops.resize_nearest(self.base, d)
        return self._levels[d]


class SPADE(nn.Module, _Cached):
    def __init__(self, label_nc: int, norm_nc: int, kernel_size: int = 3, spatial_dims: int = 2,
                 hidden_channels: int = 64, norm: str | tuple = "INSTANCE", norm_params: dict | None = None) -> None:
        super().__init__()
        norm_params = dict(norm_params or {})
        kind = str(norm).upper()
        if kind == "INSTANCE" and norm_params:
            raise NotImplementedError(f"SPADE with an INSTANCE base norm takes no norm_params (got {norm_params!r})")
        if kind not in ("GROUP", "INSTANCE"):
            raise NotImplementedError(f"SPADE base norm {norm!r} is not supported: GROUP (with its norm_params) or "
                                      "INSTANCE (default parameters)")
        self.param_free_norm = nn.Sequential()
        if kind == "GROUP":
            self.param_free_norm.add_module("N", nn.GroupNorm(num_channels=norm_nc, **norm_params))
        else:
            inorm = nn.InstanceNorm2d if spatial_dims == 2 else nn.InstanceNorm3d
            self.param_free_norm.add_module("N", inorm(norm_nc))
        self.mlp_shared = Convolution(spatial_dims, label_nc, hidden_channels, kernel_size=kernel_size,
                                      padding=kernel_size // 2, conv_only=False, act="LEAKYRELU")
        self.mlp_gamma = Convolution(spatial_dims, hidden_channels, norm_nc, kernel_size=kernel_size,
                                     padding=kernel_size // 2)
        self.mlp_beta = Convolution(spatial_dims, hidden_channels, norm_nc, kernel_size=kernel_size,
                                    padding=kernel_size // 2)
        self.norm_nc = norm_nc

    def _packed_gamma_beta(self) -> ops.PackedConv:
        g, b = self.mlp_gamma.conv, self.mlp_beta.conv
        return self._cached(("gamma|beta",), (g.weight, g.bias, b.weight, b.bias), lambda: ops.PackedConv(
            torch.cat([g.weight, b.weight], 0), torch.cat([g.bias, b.bias], 0), 1, self.mlp_gamma.padding))

    def forward(self, x: CL | Sequence[CL], seg: SegPyramid, act: int = ACT_NONE) -> CL:
        srcs = [x] if isinstance(x, CL) else list(x)
        a0 = srcs[0]
        if seg.base.C != self.mlp_shared.in_channels:
            # the reference fails inside F.conv with a RuntimeError (tests/test_spade_diffusion_model_unet.py:293-306)
            raise RuntimeError(f"segmentation map has {seg.base.C} channels but this SPADE block was built for "
                               f"label_nc = {self.mlp_shared.in_channels}")
        gn = self.param_free_norm.N
        if isinstance(gn, nn.GroupNorm):
            affine = ops.groupnorm_affine(srcs, gn.num_groups, gn.eps, gn.weight, gn.bias)
        else:       # InstanceNorm without affine: GroupNorm with one channel per group
            affine = ops.groupnorm_affine(srcs, sum(a.C for a in srcs), gn.eps, None, None)
        dims = (a0.H, a0.W) if a0.spatial_dims == 2 else (a0.D, a0.H, a0.W)
        actv = self.mlp_shared(seg.at(dims), act1=ACT_LEAKYRELU)
        gb = ops.conv(actv, self._packed_gamma_beta())
        # InstanceNorm{2,3}d defaults: eps 1e-5, no affine -> GroupNorm with one channel per group
        gb_affine = ops.groupnorm_affine(gb, gb.C, 1e-5, None, None)
        return ops.spade_modulate(srcs, affine, gb, gb_affine, act=act)

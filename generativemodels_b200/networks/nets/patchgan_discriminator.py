"""PatchDiscriminator / MultiScalePatchDiscriminator — ``generative/networks/nets/patchgan_discriminator.py`` on the H100
kernels, forward only: a trained critic scores samples (realism ranking, rejection sampling) and returns the
intermediate features its feature-matching distances are computed from.

Same constructor signatures and defaults, module tree (``state_dict`` keys, BatchNorm buffers included) and parameter
initialisation as the reference, so one seed gives the same parameters and reference checkpoints load with
``strict=True``.  The reference's quirks are kept: with ``pooling_method=None`` an integer ``num_layers_d`` becomes
``[num_layers_d * i for i in 1..num_d]``; ``AssertionError`` for an image too small for the deepest discriminator and
for a ``num_layers_d`` list of the wrong length; ``norm.lower()`` runs unconditionally, so a non-string ``norm`` raises
``AttributeError``; the warning about BatchNorm under DDP.

Where the work goes:
- every convolution runs on igemm.  BATCH layers use the eval-mode BatchNorm folded into the packed weights
  (b200_batchnorm_fold, cached against gamma, beta and the running statistics, so ``load_state_dict`` repacks), with
  the activation in the epilogue; INSTANCE layers run the convolution, then InstanceNorm + activation in one
  normalisation pass; dropout is the identity in eval mode;
- the intermediate features go back to NC[D]HW in the caller's dtype; the last convolution stores fp32;
- ``MultiScalePatchDiscriminator`` pools the input pyramid once per level (b200_pool_s2) and discriminator i reads
  level i, where the reference pools the input i times for discriminator i.

Mode rule (as VQVAE's): ``forward`` in train mode raises ``RuntimeError`` exactly when the result would depend on the
mode, i.e. the network has BatchNorm layers or dropout with p > 0.  An INSTANCE network without dropout runs as
constructed.
"""
from __future__ import annotations

import warnings
from typing import Sequence

import torch
import torch.nn as nn

from ... import ops
from ...ops import CL
from .._holders import Convolution, act_code, on_input_device, require_cuda

__all__ = ["MultiScalePatchDiscriminator", "PatchDiscriminator"]

_LEAKY02 = ("LEAKYRELU", {"negative_slope": 0.2})
# activations the InstanceNorm pass applies (b200_groupnorm_apply / b200_groupnorm_fused)
_INSTANCE_ACTS = (ops.ACT_NONE, ops.ACT_SILU, ops.ACT_LEAKYRELU, ops.ACT_LEAKYRELU02)
_POOLS = {"AVG": (nn.AvgPool2d, nn.AvgPool3d), "MAX": (nn.MaxPool2d, nn.MaxPool3d)}
_DROPOUTS = ("DROPOUT", "ALPHADROPOUT")


def _dropout_p(dropout) -> float:
    """monai ADN's ``dropout`` argument -> the probability of its (eval-mode identity) dropout layer."""
    if dropout is None:
        return 0.0
    if isinstance(dropout, (int, float)):
        return float(dropout)
    if isinstance(dropout, (tuple, list)) and len(dropout) == 2 and str(dropout[0]).upper() in _DROPOUTS:
        return float(dict(dropout[1]).get("p", 0.5))
    raise NotImplementedError(f"dropout {dropout!r} is not supported: a probability, or a tuple "
                              "('DROPOUT' | 'ALPHADROPOUT', {'p': ...})")


def _check_supported(spatial_dims: int, norm: str, activation, dropout) -> float:
    """Refuse what the CUDA path does not run, naming the supported set; returns the dropout probability."""
    if spatial_dims not in (2, 3):
        raise NotImplementedError(f"spatial_dims={spatial_dims} is not supported on the CUDA path (2 or 3)")
    if norm.lower() not in ("batch", "instance"):
        raise NotImplementedError(f"norm {norm!r} is not supported on the CUDA path: 'BATCH' or 'INSTANCE' (any case)")
    code = ops.ACT_NONE if activation is None else act_code(activation)
    if norm.lower() == "instance" and code not in _INSTANCE_ACTS:
        raise NotImplementedError(f"activation {activation!r} after norm='INSTANCE' is not supported: the normalisation "
                                  "pass applies 'LEAKYRELU', ('LEAKYRELU', {'negative_slope': 0.2}), 'SILU' / 'SWISH' "
                                  "or None (norm='BATCH' takes every activation)")
    return _dropout_p(dropout)


def _inference_only(module: nn.Module):
    raise RuntimeError(f"{type(module).__name__}.forward on the H100 kernels is inference-only for a network with "
                       "BatchNorm or dropout (p > 0), whose result depends on the mode; call .eval() first")


class PatchDiscriminator(nn.Sequential):
    """Patch-GAN discriminator (reference lines 158-301): ``forward(x)`` returns the output of every layer, the last
    one being the patch scores."""

    def __init__(self, spatial_dims: int, num_channels: int, in_channels: int, out_channels: int = 1,
                 num_layers_d: int = 3, kernel_size: int = 4, activation: str | tuple = _LEAKY02,
                 norm: str | tuple = "BATCH", bias: bool = False, padding: int | Sequence[int] = 1,
                 dropout: float | tuple = 0.0, last_conv_kernel_size: int | None = None) -> None:
        super().__init__()
        norm.lower()                     # the reference's unconditional norm.lower(): AttributeError for a non-string
        p = _check_supported(spatial_dims, norm, activation, dropout)
        self.num_layers_d = num_layers_d
        self.num_channels = num_channels
        if last_conv_kernel_size is None:
            last_conv_kernel_size = kernel_size
        self.add_module("initial_conv", Convolution(spatial_dims, in_channels, num_channels, strides=2,
                                                    kernel_size=kernel_size, padding=padding, bias=True,
                                                    conv_only=False, act=activation))
        input_channels = num_channels
        output_channels = num_channels * 2
        for l_ in range(self.num_layers_d):
            stride = 1 if l_ == self.num_layers_d - 1 else 2
            self.add_module("%d" % l_, Convolution(spatial_dims, input_channels, output_channels, strides=stride,
                                                   kernel_size=kernel_size, padding=padding, bias=bias,
                                                   conv_only=False, act=activation, norm=norm))
            input_channels = output_channels
            output_channels = output_channels * 2
        self.add_module("final_conv", Convolution(spatial_dims, input_channels, out_channels, strides=1,
                                                  kernel_size=last_conv_kernel_size,
                                                  padding=int((last_conv_kernel_size - 1) / 2), bias=True,
                                                  conv_only=True))
        self.apply(self.initialise_weights)
        self.mode_dependent = norm.lower() == "batch" or p > 0
        if norm.lower() == "batch" and torch.distributed.is_initialized():
            warnings.warn(
                "WARNING: Discriminator is using BatchNorm and a distributed training environment has been detected. "
                "To train with DDP, convert discriminator to SyncBatchNorm using "
                "torch.nn.SyncBatchNorm.convert_sync_batchnorm(model).)")

    def initialise_weights(self, m: nn.Module) -> None:
        """N(0, 0.02) convolution weights, N(1, 0.02) BatchNorm weights and zero BatchNorm biases (reference)."""
        classname = m.__class__.__name__
        if classname.find("Conv2d") != -1:
            nn.init.normal_(m.weight.data, 0.0, 0.02)
        elif classname.find("Conv3d") != -1:
            nn.init.normal_(m.weight.data, 0.0, 0.02)
        elif classname.find("Conv1d") != -1:
            nn.init.normal_(m.weight.data, 0.0, 0.02)
        elif classname.find("BatchNorm") != -1:
            nn.init.normal_(m.weight.data, 1.0, 0.02)
            nn.init.constant_(m.bias.data, 0)

    def forward_cl(self, h: CL, dtype: torch.dtype) -> list[torch.Tensor]:
        """The layer outputs for a channels-last input: features as NC[D]HW ``dtype`` tensors, then the fp32 scores."""
        *layers, final = self.children()
        out = []
        for layer in layers:
            h = layer(h)
            out.append(ops.from_cl(h, dtype))
        y = final(h, out_f32=True)
        out.append(ops.from_cl_f32(y, final.out_channels, h.spatial_dims).to(dtype))
        return out

    @on_input_device
    def forward(self, x: torch.Tensor) -> list[torch.Tensor]:
        require_cuda(x, self)
        if self.training and self.mode_dependent:
            _inference_only(self)
        return self.forward_cl(ops.to_cl(x), x.dtype)


class MultiScalePatchDiscriminator(nn.Sequential):
    """Multi-scale Patch-GAN discriminator (reference lines 23-155): ``num_d`` PatchDiscriminators, discriminator i
    seeing the input pooled i times (``pooling_method`` "avg" / "max") or, without pooling, the full input through
    more layers.  ``forward(i)`` returns ``(outputs, features)``."""

    def __init__(self, num_d: int, num_layers_d: int | list[int], spatial_dims: int, num_channels: int,
                 in_channels: int, pooling_method: str = None, out_channels: int = 1, kernel_size: int = 4,
                 activation: str | tuple = _LEAKY02, norm: str | tuple = "BATCH", bias: bool = False,
                 dropout: float | tuple = 0.0, minimum_size_im: int = 256, last_conv_kernel_size: int = 1) -> None:
        super().__init__()
        self.num_d = num_d
        if isinstance(num_layers_d, int) and pooling_method is None:
            # the reference multiplies by the discriminator's index when there is no pooling
            num_layers_d = [num_layers_d * i for i in range(1, num_d + 1)]
        elif isinstance(num_layers_d, int) and pooling_method is not None:
            num_layers_d = [num_layers_d] * num_d
        self.num_layers_d = num_layers_d
        if len(self.num_layers_d) != self.num_d:
            raise AssertionError(f"MultiScalePatchDiscriminator: num_d {num_d} must match the number of "
                                 f"num_layers_d. {num_layers_d}")
        self.padding = tuple([int((kernel_size - 1) / 2)] * spatial_dims)
        if pooling_method is None:
            pool = None
        else:
            pools = _POOLS.get(str(pooling_method).upper())
            if pools is None or spatial_dims not in (2, 3):
                raise NotImplementedError(f"pooling_method {pooling_method!r} with spatial_dims={spatial_dims} is not "
                                          "supported on the CUDA path: 'avg' or 'max', 2-D or 3-D")
            pool = pools[spatial_dims == 3](kernel_size=kernel_size, stride=2, padding=self.padding)
            self._pool_args = (kernel_size, self.padding[0], str(pooling_method).lower())
        self.num_channels = num_channels
        for i_ in range(self.num_d):
            num_layers_d_i = self.num_layers_d[i_]
            output_size = float(minimum_size_im) / (2 ** num_layers_d_i)
            if output_size < 1:
                raise AssertionError(
                    "Your image size is too small to take in up to %d discriminators with num_layers = %d."
                    "Please reduce num_layers, reduce num_D or enter bigger images." % (i_, num_layers_d_i))
            subnet_d = PatchDiscriminator(spatial_dims=spatial_dims, num_channels=self.num_channels,
                                          in_channels=in_channels, out_channels=out_channels,
                                          num_layers_d=num_layers_d_i, kernel_size=kernel_size, activation=activation,
                                          norm=norm, bias=bias, padding=self.padding, dropout=dropout,
                                          last_conv_kernel_size=last_conv_kernel_size)
            if i_ > 0 and pool is not None:
                subnet_d = nn.Sequential(*[pool] * i_, subnet_d)
            self.add_module("discriminator_%d" % i_, subnet_d)

    @on_input_device
    def forward(self, i: torch.Tensor) -> tuple[list[torch.Tensor], list[list[torch.Tensor]]]:
        require_cuda(i, self)
        discs = [d if isinstance(d, PatchDiscriminator) else d[-1] for d in self.children()]
        if self.training and any(d.mode_dependent for d in discs):
            _inference_only(self)
        levels = [ops.to_cl(i)]
        out: list[torch.Tensor] = []
        intermediate_features: list[list[torch.Tensor]] = []
        for disc, d in zip(self.children(), discs):
            n_pool = 0 if disc is d else len(disc) - 1
            while len(levels) <= n_pool:
                levels.append(ops.pool_s2(levels[-1], *self._pool_args))
            out_d = d.forward_cl(levels[n_pool], i.dtype)
            out.append(out_d[-1])
            intermediate_features.append(out_d[:-1])
        return out, intermediate_features

"""Parameter holders shared by the network modules.

The modules keep the reference's module tree and ``state_dict`` keys (SURVEY.md §8b) by holding their parameters in
ordinary ``torch.nn`` layers that are never *called*: ``forward`` hands the weights — repacked once into the K-major
h16 layout the wgmma kernel wants and cached against the parameter's version — to the C-ABI operators.
"""
from __future__ import annotations

import functools
from typing import Sequence

import torch
import torch.nn as nn

from .. import ops
from ..ops import CL


def _key(*params):
    return tuple((p.data_ptr(), p._version, p.device) if p is not None else None for p in params)


class _Cached:
    """Mixin: cache of packed weights keyed by (data_ptr, version, device, extra)."""

    def _cached(self, extra, params, build):
        cache = self.__dict__.setdefault("_pack_cache", {})
        k = (extra, _key(*params))
        hit = cache.get(extra)
        if hit is None or hit[0] != k:
            hit = (k, build())
            cache[extra] = hit
        return hit[1]


_ACT_CODES = {"RELU": ops.ACT_RELU, "SILU": ops.ACT_SILU, "SWISH": ops.ACT_SILU, "LEAKYRELU": ops.ACT_LEAKYRELU,
              "GELU": ops.ACT_GELU, "TANH": ops.ACT_TANH, "SIGMOID": ops.ACT_SIGMOID}


def act_code(act) -> int:
    """monai ``Act[...]`` name (or (name, kwargs) tuple with default kwargs) -> epilogue activation code.  The one
    non-default argument set with a code of its own is ``("LEAKYRELU", {"negative_slope": 0.2})`` (SPADENet)."""
    name = act[0] if isinstance(act, (tuple, list)) else act
    if isinstance(act, (tuple, list)) and len(act) > 1 and act[1]:
        if str(name).upper() == "LEAKYRELU" and dict(act[1]) == {"negative_slope": 0.2}:
            return ops.ACT_LEAKYRELU02
        raise NotImplementedError(f"activation {act!r} with non-default arguments is not supported "
                                  "(the only one is ('LEAKYRELU', {'negative_slope': 0.2}))")
    code = _ACT_CODES.get(str(name).upper())
    if code is None:
        raise NotImplementedError(f"activation {name!r} is not supported on the CUDA path ({sorted(_ACT_CODES)})")
    return code


def _same_padding(kernel_size: int, dilation: int = 1) -> int:
    return (kernel_size - 1) // 2 * dilation


class Convolution(nn.Module, _Cached):
    """Holder with the key layout of ``monai.networks.blocks.Convolution``: child ``conv`` is the nn.Conv /
    nn.ConvTranspose whose parameters are used (monai semantics restated in SURVEY.md §8c: padding=None -> same
    padding, output_padding=None -> stride - 1).  ``act`` is the ADN activation ("RELU") applied in the epilogue.
    ``norm="INSTANCE"`` (with ``conv_only=False``) is monai's ADN order "NDA": conv, then InstanceNorm (eps 1e-5, no
    affine, child ``adn.N`` without parameters), then ``act`` applied by the normalisation pass.
    ``norm="BATCH"`` is the same order with an ``nn.BatchNorm{2,3}d`` child ``adn.N``; in eval mode it is folded into the
    packed weights (b200_batchnorm_fold: w * s, beta + (b - mean) * s with s = gamma / sqrt(var + eps)) and ``act``
    runs in the convolution's epilogue.  Its batch statistics are not computed: forward in train mode raises."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int, strides: int = 1, kernel_size: int = 3,
                 padding: int | None = None, dilation: int = 1, bias: bool = True, conv_only: bool = True,
                 is_transposed: bool = False, output_padding: int | None = None, act: str | None = None,
                 norm: str | None = None, **_ignored):
        super().__init__()
        self.spatial_dims, self.in_channels, self.out_channels = spatial_dims, in_channels, out_channels
        self.strides, self.kernel_size, self.dilation = strides, kernel_size, dilation
        self.padding = _same_padding(kernel_size, dilation) if padding is None else padding
        self.is_transposed = is_transposed
        if dilation != 1:
            raise NotImplementedError("dilated convolutions are not on the sampling path")
        if is_transposed:
            self.output_padding = strides - 1 if output_padding is None else output_padding
            ctor = nn.ConvTranspose2d if spatial_dims == 2 else nn.ConvTranspose3d
            self.conv = ctor(in_channels, out_channels, kernel_size, stride=strides, padding=self.padding,
                             output_padding=self.output_padding, bias=bias)
        else:
            ctor = nn.Conv1d if spatial_dims == 1 else nn.Conv2d if spatial_dims == 2 else nn.Conv3d
            self.conv = ctor(in_channels, out_channels, kernel_size, stride=strides, padding=self.padding, bias=bias)
        self.act = ops.ACT_NONE if (conv_only or act is None) else act_code(act)
        self.norm = None if (conv_only or norm is None) else str(norm).upper()
        self.instance_norm = self.norm == "INSTANCE"
        if self.norm is not None:
            if self.norm not in ("INSTANCE", "BATCH") or is_transposed:
                raise NotImplementedError(f"Convolution norm {norm!r} is not supported (INSTANCE or BATCH after a "
                                          "convolution)")
            norms = {"INSTANCE": (nn.InstanceNorm2d, nn.InstanceNorm3d), "BATCH": (nn.BatchNorm2d, nn.BatchNorm3d)}
            self.adn = nn.Sequential()
            self.adn.add_module("N", norms[self.norm][spatial_dims == 3](out_channels))

    def packed(self, splits: Sequence[int] | None = None, padding=None):
        pad = self.padding if padding is None else padding
        extra = ("conv", tuple(splits) if splits else None, str(pad))
        if self.is_transposed:
            return self._cached(extra, (self.conv.weight, self.conv.bias), lambda: ops.PackedConvTranspose(
                self.conv.weight, self.conv.bias, self.strides, self.padding, self.output_padding))
        if self.norm == "BATCH":
            bn = self.adn.N
            stats = (bn.weight, bn.bias, bn.running_mean, bn.running_var)
            return self._cached(extra + ("bn", bn.eps), (self.conv.weight, self.conv.bias, *stats),
                                lambda: ops.PackedConv(*ops.batchnorm_fold(self.conv.weight, self.conv.bias, *stats,
                                                                           bn.eps), self.strides, pad, splits=splits))
        return self._cached(extra, (self.conv.weight, self.conv.bias), lambda: ops.PackedConv(
            self.conv.weight, self.conv.bias, self.strides, pad, splits=splits))

    def packed_upsample(self) -> ops.PackedUpsampleConv:
        return self._cached(("up2x",), (self.conv.weight, self.conv.bias),
                            lambda: ops.PackedUpsampleConv(self.conv.weight, self.conv.bias))

    def forward_upsampled(self, x: CL) -> CL:
        """conv(nearest_upsample_x2(x)) for a k3 s1 p1 convolution, as phase convolutions on the low-res input."""
        if self.is_transposed or self.kernel_size != 3 or self.strides != 1 or self.padding != 1:
            return self.forward(ops.upsample_nearest2x(x))
        return ops.conv_upsample2x(x, self.packed_upsample())

    def forward(self, x: CL | Sequence[CL], **epilogue):
        if self.is_transposed:
            return ops.conv_transpose(x, self.packed(), act1=self.act)
        srcs = [x] if isinstance(x, CL) else list(x)
        if self.norm == "BATCH" and self.training:
            raise RuntimeError("Convolution with norm='BATCH' runs the eval-mode BatchNorm (running statistics) only; "
                               "call .eval()")
        if self.instance_norm:
            y = ops.conv(srcs, self.packed([a.C for a in srcs]), **epilogue)
            dev = y.t.device
            return ops.groupnorm(y, y.C, self.adn.N.eps, ops._const_vec(y.C, 1.0, dev), ops._const_vec(y.C, 0.0, dev),
                                 act=self.act)
        if self.act != ops.ACT_NONE:
            epilogue.setdefault("act1", self.act)
        return ops.conv(srcs, self.packed([a.C for a in srcs]), **epilogue)

    def empty_output(self, x: CL | Sequence[CL]) -> CL:
        """The output tensor ``forward(x, out=...)`` would fill (plain convolutions only) — allocated by the caller on
        the main stream before it forks the convolution onto a side stream (ops.fork)."""
        srcs = [x] if isinstance(x, CL) else list(x)
        a0 = srcs[0]
        pc = self.packed([a.C for a in srcs])
        return ops.new_cl(a0.N, pc.out_dims(a0.D, a0.H, a0.W), pc.cout, a0.t.device, a0.spatial_dims)


class LinearHolder(_Cached):
    """Packs an nn.Linear for the tensor-core GEMM path (the nn.Linear itself lives in the owning module)."""

    def __init__(self, lin: nn.Linear):
        self.lin = lin

    def packed(self) -> ops.PackedLinear:
        return self._cached("lin", (self.lin.weight, self.lin.bias),
                            lambda: ops.PackedLinear(self.lin.weight, self.lin.bias))


def packed_linear(owner: nn.Module, name: str) -> ops.PackedLinear:
    holders = owner.__dict__.setdefault("_lin_holders", {})
    h = holders.get(name)
    lin = getattr(owner, name) if "." not in name else owner.get_submodule(name)
    if h is None or h.lin is not lin:
        h = holders[name] = LinearHolder(lin)
    return h.packed()


def packed_linear_geglu(owner: nn.Module, name: str) -> ops.PackedLinear:
    """``owner.name`` (linear1 of a GEGLU feed-forward) packed with interleaved a / gate rows (ops.PackedLinear.geglu),
    cached like packed_linear."""
    lin = getattr(owner, name)
    cache = owner.__dict__.setdefault("_pack_cache", {})
    key = ("geglu", name)
    k = (key, _key(lin.weight, lin.bias))
    hit = cache.get(key)
    if hit is None or hit[0] != k:
        hit = (k, ops.PackedLinear.geglu(lin.weight, lin.bias))
        cache[key] = hit
    return hit[1]


def packed_linear_stack(owner: nn.Module, names: Sequence[str]) -> ops.PackedLinear:
    """The linears ``names`` of ``owner`` (same input) as one stacked GEMM weight, cached like packed_linear."""
    lins = [getattr(owner, n) for n in names]
    cache = owner.__dict__.setdefault("_pack_cache", {})
    key = ("stack", tuple(names))
    k = (key, _key(*[t for lin in lins for t in (lin.weight, lin.bias)]))      # same entry layout as _Cached
    hit = cache.get(key)
    if hit is None or hit[0] != k:
        hit = (k, ops.PackedLinear.stacked([lin.weight for lin in lins], [lin.bias for lin in lins]))
        cache[key] = hit
    return hit[1]


def f32(p: torch.Tensor) -> torch.Tensor:
    return p if p.dtype == torch.float32 else p.float()


def require_cuda(x: torch.Tensor, module: nn.Module):
    if not x.is_cuda:
        raise RuntimeError(f"{type(module).__name__}: generativemodels_b200 runs on sm_90a (H100) CUDA devices only "
                           "(input tensor is on the CPU and there is no CPU path)")


def on_input_device(fn):
    """Run a module / scheduler entry point with the CUDA device of its first tensor argument current: the C-ABI
    launches on the current device and allocates workspaces there, so a model living on cuda:1 while cuda:0 is current
    would otherwise read its tensors across the peer link or fault (PyTorch modules do not require set_device)."""
    @functools.wraps(fn)
    def wrapped(self, *args, **kwargs):
        x = args[0] if args else next((v for v in kwargs.values() if torch.is_tensor(v)), None)
        if torch.is_tensor(x) and x.is_cuda and x.device.index != torch.cuda.current_device():
            with torch.cuda.device(x.device):
                return fn(self, *args, **kwargs)
        return fn(self, *args, **kwargs)
    return wrapped


def invalidate_packed(module: nn.Module) -> None:
    """Drop every packed-weight / concatenated-projection / captured-graph cache under ``module``.

    The caches are keyed by ``(data_ptr, _version, device)`` of the parameters, which catches ``load_state_dict``,
    optimiser steps, ``.to()`` and any in-place op on the parameter itself — but NOT writes through ``param.data``
    (``p.data.copy_(ema)``, ``p.data.mul_()``: PyTorch does not bump ``p._version`` for those).  Call this after such
    weight surgery (EMA swaps) and the next forward repacks from the live parameters."""
    for m in module.modules():
        for key in ("_pack_cache", "_lin_holders", "_temb_cat", "_temb_blocks", "_bare_cache"):
            m.__dict__.pop(key, None)
        g = m.__dict__.get("_b200_auto_graph")
        if g is not None:
            g._entries.clear()
        if hasattr(m, "_entries") and hasattr(m, "_weights_sig"):      # a GraphedModule
            m._entries.clear()
            m._weights_sig = None

"""DiffusionModelUNet on the H100 kernels — same classes, constructor arguments, attribute names and ``state_dict``
keys as generative/networks/nets/diffusion_model_unet.py (reference lines cited per class), different insides:

* activations stay channels-last h16 (:class:`~generativemodels_b200.ops.CL`) from ``conv_in`` to the output head;
* every ResnetBlock is  GN-stats -> GN-apply+SiLU -> wgmma conv (+bias +time-embedding row vector in the epilogue)
  -> GN -> wgmma conv (+bias +skip/residual in the epilogue);
* the up path never materialises ``torch.cat([h, skip])`` raw: GroupNorm and the 1x1 skip conv read both tensors;
* attention runs as the flash-style wgmma kernel, as wgmma GEMMs (QK^T, PV with V^T from an operand-swapped projection) or, for tiny heads /
  a handful of context tokens, the CUDA-core online-softmax kernel.
DiffusionModelEncoder, the reference's classifier built on the same down path, lives here as it does in the reference.
Inference only (``torch.no_grad`` semantics); there is no CPU path.
"""
from __future__ import annotations

import math
from collections.abc import Sequence

import torch
import torch.nn as nn

from ... import ops
from ...losses._common import forward_only
from ...ops import ACT_RELU, ACT_SILU, CL
from ..blocks.spade_norm import SPADE
from .._holders import (Convolution, _Cached, f32, on_input_device, packed_linear, packed_linear_geglu,
                        packed_linear_stack, require_cuda)

__all__ = ["DiffusionModelUNet"]


def zero_module(module: nn.Module) -> nn.Module:
    for p in module.parameters():
        p.detach().zero_()
    return module


def ensure_tuple_rep(v, n):
    if isinstance(v, (tuple, list)):
        if len(v) != n:
            raise ValueError(f"Sequence must have length {n}, got {len(v)}.")
        return tuple(v)
    return (v,) * n


def _rows(a: CL) -> torch.Tensor:
    """CL -> packed token rows [N, T, pitch]."""
    return a.t.reshape(a.N, a.spatial, a.pitch)


def _context_cl(context: torch.Tensor) -> CL:
    """(N, S, ctx_dim) float context -> CL rows [N, 1, 1, S, pitch]."""
    return ops.to_cl(context.permute(0, 2, 1).unsqueeze(2).contiguous())


def _few_rows_linear(x: CL, pl, act: int = ops.ACT_NONE, out_f32: bool = False) -> torch.Tensor:
    """act(projection) of a token matrix to packed rows [N, S, pitch] (h16, or fp32 with ``out_f32``).  A handful of
    tokens in total (the context of a classifier-free-guidance step: one token per sample) goes through the GEMV
    kernel — a 128-row tensor-core tile spends its pipeline latency on two rows, 14 of them per C5 UNet forward."""
    rows = x.N * x.spatial
    if rows <= 8 and x.C * rows * 2 <= 32 * 1024:
        y = ops.rows_linear(x.t.reshape(rows, x.pitch), x.C, pl, act=act, out_f32=out_f32)
    else:
        y = ops.linear(x, pl, act1=act, out_f32=out_f32)
        y = y if out_f32 else y.t
    return y.reshape(x.N, x.spatial, y.shape[-1])


def _sdp(owner: nn.Module, xq: CL, xkv: CL, heads: int, dh: int, scale: float, residual: CL | None,
         bias_qkv: bool) -> CL:
    """scaled-dot-product attention of ``xq`` over ``xkv`` with this module's to_q/to_k/to_v."""
    S = xkv.spatial
    inner = heads * dh
    use_tc = dh % 64 == 0 and S >= 64
    vt = vt_fork = None
    if use_tc:
        # V^T does not depend on q / k: inside a CUDA-graph capture it runs on a side stream next to their GEMM
        to_v = packed_linear(owner, "to_v")
        vt = ops.linear_transposed_out(_rows(xkv), to_v)
        with ops.fork() as vt_fork:
            ops.linear_transposed(_rows(xkv), xkv.C, to_v, out=vt)
    if xq is xkv and inner % 16 == 0:
        # self-attention: q and k from ONE GEMM over the stacked [to_q; to_k] weights; the attention kernels read
        # them as column slices of the [N, T, 2C] result (row pitch from the stride)
        qk = ops.linear(xq, packed_linear_stack(owner, ("to_q", "to_k")))
        qk_rows = _rows(qk)
        q_rows, k_rows = qk_rows[:, :, :inner], qk_rows[:, :, inner:2 * inner]
    else:
        q_rows = _rows(ops.linear(xq, packed_linear(owner, "to_q")))
        k_rows = _few_rows_linear(xkv, packed_linear(owner, "to_k"))
    if use_tc:
        vt_fork.join()
        o = ops.attention(q_rows, k_rows, None, heads, dh, scale, vt=vt,
                          residual=None if residual is None else _rows(residual))
        return CL(o.reshape(xq.t.shape[0], xq.D, xq.H, xq.W, o.shape[-1]), heads * dh, xq.spatial_dims)
    o = ops.attention(q_rows, k_rows, _few_rows_linear(xkv, packed_linear(owner, "to_v")), heads, dh, scale)
    out = CL(o.reshape(xq.t.shape[0], xq.D, xq.H, xq.W, o.shape[-1]), heads * dh, xq.spatial_dims)
    if residual is not None:
        out = ops.axpy(out, residual, 1.0, inplace=True)
    return out


class CrossAttention(nn.Module):
    """diffusion_model_unet.py:72-175 (to_q/to_k/to_v without bias, to_out = Linear + Dropout)."""

    def __init__(self, query_dim: int, cross_attention_dim: int | None = None, num_attention_heads: int = 8,
                 num_head_channels: int = 64, dropout: float = 0.0, upcast_attention: bool = False,
                 use_flash_attention: bool = False) -> None:
        super().__init__()
        inner_dim = num_head_channels * num_attention_heads
        cross_attention_dim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.scale = 1 / math.sqrt(num_head_channels)
        self.num_heads = num_attention_heads
        self.num_head_channels = num_head_channels
        self.upcast_attention = upcast_attention      # scores/softmax are always fp32 here
        self.use_flash_attention = use_flash_attention
        self.to_q = nn.Linear(query_dim, inner_dim, bias=False)
        self.to_k = nn.Linear(cross_attention_dim, inner_dim, bias=False)
        self.to_v = nn.Linear(cross_attention_dim, inner_dim, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, query_dim), nn.Dropout(dropout))

    def forward(self, x: CL, context: CL | None = None, residual: CL | None = None) -> CL:
        o = _sdp(self, x, x if context is None else context, self.num_heads, self.num_head_channels, self.scale,
                 None, False)
        return ops.linear(o, packed_linear(self, "to_out.0"), residual=residual)


class GEGLUFeedForward(nn.Module):
    """Key layout of monai ``MLPBlock(hidden, mlp_dim, act="GEGLU")``: linear1 (hidden -> 2*mlp_dim), linear2."""

    def __init__(self, hidden_size: int, mlp_dim: int, dropout_rate: float = 0.0) -> None:
        super().__init__()
        self.linear1 = nn.Linear(hidden_size, mlp_dim * 2)
        self.linear2 = nn.Linear(mlp_dim, hidden_size)

    def forward(self, x: CL, residual: CL | None = None) -> CL:
        if self.linear2.in_features % 32 == 0:
            # linear1 + gating as one GEMM (a * gelu(gate) in the epilogue, on the fp32 accumulators)
            f = ops.linear_geglu(x, packed_linear_geglu(self, "linear1"))
        else:
            f = ops.geglu(ops.linear(x, packed_linear(self, "linear1")))
        return ops.linear(f, packed_linear(self, "linear2"), residual=residual)


class BasicTransformerBlock(nn.Module):
    """diffusion_model_unet.py:178-234."""

    def __init__(self, num_channels: int, num_attention_heads: int, num_head_channels: int, dropout: float = 0.0,
                 cross_attention_dim: int | None = None, upcast_attention: bool = False,
                 use_flash_attention: bool = False) -> None:
        super().__init__()
        self.attn1 = CrossAttention(num_channels, None, num_attention_heads, num_head_channels, dropout,
                                    upcast_attention, use_flash_attention)
        self.ff = GEGLUFeedForward(num_channels, num_channels * 4, dropout)
        self.attn2 = CrossAttention(num_channels, cross_attention_dim, num_attention_heads, num_head_channels,
                                    dropout, upcast_attention, use_flash_attention)
        self.norm1 = nn.LayerNorm(num_channels)
        self.norm2 = nn.LayerNorm(num_channels)
        self.norm3 = nn.LayerNorm(num_channels)

    def _ln(self, norm: nn.LayerNorm, x: CL) -> CL:
        return ops.layernorm(x, f32(norm.weight), f32(norm.bias), norm.eps)

    def forward(self, x: CL, context: CL | None = None) -> CL:
        x = self.attn1(self._ln(self.norm1, x), residual=x)
        x = self.attn2(self._ln(self.norm2, x), context=context, residual=x)
        return self.ff(self._ln(self.norm3, x), residual=x)


class SpatialTransformer(nn.Module):
    """diffusion_model_unet.py:237-342."""

    def __init__(self, spatial_dims: int, in_channels: int, num_attention_heads: int, num_head_channels: int,
                 num_layers: int = 1, dropout: float = 0.0, norm_num_groups: int = 32, norm_eps: float = 1e-6,
                 cross_attention_dim: int | None = None, upcast_attention: bool = False,
                 use_flash_attention: bool = False) -> None:
        super().__init__()
        self.spatial_dims, self.in_channels = spatial_dims, in_channels
        inner_dim = num_attention_heads * num_head_channels
        self.norm = nn.GroupNorm(num_groups=norm_num_groups, num_channels=in_channels, eps=norm_eps, affine=True)
        self.proj_in = Convolution(spatial_dims, in_channels, inner_dim, strides=1, kernel_size=1, padding=0)
        self.transformer_blocks = nn.ModuleList([
            BasicTransformerBlock(inner_dim, num_attention_heads, num_head_channels, dropout, cross_attention_dim,
                                  upcast_attention, use_flash_attention) for _ in range(num_layers)])
        self.proj_out = zero_module(Convolution(spatial_dims, inner_dim, in_channels, strides=1, kernel_size=1,
                                                padding=0))

    def forward(self, x: CL, context: CL | None = None) -> CL:
        h = ops.groupnorm(x, self.norm.num_groups, self.norm.eps, self.norm.weight, self.norm.bias)
        h = self.proj_in(h)
        for block in self.transformer_blocks:
            h = block(h, context=context)
        return self.proj_out(h, residual=x)


class AttentionBlock(nn.Module):
    """diffusion_model_unet.py:345-458.  ``proj_attn`` is part of the state_dict but, as in the reference's forward
    (418-458), never applied."""

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


class Downsample(nn.Module):
    """diffusion_model_unet.py:488-531."""

    def __init__(self, spatial_dims: int, num_channels: int, use_conv: bool, out_channels: int | None = None,
                 padding: int = 1) -> None:
        super().__init__()
        self.num_channels = num_channels
        self.out_channels = out_channels or num_channels
        self.use_conv = use_conv
        if use_conv:
            self.op = Convolution(spatial_dims, self.num_channels, self.out_channels, strides=2, kernel_size=3,
                                  padding=padding)
        else:
            if self.num_channels != self.out_channels:
                raise ValueError("num_channels and out_channels must be equal when use_conv=False")
            self.op = nn.AvgPool2d(2, 2) if spatial_dims == 2 else nn.AvgPool3d(2, 2)   # holder only

    def forward(self, x: CL, emb=None) -> CL:
        if x.C != self.num_channels:
            raise ValueError(f"Input number of channels ({x.C}) is not equal to expected number of channels "
                             f"({self.num_channels})")
        return self.op(x) if self.use_conv else ops.avgpool2(x)


class Upsample(nn.Module):
    """diffusion_model_unet.py:534-586 (nearest x2, optional k3 conv)."""

    def __init__(self, spatial_dims: int, num_channels: int, use_conv: bool, out_channels: int | None = None,
                 padding: int = 1) -> None:
        super().__init__()
        self.num_channels = num_channels
        self.out_channels = out_channels or num_channels
        self.use_conv = use_conv
        self.conv = Convolution(spatial_dims, self.num_channels, self.out_channels, strides=1, kernel_size=3,
                                padding=padding) if use_conv else None

    def forward(self, x: CL, emb=None) -> CL:
        if x.C != self.num_channels:
            raise ValueError("Input channels should be equal to num_channels")
        if self.use_conv:
            return self.conv.forward_upsampled(x)      # upsample folded into the conv: no 8x larger intermediate
        return ops.upsample_nearest2x(x)


class TimeEmb:
    """The time embedding of one forward together with every ResnetBlock's ``time_emb_proj(silu(emb))`` row
    (diffusion_model_unet.py:686-689), which depend on the timestep only: all of them come out of ONE GEMV launch over
    the row-concatenated projection weights instead of one launch per block (a latent UNet step is ~300-500 dependent
    launches of a few microseconds each).  ``proj[id(block)]`` is a
    column slice ``[rows, out_channels]`` of that result; the conv epilogue reads it through its row stride."""

    __slots__ = ("emb", "proj")

    def __init__(self, emb: torch.Tensor, proj: dict) -> None:
        self.emb, self.proj = emb, proj


def project_time_embedding(root: nn.Module, emb: torch.Tensor) -> TimeEmb:
    """Batch the time-embedding projections of all ResnetBlocks under ``root``.  The concatenated fp32 weights are
    cached on ``root`` against the (data_ptr, version) of every projection parameter."""
    blocks = root.__dict__.get("_temb_blocks")
    if blocks is None:
        blocks = root.__dict__["_temb_blocks"] = [m for m in root.modules() if isinstance(m, ResnetBlock)]
    if len(blocks) < 2:
        return TimeEmb(emb, {})
    params = []
    for b in blocks:
        params += [b.time_emb_proj.weight, b.time_emb_proj.bias]
    key = tuple((p.data_ptr(), p._version) for p in params)
    cache = root.__dict__.get("_temb_cat")
    if cache is None or cache[0] != key:
        w = torch.cat([b.time_emb_proj.weight.detach().float() for b in blocks], 0).contiguous()
        bias = torch.cat([b.time_emb_proj.bias.detach().float() for b in blocks], 0).contiguous()
        cache = root.__dict__["_temb_cat"] = (key, w, bias)
    rows = ops.small_linear(emb, cache[1], cache[2], act_in=ACT_SILU)
    proj, off = {}, 0
    for b in blocks:
        proj[id(b)] = rows[:, off:off + b.out_channels]
        off += b.out_channels
    return TimeEmb(emb, proj)


class ResnetBlock(nn.Module):
    """diffusion_model_unet.py:589-696; with ``label_nc`` the two norms are SPADE blocks and this is
    SPADEResnetBlock (spade_diffusion_model_unet.py:72-200; same keys, ``forward(x, emb, seg)``)."""

    def __init__(self, spatial_dims: int, in_channels: int, temb_channels: int, out_channels: int | None = None,
                 up: bool = False, down: bool = False, norm_num_groups: int = 32, norm_eps: float = 1e-6,
                 label_nc: int | None = None, spade_intermediate_channels: int = 128) -> None:
        super().__init__()
        self.spatial_dims = spatial_dims
        self.channels = in_channels
        self.emb_channels = temb_channels
        self.out_channels = out_channels or in_channels
        self.up, self.down = up, down
        self.spade = label_nc is not None

        def make_norm(ch):
            if self.spade:
                return SPADE(label_nc=label_nc, norm_nc=ch, norm="GROUP",
                             norm_params={"num_groups": norm_num_groups, "eps": norm_eps, "affine": True},
                             hidden_channels=spade_intermediate_channels, kernel_size=3, spatial_dims=spatial_dims)
            return nn.GroupNorm(num_groups=norm_num_groups, num_channels=ch, eps=norm_eps, affine=True)

        self.norm1 = make_norm(in_channels)
        self.nonlinearity = nn.SiLU()
        self.conv1 = Convolution(spatial_dims, in_channels, self.out_channels, strides=1, kernel_size=3, padding=1)
        self.upsample = self.downsample = None
        if self.up:
            self.upsample = Upsample(spatial_dims, in_channels, use_conv=False)
        elif down:
            self.downsample = Downsample(spatial_dims, in_channels, use_conv=False)
        self.time_emb_proj = nn.Linear(temb_channels, self.out_channels)
        self.norm2 = make_norm(self.out_channels)
        self.conv2 = zero_module(Convolution(spatial_dims, self.out_channels, self.out_channels, strides=1,
                                             kernel_size=3, padding=1))
        if self.out_channels == in_channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = Convolution(spatial_dims, in_channels, self.out_channels, strides=1, kernel_size=1,
                                               padding=0)

    def _norm(self, norm, srcs, seg):
        if self.spade:
            if seg is None:
                raise ValueError("a SPADE ResnetBlock needs the segmentation map (seg)")
            return norm(srcs, seg, act=ACT_SILU)
        return ops.groupnorm(srcs, norm.num_groups, norm.eps, norm.weight, norm.bias, act=ACT_SILU)

    def forward(self, x: CL | Sequence[CL], emb: torch.Tensor, seg=None) -> CL:
        srcs = [x] if isinstance(x, CL) else list(x)
        h = self._norm(self.norm1, srcs, seg)
        if self.up or self.down:
            if len(srcs) != 1:
                raise ValueError("resampling ResnetBlock takes a single input tensor")
            resample = ops.upsample_nearest2x if self.up else ops.avgpool2
            srcs = [resample(srcs[0])]
            h = resample(h)
        skip_fork = None
        if isinstance(self.skip_connection, nn.Identity):
            skip = srcs[0] if len(srcs) == 1 else ops.concat(srcs)
        else:
            # the 1x1 skip convolution only needs the block's input: inside a CUDA-graph capture it runs on a side
            # stream next to conv1 / norm2 (its output is allocated here, on the main stream)
            skip = self.skip_connection.empty_output(srcs)
            with ops.fork() as skip_fork:
                self.skip_connection(srcs, out=skip)
        temb = emb.proj.get(id(self)) if isinstance(emb, TimeEmb) else None
        if temb is None:
            e = emb.emb if isinstance(emb, TimeEmb) else emb
            temb = ops.small_linear(e, self.time_emb_proj.weight, self.time_emb_proj.bias, act_in=ACT_SILU)
        h = self.conv1(h, rowvec=temb)
        h = self._norm(self.norm2, [h], seg)
        if skip_fork is not None:
            skip_fork.join()
        return self.conv2(h, residual=skip)


def _downsampler(spatial_dims, out_channels, temb_channels, norm_num_groups, norm_eps, resblock_updown,
                 downsample_padding):
    if resblock_updown:
        return ResnetBlock(spatial_dims, out_channels, temb_channels, out_channels, down=True,
                           norm_num_groups=norm_num_groups, norm_eps=norm_eps)
    return Downsample(spatial_dims, out_channels, use_conv=True, out_channels=out_channels,
                      padding=downsample_padding)


def _upsampler(spatial_dims, out_channels, temb_channels, norm_num_groups, norm_eps, resblock_updown):
    if resblock_updown:
        return ResnetBlock(spatial_dims, out_channels, temb_channels, out_channels, up=True,
                           norm_num_groups=norm_num_groups, norm_eps=norm_eps)
    return Upsample(spatial_dims, out_channels, use_conv=True, out_channels=out_channels)


class _DownBase(nn.Module):
    """Shared body of DownBlock / AttnDownBlock / CrossAttnDownBlock (diffusion_model_unet.py:699-1061)."""

    def forward(self, hidden_states: CL, temb: torch.Tensor, context: CL | None = None):
        output_states = []
        attentions = self._modules.get("attentions")      # absent on the plain DownBlock
        for i, resnet in enumerate(self.resnets):
            hidden_states = resnet(hidden_states, temb)
            if attentions is not None:
                attn = attentions[i]
                hidden_states = attn(hidden_states, context=context) if isinstance(attn, SpatialTransformer) \
                    else attn(hidden_states)
            output_states.append(hidden_states)
        if self.downsampler is not None:
            hidden_states = self.downsampler(hidden_states, temb)
            output_states.append(hidden_states)
        return hidden_states, output_states


class DownBlock(_DownBase):
    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int, temb_channels: int,
                 num_res_blocks: int = 1, norm_num_groups: int = 32, norm_eps: float = 1e-6,
                 add_downsample: bool = True, resblock_updown: bool = False, downsample_padding: int = 1) -> None:
        super().__init__()
        self.resblock_updown = resblock_updown
        self.resnets = nn.ModuleList([
            ResnetBlock(spatial_dims, in_channels if i == 0 else out_channels, temb_channels, out_channels,
                        norm_num_groups=norm_num_groups, norm_eps=norm_eps) for i in range(num_res_blocks)])
        self.downsampler = _downsampler(spatial_dims, out_channels, temb_channels, norm_num_groups, norm_eps,
                                        resblock_updown, downsample_padding) if add_downsample else None


class AttnDownBlock(_DownBase):
    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int, temb_channels: int,
                 num_res_blocks: int = 1, norm_num_groups: int = 32, norm_eps: float = 1e-6,
                 add_downsample: bool = True, resblock_updown: bool = False, downsample_padding: int = 1,
                 num_head_channels: int = 1, use_flash_attention: bool = False) -> None:
        super().__init__()
        self.resblock_updown = resblock_updown
        resnets, attentions = [], []
        for i in range(num_res_blocks):
            resnets.append(ResnetBlock(spatial_dims, in_channels if i == 0 else out_channels, temb_channels,
                                       out_channels, norm_num_groups=norm_num_groups, norm_eps=norm_eps))
            attentions.append(AttentionBlock(spatial_dims, out_channels, num_head_channels, norm_num_groups, norm_eps,
                                             use_flash_attention))
        self.attentions = nn.ModuleList(attentions)
        self.resnets = nn.ModuleList(resnets)
        self.downsampler = _downsampler(spatial_dims, out_channels, temb_channels, norm_num_groups, norm_eps,
                                        resblock_updown, downsample_padding) if add_downsample else None


class CrossAttnDownBlock(_DownBase):
    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int, temb_channels: int,
                 num_res_blocks: int = 1, norm_num_groups: int = 32, norm_eps: float = 1e-6,
                 add_downsample: bool = True, resblock_updown: bool = False, downsample_padding: int = 1,
                 num_head_channels: int = 1, transformer_num_layers: int = 1,
                 cross_attention_dim: int | None = None, upcast_attention: bool = False,
                 use_flash_attention: bool = False, dropout_cattn: float = 0.0) -> None:
        super().__init__()
        self.resblock_updown = resblock_updown
        resnets, attentions = [], []
        for i in range(num_res_blocks):
            resnets.append(ResnetBlock(spatial_dims, in_channels if i == 0 else out_channels, temb_channels,
                                       out_channels, norm_num_groups=norm_num_groups, norm_eps=norm_eps))
            attentions.append(SpatialTransformer(
                spatial_dims, out_channels, out_channels // num_head_channels, num_head_channels,
                num_layers=transformer_num_layers, norm_num_groups=norm_num_groups, norm_eps=norm_eps,
                cross_attention_dim=cross_attention_dim, upcast_attention=upcast_attention,
                use_flash_attention=use_flash_attention, dropout=dropout_cattn))
        self.attentions = nn.ModuleList(attentions)
        self.resnets = nn.ModuleList(resnets)
        self.downsampler = _downsampler(spatial_dims, out_channels, temb_channels, norm_num_groups, norm_eps,
                                        resblock_updown, downsample_padding) if add_downsample else None


class AttnMidBlock(nn.Module):
    """diffusion_model_unet.py:1064-1127."""

    def __init__(self, spatial_dims: int, in_channels: int, temb_channels: int, norm_num_groups: int = 32,
                 norm_eps: float = 1e-6, num_head_channels: int = 1, use_flash_attention: bool = False) -> None:
        super().__init__()
        self.resnet_1 = ResnetBlock(spatial_dims, in_channels, temb_channels, in_channels,
                                    norm_num_groups=norm_num_groups, norm_eps=norm_eps)
        self.attention = AttentionBlock(spatial_dims, in_channels, num_head_channels, norm_num_groups, norm_eps,
                                        use_flash_attention)
        self.resnet_2 = ResnetBlock(spatial_dims, in_channels, temb_channels, in_channels,
                                    norm_num_groups=norm_num_groups, norm_eps=norm_eps)

    def forward(self, hidden_states: CL, temb: torch.Tensor, context: CL | None = None) -> CL:
        hidden_states = self.resnet_1(hidden_states, temb)
        hidden_states = self.attention(hidden_states)
        return self.resnet_2(hidden_states, temb)


class CrossAttnMidBlock(nn.Module):
    """diffusion_model_unet.py:1130-1210."""

    def __init__(self, spatial_dims: int, in_channels: int, temb_channels: int, norm_num_groups: int = 32,
                 norm_eps: float = 1e-6, num_head_channels: int = 1, transformer_num_layers: int = 1,
                 cross_attention_dim: int | None = None, upcast_attention: bool = False,
                 use_flash_attention: bool = False, dropout_cattn: float = 0.0) -> None:
        super().__init__()
        self.resnet_1 = ResnetBlock(spatial_dims, in_channels, temb_channels, in_channels,
                                    norm_num_groups=norm_num_groups, norm_eps=norm_eps)
        self.attention = SpatialTransformer(
            spatial_dims, in_channels, in_channels // num_head_channels, num_head_channels,
            num_layers=transformer_num_layers, norm_num_groups=norm_num_groups, norm_eps=norm_eps,
            cross_attention_dim=cross_attention_dim, upcast_attention=upcast_attention,
            use_flash_attention=use_flash_attention, dropout=dropout_cattn)
        self.resnet_2 = ResnetBlock(spatial_dims, in_channels, temb_channels, in_channels,
                                    norm_num_groups=norm_num_groups, norm_eps=norm_eps)

    def forward(self, hidden_states: CL, temb: torch.Tensor, context: CL | None = None) -> CL:
        hidden_states = self.resnet_1(hidden_states, temb)
        hidden_states = self.attention(hidden_states, context=context)
        return self.resnet_2(hidden_states, temb)


class _UpBase(nn.Module):
    """Shared body of UpBlock / AttnUpBlock / CrossAttnUpBlock (diffusion_model_unet.py:1213-1469).  The
    ``torch.cat([hidden_states, res_hidden_states], dim=1)`` (1232/1340/1461) is virtual: the pair goes to the
    ResnetBlock, whose GroupNorm and 1x1 skip conv read both tensors."""

    def forward(self, hidden_states: CL, res_hidden_states_list: list[CL], temb: torch.Tensor,
                context: CL | None = None, seg=None) -> CL:
        attentions = self._modules.get("attentions")      # absent on the plain UpBlock
        for i, resnet in enumerate(self.resnets):
            res_hidden_states = res_hidden_states_list[-1]
            res_hidden_states_list = res_hidden_states_list[:-1]
            hidden_states = resnet([hidden_states, res_hidden_states], temb, seg)
            if attentions is not None:
                attn = attentions[i]
                hidden_states = attn(hidden_states, context=context) if isinstance(attn, SpatialTransformer) \
                    else attn(hidden_states)
        if self.upsampler is not None:
            hidden_states = self.upsampler(hidden_states, temb)
        return hidden_states


def _up_resnets(spatial_dims, in_channels, prev_output_channel, out_channels, temb_channels, num_res_blocks,
                norm_num_groups, norm_eps, label_nc=None, spade_intermediate_channels=128):
    resnets = []
    for i in range(num_res_blocks):
        res_skip_channels = in_channels if (i == num_res_blocks - 1) else out_channels
        resnet_in_channels = prev_output_channel if i == 0 else out_channels
        resnets.append(ResnetBlock(spatial_dims, resnet_in_channels + res_skip_channels, temb_channels, out_channels,
                                   norm_num_groups=norm_num_groups, norm_eps=norm_eps, label_nc=label_nc,
                                   spade_intermediate_channels=spade_intermediate_channels))
    return resnets


class UpBlock(_UpBase):
    def __init__(self, spatial_dims: int, in_channels: int, prev_output_channel: int, out_channels: int,
                 temb_channels: int, num_res_blocks: int = 1, norm_num_groups: int = 32, norm_eps: float = 1e-6,
                 add_upsample: bool = True, resblock_updown: bool = False, label_nc: int | None = None,
                 spade_intermediate_channels: int = 128) -> None:
        super().__init__()
        self.resblock_updown = resblock_updown
        self.resnets = nn.ModuleList(_up_resnets(spatial_dims, in_channels, prev_output_channel, out_channels,
                                                 temb_channels, num_res_blocks, norm_num_groups, norm_eps, label_nc,
                                                 spade_intermediate_channels))
        self.upsampler = _upsampler(spatial_dims, out_channels, temb_channels, norm_num_groups, norm_eps,
                                    resblock_updown) if add_upsample else None


class AttnUpBlock(_UpBase):
    def __init__(self, spatial_dims: int, in_channels: int, prev_output_channel: int, out_channels: int,
                 temb_channels: int, num_res_blocks: int = 1, norm_num_groups: int = 32, norm_eps: float = 1e-6,
                 add_upsample: bool = True, resblock_updown: bool = False, num_head_channels: int = 1,
                 use_flash_attention: bool = False, label_nc: int | None = None,
                 spade_intermediate_channels: int = 128) -> None:
        super().__init__()
        self.resblock_updown = resblock_updown
        self.resnets = nn.ModuleList(_up_resnets(spatial_dims, in_channels, prev_output_channel, out_channels,
                                                 temb_channels, num_res_blocks, norm_num_groups, norm_eps, label_nc,
                                                 spade_intermediate_channels))
        self.attentions = nn.ModuleList([
            AttentionBlock(spatial_dims, out_channels, num_head_channels, norm_num_groups, norm_eps,
                           use_flash_attention) for _ in range(num_res_blocks)])
        self.upsampler = _upsampler(spatial_dims, out_channels, temb_channels, norm_num_groups, norm_eps,
                                    resblock_updown) if add_upsample else None


class CrossAttnUpBlock(_UpBase):
    def __init__(self, spatial_dims: int, in_channels: int, prev_output_channel: int, out_channels: int,
                 temb_channels: int, num_res_blocks: int = 1, norm_num_groups: int = 32, norm_eps: float = 1e-6,
                 add_upsample: bool = True, resblock_updown: bool = False, num_head_channels: int = 1,
                 transformer_num_layers: int = 1, cross_attention_dim: int | None = None,
                 upcast_attention: bool = False, use_flash_attention: bool = False,
                 dropout_cattn: float = 0.0, label_nc: int | None = None,
                 spade_intermediate_channels: int = 128) -> None:
        super().__init__()
        self.resblock_updown = resblock_updown
        self.resnets = nn.ModuleList(_up_resnets(spatial_dims, in_channels, prev_output_channel, out_channels,
                                                 temb_channels, num_res_blocks, norm_num_groups, norm_eps, label_nc,
                                                 spade_intermediate_channels))
        self.attentions = nn.ModuleList([
            SpatialTransformer(spatial_dims, out_channels, out_channels // num_head_channels, num_head_channels,
                               num_layers=transformer_num_layers, norm_num_groups=norm_num_groups, norm_eps=norm_eps,
                               cross_attention_dim=cross_attention_dim, upcast_attention=upcast_attention,
                               use_flash_attention=use_flash_attention, dropout=dropout_cattn)
            for _ in range(num_res_blocks)])
        self.upsampler = _upsampler(spatial_dims, out_channels, temb_channels, norm_num_groups, norm_eps,
                                    resblock_updown) if add_upsample else None


def get_down_block(spatial_dims, in_channels, out_channels, temb_channels, num_res_blocks, norm_num_groups, norm_eps,
                   add_downsample, resblock_updown, with_attn, with_cross_attn, num_head_channels,
                   transformer_num_layers, cross_attention_dim, upcast_attention=False, use_flash_attention=False,
                   dropout_cattn=0.0) -> nn.Module:
    """diffusion_model_unet.py:1472-1537."""
    common = dict(spatial_dims=spatial_dims, in_channels=in_channels, out_channels=out_channels,
                  temb_channels=temb_channels, num_res_blocks=num_res_blocks, norm_num_groups=norm_num_groups,
                  norm_eps=norm_eps, add_downsample=add_downsample, resblock_updown=resblock_updown)
    if with_attn:
        return AttnDownBlock(**common, num_head_channels=num_head_channels, use_flash_attention=use_flash_attention)
    if with_cross_attn:
        return CrossAttnDownBlock(**common, num_head_channels=num_head_channels,
                                  transformer_num_layers=transformer_num_layers,
                                  cross_attention_dim=cross_attention_dim, upcast_attention=upcast_attention,
                                  use_flash_attention=use_flash_attention, dropout_cattn=dropout_cattn)
    return DownBlock(**common)


def get_mid_block(spatial_dims, in_channels, temb_channels, norm_num_groups, norm_eps, with_conditioning,
                  num_head_channels, transformer_num_layers, cross_attention_dim, upcast_attention=False,
                  use_flash_attention=False, dropout_cattn=0.0) -> nn.Module:
    """diffusion_model_unet.py:1540-1574 — the mid block always has attention."""
    if with_conditioning:
        return CrossAttnMidBlock(spatial_dims, in_channels, temb_channels, norm_num_groups, norm_eps,
                                 num_head_channels, transformer_num_layers, cross_attention_dim, upcast_attention,
                                 use_flash_attention, dropout_cattn)
    return AttnMidBlock(spatial_dims, in_channels, temb_channels, norm_num_groups, norm_eps, num_head_channels,
                        use_flash_attention)


def get_up_block(spatial_dims, in_channels, prev_output_channel, out_channels, temb_channels, num_res_blocks,
                 norm_num_groups, norm_eps, add_upsample, resblock_updown, with_attn, with_cross_attn,
                 num_head_channels, transformer_num_layers, cross_attention_dim, upcast_attention=False,
                 use_flash_attention=False, dropout_cattn=0.0, label_nc=None,
                 spade_intermediate_channels=128) -> nn.Module:
    """diffusion_model_unet.py:1577-1643; with ``label_nc`` the SPADE variants (spade_diffusion_model_unet.py:540-609)."""
    common = dict(spatial_dims=spatial_dims, in_channels=in_channels, prev_output_channel=prev_output_channel,
                  out_channels=out_channels, temb_channels=temb_channels, num_res_blocks=num_res_blocks,
                  norm_num_groups=norm_num_groups, norm_eps=norm_eps, add_upsample=add_upsample,
                  resblock_updown=resblock_updown, label_nc=label_nc,
                  spade_intermediate_channels=spade_intermediate_channels)
    if with_attn:
        return AttnUpBlock(**common, num_head_channels=num_head_channels, use_flash_attention=use_flash_attention)
    if with_cross_attn:
        return CrossAttnUpBlock(**common, num_head_channels=num_head_channels,
                                transformer_num_layers=transformer_num_layers,
                                cross_attention_dim=cross_attention_dim, upcast_attention=upcast_attention,
                                use_flash_attention=use_flash_attention, dropout_cattn=dropout_cattn)
    return UpBlock(**common)


def time_embedding(module: nn.Module, x: torch.Tensor, timesteps: torch.Tensor,
                   class_labels: torch.Tensor | None) -> torch.Tensor:
    """Sinusoidal embedding -> time_embed MLP (+ class embedding): diffusion_model_unet.py:1888-1902.
    Returns fp32 [len(timesteps), 4*C0]; a single timestep broadcasts over the batch in the conv epilogue."""
    if timesteps.ndim != 1:
        raise ValueError("Timesteps should be a 1d-array")
    t = timesteps.to(device=x.device, dtype=torch.float32)
    t_emb = ops.timestep_embedding(t, module.block_out_channels[0])
    l0, l2 = module.time_embed[0], module.time_embed[2]
    emb = ops.small_linear(t_emb, l0.weight, l0.bias, act_out=ACT_SILU)
    emb = ops.small_linear(emb, l2.weight, l2.bias)
    if module.num_class_embeds is not None:
        if class_labels is None:
            raise ValueError("class_labels should be provided when num_class_embeds > 0")
        # nn.Embedding gather of a handful of rows: index_select is allocation plumbing, not arithmetic
        class_emb = module.class_embedding.weight.index_select(0, class_labels.to(x.device).long()).float()
        if class_emb.shape[0] != emb.shape[0]:
            emb = emb.expand(class_emb.shape[0], -1)
        emb = ops.add_f32(emb, class_emb)
    return emb


def _down_path(module: nn.Module, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor | None,
               class_labels: torch.Tensor | None) -> tuple[CL, list[CL], TimeEmb, CL | None]:
    """Time (+ class) embedding, ``conv_in`` and the down blocks of the UNet (diffusion_model_unet.py:1887-1916) and
    of DiffusionModelEncoder (2087-2111) -> (h, skip list, embedding, context rows)."""
    require_cuda(x, module)
    emb = project_time_embedding(module, time_embedding(module, x, timesteps, class_labels))
    if context is not None and module.with_conditioning is False:
        raise ValueError("model should have with_conditioning = True if context is provided")
    ctx = _context_cl(context) if context is not None else None
    h = module.conv_in(ops.to_cl(x))
    down_block_res_samples: list[CL] = [h]
    for downsample_block in module.down_blocks:
        h, res_samples = downsample_block(hidden_states=h, temb=emb, context=ctx)
        down_block_res_samples.extend(res_samples)
    return h, down_block_res_samples, emb, ctx


class DiffusionModelUNet(nn.Module):
    """diffusion_model_unet.py:1646-1943 — same constructor, same forward signature, same state_dict."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int,
                 num_res_blocks: Sequence[int] | int = (2, 2, 2, 2), num_channels: Sequence[int] = (32, 64, 64, 64),
                 attention_levels: Sequence[bool] = (False, False, True, True), norm_num_groups: int = 32,
                 norm_eps: float = 1e-6, resblock_updown: bool = False, num_head_channels: int | Sequence[int] = 8,
                 with_conditioning: bool = False, transformer_num_layers: int = 1,
                 cross_attention_dim: int | None = None, num_class_embeds: int | None = None,
                 upcast_attention: bool = False, use_flash_attention: bool = False,
                 dropout_cattn: float = 0.0, _label_nc: int | None = None,
                 _spade_intermediate_channels: int = 128) -> None:
        super().__init__()
        if with_conditioning is True and cross_attention_dim is None:
            raise ValueError("DiffusionModelUNet expects dimension of the cross-attention conditioning "
                             "(cross_attention_dim) when using with_conditioning.")
        if cross_attention_dim is not None and with_conditioning is False:
            raise ValueError("DiffusionModelUNet expects with_conditioning=True when specifying the "
                             "cross_attention_dim.")
        if dropout_cattn > 1.0 or dropout_cattn < 0.0:
            raise ValueError("Dropout cannot be negative or >1.0!")
        if any((out_channel % norm_num_groups) != 0 for out_channel in num_channels):
            raise ValueError("DiffusionModelUNet expects all num_channels being multiple of norm_num_groups")
        if len(num_channels) != len(attention_levels):
            raise ValueError("DiffusionModelUNet expects num_channels being same size of attention_levels")
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
        # use_flash_attention (xformers) has no meaning here: attention already never materialises more than a
        # bounded score slab; the flag is accepted and ignored.
        self.spatial_dims = spatial_dims
        self.in_channels = in_channels
        self.block_out_channels = num_channels
        self.out_channels = out_channels
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

        self.down_blocks = nn.ModuleList([])
        output_channel = num_channels[0]
        for i in range(len(num_channels)):
            input_channel = output_channel
            output_channel = num_channels[i]
            is_final_block = i == len(num_channels) - 1
            self.down_blocks.append(get_down_block(
                spatial_dims, input_channel, output_channel, time_embed_dim, num_res_blocks[i], norm_num_groups,
                norm_eps, not is_final_block, resblock_updown, attention_levels[i] and not with_conditioning,
                attention_levels[i] and with_conditioning, num_head_channels[i], transformer_num_layers,
                cross_attention_dim, upcast_attention, use_flash_attention, dropout_cattn))

        self.middle_block = get_mid_block(spatial_dims, num_channels[-1], time_embed_dim, norm_num_groups, norm_eps,
                                          with_conditioning, num_head_channels[-1], transformer_num_layers,
                                          cross_attention_dim, upcast_attention, use_flash_attention, dropout_cattn)

        self.up_blocks = nn.ModuleList([])
        rev_ch = list(reversed(num_channels))
        rev_res = list(reversed(num_res_blocks))
        rev_attn = list(reversed(attention_levels))
        rev_heads = list(reversed(num_head_channels))
        output_channel = rev_ch[0]
        for i in range(len(rev_ch)):
            prev_output_channel = output_channel
            output_channel = rev_ch[i]
            input_channel = rev_ch[min(i + 1, len(num_channels) - 1)]
            is_final_block = i == len(num_channels) - 1
            self.up_blocks.append(get_up_block(
                spatial_dims, input_channel, prev_output_channel, output_channel, time_embed_dim, rev_res[i] + 1,
                norm_num_groups, norm_eps, not is_final_block, resblock_updown,
                rev_attn[i] and not with_conditioning, rev_attn[i] and with_conditioning, rev_heads[i],
                transformer_num_layers, cross_attention_dim, upcast_attention, use_flash_attention, dropout_cattn,
                _label_nc, _spade_intermediate_channels))

        self.out = nn.Sequential(
            nn.GroupNorm(num_groups=norm_num_groups, num_channels=num_channels[0], eps=norm_eps, affine=True),
            nn.SiLU(),
            zero_module(Convolution(spatial_dims, num_channels[0], out_channels, strides=1, kernel_size=3,
                                    padding=1)))

    @torch.no_grad()
    def forward(self, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor | None = None,
                class_labels: torch.Tensor | None = None,
                down_block_additional_residuals: tuple[torch.Tensor] | None = None,
                mid_block_additional_residual: torch.Tensor | None = None) -> torch.Tensor:
        return self._forward(x, timesteps, context, class_labels, down_block_additional_residuals,
                             mid_block_additional_residual, None)

    @on_input_device
    def _forward(self, x, timesteps, context, class_labels, down_block_additional_residuals,
                 mid_block_additional_residual, seg):
        h, down_block_res_samples, emb, ctx = _down_path(self, x, timesteps, context, class_labels)
        if down_block_additional_residuals is not None:
            down_block_res_samples = [
                ops.axpy(s, r if isinstance(r, CL) else ops.to_cl(r), 1.0)
                for s, r in zip(down_block_res_samples, down_block_additional_residuals)]
        h = self.middle_block(hidden_states=h, temb=emb, context=ctx)
        if mid_block_additional_residual is not None:
            r = mid_block_additional_residual
            h = ops.axpy(h, r if isinstance(r, CL) else ops.to_cl(r), 1.0)
        for upsample_block in self.up_blocks:
            n = len(upsample_block.resnets)
            res_samples = down_block_res_samples[-n:]
            down_block_res_samples = down_block_res_samples[:-n]
            h = upsample_block(hidden_states=h, res_hidden_states_list=res_samples, temb=emb, context=ctx, seg=seg)
        norm = self.out[0]
        h = ops.groupnorm(h, norm.num_groups, norm.eps, norm.weight, norm.bias, act=ACT_SILU)
        y = self.out[2](h, out_f32=True)
        out = ops.from_cl_f32(y, self.out_channels, self.spatial_dims)
        return out if x.dtype == torch.float32 else out.to(x.dtype)


class DiffusionModelEncoder(nn.Module, _Cached):
    """diffusion_model_unet.py:1946-2115 — the classifier of Wolleb et al. 2022 ("Diffusion Models for Medical Anomaly
    Detection"): the UNet's time embedding and down path followed by ``out = Sequential(Linear(4096, 512), ReLU,
    Dropout(0.1), Linear(512, out_channels))`` on the flattened last feature map.  Same constructor, attributes and
    ``state_dict`` as the reference, including its quirks: every level downsamples, the last one too
    (``is_final_block`` compares ``i`` with ``len(num_channels)``); there is no middle block; the head takes exactly
    4096 features; an integer ``num_res_blocks`` is not expanded (the reference indexes it and raises ``TypeError``).

    Inference only, like every network here: ``forward`` computes no gradients, and a call with grad enabled on an
    ``x`` that requires grad raises ``RuntimeError`` (classifier guidance needs d logits / d x, which this library does
    not compute).  Dropout is never applied, so train mode computes what eval mode does.  CPU tensors raise.

    ``forward`` returns fp32 logits ``[N, out_channels]`` cast to ``x.dtype``.  The head reads the channels-last
    feature map directly: the first Linear's weight columns are permuted once, when packed, from the reference's
    channels-first flattening; Linear + bias + ReLU and Linear + bias run as GEMV (a few samples) or GEMM launches."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int,
                 num_res_blocks: Sequence[int] | int = (2, 2, 2, 2), num_channels: Sequence[int] = (32, 64, 64, 64),
                 attention_levels: Sequence[bool] = (False, False, True, True), norm_num_groups: int = 32,
                 norm_eps: float = 1e-6, resblock_updown: bool = False, num_head_channels: int | Sequence[int] = 8,
                 with_conditioning: bool = False, transformer_num_layers: int = 1,
                 cross_attention_dim: int | None = None, num_class_embeds: int | None = None,
                 upcast_attention: bool = False) -> None:
        super().__init__()
        if with_conditioning is True and cross_attention_dim is None:
            raise ValueError("DiffusionModelEncoder expects dimension of the cross-attention conditioning "
                             "(cross_attention_dim) when using with_conditioning.")
        if cross_attention_dim is not None and with_conditioning is False:
            raise ValueError("DiffusionModelEncoder expects with_conditioning=True when specifying the "
                             "cross_attention_dim.")
        if any((out_channel % norm_num_groups) != 0 for out_channel in num_channels):
            raise ValueError("DiffusionModelEncoder expects all num_channels being multiple of norm_num_groups")
        if len(num_channels) != len(attention_levels):
            raise ValueError("DiffusionModelEncoder expects num_channels being same size of attention_levels")
        if isinstance(num_head_channels, int):
            num_head_channels = ensure_tuple_rep(num_head_channels, len(attention_levels))
        if len(num_head_channels) != len(attention_levels):
            raise ValueError("num_head_channels should have the same length as attention_levels. For the i levels "
                             "without attention, i.e. `attention_level[i]=False`, the num_head_channels[i] will be "
                             "ignored.")
        self.in_channels = in_channels
        self.block_out_channels = num_channels
        self.out_channels = out_channels
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

        self.down_blocks = nn.ModuleList([])
        output_channel = num_channels[0]
        for i in range(len(num_channels)):
            input_channel = output_channel
            output_channel = num_channels[i]
            is_final_block = i == len(num_channels)      # never true: the reference downsamples at every level
            self.down_blocks.append(get_down_block(
                spatial_dims, input_channel, output_channel, time_embed_dim, num_res_blocks[i], norm_num_groups,
                norm_eps, not is_final_block, resblock_updown, attention_levels[i] and not with_conditioning,
                attention_levels[i] and with_conditioning, num_head_channels[i], transformer_num_layers,
                cross_attention_dim, upcast_attention))

        self.out = nn.Sequential(nn.Linear(4096, 512), nn.ReLU(), nn.Dropout(0.1), nn.Linear(512, self.out_channels))

    def forward(self, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor | None = None,
                class_labels: torch.Tensor | None = None) -> torch.Tensor:
        forward_only(type(self).__name__, x)
        with torch.no_grad():
            return self._forward(x, timesteps, context, class_labels)

    @on_input_device
    def _forward(self, x, timesteps, context, class_labels):
        h, _, _, _ = _down_path(self, x, timesteps, context, class_labels)
        fc1, fc2 = self.out[0], self.out[3]
        S = h.spatial
        if S * h.C != fc1.in_features:
            raise RuntimeError(f"mat1 and mat2 shapes cannot be multiplied ({h.N}x{S * h.C} and "
                               f"{fc1.in_features}x{fc1.out_features})")
        pl1 = self._cached(("out.0", h.C, h.pitch, S), (fc1.weight, fc1.bias),
                           lambda: ops.PackedLinear.channels_first_input(fc1.weight, fc1.bias, h.C, h.pitch, S))
        pl2 = self._cached(("out.3",), (fc2.weight, fc2.bias), lambda: ops.PackedLinear(fc2.weight, fc2.bias))
        hidden = _few_rows_linear(ops.as_rows(h.t.reshape(h.N, S * h.pitch), S * h.pitch), pl1, act=ACT_RELU)
        logits = _few_rows_linear(ops.as_rows(hidden.reshape(h.N, -1), fc1.out_features), pl2, out_f32=True)
        out = logits.reshape(h.N, -1)[:, :self.out_channels].contiguous()
        return out if x.dtype == torch.float32 else out.to(x.dtype)

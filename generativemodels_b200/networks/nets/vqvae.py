"""VQVAE on the H100 kernels — classes, arguments and state_dict keys of generative/networks/nets/vqvae.py."""
from __future__ import annotations

from collections.abc import Sequence

import torch
import torch.nn as nn

from ... import _lib, ops
from ...ops import ACT_RELU, CL
from .._holders import Convolution, act_code, on_input_device, require_cuda
from ..layers.vector_quantizer import EMAQuantizer, VectorQuantizer
from .diffusion_model_unet import ensure_tuple_rep

__all__ = ["VQVAE"]


class VQVAEResidualUnit(nn.Module):
    """vqvae.py:27-80: relu(x + conv2(relu(conv1(x)))) — both ReLUs and the add run in the conv epilogues."""

    def __init__(self, spatial_dims: int, num_channels: int, num_res_channels: int, act="RELU", dropout: float = 0.0,
                 bias: bool = True) -> None:
        super().__init__()
        self.spatial_dims, self.num_channels, self.num_res_channels = spatial_dims, num_channels, num_res_channels
        self.act, self.dropout, self.bias = act, dropout, bias
        self.conv1 = Convolution(spatial_dims, num_channels, num_res_channels, bias=bias, conv_only=False, act=act)
        self.conv2 = Convolution(spatial_dims, num_res_channels, num_channels, bias=bias)

    def forward(self, x: CL) -> CL:
        return self.conv2(self.conv1(x), residual=x, act2=ACT_RELU)


class Encoder(nn.Module):
    """vqvae.py:83-170."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int, num_channels: Sequence[int],
                 num_res_layers: int, num_res_channels: Sequence[int], downsample_parameters, dropout: float,
                 act) -> None:
        super().__init__()
        blocks: list[nn.Module] = []
        for i in range(len(num_channels)):
            s, k, d, p = downsample_parameters[i]
            blocks.append(Convolution(spatial_dims, in_channels if i == 0 else num_channels[i - 1], num_channels[i],
                                      strides=s, kernel_size=k, dilation=d, padding=p, conv_only=False, act=act))
            for _ in range(num_res_layers):
                blocks.append(VQVAEResidualUnit(spatial_dims, num_channels[i], num_res_channels[i], act=act,
                                                dropout=dropout))
        blocks.append(Convolution(spatial_dims, num_channels[-1], out_channels, strides=1, kernel_size=3, padding=1))
        self.blocks = nn.ModuleList(blocks)

    def forward(self, x: CL) -> torch.Tensor:
        """-> fp32 channels-last [N, D, H, W, round_up(C, 4)] (the quantiser works in fp32, vector_quantizer.py:102)."""
        for block in self.blocks[:-1]:
            x = block(x)
        return self.blocks[-1](x, out_f32=True)


class Decoder(nn.Module):
    """vqvae.py:173-271."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int, num_channels: Sequence[int],
                 num_res_layers: int, num_res_channels: Sequence[int], upsample_parameters, dropout: float, act,
                 output_act) -> None:
        super().__init__()
        rev_ch = list(reversed(num_channels))
        rev_res = list(reversed(num_res_channels))
        blocks: list[nn.Module] = [Convolution(spatial_dims, in_channels, rev_ch[0], strides=1, kernel_size=3,
                                               padding=1)]
        for i in range(len(num_channels)):
            for _ in range(num_res_layers):
                blocks.append(VQVAEResidualUnit(spatial_dims, rev_ch[i], rev_res[i], act=act, dropout=dropout))
            s, k, d, p, op = upsample_parameters[i]
            last = i == len(num_channels) - 1
            blocks.append(Convolution(spatial_dims, rev_ch[i], out_channels if last else rev_ch[i + 1], strides=s,
                                      kernel_size=k, dilation=d, padding=p, output_padding=op, is_transposed=True,
                                      conv_only=last, act=act))
        if output_act:
            # vqvae.py:263-264 appends Act[output_act]() after the last (conv_only) transposed convolution: here it
            # rides in that convolution's epilogue
            blocks[-1].act = act_code(output_act)
        self.blocks = nn.ModuleList(blocks)

    def forward(self, x: CL) -> CL:
        for block in self.blocks:
            x = block(x)
        return x


class VQVAE(nn.Module):
    """vqvae.py:274-455."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int,
                 num_channels: Sequence[int] | int = (96, 96, 192), num_res_layers: int = 3,
                 num_res_channels: Sequence[int] | int = (96, 96, 192),
                 downsample_parameters=((2, 4, 1, 1), (2, 4, 1, 1), (2, 4, 1, 1)),
                 upsample_parameters=((2, 4, 1, 1, 0), (2, 4, 1, 1, 0), (2, 4, 1, 1, 0)), num_embeddings: int = 32,
                 embedding_dim: int = 64, embedding_init: str = "normal", commitment_cost: float = 0.25,
                 decay: float = 0.5, epsilon: float = 1e-5, dropout: float = 0.0, act="RELU", output_act=None,
                 ddp_sync: bool = True, use_checkpointing: bool = False):
        super().__init__()
        self.in_channels, self.out_channels, self.spatial_dims = in_channels, out_channels, spatial_dims
        self.num_channels, self.num_embeddings, self.embedding_dim = num_channels, num_embeddings, embedding_dim
        self.use_checkpointing = use_checkpointing
        if isinstance(num_res_channels, int):
            num_res_channels = ensure_tuple_rep(num_res_channels, len(num_channels))
        if len(num_res_channels) != len(num_channels):
            raise ValueError("`num_res_channels` should be a single integer or a tuple of integers with the same "
                             "length as `num_channels`.")
        if not all(isinstance(values, (int, Sequence)) for values in downsample_parameters):
            raise ValueError("`downsample_parameters` should be a single tuple of integer or a tuple of tuples.")
        if not all(isinstance(values, (int, Sequence)) for values in upsample_parameters):
            raise ValueError("`upsample_parameters` should be a single tuple of integer or a tuple of tuples.")
        if all(isinstance(values, int) for values in upsample_parameters):
            upsample_parameters = (upsample_parameters,) * len(num_channels)
        if all(isinstance(values, int) for values in downsample_parameters):
            downsample_parameters = (downsample_parameters,) * len(num_channels)
        for parameter in downsample_parameters:
            if len(parameter) != 4:
                raise ValueError("`downsample_parameters` should be a tuple of tuples with 4 integers.")
        for parameter in upsample_parameters:
            if len(parameter) != 5:
                raise ValueError("`upsample_parameters` should be a tuple of tuples with 5 integers.")
        if len(downsample_parameters) != len(num_channels):
            raise ValueError("`downsample_parameters` should be a tuple of tuples with the same length as "
                             "`num_channels`.")
        if len(upsample_parameters) != len(num_channels):
            raise ValueError("`upsample_parameters` should be a tuple of tuples with the same length as "
                             "`num_channels`.")
        self.num_res_layers = num_res_layers
        self.num_res_channels = num_res_channels
        self.encoder = Encoder(spatial_dims, in_channels, embedding_dim, num_channels, num_res_layers,
                               num_res_channels, downsample_parameters, dropout, act)
        self.decoder = Decoder(spatial_dims, embedding_dim, out_channels, num_channels, num_res_layers,
                               num_res_channels, upsample_parameters, dropout, act, output_act)
        self.quantizer = VectorQuantizer(quantizer=EMAQuantizer(
            spatial_dims=spatial_dims, num_embeddings=num_embeddings, embedding_dim=embedding_dim,
            commitment_cost=commitment_cost, decay=decay, epsilon=epsilon, embedding_init=embedding_init,
            ddp_sync=ddp_sync))

    # ---- channels-last internals -----------------------------------------------------------------
    def _encode_cl(self, images: torch.Tensor) -> torch.Tensor:
        require_cuda(images, self)
        return self.encoder(ops.to_cl(images))

    def _z_to_nchw(self, z: torch.Tensor) -> torch.Tensor:
        return ops.from_cl_f32(z, self.embedding_dim, self.spatial_dims)

    def _decode_cl(self, q: CL) -> torch.Tensor:
        return ops.from_cl(self.decoder(q))

    # ---- reference interface (vqvae.py:417-455) --------------------------------------------------
    @on_input_device
    @torch.no_grad()
    def encode(self, images: torch.Tensor) -> torch.Tensor:
        return self._z_to_nchw(self._encode_cl(images))

    def quantize(self, encodings: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        x_loss, x = self.quantizer(encodings)
        return x, x_loss

    @on_input_device
    @torch.no_grad()
    def decode(self, quantizations: torch.Tensor) -> torch.Tensor:
        require_cuda(quantizations, self)
        return self._decode_cl(ops.to_cl(quantizations))

    @on_input_device
    @torch.no_grad()
    def index_quantize(self, images: torch.Tensor) -> torch.Tensor:
        r = self.quantizer.forward_cl(self._encode_cl(images), want_f32=False)
        return self.quantizer.quantizer._indices_view(r["indices"])

    @on_input_device
    @torch.no_grad()
    def decode_samples(self, embedding_indices: torch.Tensor) -> torch.Tensor:
        require_cuda(embedding_indices, self)
        lib = _lib.require_device()
        q = self.quantizer.quantizer
        idx = embedding_indices.long().contiguous()
        dims = (1, *idx.shape[1:]) if self.spatial_dims == 2 else tuple(idx.shape[1:])
        out = ops.new_cl(idx.shape[0], dims, self.embedding_dim, idx.device, self.spatial_dims)
        cb = q.embedding.weight.detach().float().contiguous()
        _lib.check(lib.b200_vq_gather(idx.data_ptr(), idx.numel(), cb.data_ptr(), q.num_embeddings, self.embedding_dim,
                                      out.t.data_ptr(), out.pitch, ops._stream()),
                   "b200_vq_gather")
        return self._decode_cl(out)

    @on_input_device
    @torch.no_grad()
    def forward(self, images: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        if self.training:
            raise RuntimeError("VQVAE.forward on the H100 kernels is inference-only; call .eval() first")
        r = self.quantizer.forward_cl(self._encode_cl(images), want_f32=False)
        return self._decode_cl(r["q"]), r["loss"]

    @on_input_device
    @torch.no_grad()
    def encode_stage_2_inputs(self, x: torch.Tensor, quantized: bool = True) -> torch.Tensor:
        z = self._encode_cl(x)
        if not quantized:
            return self._z_to_nchw(z)
        r = self.quantizer.forward_cl(z, want_f32=True)
        return ops.from_cl_f32(r["q_f32"].contiguous(), self.embedding_dim, self.spatial_dims)

    @on_input_device
    @torch.no_grad()
    def decode_stage_2_outputs(self, z: torch.Tensor) -> torch.Tensor:
        """Re-quantises the latent before decoding (vqvae.py:452-455)."""
        require_cuda(z, self)
        q = self.quantizer.quantizer
        zc = q._z_channels_last(z)
        r = self.quantizer.forward_cl(zc, want_f32=False)
        return self._decode_cl(r["q"])

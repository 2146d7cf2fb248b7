"""SABlock — ``generative/networks/blocks/selfattention.py:33-148`` on the H100 kernels: multi-head (causal) self- or
cross-attention with bias-free q / k / v projections and an output projection.  Token rows stay packed
[B*T, hidden]; heads are channel slices, the causal mask is an index comparison inside the attention kernel (the
``causal_mask`` buffer is kept only so that reference state_dicts load strictly)."""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from ... import ops
from ...ops import CL
from .._holders import packed_linear


class SABlock(nn.Module):
    def __init__(self, hidden_size: int, num_heads: int, dropout_rate: float = 0.0, qkv_bias: bool = False,
                 causal: bool = False, sequence_length: int | None = None, with_cross_attention: bool = False,
                 use_flash_attention: bool = False) -> None:
        super().__init__()
        self.hidden_size, self.num_heads = hidden_size, num_heads
        self.head_dim = hidden_size // num_heads
        self.scale = 1.0 / math.sqrt(self.head_dim)
        self.causal, self.sequence_length = causal, sequence_length
        self.with_cross_attention = with_cross_attention
        self.use_flash_attention = use_flash_attention          # xformers switch of the reference: no meaning here
        if not (0 <= dropout_rate <= 1):
            raise ValueError("dropout_rate should be between 0 and 1.")
        self.dropout_rate = dropout_rate
        if hidden_size % num_heads != 0:
            raise ValueError("hidden size should be divisible by num_heads.")
        if causal and sequence_length is None:
            raise ValueError("sequence_length is necessary for causal attention.")
        self.to_q = nn.Linear(hidden_size, hidden_size, bias=qkv_bias)
        self.to_k = nn.Linear(hidden_size, hidden_size, bias=qkv_bias)
        self.to_v = nn.Linear(hidden_size, hidden_size, bias=qkv_bias)
        self.drop_weights = nn.Dropout(dropout_rate)
        self.drop_output = nn.Dropout(dropout_rate)
        self.out_proj = nn.Linear(hidden_size, hidden_size)
        if causal and sequence_length is not None:
            self.register_buffer("causal_mask", torch.tril(torch.ones(sequence_length, sequence_length)).view(
                1, 1, sequence_length, sequence_length))

    # ------------------------------------------------------------------------------------------
    def project_kv(self, rows: CL) -> tuple[CL, CL]:
        return ops.linear(rows, packed_linear(self, "to_k")), ops.linear(rows, packed_linear(self, "to_v"))

    def attend(self, x: CL, B: int, T: int, k: torch.Tensor, v: torch.Tensor, S: int, q_pos0: int,
               residual: CL | None, pos_dev: torch.Tensor | None = None) -> CL:
        """x: rows [B*T, hidden]; k, v: [B, rows >= S, pitch] (a cache or fresh projections); with ``pos_dev`` the
        prefix length is read on the device instead of (S, q_pos0)."""
        q = ops.linear(x, packed_linear(self, "to_q")).t.reshape(B, T, -1)
        o = ops.attention_causal(q, k, v, self.num_heads, self.head_dim, self.scale, S, causal=self.causal,
                                 q_pos0=q_pos0, pos_dev=pos_dev)
        return ops.linear(ops.as_rows(o, self.hidden_size), packed_linear(self, "out_proj"), residual=residual)

    def forward(self, x: CL, B: int, T: int, context: CL | None = None, context_len: int = 0,
                residual: CL | None = None) -> CL:
        """Full-sequence form (selfattention.py:101-148): rows of B sequences of T tokens; ``context`` rows of B
        sequences of ``context_len`` tokens for cross-attention."""
        kv, S = (x, T) if context is None else (context, context_len)
        k, v = self.project_kv(kv)
        return self.attend(x, B, T, k.t.reshape(B, S, -1), v.t.reshape(B, S, -1), S, 0, residual)

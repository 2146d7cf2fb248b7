"""DecoderOnlyTransformer — ``generative/networks/nets/transformer.py:20-106`` on the H100 kernels (SURVEY.md §8f rank 3).

Same constructor, ``forward(x, context)`` -> logits [B, T, num_tokens] (fp32) and state_dict keys as the reference.
Beyond that interface the class offers the incremental form the sampler wants: ``new_cache`` / ``step`` keep every
layer's keys and values of the tokens seen so far (the reference recomputes the whole prefix for every new token,
inferer.py:1219-1225 — O(n^3) over a sequence; with the cache each step is one row through the GEMMs plus attention of
one query over the cached keys).  Absolute position embeddings make the cache valid only while the sequence still
fits ``max_seq_len`` (after that the window slides and every position changes); ``step`` refuses beyond that and the
inferer falls back to the full forward, exactly the reference's behaviour.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ... import cuda_graph, ops
from ...ops import CL
from .._holders import f32, packed_linear, on_input_device, require_cuda
from ..blocks.transformerblock import TransformerBlock

__all__ = ["DecoderOnlyTransformer", "AbsolutePositionalEmbedding"]


class AbsolutePositionalEmbedding(nn.Module):
    """nets/transformer.py:20-37 (a learnt table indexed by position; used through the fused embedding kernel)."""

    def __init__(self, max_seq_len: int, embedding_dim: int) -> None:
        super().__init__()
        self.max_seq_len = max_seq_len
        self.embedding_dim = embedding_dim
        self.embedding = nn.Embedding(max_seq_len, embedding_dim)


class _Cache:
    """Keys / values of the tokens processed so far, per layer: h16 [B, max_seq_len, pitch]; cross-attention keys
    and values of the conditioning are projected once."""

    def __init__(self, model: "DecoderOnlyTransformer", batch: int, device, context: torch.Tensor | None,
                 graph: bool = False):
        # ``graph``: single-token steps are captured once in a CUDA graph and replayed (the prefix length then lives
        # in device memory, ``pos_dev``); the first two single-token steps run eagerly as the capture's warm-up
        self.use_graph = graph
        self.pos_dev = torch.zeros(1, dtype=torch.int32, device=device)
        self.graph = None
        self.static_tokens = None
        self.static_logits = None
        self.dyn_steps = 0
        P = ops.round_up(model.attn_layers_dim, 8)
        mk = lambda: torch.zeros((batch, model.max_seq_len, P), dtype=ops.H16, device=device)
        self.k = [mk() for _ in model.blocks]
        self.v = [mk() for _ in model.blocks]
        self.length = 0
        self.batch = batch
        self.cross = None
        self.context_len = 0
        if model.with_cross_attention:
            if context is None:
                raise ValueError("this transformer was built with cross attention: a context is required")
            ctx = ops.as_rows(ops.to_cl(context.permute(0, 2, 1).unsqueeze(2).contiguous()).t, context.shape[2])
            self.context_len = context.shape[1]
            self.cross = []
            for blk in model.blocks:
                k, v = blk.cross_attn.project_kv(ctx)
                self.cross.append((k.t.reshape(batch, self.context_len, -1), v.t.reshape(batch, self.context_len, -1)))


class DecoderOnlyTransformer(nn.Module):
    def __init__(self, num_tokens: int, max_seq_len: int, attn_layers_dim: int, attn_layers_depth: int,
                 attn_layers_heads: int, with_cross_attention: bool = False, embedding_dropout_rate: float = 0.0,
                 use_flash_attention: bool = False) -> None:
        super().__init__()
        self.num_tokens = num_tokens
        self.max_seq_len = max_seq_len
        self.attn_layers_dim = attn_layers_dim
        self.attn_layers_depth = attn_layers_depth
        self.attn_layers_heads = attn_layers_heads
        self.with_cross_attention = with_cross_attention
        self.token_embeddings = nn.Embedding(num_tokens, attn_layers_dim)
        self.position_embeddings = AbsolutePositionalEmbedding(max_seq_len=max_seq_len, embedding_dim=attn_layers_dim)
        self.embedding_dropout = nn.Dropout(embedding_dropout_rate)
        self.blocks = nn.ModuleList([
            TransformerBlock(hidden_size=attn_layers_dim, mlp_dim=attn_layers_dim * 4, num_heads=attn_layers_heads,
                             dropout_rate=0.0, qkv_bias=False, causal=True, sequence_length=max_seq_len,
                             with_cross_attention=with_cross_attention, use_flash_attention=use_flash_attention)
            for _ in range(attn_layers_depth)])
        self.to_logits = nn.Linear(attn_layers_dim, num_tokens)

    # ------------------------------------------------------------------------------------------
    def _embed(self, x: torch.Tensor, pos0: int) -> CL:
        return ops.embed_tokens(x, f32(self.token_embeddings.weight), f32(self.position_embeddings.embedding.weight),
                                pos0)

    def _logits(self, h: CL, B: int, T: int) -> torch.Tensor:
        y = ops.linear(h, packed_linear(self, "to_logits"), out_f32=True)
        return y.reshape(B, T, -1)[:, :, : self.num_tokens]

    @on_input_device
    @torch.no_grad()
    def forward(self, x: torch.Tensor, context: torch.Tensor | None = None) -> torch.Tensor:
        require_cuda(x, self)
        B, T = x.shape
        if T > self.max_seq_len:
            raise IndexError(f"sequence of {T} tokens exceeds max_seq_len {self.max_seq_len}")
        ctx, ctx_len = None, 0
        if self.with_cross_attention:
            if context is None:
                raise ValueError("this transformer was built with cross attention: a context is required")
            ctx = ops.as_rows(ops.to_cl(context.permute(0, 2, 1).unsqueeze(2).contiguous()).t, context.shape[2])
            ctx_len = context.shape[1]
        h = self._embed(x, 0)
        for blk in self.blocks:
            h = blk(h, B, T, context=ctx, context_len=ctx_len)
        return self._logits(h, B, T)

    # ---- incremental decoding -------------------------------------------------------------------
    def new_cache(self, batch: int, device, context: torch.Tensor | None = None, graph: bool = False) -> _Cache:
        return _Cache(self, batch, device, context, graph)

    def _step_dyn(self, x: torch.Tensor, cache: _Cache) -> torch.Tensor:
        """One single-token step whose only notion of "where" is ``cache.pos_dev`` in device memory: the same kernel
        sequence serves every position, which is what lets it be captured in a CUDA graph."""
        B = x.shape[0]
        pos = cache.pos_dev
        h = ops.embed_tokens(x, f32(self.token_embeddings.weight), f32(self.position_embeddings.embedding.weight),
                             pos_dev=pos)
        if B <= 8:
            return self._step_rows(h.t.reshape(B, -1), cache)
        for i, blk in enumerate(self.blocks):
            n1 = blk._ln(blk.norm1, h)
            k, v = blk.attn.project_kv(n1)
            ops.cache_append(k.t, cache.k[i], 1, pos)
            ops.cache_append(v.t, cache.v[i], 1, pos)
            h = blk.attn.attend(n1, B, 1, cache.k[i], cache.v[i], 1, 0, residual=h, pos_dev=pos)
            if self.with_cross_attention:
                ck, cv = cache.cross[i]
                h = blk.cross_attn.attend(blk._ln(blk.norm2, h), B, 1, ck, cv, cache.context_len, 0, residual=h)
            h = blk.mlp(blk._ln(blk.norm3, h), residual=h)
        logits = self._logits(h, B, 1)
        ops.advance_i32(pos, 1)
        return logits

    def _step_rows(self, h: torch.Tensor, cache: _Cache) -> torch.Tensor:
        """The same step for at most 8 sequences: every linear layer is a GEMV (b200_rows_linear, LayerNorm fused into
        its prologue, GELU / residual into its epilogue) and attention is one query per (sequence, head) over the
        cache (b200_attention_decode) — ~9 small launches per layer instead of 128-row tensor-core tiles."""
        B, C_ = h.shape[0], self.attn_layers_dim
        pos = cache.pos_dev
        for i, blk in enumerate(self.blocks):
            a = blk.attn
            ln1 = (f32(blk.norm1.weight), f32(blk.norm1.bias), blk.norm1.eps)
            q = ops.rows_linear(h, C_, packed_linear(a, "to_q"), ln=ln1)
            k = ops.rows_linear(h, C_, packed_linear(a, "to_k"), ln=ln1)
            v = ops.rows_linear(h, C_, packed_linear(a, "to_v"), ln=ln1)
            ops.cache_append(k, cache.k[i], 1, pos)
            ops.cache_append(v, cache.v[i], 1, pos)
            o = ops.attention_decode(q, cache.k[i], cache.v[i], a.num_heads, a.head_dim, a.scale, 1, pos_dev=pos)
            h = ops.rows_linear(o, C_, packed_linear(a, "out_proj"), residual=h)
            if self.with_cross_attention:
                c = blk.cross_attn
                ck, cv = cache.cross[i]
                ln2 = (f32(blk.norm2.weight), f32(blk.norm2.bias), blk.norm2.eps)
                q = ops.rows_linear(h, C_, packed_linear(c, "to_q"), ln=ln2)
                o = ops.attention_decode(q, ck, cv, c.num_heads, c.head_dim, c.scale, cache.context_len)
                h = ops.rows_linear(o, C_, packed_linear(c, "out_proj"), residual=h)
            ln3 = (f32(blk.norm3.weight), f32(blk.norm3.bias), blk.norm3.eps)
            m = ops.rows_linear(h, C_, packed_linear(blk.mlp, "linear1"), ln=ln3, act=ops.ACT_GELU)
            h = ops.rows_linear(m, blk.mlp.linear1.out_features, packed_linear(blk.mlp, "linear2"), residual=h)
        logits = ops.rows_linear(h, C_, packed_linear(self, "to_logits"), out_f32=True)
        ops.advance_i32(pos, 1)
        return logits[:, : self.num_tokens].reshape(B, 1, self.num_tokens)

    def _step_graph(self, x: torch.Tensor, cache: _Cache) -> torch.Tensor:
        if cache.graph is None:
            if cache.dyn_steps < 2:                         # real steps that double as the capture's warm-up
                cache.dyn_steps += 1
                return self._step_dyn(x.long().contiguous(), cache)
            cache.static_tokens = x.long().contiguous().clone()
            torch.cuda.synchronize()
            cache.graph = torch.cuda.CUDAGraph()
            with cuda_graph.capture(cache.graph):
                cache.static_logits = self._step_dyn(cache.static_tokens, cache)
        cache.static_tokens.copy_(x, non_blocking=True)
        cache.graph.replay()
        return cache.static_logits

    @on_input_device
    @torch.no_grad()
    def step(self, x: torch.Tensor, cache: _Cache) -> torch.Tensor:
        """Logits [B, T_new, num_tokens] of ``x`` ([B, T_new] tokens that extend the cached prefix), identical to the
        last T_new rows of ``forward`` on the whole sequence.  (With a graph cache the returned tensor of a
        single-token step is a static buffer, valid until the next step.)"""
        require_cuda(x, self)
        B, T = x.shape
        L = cache.length
        if B != cache.batch or L + T > self.max_seq_len:
            raise IndexError("key/value cache exhausted: the sequence no longer fits max_seq_len")
        if cache.use_graph and T == 1:
            cache.length = L + 1
            return self._step_graph(x, cache)
        h = self._embed(x, L)
        for i, blk in enumerate(self.blocks):
            n1 = blk._ln(blk.norm1, h)
            ops.linear_into_cache(n1, B, T, packed_linear(blk.attn, "to_k"), cache.k[i], L)
            ops.linear_into_cache(n1, B, T, packed_linear(blk.attn, "to_v"), cache.v[i], L)
            h = blk.attn.attend(n1, B, T, cache.k[i], cache.v[i], L + T, L, residual=h)
            if self.with_cross_attention:
                ck, cv = cache.cross[i]
                h = blk.cross_attn.attend(blk._ln(blk.norm2, h), B, T, ck, cv, cache.context_len, 0, residual=h)
            h = blk.mlp(blk._ln(blk.norm3, h), residual=h)
        cache.length = L + T
        if cache.use_graph:
            cache.pos_dev.fill_(L + T)                       # keep the device-side position in step with eager steps
        return self._logits(h, B, T)

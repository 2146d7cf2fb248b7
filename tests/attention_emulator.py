"""Float64 reading of the attention entry points of include/b200gen.h (CPU only; test infrastructure).

One function per entry point.  Each takes flat host tensors laid out as the C ABI describes them (row pitches, key /
value caches of kv_rows rows per batch item, V transposed for the tensor-core kernels, a residual with its own pitch)
and returns a Result: the float64 value before the final 16-bit rounding (`exact`), the rounded value (`out`) and the
accuracy term of the bound (`err`).  Each function mirrors the rounding its kernel documents, so the differences left
between a correct kernel and `out` are fp32 accumulation order, `ex2.approx` / `__expf`, and the last-bit rounding
of the store:

  flash (head_dim 64..256)  sigma_s = c q.k with c = fp32(scale * fp32(log2 e)); the running row maximum m_blk(s)
                            advances once per 64-key block; P~_s = h16(fp32(2^(sigma_s - m_blk(s)))) (ex2.approx.ftz:
                            below 2^-126 is 0); l = sum_s 2^(sigma_s - m_T) from the UNROUNDED p (m_T = final max);
                            out = h16((sum_s P~_s 2^(m_blk(s) - m_T) v_s) / l + res), the residual added in fp32
                            before the single rounding.
  flash (head_dim 512)      the same with 128-key blocks (both consumers share the maximum over the whole block).
  unfused (ops.attention)   fp32 scores; P = h16(exp(s - max) / sum), normalised before rounding; P V in fp32 + res,
                            one rounding.
  attention_small(_ex)      fp32 throughout, nothing rounded but the output; the causal horizon s <= q_pos0 + t,
  attention_decode          kv_rows, and pos_dev (q_pos0 = *pos, S = *pos + T; decode: S = *pos + 1).
  softmax_rows(_partials)   p = h16(fp32(exp(s - max) * (1 / sum))); pad columns [S, p_pitch) are +0.

16-bit rounding goes through fp32 (`.to(torch.float32).to(H16)`), as the kernels round their fp32 values with RN; a
direct float64 -> 16-bit conversion can round differently.  fp16 stores saturate at +-65504 (cvt.rn.satfinite).

Value bound, per output element (tolerance()):

    |got - want| <= ulp16(max(|got|, |want|)) + err + REL (|want| + floor)

with REL = 2^-17 for the fp32 rounding of the final additions, floor = 1 for attention and 0 for the softmax rows,
and err = (sum_s w_s |v_s|) / l built from:

  eps_s   relative error of the kernel's p_s.  The score q.k is an fp32 sum of exactly representable 16-bit products:
          within ACC |scale| sum_c |q_c k_c| with ACC = 2^-16 on the tensor cores (the bound tests/
          test_igemm_contract_gpu.py holds wgmma to) and 2^-17 on the CUDA cores (a <= 32-term fma chain and a 5-level
          warp tree); an absolute score error d moves p by a factor e^d, so ACC |scale| sum|q k| is also p's relative
          error (for flash: ln 2 * c = scale).  fp32 rounding of the scaled score and of the max subtraction adds
          2^-23 ln2 (|sigma_s| + |m|) (flash; 2^-22 (|s| + |m|) on the CUDA cores), ex2.approx 2^-22 and the fp32 p
          another 2^-24: 2^-21 covers both.  __expf(x) is within (2 + 1.2 |x|) ulp; the CUDA-core kernels re-scale
          their running sums at every new maximum, adding (2 n_inc + 16 + 2.4 (m - min s)) 2^-24 for n_inc increases.
  fragile the kernel rounds P~ from its own fp32 p.  Where p (1 - eps) and p (1 + eps) round to different 16-bit
          values, the kernel may land on the neighbour: that key gets its rounding step |h16(p(1+eps)) -
          h16(p(1-eps))| 2^(m_blk - m_T) as extra weight.
  acc     fp32 accumulation of l and of sum p v: 2^-17 + (S + 64) 2^-24 relative on the tensor cores, (2 S + 40) 2^-24
          on the CUDA cores.

An error in p_s moves both the numerator and l, so the eps term is sum_s eps_s p_s (|v_s| + |o|) / l.  With fp16 the
bound is one to a few output ulps; a key of weight 1/1000 dropped, a zero-filled key counted in l, or a late rescale
is several times over it (tests/test_attention_emulator_cpu.py shows each such mutant failing it).
"""
from __future__ import annotations

import contextlib
import math
from dataclasses import dataclass

import numpy as np
import torch

from generativemodels_b200._lib import ACT_DTYPE

F64 = torch.float64
LN2 = math.log(2.0)
ACC_TC, ACC_CC = 2.0 ** -16, 2.0 ** -17
REL = 2.0 ** -17
FTZ = 2.0 ** -126

H16 = torch.float16 if ACT_DTYPE == "fp16" else torch.bfloat16


@contextlib.contextmanager
def storage(dtype):
    """Emulate the library flavour whose 16-bit type is `dtype` (torch.float16 or torch.bfloat16) inside the block."""
    global H16
    old, H16 = H16, dtype
    try:
        yield
    finally:
        H16 = old


def _mant():
    return 10 if H16 is torch.float16 else 7


def f32(x):
    return x.to(torch.float32).to(F64)


def h16(x):
    """fp32 -> 16-bit with round-to-nearest-even, as the kernels store; fp16 saturates at +-65504."""
    x = x.to(torch.float32)
    if H16 is torch.float16:
        x = x.clamp(-65504.0, 65504.0)
    return x.to(H16).to(F64)


def ulp16(x):
    emin = -14 if H16 is torch.float16 else -126
    m = x.abs().clamp_min(2.0 ** emin)
    return torch.exp2(torch.floor(torch.log2(m)) - _mant())


@dataclass
class Result:
    exact: torch.Tensor       # float64 before the final 16-bit rounding
    out: torch.Tensor         # the rounded result, as float64
    err: torch.Tensor         # accuracy term of the bound (see the module docstring)
    floor: float = 1.0


def tolerance(r: Result, got: torch.Tensor) -> torch.Tensor:
    return ulp16(torch.maximum(got.abs(), r.out.abs())) + r.err + REL * (r.out.abs() + r.floor)


def excess(r: Result, got: torch.Tensor) -> torch.Tensor:
    """err / tolerance per element (> 1 is outside the bound; a NaN or inf that the emulator does not have is inf)."""
    got = got.to(F64)
    ratio = (got - r.out).abs() / tolerance(r, got)
    bad = ~torch.isfinite(got) & torch.isfinite(r.out)
    return torch.where(bad, torch.full_like(ratio, math.inf), ratio.nan_to_num(0.0))


def fp32_scale_log2e(scale: float) -> float:
    """The kernel's score multiplier: scale * log2(e), one fp32 product computed on the host."""
    return float(np.float32(scale) * np.float32(1.4426950408889634))


# ----------------------------------------------------------------------------------------------------------------
# one (batch, head): Q [T, d], K [S, d], V [S, dv] float64 -> attention without residual and its err term
# ----------------------------------------------------------------------------------------------------------------
def flash_head(Q, K, V, scale, block):
    """The flash kernels' arithmetic; returns a dict with o, err and the per-key pieces (p, l, ptil, m_blk, m_T)."""
    T, S = Q.shape[0], K.shape[0]
    dot, mag = Q @ K.T, Q.abs() @ K.abs().T
    sig = fp32_scale_log2e(scale) * dot
    nb = -(-S // block)
    padded = torch.full((T, nb * block), -math.inf, dtype=F64)
    padded[:, :S] = sig
    mb = padded.view(T, nb, block).amax(2).cummax(1).values          # running max after each key block
    m_blk = mb.repeat_interleave(block, 1)[:, :S]
    m_T = mb[:, -1:]
    pb = torch.exp2(sig - m_blk)
    p32 = f32(pb)
    p32[p32 < FTZ] = 0.0                                              # ex2.approx.ftz
    down = torch.exp2(m_blk - m_T)
    ptil = h16(p32) * down
    p = torch.exp2(sig - m_T)
    l = p.sum(1, keepdim=True)
    o = ptil @ V / l
    eps = abs(scale) * ACC_TC * mag + LN2 * 2.0 ** -23 * (sig.abs() + m_T.abs()) + 2.0 ** -21
    frag = (h16(pb * (1 + eps)) - h16(pb * (1 - eps))).abs() * down
    acc = 2.0 ** -17 + (S + 64) * 2.0 ** -24
    aV, ep = V.abs(), eps * p
    err = (ep @ aV + ep.sum(1, keepdim=True) * o.abs() + frag @ aV + acc * (p @ aV + l * o.abs())) / l
    return dict(o=o, err=err, p=p, l=l, ptil=ptil, m_blk=m_blk, m_T=m_T)


def unfused_head(Q, K, V, scale):
    """Score GEMM (fp32) -> row softmax normalised before the 16-bit rounding -> P V GEMM (fp32)."""
    S = K.shape[0]
    dot, mag = Q @ K.T, Q.abs() @ K.abs().T
    s = f32(scale * dot)
    m = s.amax(1, keepdim=True)
    e = torch.exp(s - m)
    e[e < FTZ] = 0.0                                                  # __expf flushes to zero
    tot = e.sum(1, keepdim=True)
    Pex = e / tot
    P = h16(Pex)
    o = P @ V
    eps = abs(scale) * ACC_TC * mag + 2.0 ** -22 * (s.abs() + m.abs()) + (2 + 1.2 * (s - m).abs()) * 2.0 ** -24
    eps = eps + (eps * Pex).sum(1, keepdim=True) + (S + 64) * 2.0 ** -24 + 2.0 ** -22
    frag = (h16(Pex * (1 + eps)) - h16(Pex * (1 - eps))).abs()
    aV = V.abs()
    err = (eps * Pex) @ aV + frag @ aV + (2.0 ** -17 + (S + 64) * 2.0 ** -24) * (P @ aV)
    return dict(o=o, err=err, P=P)


def fp32_head(Q, K, V, scale, end=None, chain=None):
    """The CUDA-core online softmax: fp32 throughout.  end[t] = keys row t sees (causal horizon), None = all;
    chain = re-scales of the running sums per row (None: count the running-max increases of a sequential scan)."""
    T, S = Q.shape[0], K.shape[0]
    s = scale * (Q @ K.T)
    mag = Q.abs() @ K.abs().T
    valid = torch.ones(T, S, dtype=torch.bool) if end is None else torch.arange(S)[None, :] < end[:, None]
    s = torch.where(valid, s, -math.inf)
    m = s.amax(1, keepdim=True)
    p = torch.exp(s - m)
    l = p.sum(1, keepdim=True)
    o = p @ V / l
    smin = torch.where(valid, s, math.inf).amin(1, keepdim=True)
    if chain is None:
        cm = s.cummax(1).values
        chain = ((s[:, 1:] > cm[:, :-1]) & valid[:, 1:]).sum(1, keepdim=True).to(F64)
    n = valid.sum(1, keepdim=True).to(F64)
    d = torch.where(valid, (s - m).abs(), 0.0)
    eps = (abs(scale) * ACC_CC * mag + 2.0 ** -22 * (d + m.abs()) + (2 + 1.2 * d) * 2.0 ** -24
           + (2 * chain + 16 + 2.4 * (m - smin)) * 2.0 ** -24)
    acc = (2 * n + 40) * 2.0 ** -24
    aV, ep = V.abs(), torch.where(valid, eps * p, 0.0)
    err = (ep @ aV + ep.sum(1, keepdim=True) * o.abs() + acc * (p @ aV + l * o.abs())) / l
    return dict(o=o, err=err, p=p, l=l)


# ----------------------------------------------------------------------------------------------------------------
# the entry points
# ----------------------------------------------------------------------------------------------------------------
def _rows(buf, row0, n, pitch):
    """Rows [row0, row0 + n) of a flat buffer of `pitch`-element rows, as a 2-D view."""
    return buf[row0 * pitch:(row0 + n) * pitch].view(n, pitch)


def _finish(exact, err, res_rows=None):
    if res_rows is not None:
        exact = exact + res_rows
    return Result(exact, h16(exact), err)


def _tensor_core(head_fn, q, k, vt, res, B, T, S, heads, dh, q_pitch, k_pitch, vt_pitch, res_pitch, rows):
    C = heads * dh
    rows = torch.arange(T) if rows is None else torch.as_tensor(rows)
    exact = torch.zeros(B, len(rows), C, dtype=F64)
    err = torch.zeros_like(exact)
    for b in range(B):
        Qb = _rows(q, b * T, T, q_pitch)[rows]
        Kb = _rows(k, b * S, S, k_pitch)
        for h in range(heads):
            cs = slice(h * dh, (h + 1) * dh)
            V = _rows(vt, b * C + h * dh, dh, vt_pitch)[:, :S].T.to(F64)
            r = head_fn(Qb[:, cs].to(F64), Kb[:, cs].to(F64), V)
            exact[b, :, cs], err[b, :, cs] = r["o"], r["err"]
    R = None
    if res is not None:
        R = torch.stack([_rows(res, b * T, T, res_pitch)[rows, :C].to(F64) for b in range(B)])
    return _finish(exact, err, R)


def flash(q, k, vt, res, B, T, S, heads, dh, q_pitch, k_pitch, vt_pitch, res_pitch, scale, rows=None):
    """b200_attention_flash: q [B][T][q_pitch], k [B][S][k_pitch], vt [B][heads*dh][vt_pitch], res [B][T][res_pitch]
    or None.  Returns [B, len(rows), heads*dh] (rows: the query rows to emulate, default all)."""
    block = 128 if dh == 512 else 64
    fn = lambda Q, K, V: flash_head(Q, K, V, scale, block)
    return _tensor_core(fn, q, k, vt, res, B, T, S, heads, dh, q_pitch, k_pitch, vt_pitch, res_pitch, rows)


def unfused(q, k, vt, res, B, T, S, heads, dh, q_pitch, k_pitch, vt_pitch, res_pitch, scale, rows=None):
    """ops.attention's score GEMM + softmax_rows_partials + PV GEMM path, same layout as flash()."""
    fn = lambda Q, K, V: unfused_head(Q, K, V, scale)
    return _tensor_core(fn, q, k, vt, res, B, T, S, heads, dh, q_pitch, k_pitch, vt_pitch, res_pitch, rows)


def small(q, k, v, B, T, S, heads, dh, q_pitch, k_pitch, v_pitch, scale, kv_rows=None, causal=0, q_pos0=0, pos=None):
    """b200_attention_small(_ex): q [B][T][q_pitch]; k, v [B][kv_rows][pitch] (S valid rows); pos = *pos_dev or None.
    Returns [B, T, heads*dh]."""
    if pos is not None:
        q_pos0, S = pos, pos + T
    kv_rows = S if kv_rows is None else kv_rows
    C = heads * dh
    end = torch.clamp(q_pos0 + torch.arange(T) + 1, max=S) if causal else None
    exact = torch.zeros(B, T, C, dtype=F64)
    err = torch.zeros_like(exact)
    for b in range(B):
        Qb, Kb, Vb = _rows(q, b * T, T, q_pitch), _rows(k, b * kv_rows, S, k_pitch), _rows(v, b * kv_rows, S, v_pitch)
        for h in range(heads):
            cs = slice(h * dh, (h + 1) * dh)
            r = fp32_head(Qb[:, cs].to(F64), Kb[:, cs].to(F64), Vb[:, cs].to(F64), scale, end)
            exact[b, :, cs], err[b, :, cs] = r["o"], r["err"]
    return _finish(exact, err)


def decode(q, k, v, B, S, heads, dh, q_pitch, k_pitch, v_pitch, scale, kv_rows, pos=None):
    """b200_attention_decode: one query row per batch item (q [B][q_pitch]) over S keys of [B][kv_rows][pitch] caches
    (S = *pos + 1 with pos given).  The keys are split over 8 warps whose states are merged.  Returns [B, heads*dh]."""
    if pos is not None:
        S = pos + 1
    C = heads * dh
    chain = torch.full((1, 1), float(-(-S // 8) + 8), dtype=F64)      # per-warp re-scales + the 8-way merge
    exact = torch.zeros(B, C, dtype=F64)
    err = torch.zeros_like(exact)
    for b in range(B):
        Qb, Kb, Vb = _rows(q, b, 1, q_pitch), _rows(k, b * kv_rows, S, k_pitch), _rows(v, b * kv_rows, S, v_pitch)
        for h in range(heads):
            cs = slice(h * dh, (h + 1) * dh)
            r = fp32_head(Qb[:, cs].to(F64), Kb[:, cs].to(F64), Vb[:, cs].to(F64), scale, chain=chain)
            exact[b, cs], err[b, cs] = r["o"][0], r["err"][0]
    return _finish(exact, err)


def _softmax_result(x, m, tot, sum_err, S, p_pitch):
    """p = exp(x - m) / tot over [M, S] float64 scores -> Result over [M, p_pitch] (pad columns +0)."""
    M = x.shape[0]
    e = torch.exp(x - m)
    tiny = e < FTZ
    e[tiny] = 0.0                                                     # __expf flushes to zero
    Pex = e / tot
    d = (x - m).abs()
    eps = (2 + 1.2 * d) * 2.0 ** -24 + sum_err + 2.0 ** -22
    exact = torch.zeros(M, p_pitch, dtype=F64)
    err = torch.zeros_like(exact)
    exact[:, :S] = Pex
    err[:, :S] = torch.where(d.isfinite(), eps * Pex, 0.0) + torch.where(e < 2 * FTZ, torch.exp(x - m) / tot, 0.0)
    return Result(exact, h16(exact), err, floor=0.0)


def softmax_rows(s, M, S, s_pitch, p_pitch):
    """b200_softmax_rows: fp32 scores [M][s_pitch] -> [M, p_pitch]."""
    x = _rows(s, 0, M, s_pitch)[:, :S].to(F64)
    m = x.amax(1, keepdim=True)
    e = torch.exp(x - m)
    e[e < FTZ] = 0.0
    tot = e.sum(1, keepdim=True)
    sum_err = ((2 + 1.2 * (x - m).abs()) * e).sum(1, keepdim=True) / tot * 2.0 ** -24 + (S / 32 + 16) * 2.0 ** -24
    return _softmax_result(x, m, tot, sum_err, S, p_pitch)


def softmax_rows_partials(s, M, S, s_pitch, partials, n_tiles, p_pitch):
    """b200_softmax_rows_partials: the row maximum and sum come from partials [M][n_tiles] of (max, sum exp(v - max))
    per 128-column tile ((-inf, 0) for a tile without columns), the scores are read once."""
    x = _rows(s, 0, M, s_pitch)[:, :S].to(F64)
    part = partials[:M * n_tiles * 2].view(M, n_tiles, 2).to(F64)
    pm, ps = part[..., 0], part[..., 1]
    m = pm.amax(1, keepdim=True)
    live = pm > -math.inf
    w = torch.where(live, torch.exp(pm - m), 0.0)
    w[w < FTZ] = 0.0
    tot = (ps * w).sum(1, keepdim=True)
    d = torch.where(live, (pm - m).abs(), 0.0)
    sum_err = ((2 + 1.2 * d) * ps * w).sum(1, keepdim=True) / tot * 2.0 ** -24 + (n_tiles + 16) * 2.0 ** -24
    return _softmax_result(x, m, tot, sum_err, S, p_pitch)

"""tests/attention_emulator.py on the CPU: it agrees with plain float64 softmax attention up to the roundings it
documents, and its value bound rejects the subtle bugs an attention kernel can have (each mutant below is one, applied
to the emulator and compared against the unmutated emulator), in both 16-bit formats."""
import math

import pytest
import torch

from tests import attention_emulator as E

FORMATS = [torch.float16, torch.bfloat16]
NAN = float("nan")


@pytest.fixture(params=FORMATS, ids=["fp16", "bf16"])
def fmt(request):
    with E.storage(request.param):
        yield request.param


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def pack_rows(X, pitch, extra_rows=3):
    """[N, R, C] -> flat [N*R + extra][pitch] buffer, columns past C and the trailing rows NaN."""
    N, R, C = X.shape
    buf = torch.full(((N * R + extra_rows) * pitch,), NAN, dtype=X.dtype)
    buf[:N * R * pitch].view(N, R, pitch)[..., :C] = X
    return buf


def flash_buffers(Q, K, V, R, pad=8, vt_pad=16):
    """Logical [B, T, C] / [B, S, C] tensors -> the flash ABI buffers and pitches."""
    C, S = Q.shape[2], K.shape[1]
    qp, kp, rp = C + pad, 3 * C, C + 2 * pad
    vtp = (S + 7) // 8 * 8 + vt_pad
    vt = pack_rows(V.transpose(1, 2).contiguous(), vtp)
    res = None if R is None else pack_rows(R, rp)
    return pack_rows(Q, qp), pack_rows(K, kp), vt, res, qp, kp, vtp, rp


def rand_inputs(B, T, S, C, seed, dtype, res=True):
    g = _gen(seed)
    mk = lambda *s: torch.randn(*s, generator=g).to(dtype)
    return mk(B, T, C), mk(B, S, C), mk(B, S, C), (mk(B, T, C) if res else None)


def run_flash(Q, K, V, R, heads, dh, scale, S=None):
    q, k, vt, res, qp, kp, vtp, rp = flash_buffers(Q, K, V, R)
    B, T = Q.shape[:2]
    return E.flash(q, k, vt, res, B, T, S or K.shape[1], heads, dh, qp, kp, vtp, rp, scale)


def heads_view(X, heads, dh):
    B, N, _ = X.shape
    return X.to(torch.float64).view(B, N, heads, dh).transpose(1, 2)


def plain(Q, K, V, R, heads, dh, scale, end=None):
    """softmax(scale Q K^T) V (+ R) in float64; also the normalised P and |V| per head for the bounds."""
    q, k, v = heads_view(Q, heads, dh), heads_view(K, heads, dh), heads_view(V, heads, dh)
    s = scale * q @ k.transpose(-1, -2)
    if end is not None:
        s = torch.where(torch.arange(K.shape[1])[None, :] < end[:, None], s, -math.inf)
    P = torch.softmax(s, -1)
    o = (P @ v).transpose(1, 2).reshape(Q.shape[0], Q.shape[1], -1)
    if R is not None:
        o = o + R.to(torch.float64)
    return o, P, v, s


def _merge_heads(x):
    B, H, T, d = x.shape
    return x.transpose(1, 2).reshape(B, T, H * d)


def half_ulp_bound(P, v, s):
    """What rounding each normalised or block-scaled probability to 16 bits may move an output by: half a 16-bit step
    of P_s (relative 2^-(mant + 1), absolute 2^-25 below fp16's normal range, 2^-126 for the flush to zero), plus the
    float64 difference of exp2 against exp."""
    rel = 2.0 ** -(E._mant() + 1) + 2.0 ** -23
    floor = 2.0 ** -25 if E.H16 is torch.float16 else 2.0 ** -126
    l = torch.exp(s - s.amax(-1, keepdim=True)).sum(-1, keepdim=True)
    return _merge_heads(rel * (P @ v.abs()) + floor * v.abs().sum(-2, keepdim=True) / l) + 1e-12


# ----------------------------------------------------------------------------------------------------------------
# the emulator agrees with plain float64 softmax attention
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dh,heads,B,T,S,scale", [
    (64, 3, 2, 70, 65, 0.125), (64, 1, 1, 5, 1021, 0.125), (128, 2, 1, 33, 129, -0.09), (256, 1, 2, 9, 7, 2.5),
    (512, 2, 1, 20, 129, 0.044), (512, 1, 1, 8, 300, 0.0)])
def test_flash_emulator_is_softmax_attention(fmt, dh, heads, B, T, S, scale):
    Q, K, V, R = rand_inputs(B, T, S, heads * dh, dh + S, fmt)
    r = run_flash(Q, K, V, R, heads, dh, scale)
    # the kernel's multiplier is fp32(scale * fp32(log2 e)): the plain reference uses the same effective scale
    want, P, v, s = plain(Q, K, V, R, heads, dh, E.fp32_scale_log2e(scale) * math.log(2.0))
    assert ((r.exact - want).abs() <= half_ulp_bound(P, v, s)).all()


@pytest.mark.parametrize("dh,heads,S,scale", [(192, 2, 100, 0.07), (768, 1, 37, 0.036), (64, 1, 300, 0.5)])
def test_unfused_emulator_is_softmax_attention(fmt, dh, heads, S, scale):
    B, T = 2, 11
    Q, K, V, R = rand_inputs(B, T, S, heads * dh, dh + 7, fmt)
    q, k, vt, res, qp, kp, vtp, rp = flash_buffers(Q, K, V, R)
    r = E.unfused(q, k, vt, res, B, T, S, heads, dh, qp, kp, vtp, rp, scale)
    want, P, v, s = plain(Q, K, V, R, heads, dh, scale)
    # P is normalised before its rounding; the scores themselves are fp32 (relative 2^-24 of |s|)
    smax = s.abs().amax(-1, keepdim=True)
    bound = half_ulp_bound(P, v, s) + _merge_heads(2.0 ** -23 * smax * (P @ v.abs()))
    assert ((r.exact - want).abs() <= bound).all()


def test_cuda_core_emulators_are_softmax_attention(fmt):
    B, T, S, heads, dh, kv_rows = 2, 5, 9, 3, 33, 12
    Q, K, V, _ = rand_inputs(B, T, kv_rows, heads * dh, 3, fmt, res=False)
    C = heads * dh
    q, k, v = pack_rows(Q, C + 1), pack_rows(K, C + 3), pack_rows(V, C + 5)
    for causal, q_pos0 in ((0, 0), (1, 4)):
        r = E.small(q, k, v, B, T, S, heads, dh, C + 1, C + 3, C + 5, 0.3, kv_rows, causal, q_pos0)
        end = torch.clamp(q_pos0 + torch.arange(T) + 1, max=S) if causal else None
        want = plain(Q, K[:, :S], V[:, :S], None, heads, dh, 0.3, end)[0]
        assert torch.allclose(r.exact, want, rtol=1e-10, atol=1e-12)
    r2 = E.small(q, k, v, B, T, 0, heads, dh, C + 1, C + 3, C + 5, 0.3, kv_rows, 1, 0, pos=S - T)
    want = plain(Q, K[:, :S], V[:, :S], None, heads, dh, 0.3, S - T + torch.arange(T) + 1)[0]
    assert torch.allclose(r2.exact, want, rtol=1e-10, atol=1e-12)
    qd = pack_rows(Q[:, :1].reshape(1, B, C), C + 1)
    for S_, pos in ((7, None), (0, 6)):
        d = E.decode(qd, k, v, B, S_, heads, dh, C + 1, C + 3, C + 5, 0.3, kv_rows, pos=pos)
        want = plain(Q[:, :1], K[:, :7], V[:, :7], None, heads, dh, 0.3)[0][:, 0]
        assert torch.allclose(d.exact, want, rtol=1e-10, atol=1e-12)


def test_softmax_emulators_are_softmax(fmt):
    M, S, sp, pp = 6, 300, 301, 304
    g = _gen(5)
    x = torch.randn(M, S, generator=g) * 4
    x[1] = 2.5
    x[2, ::2] = 1e4
    x[2, 1::2] = -1e4
    s = torch.full((M * sp,), NAN)
    s.view(M, sp)[:, :S] = x
    want = torch.zeros(M, pp, dtype=torch.float64)
    want[:, :S] = torch.softmax(x.double(), -1)
    r = E.softmax_rows(s, M, S, sp, pp)
    assert torch.allclose(r.exact, want, rtol=1e-12, atol=0)
    nt = (S + 127) // 128 + 1
    part = torch.zeros(M, nt, 2)
    for t in range(nt):
        seg = x[:, t * 128:min((t + 1) * 128, S)].double()
        if seg.shape[1] == 0:
            part[:, t, 0], part[:, t, 1] = -math.inf, 0.0
            continue
        mx = seg.amax(1)
        part[:, t, 0], part[:, t, 1] = mx.float(), torch.exp(seg - mx[:, None]).sum(1).float()
    rp = E.softmax_rows_partials(s, M, S, sp, part.reshape(-1), nt, pp)
    assert torch.allclose(rp.exact, want, rtol=1e-6, atol=0)      # the partial sums are fp32
    assert (rp.out[:, S:] == 0).all() and not torch.signbit(rp.out[:, S:]).any()


# ----------------------------------------------------------------------------------------------------------------
# mutants: each is a bug an attention kernel could have; the bound must reject it on the case designed for it
# ----------------------------------------------------------------------------------------------------------------
def _zero_keys_in_l(dt):
    """Keys past S (TMA zero fill, score 0) counted in the denominator: invisible unless valid scores are 0 too."""
    Q, K, V, R = rand_inputs(1, 8, 65, 128, 11, dt)
    want = run_flash(Q, K, V, R, 2, 64, 0.0)
    Kz, Vz = (torch.cat([X, torch.zeros(1, 63, 128, dtype=dt)], 1) for X in (K, V))
    return want, run_flash(Q, Kz, Vz, R, 2, 64, 0.0).out


def _last_key_dropped(dt):
    Q, K, V, R = rand_inputs(1, 16, 65, 128, 12, dt)
    return run_flash(Q, K, V, R, 1, 128, 0.088), run_flash(Q, K, V, R, 1, 128, 0.088, S=64).out


def _causal(delta):
    def mutant(dt):
        B, T, S, heads, dh, kv = 2, 4, 7, 2, 32, 9
        Q, K, V, _ = rand_inputs(B, T, kv, heads * dh, 13, dt, res=False)
        C = heads * dh
        q, k, v = pack_rows(Q, C), pack_rows(K, C + 8), pack_rows(V, C + 8)
        run = lambda p0: E.small(q, k, v, B, T, S, heads, dh, C, C + 8, C + 8, 0.18, kv, 1, p0)
        return run(3), run(3 + delta).out
    return mutant


def _vt_halves_swapped(dt):
    Q, K, V, R = rand_inputs(1, 16, 128, 512, 14, dt)
    return run_flash(Q, K, V, R, 1, 512, 0.044), run_flash(Q, K, torch.cat([V[:, 64:], V[:, :64]], 1), R, 1, 512,
                                                           0.044).out


def _partner_sum_missing(dt):
    """d512: consumer c divides by the row sum over its own 64 keys of every block only."""
    Q, K, V, R = rand_inputs(1, 16, 128, 512, 15, dt)
    want = run_flash(Q, K, V, R, 1, 512, 0.044)
    r = E.flash_head(Q[0].double(), K[0].double(), V[0].double(), 0.044, 128)
    own = (torch.arange(128) // 64)[None, :]
    out = torch.cat([r["ptil"] @ V[0, :, 256 * c:256 * (c + 1)].double() / (r["p"] * (own == c)).sum(1, keepdim=True)
                     for c in range(2)], 1)
    return want, E.h16(out + R[0].double())[None]


def _scale_without_log2e(dt):
    Q, K, V, R = rand_inputs(1, 16, 100, 64, 16, dt)
    return run_flash(Q, K, V, R, 1, 64, 0.125), run_flash(Q, K, V, R, 1, 64, 0.125 * math.log(2.0)).out


def _head_offset(dt):
    """Every head reads its keys at head 0's channels."""
    Q, K, V, R = rand_inputs(1, 16, 70, 3 * 64, 17, dt)
    Kw = K.clone()
    Kw[..., 64:128] = K[..., :64]
    Kw[..., 128:] = K[..., :64]
    return run_flash(Q, K, V, R, 3, 64, 0.125), run_flash(Q, Kw, V, R, 3, 64, 0.125).out


def _batch_reads_batch0(dt):
    Q, K, V, R = rand_inputs(2, 16, 70, 128, 18, dt)
    Kw = K.clone()
    Kw[1] = K[0]
    return run_flash(Q, K, V, R, 1, 128, 0.088), run_flash(Q, Kw, V, R, 1, 128, 0.088).out


def _decode_empty_warp(dt):
    """S = 3 over 8 warps: the five empty warps' states counted as (max 0, sum 1, acc 0) in the merge, i.e. five
    phantom keys of score 0 and value 0."""
    B, heads, dh, kv = 2, 2, 33, 16
    C = heads * dh
    _, K, V, _ = rand_inputs(B, 1, kv, C, 19, dt, res=False)
    Qd = rand_inputs(1, B, 1, C, 20, dt, res=False)[0]
    q, k, v = pack_rows(Qd, C), pack_rows(K, C), pack_rows(V, C)
    want = E.decode(q, k, v, B, 3, heads, dh, C, C, C, 0.17, kv)
    Kz, Vz = K.clone(), V.clone()
    Kz[:, 3:8] = 0
    Vz[:, 3:8] = 0
    return want, E.decode(q, pack_rows(Kz, C), pack_rows(Vz, C), B, 8, heads, dh, C, C, C, 0.17, kv).out


def _softmax_tail_unwritten(dt):
    M, S, sp, pp = 5, 7, 8, 8
    x = torch.randn(M, S, generator=_gen(21))
    s = torch.full((M * sp,), NAN)
    s.view(M, sp)[:, :S] = x
    mx = x.double().amax(1)
    part = torch.stack([mx, torch.exp(x.double() - mx[:, None]).sum(1)], -1).float()
    want = E.softmax_rows_partials(s, M, S, sp, part.reshape(-1), 1, pp)
    got = want.out.clone()
    got[:, 4:S] = NAN                       # the sentinel the GPU test prefills
    return want, got


MUTANTS = {
    "zero_filled_keys_in_l": _zero_keys_in_l,
    "last_valid_key_dropped": _last_key_dropped,
    "causal_horizon_one_short": _causal(-1),
    "causal_horizon_one_long": _causal(+1),
    "d512_vt_key_halves_swapped": _vt_halves_swapped,
    "d512_partner_row_sum_missing": _partner_sum_missing,
    "scale_without_log2e": _scale_without_log2e,
    "head_channel_offset_wrong": _head_offset,
    "batch1_reads_batch0_keys": _batch_reads_batch0,
    "decode_merge_counts_empty_warps": _decode_empty_warp,
    "softmax_tail_not_written": _softmax_tail_unwritten,
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_bound_rejects_mutant(fmt, name):
    want, got = MUTANTS[name](fmt)
    assert torch.isfinite(want.out).all()
    assert E.excess(want, got).max() > 1, f"{name}: the bound does not see this bug"

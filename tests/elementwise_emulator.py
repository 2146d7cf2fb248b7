"""Float64 reading of the elementwise, scheduler and vector-quantiser entry points of include/b200gen.h (CPU only; test
infrastructure).

One function per entry point.  Each takes flat host tensors laid out as the C ABI describes them and returns a Result:
the float64 value before the final rounding (`exact`), the value as the entry point stores it (`out`: 16-bit or fp32,
as float64) and the accuracy term of the bound (`err`), one per element of the written region.  `kind` says how the
bound reads:

  copy   the kernel moves data, or runs an fp32 sequence the emulator reproduces exactly (embed_tokens' one fp32
         add): the bound is zero and the GPU test compares bits.  16-bit stores are fp32 -> 16-bit RN; fp16
         saturates at +-65504 (cvt.rn.satfinite), which is part of the rounding.
  h16    |got - out| <= ulp16(max(|got|, |out|)) + err;
  f32    |got - out| <= ulp32(max(|got|, |out|)) + err;
  f64    |got - out| <= ulp64(max(|got|, |out|)) + err (the double outputs of the metric and loss entry points).

err collects the fp32 terms of each kernel's arithmetic, with u = 2^-24 the unit roundoff of fp32:

  a*x + b*y       one rounding per product and one per sum, or one fma (nvcc contracts at -O3; which operand pair it
                  fuses is not specified, so both readings fit): 2u (|a x| + |b y|).  add_noise, ddim_one, the DDPM
                  and PNDM updates and the likelihood means are all of this form.
  a / b           one IEEE rounding (-prec-div): u |a / b|.
  sequential sums n terms added in fp32 in a fixed order: (n + 1) u sum |terms| (tap_sum; small_linear's lane chain
                  of ceil(K / 32) fmas plus the 5 levels of the warp tree).
  libm            CUDA's documented maximum errors: expf, cosf, sinf, tanhf, erff 2 ulp (2^-22 relative), logf 1 ulp;
                  the intrinsic __expf of SiLU / sigmoid 2 + floor(1.17 |x|) ulp, carried as (8 + 1.2 |x|) u relative as
                  tests/norm_emulator.py does.  An error d on an argument moves a function by its slope times d (SiLU
                  1.1, GELU 1.13, sigmoid 0.25, tanh 1, exp its own value).
  fp64 sums       n terms summed in fp64 in any order: n 2^-52 sum |terms| (vae_reparam_kld, ddpm_kl's sample_sum, the
                  VQ commitment numerator).

The VQ search is reproduced, not bounded: |x|^2, |e|^2 and x.e are fp32 fma chains over d from 0 (each fma computed as
the float64 product plus the addend, rounded once to fp32: exact except when the float64 sum itself rounds), then
d = (|x|^2 + |e|^2) - 2 x.e, NaN distances never win, ties go to the lowest index and a row without a finite distance
gets index 0.  tests/test_elementwise_emulator_cpu.py shows the bound rejecting the kernel-shaped mutants it lists.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from tests import norm_emulator as N
from tests.norm_emulator import F64, f32, h16, storage, ulp16  # noqa: F401  (storage: the flavour switch)

U = 2.0 ** -24                     # fp32 unit roundoff
LIBM = 2.0 ** -22                  # 2 ulp relative: expf, cosf, sinf, tanhf, erff
U52 = 2.0 ** -52                   # fp64 unit roundoff (one term of a sum)
ACT_NONE, ACT_RELU, ACT_SILU, ACT_LEAKYRELU, ACT_GELU, ACT_TANH, ACT_SIGMOID, ACT_LEAKYRELU02 = 0, 1, 2, 3, 4, 5, 6, 8
PRED_EPSILON, PRED_SAMPLE, PRED_V = 0, 1, 2
KL_EDGE = float(torch.tensor(0.999, dtype=torch.float32))     # the fp32 constant of the t = 0 thresholds


def ulp32(x):
    m = x.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(m)) - 23)


def ulp64(x):
    m = x.abs().clamp_min(2.0 ** -1022)
    return torch.exp2(torch.floor(torch.log2(m)) - 52)


@dataclass
class Result:
    exact: torch.Tensor
    out: torch.Tensor
    err: torch.Tensor
    kind: str                      # "copy", "h16", "f32" or "f64"


def _res(exact, err, kind):
    out = exact if kind in ("copy", "f64") else (h16(exact) if kind == "h16" else f32(exact))
    return Result(exact, out, err, kind)


def copy(out):
    return Result(out, out, torch.zeros_like(out), "copy")


def tolerance(r: Result, got):
    if r.kind == "copy":
        return r.err
    ulp = {"h16": ulp16, "f32": ulp32, "f64": ulp64}[r.kind]
    return ulp(torch.maximum(got.abs(), r.out.abs())) + r.err


def excess(r: Result, got):
    """|got - out| / tolerance per element (> 1 is outside the bound).  Equal values, NaN included, are 0; a value
    that differs from a copy, or a NaN / inf the emulator does not have, is inf."""
    got = got.to(F64)
    same = (got == r.out) | (torch.isnan(got) & torch.isnan(r.out))
    ratio = (got - r.out).abs() / tolerance(r, got)
    ratio = torch.where(same, torch.zeros_like(ratio), ratio.nan_to_num(math.inf, math.inf))
    bad = (~torch.isfinite(got) | ~torch.isfinite(r.out)) & ~same
    return torch.where(bad, torch.full_like(ratio, math.inf), ratio)


def rows_of(buf, n, pitch, c=None):
    return N.rows_of(buf, n, pitch, c)


# ----------------------------------------------------------------------------------------------------------------
# layout, resampling, data movement (16-bit storage)
# ----------------------------------------------------------------------------------------------------------------
def nchw_to_nhwc(x, n, C, spatial, pitch):
    """[N][C][spatial] fp32 -> rows [N * spatial][pitch] h16, pad channels +0."""
    X = x[:n * C * spatial].view(n, C, spatial).to(F64).permute(0, 2, 1).reshape(-1, C)
    out = torch.zeros(n * spatial, pitch, dtype=F64)
    out[:, :C] = h16(X)
    return copy(out)


def nhwc_to_nchw(x, n, C, spatial, pitch):
    """rows [N * spatial][pitch] (h16 or fp32) -> [N][C][spatial] fp32: columns [C, pitch) not read."""
    X = rows_of(x, n * spatial, pitch, C).view(n, spatial, C)
    return copy(X.permute(0, 2, 1).reshape(-1))


def axpy_h16(a, b, alpha, n):
    """h16(fma(alpha, b, a)) over n elements."""
    A, B = a[:n].to(F64), b[:n].to(F64)
    exact = A + f32(torch.tensor(alpha, dtype=F64)) * B
    return _res(exact, U * exact.abs(), "h16")


def copy_channels(src, C, src_pitch, rows):
    """The [rows, C] block the kernel copies into columns [dst_off, dst_off + C) of the destination."""
    return copy(rows_of(src, rows, src_pitch, C))


def gelu_erf(g):
    return 0.5 * g * (1.0 + torch.erf(g / math.sqrt(2.0)))


def geglu(x, M, H, x_pitch):
    """h16(a * 0.5 g (1 + erff(g / sqrt 2))) over [M, H]; erff 2 ulp and four fp32 roundings."""
    X = rows_of(x, M, x_pitch, 2 * H)
    a, g = X[:, :H], X[:, H:]
    exact = a * gelu_erf(g)
    err = (a * 0.5 * g).abs() * (2 * LIBM) + 4 * U * exact.abs()
    return _res(exact, err, "h16")


def _tap_offsets(geom):
    n, D, H, W, OD, OH, OW, kd, kh, kw, sd, sh, sw, pd, ph, pw = geom
    for a in range(kd):
        for b in range(kh):
            for c in range(kw):
                yield (a * kh + b) * kw + c, a, b, c


def _grid(n, OD, OH, OW):
    nn, od, oh, ow = torch.meshgrid(torch.arange(n), torch.arange(OD), torch.arange(OH), torch.arange(OW),
                                    indexing="ij")
    return nn.reshape(-1), od.reshape(-1), oh.reshape(-1), ow.reshape(-1)


def tap_gather(x, C, x_pitch, geom, out_pitch):
    """out[v][tap * C + c] = x[in_voxel(v, tap)][c] (0 outside), tap = (a kh + b) kw + c; columns past taps*C zero."""
    n, D, H, W, OD, OH, OW, kd, kh, kw, sd, sh, sw, pd, ph, pw = geom
    X = rows_of(x, n * D * H * W, x_pitch, C).view(n, D, H, W, C)
    nn, od, oh, ow = _grid(n, OD, OH, OW)
    out = torch.zeros(nn.numel(), out_pitch, dtype=F64)
    for tap, a, b, c in _tap_offsets(geom):
        i_d, i_h, i_w = od * sd + a - pd, oh * sh + b - ph, ow * sw + c - pw
        ok = (i_d >= 0) & (i_d < D) & (i_h >= 0) & (i_h < H) & (i_w >= 0) & (i_w < W)
        v = X[nn, i_d.clamp(0, D - 1), i_h.clamp(0, H - 1), i_w.clamp(0, W - 1)]
        out[:, tap * C:(tap + 1) * C] = torch.where(ok[:, None], v, torch.zeros_like(v))
    return copy(out)


def tap_sum(y, y_pitch, geom, cout, bias, out_pitch, out_h16):
    """out[v][co] = bias[co] + sum_tap y[v + off(tap)][tap * cout + co] over the taps inside the input grid (stride 1),
    fp32 in tap order; columns [cout, out_pitch) zero."""
    n, D, H, W, OD, OH, OW, kd, kh, kw, sd, sh, sw, pd, ph, pw = geom
    taps = kd * kh * kw
    Y = rows_of(y, n * D * H * W, y_pitch, taps * cout).view(n, D, H, W, taps * cout)
    nn, od, oh, ow = _grid(n, OD, OH, OW)
    b = torch.zeros(cout, dtype=F64) if bias is None else bias[:cout].to(F64)
    acc = b[None].repeat(nn.numel(), 1)
    mag = acc.abs()
    for tap, a, bb, c in _tap_offsets(geom):
        i_d, i_h, i_w = od + a - pd, oh + bb - ph, ow + c - pw
        ok = (i_d >= 0) & (i_d < D) & (i_h >= 0) & (i_h < H) & (i_w >= 0) & (i_w < W)
        v = Y[nn, i_d.clamp(0, D - 1), i_h.clamp(0, H - 1), i_w.clamp(0, W - 1), tap * cout:(tap + 1) * cout]
        v = torch.where(ok[:, None], v, torch.zeros_like(v))
        acc, mag = acc + v, mag + v.abs()
    exact = torch.zeros(nn.numel(), out_pitch, dtype=F64)
    err = torch.zeros_like(exact)
    exact[:, :cout], err[:, :cout] = acc, (taps + 1) * U * mag
    return _res(exact, err, "h16" if out_h16 else "f32")


def embed_tokens(tokens, M, seq_len, pos0, tok_emb, pos_emb, C, pitch):
    """h16(fp32(tok_emb[tokens[m]] + pos_emb[pos0 + m % seq_len])); pad columns +0."""
    T = tok_emb.float().view(-1, C)[tokens[:M].long()]
    P = pos_emb.float().view(-1, C)[pos0 + torch.arange(M) % seq_len]
    out = torch.zeros(M, pitch, dtype=F64)
    out[:, :C] = h16((T + P).to(F64))
    return copy(out)


def cache_append(src, cache, B, T, L, pitch, pos):
    """The whole [B, L, pitch] cache after the call: rows with 0 <= pos + t < L replaced, the others untouched."""
    out = cache[:B * L * pitch].to(F64).view(B, L, pitch).clone()
    S = src[:B * T * pitch].to(F64).view(B, T, pitch)
    for t in range(T):
        if 0 <= pos + t < L:
            out[:, pos + t] = S[:, t]
    return copy(out.reshape(-1))


def vq_gather(idx, M, cb, K, D, q_pitch):
    """h16 rows of the codebook at clamp(idx, 0, K - 1); pad columns +0."""
    k = idx[:M].long().clamp(0, K - 1)
    out = torch.zeros(M, q_pitch, dtype=F64)
    out[:, :D] = h16(cb.to(F64).view(K, D)[k])
    return copy(out)


# ----------------------------------------------------------------------------------------------------------------
# fp32 sampler path
# ----------------------------------------------------------------------------------------------------------------
def timestep_embedding(t, n, dim, max_period):
    """[cos(t f_k), sin(t f_k)], f_k = exp(-ln(max_period) k / half), the last column 0 when dim is odd.  The exponent
    carries logf (1 ulp), a product and a division (u each), expf 2 ulp more, the argument one rounding more: d arg =
    |arg| (|e| (2^-23 + 2u) + 2^-22 + u), then cosf / sinf 2 ulp."""
    half = dim // 2
    exact = torch.zeros(n, dim, dtype=F64)
    err = torch.zeros_like(exact)
    if half:
        k = torch.arange(half, dtype=F64)
        e = -math.log(float(f32(torch.tensor(max_period, dtype=F64)))) * k / half
        arg = t[:n].to(F64)[:, None] * torch.exp(e)[None]
        d_arg = arg.abs() * (e.abs() * (2.0 ** -23 + 2 * U) + LIBM + U)[None]
        c, s = torch.cos(arg), torch.sin(arg)
        exact[:, :half], exact[:, half:2 * half] = c, s
        err[:, :half] = d_arg + LIBM * c.abs()
        err[:, half:2 * half] = d_arg + LIBM * s.abs()
    return _res(exact, err, "f32")


_SLOPE = {ACT_NONE: 1.0, ACT_RELU: 1.0, ACT_LEAKYRELU: 1.0, ACT_LEAKYRELU02: 1.0, ACT_SILU: 1.1, ACT_GELU: 1.13,
          ACT_TANH: 1.0, ACT_SIGMOID: 0.25}


def act(t, t_err, code):
    """act(t) in float64 and its error given |d t| <= t_err: the slope carries t_err, the kernel's own arithmetic
    adds its fp32 / libm error."""
    if code == ACT_NONE:
        return t, t_err
    if code == ACT_RELU:
        return t.clamp_min(0.0), t_err
    if code in (ACT_LEAKYRELU, ACT_LEAKYRELU02):
        y = torch.where(t > 0, t, (0.01 if code == ACT_LEAKYRELU else 0.2) * t)
        return y, t_err + 2 * U * y.abs()
    if code == ACT_SILU:
        y = t * torch.sigmoid(t)
        return y, 1.1 * t_err + (8 + 1.2 * t.abs()) * U * y.abs()
    if code == ACT_SIGMOID:
        y = torch.sigmoid(t)
        return y, 0.25 * t_err + (8 + 1.2 * t.abs()) * U * y.abs()
    if code == ACT_GELU:
        y = gelu_erf(t)
        return y, 1.13 * t_err + (0.5 * t).abs() * 2 * LIBM + 4 * U * y.abs()
    if code == ACT_TANH:
        y = torch.tanh(t)
        return y, t_err + LIBM * y.abs() + U
    raise ValueError(f"activation {code} is not one small_linear takes")


def small_linear(x, M, K, W, b, O, act_in, act_out):
    """act_out(b + sum_k act_in(x) W) per [M, O]: each lane an fp32 fma chain of ceil(K / 32) terms, a 5-level warp
    tree, the bias add: (ceil(K / 32) + 7) u sum |act_in(x) w| + the activations' own terms."""
    X = x[:M * K].to(F64).view(M, K)
    Wm = W[:O * K].to(F64).view(O, K)
    a, a_err = act(X, torch.zeros_like(X), act_in)
    dot = a @ Wm.t()
    mag = a.abs() @ Wm.abs().t()
    bb = torch.zeros(O, dtype=F64) if b is None else b[:O].to(F64)
    t = dot + bb[None]
    t_err = (math.ceil(K / 32) + 7) * U * (mag + bb.abs()[None]) + a_err @ Wm.abs().t()
    y, y_err = act(t, t_err, act_out)
    return _res(y, y_err, "f32")


def rows_linear(x, x_pitch, M, K, ln_g, ln_b, eps, w, w_pitch, O, bias, act_code, res, r_pitch, out_h16):
    """b200_rows_linear over [M, O]: act(LN?(x) . w[o, :K] + bias[o]) + res[m, o].  The staged row is
    norm_emulator.rows_linear_ln's h16 row (its bound plus one 16-bit step) or x itself; each lane runs an fp32 fma
    chain of 8 ceil(K / 256) terms, a 5-level warp butterfly folds the lanes and the bias adds once:
    (8 ceil(K / 256) + 7) u (sum |x w| + |bias|); the residual add one rounding more.  Not read: x columns [K, x_pitch),
    w columns [K, w_pitch), res columns [O, r_pitch)."""
    if ln_g is not None:
        ln = N.rows_linear_ln(x, M, K, x_pitch, ln_g, ln_b, eps)
        X, X_err = ln.exact, ln.err + ulp16(ln.exact.abs() + ln.err)
    else:
        X = rows_of(x, M, x_pitch, K)
        X_err = torch.zeros_like(X)
    Wm = rows_of(w, O, w_pitch, K)
    bb = torch.zeros(O, dtype=F64) if bias is None else bias[:O].to(F64)
    t = X @ Wm.t() + bb[None]
    n = 8 * math.ceil(K / 256) + 5
    t_err = (n + 2) * U * (X.abs() @ Wm.abs().t() + bb.abs()[None]) + X_err @ Wm.abs().t()
    y, y_err = act(t, t_err, act_code)
    if res is not None:
        y = y + rows_of(res, M, r_pitch, O)
        y_err = y_err + U * y.abs()
    return _res(y, y_err, "h16" if out_h16 else "f32")


def batchnorm_fold(w, b, gamma, beta, mean, var, eps, cout, per_out):
    """(w_out, b_out) of b200_batchnorm_fold: s = gamma / sqrt(var + eps) in IEEE double, w_out = fp32(w s) bit for bit;
    b_out = fp32(beta + (b - mean) s) or one fp32 neighbour (nvcc may contract the double multiply-add into an fma,
    which can move a midpoint)."""
    s = gamma[:cout].to(F64) / torch.sqrt(var[:cout].to(F64) + float(f32(torch.tensor(eps, dtype=F64))))
    wo = f32(w[:cout * per_out].to(F64).view(cout, per_out) * s[:, None])
    bb = torch.zeros(cout, dtype=F64) if b is None else b[:cout].to(F64)
    bo = beta[:cout].to(F64) + (bb - mean[:cout].to(F64)) * s
    return copy(wo.reshape(-1)), _res(bo, torch.zeros_like(bo), "f32")


def pred_x0(m, s, c):
    """x0 and its error from the model output m and the sample s per prediction type (before any clip)."""
    sa, sb = c.sqrt_alpha_prod_t, c.sqrt_beta_prod_t
    if c.prediction_type == PRED_EPSILON:
        v = (s - sb * m) / sa
        return v, 2 * U * (s.abs() + abs(sb) * m.abs()) / abs(sa) + U * v.abs()
    if c.prediction_type == PRED_SAMPLE:
        return m.clone(), torch.zeros_like(m)
    return sa * s - sb * m, 2 * U * (abs(sa) * s.abs() + abs(sb) * m.abs())


def _clip(v, c, lo, hi):
    return v.clamp(lo, hi) if c.clip else v


def ddim_step(m, s, noise, c, n):
    """DDIMScheduler.step: (prev_sample, pred_x0) Results.  eps from the unclipped x0 (sample prediction:
    (s - sa x0) / sb; v: sa m + sb s), x0 clipped, prev = sa_prev x0 + dir eps (+ sigma noise)."""
    m, s = m[:n].to(F64), s[:n].to(F64)
    x0, e0 = pred_x0(m, s, c)
    sa, sb = c.sqrt_alpha_prod_t, c.sqrt_beta_prod_t
    if c.prediction_type == PRED_EPSILON:
        eps, ee = m, torch.zeros_like(m)
    elif c.prediction_type == PRED_SAMPLE:
        eps = (s - sa * x0) / sb
        ee = 2 * U * (s.abs() + abs(sa) * x0.abs()) / abs(sb) + U * eps.abs()
    else:
        eps = sa * m + sb * s
        ee = 2 * U * (abs(sa) * m.abs() + abs(sb) * s.abs())
    x0 = _clip(x0, c, c.clip_min, c.clip_max)
    ap, dc = c.sqrt_alpha_prod_prev, c.dir_coef
    p = ap * x0 + dc * eps
    pe = abs(ap) * e0 + abs(dc) * ee + 2 * U * (abs(ap) * x0.abs() + abs(dc) * eps.abs())
    if noise is not None:
        z = c.sigma * noise[:n].to(F64)
        pe = pe + 2 * U * (p.abs() + z.abs())
        p = p + z
    return _res(p, pe, "f32"), _res(x0, e0, "f32")


def ddpm_variance_sigma(pv, c):
    """sigma per element for var_mode 1 (sqrt(pred_var)) and 2 (sqrt(frac max_log + (1 - frac) min_log), frac =
    (pred_var + 1) / 2: MONAI's linear-domain interpolation) with its error."""
    if c.var_mode == 1:
        sig = pv.clamp_min(0).sqrt()
        return sig, U * sig
    frac = (pv + 1.0) / 2.0
    var = frac * c.max_log + (1.0 - frac) * c.min_log
    var_err = (abs(c.max_log) + abs(c.min_log)) * 2 * U * (pv.abs() + 1) + 3 * U * (
        (frac * c.max_log).abs() + ((1.0 - frac) * c.min_log).abs())
    sig = var.clamp_min(0).sqrt()
    sig_err = torch.minimum(var_err / (2 * sig.clamp_min(1e-300)), var_err.sqrt()) + U * sig
    return sig, sig_err


def ddpm_step(m, s, noise, pv, c, n):
    """DDPMScheduler.step: prev = c_x0 clip(x0) + c_xt s, + sigma noise when noise is given (sigma from var_mode)."""
    m, s = m[:n].to(F64), s[:n].to(F64)
    x0, e0 = pred_x0(m, s, c)
    x0 = _clip(x0, c, c.clip_min, c.clip_max)
    p = c.coef_x0 * x0 + c.coef_xt * s
    pe = abs(c.coef_x0) * e0 + 2 * U * (abs(c.coef_x0) * x0.abs() + abs(c.coef_xt) * s.abs())
    if noise is not None:
        z = noise[:n].to(F64)
        if c.var_mode == 0:
            sig, se = torch.full_like(z, c.sigma), torch.zeros_like(z)
        else:
            sig, se = ddpm_variance_sigma(pv[:n].to(F64), c)
        pe = pe + se * z.abs() + 2 * U * (p.abs() + (sig * z).abs())
        p = p + sig * z
    return _res(p, pe, "f32"), _res(x0, e0, "f32")


def pndm_step(hist, s, c, n):
    """eps = sum_k w[k] h[k] as an fma chain (k < n_hist), prev = sample_coeff s - eps_coeff eps' with eps' = v_alpha
    eps + v_beta s for v-prediction.  Returns (prev or None, eps) Results."""
    e = torch.zeros(n, dtype=F64)
    ee = torch.zeros_like(e)
    for k in range(c.n_hist):
        t = c.w[k] * hist[k][:n].to(F64)
        e = e + t
        ee = ee + U * (t.abs() + e.abs())
    eps = _res(e, ee, "f32")
    if s is None:
        return None, eps
    s = s[:n].to(F64)
    if c.prediction_type == PRED_V:
        e2 = c.v_alpha * e + c.v_beta * s
        ee = abs(c.v_alpha) * ee + 2 * U * (abs(c.v_alpha) * e.abs() + abs(c.v_beta) * s.abs())
        e = e2
    p = c.sample_coeff * s - c.eps_coeff * e
    pe = abs(c.eps_coeff) * ee + 2 * U * (abs(c.sample_coeff) * s.abs() + abs(c.eps_coeff) * e.abs())
    return _res(p, pe, "f32"), eps


def add_noise(x0, noise, ca, cb, sign_b, n, per):
    """out[i] = ca[n] x0 + sign_b cb[n] noise per sample."""
    a = ca[:n].to(F64)[:, None]
    b = cb[:n].to(F64)[:, None] * sign_b
    X, Z = x0[:n * per].to(F64).view(n, per), noise[:n * per].to(F64).view(n, per)
    v = a * X + b * Z
    return _res(v.reshape(-1), (2 * U * ((a * X).abs() + (b * Z).abs())).reshape(-1), "f32")


def exp_half_clamped(x, lo, hi, n):
    """expf(clamp(x, lo, hi) / 2): the halving is exact, expf 2 ulp."""
    y = torch.exp(x[:n].to(F64).clamp(f32(torch.tensor(lo, dtype=F64)).item(), f32(torch.tensor(hi, dtype=F64)).item()) / 2)
    return _res(y, LIBM * y, "f32")


def fma_f32(a, b, c, n):
    """a + b c: one fma, or a rounded product and a sum."""
    A, B, Cc = (t[:n].to(F64) for t in (a, b, c))
    return _res(A + B * Cc, U * (B * Cc).abs(), "f32")


def scale_f32(x, mul, div, n):
    """(x mul) / div: two roundings."""
    y = x[:n].to(F64) * float(f32(torch.tensor(mul, dtype=F64))) / float(f32(torch.tensor(div, dtype=F64)))
    return _res(y, U * y.abs(), "f32")


def vae_reparam_kld(mu, logvar, eps, n):
    """(z, kld): z = fma(eps, expf(0.5 logvar), mu); kld = fp32(-0.5 sum_fp64(1 + lv - mu^2 - exp(lv)))."""
    m, lv, e = (t[:n].to(F64) for t in (mu, logvar, eps))
    E = torch.exp(0.5 * lv)
    z = e * E + m
    terms = 1.0 + lv - m * m - torch.exp(lv)
    mag = (1.0 + lv.abs() + m * m + torch.exp(lv)).sum()
    kld = (-0.5 * terms.sum()).view(1)
    return (_res(z, (e * E).abs() * (LIBM + U), "f32"),
            _res(kld, (0.5 * (n + 8) * U52 * mag).view(1), "f32"))


def approx_cdf(x):
    return 0.5 * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))


def _cdf_err(x, x_err):
    z = 0.7978845608028654 * (x + 0.044715 * x ** 3)
    sech2 = 1.0 / torch.cosh(z.clamp(-40, 40)) ** 2
    slope = 0.5 * sech2 * 0.7978845608028654 * (1 + 3 * 0.044715 * x * x)
    inner = 0.5 * sech2 * 6 * U * 0.7978845608028654 * (x.abs() + 0.044715 * x.abs() ** 3)
    return slope * x_err + inner + 2 * LIBM


def ddpm_kl(x0, xt, mo, c, n, per):
    """b200_ddpm_kl: (kl Result [n * per], sample sums [n] in float64, their error [n]).  t > 0: the KL between the
    posterior N(post, e^lpo) and the predicted N(pred, e^lpv); t = 0: -log of the discretised Gaussian with the tanh
    CDF, the edge bins at a < -0.999f and a > 0.999f.  The sums are of the kernel's own fp32 terms (n 2^-52 sum |kl|
    for the fp64 accumulation) plus, against this emulator, the terms' own errors."""
    a, s, m = (t[:n * per].to(F64) for t in (x0, xt, mo))
    p0, e0 = pred_x0(m, s, c)
    p0 = p0.clamp(-1.0, 1.0) if c.clip else p0
    pm = c.coef_x0 * p0 + c.coef_xt * s
    epm = abs(c.coef_x0) * e0 + 2 * U * (abs(c.coef_x0) * p0.abs() + abs(c.coef_xt) * s.abs())
    lpv, lpo = c.log_pred_var, c.log_post_var
    if c.is_t0:
        cen = a - pm
        ec = epm + U * cen.abs()
        inv = math.exp(-0.5 * lpv)
        einv = inv * (LIBM + U)
        hb = c.bin_width / 2
        xp, xm = inv * (cen + hb), inv * (cen - hb)
        exp_ = inv * (ec + U * (cen + hb).abs()) + (cen + hb).abs() * einv + U * xp.abs()
        exm = inv * (ec + U * (cen - hb).abs()) + (cen - hb).abs() * einv + U * xm.abs()
        cp, cm = approx_cdf(xp), approx_cdf(xm)
        ecp, ecm = _cdf_err(xp, exp_), _cdf_err(xm, exm)
        lo = a < -KL_EDGE
        hi = a > KL_EDGE
        arg = torch.where(lo, cp, torch.where(hi, 1.0 - cm, cp - cm)).clamp_min(1e-12)
        earg = torch.where(lo, ecp, torch.where(hi, ecm + U, ecp + ecm + U))
        lp = torch.log(arg)
        kl = -lp
        ekl = earg / arg + 2.0 ** -23 * lp.abs()
    else:
        post = c.coef_x0 * a + c.coef_xt * s
        epost = 2 * U * (abs(c.coef_x0) * a.abs() + abs(c.coef_xt) * s.abs())
        d = post - pm
        ed = epost + epm + U * d.abs()
        E1, E2 = math.exp(lpo - lpv), math.exp(-lpv)
        kl = 0.5 * (-1.0 + lpv - lpo + E1 + d * d * E2)
        ekl = 0.5 * (6 * U * (1 + abs(lpv) + abs(lpo) + E1 + d * d * E2) + E1 * (U * abs(lpo - lpv) + LIBM)
                     + E2 * (2 * d.abs() * ed + ed * ed) + d * d * E2 * (LIBM + 2 * U))
    r = _res(kl, ekl, "f32")
    K = kl.view(n, per)
    return r, K.sum(1), ekl.view(n, per).sum(1) + per * U52 * K.abs().sum(1)


# ----------------------------------------------------------------------------------------------------------------
# vector quantiser
# ----------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    return f32(a * b + c)


def vq_distances(X, E):
    """X [M, D], E [K, D] fp32 values as float64 -> the kernel's fp32 distances [M, K]."""
    M, D = X.shape
    K = E.shape[0]
    xx = torch.zeros(M, dtype=F64)
    ee = torch.zeros(K, dtype=F64)
    dot = torch.zeros(M, K, dtype=F64)
    for d in range(D):
        xx = fma32(X[:, d], X[:, d], xx)
        ee = fma32(E[:, d], E[:, d], ee)
        dot = fma32(X[:, d, None], E[None, :, d], dot)
    return f32(f32(xx[:, None] + ee[None]) - 2.0 * dot)


def vq_pick(dist):
    """First index of the smallest non-NaN distance; 0 when no distance is finite."""
    d = torch.where(torch.isnan(dist), torch.full_like(dist, math.inf), dist)
    best = d.min(1).values
    idx = (d == best[:, None]).to(torch.int8).argmax(1)
    return torch.where(torch.isfinite(best), idx, torch.zeros_like(idx))


@dataclass
class VQ:
    idx: torch.Tensor              # int64 [M]
    q16: torch.Tensor              # [M, q_pitch] as stored, pads +0
    q32: torch.Tensor              # [M, D] fp32 (straight-through when ste)
    sqerr: float                   # float64 sum of (q - x)^2 of the fp32 differences
    sqerr_err: float
    hist: torch.Tensor             # int64 [K]
    gap: torch.Tensor              # float64 distance from the winner to the runner-up, per row (the near-tie report)


def vq_argmin_gather(x, M, D, x_pitch, cb, K, q_pitch, ste):
    X = rows_of(x, M, x_pitch, D)
    E = cb[:K * D].to(F64).view(K, D)
    idx = vq_pick(vq_distances(X, E))
    Q = E[idx]
    q16 = torch.zeros(M, q_pitch, dtype=F64)
    q16[:, :D] = h16(Q)
    diff = f32(Q - X)
    q32 = f32(X + diff) if ste else Q
    sq = float((diff * diff).sum())
    true = ((X[:, None, :] - E[None]) ** 2).sum(-1) if K > 1 else torch.zeros(M, 1, dtype=F64)
    srt = true.sort(1).values
    gap = srt[:, 1] - srt[:, 0] if K > 1 else torch.full((M,), math.inf, dtype=F64)
    return VQ(idx, q16, q32, sq, (M * D + 8) * U52 * abs(sq), torch.bincount(idx, minlength=K), gap)

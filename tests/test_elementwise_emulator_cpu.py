"""tests/elementwise_emulator.py against independent float64 references, and its bound against kernel-shaped mutants
(CPU only).

The emulator, and tests/rescaler_oracle.py's reading of the channels-last resampling calls, have to agree with
F.interpolate(nearest), F.avg_pool{2,3}d, F.gelu, F.conv{2,3}d (for the tap pair),
float64 restatements of the DDIM / DDPM / PNDM updates and of the likelihood terms, and torch.cdist's nearest codes.  Its
bound has to reject the mistakes these kernels make: kh / kw swapped in the tap decode, tap_sum padding off by one, a
dropped last tap, the 2x average pool dividing by 4 in 3-D, the nearest index (o + 1) >> 1, GEGLU halves swapped, copy_channels
ignoring dst_off, v-prediction's eps with the wrong sign, DDPM learned_range interpolated in the log domain, sigma
noise added when noise is NULL, PNDM history weights shifted by one, add_noise ignoring sign_b, the KL t = 0
thresholds swapped, the KLD sign, VQ ties to the highest index and the VQ tiled tail written from its duplicate.  Each
mutant prints its excess factor (max err / tol; inf for a copy that differs) in both storage flavours and must exceed
MARGIN.
"""
import math
import zlib
from types import SimpleNamespace as NS

import pytest
import torch
import torch.nn.functional as F

from oracle import torch_oracle as O
from tests import elementwise_emulator as E
from tests import rescaler_oracle as R

F64 = torch.float64
FLAVOURS = [torch.float16, torch.bfloat16]
FL_IDS = ["fp16", "bf16"]
MARGIN = 4.0            # a mutant must leave the bound by at least this factor


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def worst(r, got):
    return float(E.excess(r, got).max())


def report(name, flavour, r):
    print(f"\nMUTANT {name} {flavour} excess = {r:.1f}")


def rejects(name, dt, r, got):
    ex = worst(r, got)
    report(name, FL_IDS[FLAVOURS.index(dt)], ex)
    assert ex > MARGIN, name


def h16t(x):
    """Round to the current flavour's 16-bit type and keep it there."""
    return x.float().clamp(-65504, 65504).to(E.N.H16) if E.N.H16 is torch.float16 else x.float().to(E.N.H16)


# ----------------------------------------------------------------------------------------------------------------
# resampling and GEGLU against PyTorch
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
@pytest.mark.parametrize("dims", [2, 3])
def test_upsample_and_avgpool_match_torch(dt, dims):
    with E.storage(dt):
        g = gen(f"rs{dims}")
        n, D, H, W, C, pitch = 2, 5 if dims == 3 else 3, 7, 9, 12, 16
        X = torch.randn(n, D, H, W, C, generator=g, dtype=F64)
        x = torch.zeros(n, D, H, W, pitch, dtype=E.N.H16)
        x[..., :C] = h16t(X)
        ncd = x[..., :C].to(F64).permute(0, 4, 1, 2, 3)
        OD = 2 * D if dims == 3 else D
        got = E.h16(R.resample_cl(x, (OD, 2 * H, 2 * W), R.NEAREST).to(F64))
        if dims == 3:
            want = F.interpolate(ncd, scale_factor=2.0, mode="nearest")
        else:
            want = torch.stack([F.interpolate(ncd[:, :, i], scale_factor=2.0, mode="nearest") for i in range(D)], 2)
        assert torch.equal(got[..., :C], want.permute(0, 2, 3, 4, 1)) and (got[..., C:] == 0).all()
        OD = D // 2 if dims == 3 else D
        got = E.h16(R.resample_cl(x, (OD, H // 2, W // 2), R.AREA,
                                  src=(2 * OD if dims == 3 else D, H // 2 * 2, W // 2 * 2)).to(F64))
        if dims == 3:
            want = F.avg_pool3d(ncd, 2, 2)
        else:
            want = torch.stack([F.avg_pool2d(ncd[:, :, i], 2, 2) for i in range(D)], 2)
        assert torch.equal(got[..., :C], E.h16(want.permute(0, 2, 3, 4, 1))) and (got[..., C:] == 0).all()


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_geglu_matches_f_gelu(dt):
    with E.storage(dt):
        g = gen("geglu")
        M, H, xp = 33, 40, 88
        x = torch.full((M, xp), math.nan, dtype=E.N.H16)
        x[:, :2 * H] = h16t(3 * torch.randn(M, 2 * H, generator=g))
        r = E.geglu(x.reshape(-1), M, H, xp)
        X = x[:, :2 * H].to(F64)
        want = E.h16(X[:, :H] * F.gelu(X[:, H:]))
        assert worst(r, want) <= 1


GEOMS = [  # (N, D, H, W, kd, kh, kw, pd, ph, pw, stride) ; 2-D as D = kd = 1, pd = 0
    (2, 1, 9, 11, 1, 3, 3, 0, 1, 1, 1),
    (1, 6, 7, 8, 3, 1, 2, 1, 0, 1, 1),
    (2, 5, 6, 9, 2, 3, 1, 0, 2, 0, 1),
    (1, 7, 8, 9, 3, 3, 3, 1, 1, 1, 2),
    (1, 6, 9, 7, 3, 1, 2, 2, 0, 1, 2),
]


def geom_of(n, D, H, W, kd, kh, kw, pd, ph, pw, s):
    OD, OH, OW = ((e + 2 * p - k) // s + 1 for e, p, k in ((D, pd, kd), (H, ph, kh), (W, pw, kw)))
    return [n, D, H, W, OD, OH, OW, kd, kh, kw, s, s, s, pd, ph, pw]


def conv_ref(x, w, b, pads, s):
    """x [N, C, D, H, W], w [O, C, kd, kh, kw] float64 -> F.conv3d (F.conv2d when D = kd = 1)."""
    if x.shape[2] == 1 and w.shape[2] == 1:
        return F.conv2d(x[:, :, 0], w[:, :, 0], b, stride=s, padding=pads[1:])[:, :, None]
    return F.conv3d(x, w, b, stride=s, padding=pads)


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
@pytest.mark.parametrize("gi", range(len(GEOMS)))
def test_tap_pair_matches_f_conv(dt, gi):
    with E.storage(dt):
        n, D, H, W, kd, kh, kw, pd, ph, pw, s = GEOMS[gi]
        g = gen(f"tap{gi}")
        geom = geom_of(*GEOMS[gi])
        taps = kd * kh * kw
        # tap_gather: conv of a 2-channel input = gathered rows x the [taps * C] weight vector
        C = 2
        x = h16t(torch.randn(n, D, H, W, C, generator=g)).to(F64)
        w = torch.randn(3, C, kd, kh, kw, generator=g, dtype=F64)
        xp, op = C + 3, (taps * C + 7) // 8 * 8
        xbuf = torch.full((n * D * H * W, xp), math.nan, dtype=F64)
        xbuf[:, :C] = x.reshape(-1, C)
        rows = E.tap_gather(xbuf.reshape(-1), C, xp, geom, op).out
        W2 = w.permute(0, 2, 3, 4, 1).reshape(3, taps * C)            # column tap * C + c
        got = rows[:, :taps * C] @ W2.t()
        want = conv_ref(x.permute(0, 4, 1, 2, 3), w, None, (pd, ph, pw), s).permute(0, 2, 3, 4, 1).reshape(-1, 3)
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12) and (rows[:, taps * C:] == 0).all()
        if s != 1:
            return
        # tap_sum: per-tap 1x1 products y[v][tap * cout + co] = x[v] . w[co, :, tap], summed over the shifted taps
        cout, Cin = 3, 4
        x = torch.randn(n, D, H, W, Cin, generator=g, dtype=F64)
        w = torch.randn(cout, Cin, kd, kh, kw, generator=g, dtype=F64)
        b = torch.randn(cout, generator=g, dtype=F64)
        Y = torch.einsum("ndhwc,ocabe->ndhwabeo", x, w).reshape(-1, taps * cout)
        yp = taps * cout + 5
        ybuf = torch.full((Y.shape[0], yp), math.nan, dtype=F64)
        ybuf[:, :taps * cout] = E.f32(Y)
        want = conv_ref(x.permute(0, 4, 1, 2, 3), w, b, (pd, ph, pw), 1).permute(0, 2, 3, 4, 1).reshape(-1, cout)
        for out_h16 in (True, False):
            r = E.tap_sum(ybuf.reshape(-1), yp, geom, cout, b.float(), 6, out_h16)
            full = torch.zeros(want.shape[0], 6, dtype=F64)
            full[:, :cout] = E.h16(want) if out_h16 else E.f32(want)
            assert worst(r, full) <= 1


# ----------------------------------------------------------------------------------------------------------------
# schedulers and the likelihood against float64 restatements of the reference formulas
# ----------------------------------------------------------------------------------------------------------------
def ddim_coef(pred, clip=0, sigma=0.0, t=0.3, t_prev=0.55):
    sa, sb = math.sqrt(t), math.sqrt(1 - t)
    var = sigma ** 2
    c = NS(sqrt_alpha_prod_t=sa, sqrt_beta_prod_t=sb, sqrt_alpha_prod_prev=math.sqrt(t_prev),
           dir_coef=math.sqrt(1 - t_prev - var), sigma=sigma, clip_min=-1.0, clip_max=1.0, prediction_type=pred,
           clip=clip)
    for k, v in vars(c).items():           # the fp32 values the C struct holds
        if isinstance(v, float):
            setattr(c, k, float(E.f32(torch.tensor(v, dtype=F64))))
    return c


def ddim_ref(m, s, z, c, eps_sign=1.0):
    """ddim.py's step in float64: x0 and eps per prediction type, clip, prev = sqrt(a_prev) x0 + dir eps + sigma z."""
    sa, sb = c.sqrt_alpha_prod_t, c.sqrt_beta_prod_t
    if c.prediction_type == E.PRED_EPSILON:
        x0, eps = (s - sb * m) / sa, m
    elif c.prediction_type == E.PRED_SAMPLE:
        x0, eps = m, (s - sa * m) / sb
    else:
        x0, eps = sa * s - sb * m, eps_sign * sa * m + sb * s
    if c.clip:
        x0 = x0.clamp(c.clip_min, c.clip_max)
    p = c.sqrt_alpha_prod_prev * x0 + c.dir_coef * eps
    return p + c.sigma * z if z is not None else p, x0


def operands(name, n, scale=1.0):
    g = gen(name)
    return [E.f32(scale * torch.randn(n, generator=g, dtype=F64)) for _ in range(4)]


@pytest.mark.parametrize("pred", [E.PRED_EPSILON, E.PRED_SAMPLE, E.PRED_V], ids=["eps", "sample", "v"])
@pytest.mark.parametrize("clip", [0, 1])
@pytest.mark.parametrize("noise", [False, True])
def test_ddim_matches_reference_formula(pred, clip, noise):
    m, s, z, _ = operands(f"ddim{pred}{clip}{noise}", 4000)
    c = ddim_coef(pred, clip, sigma=0.3 if noise else 0.0)
    rp, rx = E.ddim_step(m, s, z if noise else None, c, m.numel())
    p, x0 = ddim_ref(m, s, z if noise else None, c)
    assert worst(rp, E.f32(p)) <= 1 and worst(rx, E.f32(x0)) <= 1


def ddpm_coef(pred=E.PRED_EPSILON, var_mode=0, clip=0):
    a_t, a_prev, beta = 0.4, 0.45, 0.02
    var = (1 - a_prev) / (1 - a_t) * beta
    c = NS(sqrt_alpha_prod_t=math.sqrt(a_t), sqrt_beta_prod_t=math.sqrt(1 - a_t),
           coef_x0=math.sqrt(a_prev) * beta / (1 - a_t), coef_xt=math.sqrt(1 - beta) * (1 - a_prev) / (1 - a_t),
           sigma=math.sqrt(var), clip_min=-1.0, clip_max=1.0, min_log=var, max_log=beta, var_mode=var_mode,
           prediction_type=pred, clip=clip)
    for k, v in vars(c).items():
        if isinstance(v, float):
            setattr(c, k, float(E.f32(torch.tensor(v, dtype=F64))))
    return c


def ddpm_ref(m, s, z, pv, c, log_domain=False):
    """ddpm.py's step in float64 (MONAI's _get_variance: learned returns pred_var, learned_range interpolates the
    variances linearly); log_domain=True is the diffusers form, exp(frac log max + (1 - frac) log min)."""
    sa, sb = c.sqrt_alpha_prod_t, c.sqrt_beta_prod_t
    x0 = (s - sb * m) / sa if c.prediction_type == E.PRED_EPSILON else (
        m if c.prediction_type == E.PRED_SAMPLE else sa * s - sb * m)
    if c.clip:
        x0 = x0.clamp(c.clip_min, c.clip_max)
    p = c.coef_x0 * x0 + c.coef_xt * s
    if z is None:
        return p
    if c.var_mode == 0:
        var = torch.full_like(p, c.sigma ** 2)
    elif c.var_mode == 1:
        var = pv
    else:
        frac = (pv + 1) / 2
        var = (torch.exp(frac * math.log(c.max_log) + (1 - frac) * math.log(c.min_log)) if log_domain
               else frac * c.max_log + (1 - frac) * c.min_log)
    return p + var.sqrt() * z


@pytest.mark.parametrize("var_mode", [0, 1, 2], ids=["fixed", "learned", "learned_range"])
@pytest.mark.parametrize("pred", [E.PRED_EPSILON, E.PRED_SAMPLE, E.PRED_V], ids=["eps", "sample", "v"])
def test_ddpm_matches_reference_formula(var_mode, pred):
    m, s, z, pv = operands(f"ddpm{var_mode}{pred}", 4000)
    pv = E.f32(pv.abs() * 0.01) if var_mode == 1 else E.f32(pv.tanh())
    c = ddpm_coef(pred, var_mode, clip=1)
    rp, rx = E.ddpm_step(m, s, z, pv, c, m.numel())
    assert worst(rp, E.f32(ddpm_ref(m, s, z, pv, c))) <= 1
    r0, _ = E.ddpm_step(m, s, None, None, c, m.numel())                 # t = 0: no noise
    assert worst(r0, E.f32(ddpm_ref(m, s, None, pv, c))) <= 1


def pndm_coef(n_hist, pred=E.PRED_EPSILON):
    w = {1: [1.0], 2: [1.5, -0.5], 3: [23 / 12, -16 / 12, 5 / 12], 4: [55 / 24, -59 / 24, 37 / 24, -9 / 24]}[n_hist]
    c = NS(w=[float(E.f32(torch.tensor(v, dtype=F64))) for v in w + [0.0] * (4 - n_hist)], n_hist=n_hist,
           sample_coeff=1.0123, eps_coeff=0.0456, v_alpha=0.6, v_beta=0.8, prediction_type=pred)
    for k in ("sample_coeff", "eps_coeff", "v_alpha", "v_beta"):
        setattr(c, k, float(E.f32(torch.tensor(getattr(c, k), dtype=F64))))
    return c


def pndm_ref(hist, s, c, shift=0):
    """pndm.py's linear multistep (weights per history length) then _get_prev_sample's update (v pre-mix)."""
    e = sum(c.w[k + shift] * hist[k] for k in range(c.n_hist) if k + shift < 4)
    if c.prediction_type == E.PRED_V:
        e = c.v_alpha * e + c.v_beta * s
    return c.sample_coeff * s - c.eps_coeff * e


@pytest.mark.parametrize("n_hist", [1, 2, 3, 4])
@pytest.mark.parametrize("pred", [E.PRED_EPSILON, E.PRED_V], ids=["eps", "v"])
def test_pndm_matches_reference_formula(n_hist, pred):
    h = operands(f"pndm{n_hist}", 3000)
    s = operands(f"pndm_s{n_hist}", 3000)[0]
    c = pndm_coef(n_hist, pred)
    rp, re = E.pndm_step(h, s, c, 3000)
    assert worst(rp, E.f32(pndm_ref(h, s, c))) <= 1
    assert worst(re, E.f32(sum(c.w[k] * h[k] for k in range(n_hist)))) <= 1


def kl_coef(is_t0, pred=E.PRED_EPSILON, clip=1):
    c = NS(sqrt_alpha_prod_t=0.9, sqrt_beta_prod_t=math.sqrt(1 - 0.81), coef_x0=0.3, coef_xt=0.65,
           log_pred_var=math.log(0.02) if not is_t0 else math.log(1e-4), log_post_var=math.log(0.015),
           bin_width=2.0 / 255, prediction_type=pred, clip=clip, is_t0=is_t0)
    for k, v in vars(c).items():
        if isinstance(v, float):
            setattr(c, k, float(E.f32(torch.tensor(v, dtype=F64))))
    return c


def kl_inputs(name, n, per):
    g = gen(name)
    a = E.f32((torch.rand(n * per, generator=g, dtype=F64) * 2 - 1))
    a[:6] = torch.tensor([E.KL_EDGE, -E.KL_EDGE, 1.0, -1.0, 0.9999, -0.9999], dtype=F64)
    s = E.f32(0.9 * a + 0.44 * torch.randn(n * per, generator=g, dtype=F64))
    m = E.f32((s - 0.9 * a) / 0.44 + 0.01 * torch.randn(n * per, generator=g, dtype=F64))
    return a, s, m


def kl_ref(a, s, m, c, swap=False):
    """inferer.py's per-element terms in float64: normal KL (t > 0) and -decoder_log_likelihood (t = 0, the oracle's
    discretised Gaussian with the tanh CDF).  swap=True exchanges the two edge bins."""
    x0 = (s - c.sqrt_beta_prod_t * m) / c.sqrt_alpha_prod_t
    x0 = x0.clamp(-1, 1) if c.clip else x0
    pred = c.coef_x0 * x0 + c.coef_xt * s
    if not c.is_t0:
        post = c.coef_x0 * a + c.coef_xt * s
        return 0.5 * (-1.0 + c.log_pred_var - c.log_post_var + math.exp(c.log_post_var - c.log_pred_var)
                      + (post - pred) ** 2 * math.exp(-c.log_pred_var))
    if not swap:
        return -O.decoder_log_likelihood(a, pred, torch.tensor(0.5 * c.log_pred_var, dtype=F64), (0, 1),
                                         (0, c.bin_width))
    inv = math.exp(-0.5 * c.log_pred_var)
    cp = O.approx_standard_normal_cdf(inv * (a - pred + c.bin_width / 2))
    cm = O.approx_standard_normal_cdf(inv * (a - pred - c.bin_width / 2))
    lp = torch.where(a < -E.KL_EDGE, torch.log((1 - cm).clamp(min=1e-12)),
                     torch.where(a > E.KL_EDGE, torch.log(cp.clamp(min=1e-12)), torch.log((cp - cm).clamp(min=1e-12))))
    return -lp


@pytest.mark.parametrize("is_t0", [0, 1], ids=["kl", "decoder_nll"])
def test_ddpm_kl_matches_likelihood_formulas(is_t0):
    c = kl_coef(is_t0)
    a, s, m = kl_inputs(f"kl{is_t0}", 3, 500)
    r, sums, serr = E.ddpm_kl(a, s, m, c, 3, 500)
    want = kl_ref(a, s, m, c)
    assert worst(r, E.f32(want)) <= 1
    assert ((sums - want.view(3, -1).sum(1)).abs() <= serr).all()


def test_vae_kld_matches_formula():
    mu, lv, eps, _ = operands("vae", 1000)
    z, kld = E.vae_reparam_kld(mu, lv, eps, 1000)
    assert worst(z, E.f32(eps * torch.exp(0.5 * lv) + mu)) <= 1
    want = -0.5 * torch.sum(1 + lv - mu.pow(2) - lv.exp())
    assert worst(kld, E.f32(want.view(1))) <= 1


@pytest.mark.parametrize("D,K", [(1, 7), (3, 33), (32, 256), (64, 1024)])
def test_vq_codes_match_cdist(D, K):
    g = gen(f"vq{D}{K}")
    M = 300
    X = E.f32(torch.randn(M, D, generator=g, dtype=F64))
    cb = E.f32(torch.randn(K, D, generator=g, dtype=F64))
    r = E.vq_argmin_gather(X.reshape(-1), M, D, D, cb.reshape(-1), K, D + 8, True)
    want = torch.cdist(X, cb).argmin(1)
    clear = r.gap > 1e-4 * (1 + (X ** 2).sum(1))              # outside fp32 near-ties
    assert clear.float().mean() > 0.9
    assert torch.equal(r.idx[clear], want[clear])
    assert torch.equal(r.hist, torch.bincount(r.idx, minlength=K))


# ----------------------------------------------------------------------------------------------------------------
# mutants
# ----------------------------------------------------------------------------------------------------------------
def gather_swapped_decode(x, C, geom, out_pitch):
    """tap_gather with the tap decoded as w = tap % kh, h = (tap / kh) % kw: kh and kw exchanged."""
    n, D, H, W, OD, OH, OW, kd, kh, kw, sd, sh, sw, pd, ph, pw = geom
    X = x.view(n, D, H, W, C)
    nn, od, oh, ow = E._grid(n, OD, OH, OW)
    out = torch.zeros(nn.numel(), out_pitch, dtype=F64)
    for tap in range(kd * kh * kw):
        cw, bh, ad = tap % kh, (tap // kh) % kw, tap // (kh * kw)
        i_d, i_h, i_w = od * sd + ad - pd, oh * sh + bh - ph, ow * sw + cw - pw
        ok = (i_d >= 0) & (i_d < D) & (i_h >= 0) & (i_h < H) & (i_w >= 0) & (i_w < W)
        v = X[nn, i_d.clamp(0, D - 1), i_h.clamp(0, H - 1), i_w.clamp(0, W - 1)]
        out[:, tap * C:(tap + 1) * C] = torch.where(ok[:, None], v, torch.zeros_like(v))
    return out


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_tap_mutants(dt):
    with E.storage(dt):
        g = gen("tapmut")
        n, D, H, W, kd, kh, kw, pd, ph, pw, s = 1, 4, 5, 6, 2, 3, 2, 1, 1, 1, 1
        geom = geom_of(n, D, H, W, kd, kh, kw, pd, ph, pw, s)
        taps, C = kd * kh * kw, 3
        x = h16t(torch.randn(n * D * H * W * C, generator=g)).to(F64)
        r = E.tap_gather(x, C, C, geom, 40)
        rejects("tap_decode_kh_kw_swapped", dt, r, gather_swapped_decode(x, C, geom, 40))
        cout = 2
        y = E.f32(torch.randn(n * D * H * W * taps * cout, generator=g, dtype=F64))
        b = torch.randn(cout, generator=g)
        for h in (True, False):
            tag = "h16" if h else "f32"
            r = E.tap_sum(y, taps * cout, geom, cout, b, 4, h)
            off = list(geom)
            off[14] = pw + 1                                                # padding off by one (low side, w)
            rejects(f"tap_sum_padding_off_by_one_{tag}", dt, r, E.tap_sum(y, taps * cout, off, cout, b, 4, h).out)
            y2 = y.view(-1, taps * cout).clone()
            y2[:, (taps - 1) * cout:] = 0                                   # the last tap dropped
            rejects(f"tap_sum_last_tap_dropped_{tag}", dt, r,
                    E.tap_sum(y2.reshape(-1), taps * cout, geom, cout, b, 4, h).out)


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_resampling_and_copy_mutants(dt):
    with E.storage(dt):
        g = gen("rsmut")
        n, D, H, W, p = 1, 4, 6, 6, 8
        x = h16t(torch.randn(n * D * H * W * p, generator=g) + 2).to(F64)
        X = x.view(n, D, H, W, p)
        r = E.copy(E.h16(R.resample_cl(X, (D // 2, H // 2, W // 2), R.AREA).to(F64)).reshape(-1))
        rejects("avgpool2_3d_divides_by_4", dt, r, E.h16(r.out * 2))
        r = E.copy(E.h16(R.resample_cl(X, (2 * D, 2 * H, 2 * W), R.NEAREST).to(F64)).reshape(-1))
        i = lambda e: ((torch.arange(2 * e) + 1) >> 1).clamp_max(e - 1)
        m = X[:, i(D)][:, :, i(H)][:, :, :, i(W)]
        rejects("nearest_index_o_plus_1", dt, r, m.reshape(-1))
        M, Hh = 5, 16
        xg = h16t(2 * torch.randn(M * 2 * Hh, generator=g)).to(F64)
        r = E.geglu(xg, M, Hh, 2 * Hh)
        X = xg.view(M, 2 * Hh)
        rejects("geglu_halves_swapped", dt, r, E.h16(X[:, Hh:] * E.gelu_erf(X[:, :Hh])))
        # copy_channels: the destination row as the kernel leaves it, with and without dst_off
        src = h16t(torch.randn(M * 8, generator=g)).to(F64)
        dst = torch.full((M, 24), 7.0, dtype=F64)
        want = dst.clone()
        want[:, 8:16] = E.copy_channels(src, 8, 8, M).out
        got = dst.clone()
        got[:, 0:8] = src.view(M, 8)
        rejects("copy_channels_ignores_dst_off", dt, E.copy(want), got)


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_scheduler_mutants(dt):
    with E.storage(dt):
        m, s, z, pv = operands("schedmut", 2000)
        c = ddim_coef(E.PRED_V)
        rp, _ = E.ddim_step(m, s, None, c, 2000)
        rejects("ddim_v_eps_sign_flipped", dt, rp, E.f32(ddim_ref(m, s, None, c, eps_sign=-1.0)[0]))
        c = ddpm_coef(var_mode=2)
        pvr = E.f32(pv.tanh())
        rp, _ = E.ddpm_step(m, s, z, pvr, c, 2000)
        rejects("ddpm_learned_range_log_domain", dt, rp, E.f32(ddpm_ref(m, s, z, pvr, c, log_domain=True)))
        c0 = ddpm_coef(var_mode=0)
        r0, _ = E.ddpm_step(m, s, None, None, c0, 2000)
        rejects("ddpm_sigma_without_noise", dt, r0, E.f32(ddpm_ref(m, s, z, None, c0)))
        h = operands("pndmmut", 2000)
        for n_hist in (2, 3, 4):
            cp = pndm_coef(n_hist)
            rp, _ = E.pndm_step(h, s, cp, 2000)
            rejects(f"pndm_weights_shifted_n{n_hist}", dt, rp, E.f32(pndm_ref(h, s, cp, shift=1)))
        ca, cb = E.f32(torch.tensor([0.9, 0.5, 0.1], dtype=F64)), E.f32(torch.tensor([0.4, 0.8, 0.99], dtype=F64))
        x0, nz = operands("addmut", 3 * 500)[:2]
        r = E.add_noise(x0, nz, ca, cb, -1.0, 3, 500)
        rejects("add_noise_ignores_sign_b", dt, r, E.add_noise(x0, nz, ca, cb, 1.0, 3, 500).out)


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_likelihood_mutants(dt):
    with E.storage(dt):
        c = kl_coef(1)
        a, s, m = kl_inputs("klmut", 1, 400)
        r, _, _ = E.ddpm_kl(a, s, m, c, 1, 400)
        rejects("kl_t0_thresholds_swapped", dt, r, E.f32(kl_ref(a, s, m, c, swap=True)))
        mu, lv, eps, _ = operands("kldmut", 500)
        _, kld = E.vae_reparam_kld(mu, lv, eps, 500)
        rejects("kld_sign", dt, kld, -kld.out)


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_vq_mutants_differ(dt):
    with E.storage(dt):
        g = gen("vqmut")
        M, D, K = 9, 32, 64
        X = E.f32(torch.randn(M, D, generator=g, dtype=F64))
        cb = E.f32(torch.randn(K, D, generator=g, dtype=F64))
        for k in (3, 4, 35):                                # rows 3, 4 and 35 all equal to x[0]: three lanes, two of one
            cb[k] = X[0]
        r = E.vq_argmin_gather(X.reshape(-1), M, D, D, cb.reshape(-1), K, D, False)
        assert int(r.idx[0]) == 3
        dist = E.vq_distances(X, cb)
        d = torch.where(torch.isnan(dist), torch.full_like(dist, math.inf), dist)
        last = K - 1 - d.flip(1).argmin(1)                   # ties to the highest index
        bad = int((last != r.idx).sum())
        print(f"\nMUTANT vq_ties_to_highest_index {FL_IDS[FLAVOURS.index(dt)]} differs at {bad} of {M} rows")
        assert bad > 0
        # the tiled kernel's last group of 4 holds M % 4 real rows and duplicates of row M - 1: written, they land past
        # the outputs and count in the histogram
        dup = torch.cat([r.idx, r.idx[-1:].repeat((-M) % 4)])
        hist = torch.bincount(dup, minlength=K)
        bad = int((hist != r.hist).sum()) + (dup.numel() - M)
        print(f"\nMUTANT vq_tiled_tail_written_from_duplicate {FL_IDS[FLAVOURS.index(dt)]} differs at {bad} entries")
        assert bad > 0


# ------------------------------------------------------------------------------------------------------------------
# rows_linear (decode GEMV) and batchnorm_fold
# ------------------------------------------------------------------------------------------------------------------
def _rows_linear_case(M, K, O, flavour, ln=True):
    g = torch.Generator().manual_seed(1000 * M + K)
    x = (torch.randn(M, K, generator=g) + 0.5).to(flavour)
    w = (torch.randn(O, K, generator=g) / K ** 0.5).to(flavour)
    bias = (0.1 * torch.randn(O, generator=g)).float()
    gam, bet = (1 + 0.1 * torch.randn(K, generator=g)).float(), (0.1 * torch.randn(K, generator=g)).float()
    res = torch.randn(M, O, generator=g).to(flavour)
    return x, w, bias, (gam, bet) if ln else (None, None), res


@pytest.mark.parametrize("flavour", FLAVOURS, ids=["fp16", "bf16"])
@pytest.mark.parametrize("M,K,O,ln,act", [(1, 1, 8, False, E.ACT_NONE), (3, 257, 40, True, E.ACT_GELU),
                                          (8, 512, 64, True, E.ACT_NONE), (5, 3072, 16, False, E.ACT_RELU)])
def test_rows_linear_reading_against_float64_linear(flavour, M, K, O, ln, act):
    """F.linear of F.layer_norm in float64, the activation, the residual: inside the reading's bound."""
    with E.storage(flavour):
        x, w, bias, (gam, bet), res = _rows_linear_case(M, K, O, flavour, ln)
        want = E.rows_linear(x.reshape(-1), K, M, K, gam, bet, 1e-5, w.reshape(-1), K, O, bias, act, res.reshape(-1), O,
                             True)
        X = x.double()
        if ln:
            X = F.layer_norm(X, (K,), gam.double(), bet.double(), 1e-5)
        t = F.linear(X, w.double(), bias.double())
        y = {E.ACT_NONE: t, E.ACT_GELU: F.gelu(t), E.ACT_RELU: F.relu(t)}[act] + res.double()
        assert (E.excess(want, E.h16(y)) <= 1).all()


def _rl_report(name, want, got):
    r = float(E.excess(want, got).max())
    print(f"\nMUTANT rows_linear {name} rejected by {r:.3g}x")
    assert r > 1, name


@pytest.mark.parametrize("flavour", FLAVOURS, ids=["fp16", "bf16"])
def test_rows_linear_bound_rejects_mutants(flavour):
    M, K, O = 8, 257, 48
    with E.storage(flavour):
        x, w, bias, (gam, bet), res = _rows_linear_case(M, K, O, flavour)
        args = lambda xx, ww, rr: (xx.reshape(-1), K, M, K, gam, bet, 1e-5, ww.reshape(-1), K, O, bias, E.ACT_GELU,
                                   rr.reshape(-1), O, True)
        want = E.rows_linear(*args(x, w, res))
        X = E.N.rows_linear_ln(x.reshape(-1), M, K, K, gam, bet, 1e-5).out
        t = X @ w.double().t()
        b, r = bias.double(), res.double()
        # the last 8-column chunk dropped (columns 256 of 257)
        w_cut = w.clone()
        w_cut[:, 256:] = 0
        _rl_report("last chunk dropped", want, E.h16(E.gelu_erf(X @ w_cut.double().t() + b) + r))
        _rl_report("bias after act", want, E.h16(E.gelu_erf(t) + b + r))
        _rl_report("residual before act", want, E.h16(E.gelu_erf(t + b + r)))
        good = E.gelu_erf(t + b) + r
        _rl_report("lane m takes row m - 1", want, E.h16(torch.cat([good[:1], good[:-1]])))


def test_batchnorm_fold_reading_against_float64():
    g = torch.Generator().manual_seed(5)
    cout, per = 16, 27
    w, b, gamma, beta, mean = (torch.randn(n, generator=g).float() for n in (cout * per, cout, cout, cout, cout))
    var = torch.rand(cout, generator=g).float()
    rw, rb = E.batchnorm_fold(w, b, gamma, beta, mean, var, 1e-5, cout, per)
    s = gamma.double() / (var.double() + float(torch.tensor(1e-5, dtype=torch.float32))).sqrt()
    assert torch.equal(rw.out, (w.double().view(cout, per) * s[:, None]).float().double().reshape(-1))
    assert (E.excess(rb, (beta.double() + (b.double() - mean.double()) * s).float().double()) <= 1).all()
    rw0, rb0 = E.batchnorm_fold(w, None, gamma, beta, mean, var, 1e-5, cout, per)
    assert torch.equal(rb0.exact, beta.double() - mean.double() * s)

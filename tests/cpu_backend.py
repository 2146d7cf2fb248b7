"""TEST-ONLY CPU stand-in for libb200gen.so: every C-ABI entry point on HOST pointers, so that the `-m "not gpu"` suite
drives the real host code (generativemodels_b200: modules, weight packing, schedulers, inferers, ctypes marshalling) end
to end on a machine without a GPU.  It is never importable from the product package.

The stand-in is marshalling: each method views its pointers as flat host tensors, calls the float64 reading of the
entry point that the GPU contract tests hold the kernels to (tests/{igemm,norm,attention,elementwise,resample}_emulator.py)
and stores that reading's rounded result.  Only weight repacking (compared bit for bit on the GPU), the position
counter of advance_i32 and the host queries are restated here."""
import ctypes as C

import numpy as np
import torch

from generativemodels_b200 import _lib, ops
from tests import attention_emulator as A
from tests import elementwise_emulator as W
from tests import igemm_emulator as E
from tests import norm_emulator as N
from tests import resample_emulator as R

F64 = torch.float64


def _obj(ref):
    return ref._obj if hasattr(ref, "_obj") else ref


def _np(ptr, count, ctype):
    if not ptr:
        return None
    return np.ctypeslib.as_array(C.cast(int(ptr), C.POINTER(ctype)), shape=(int(count),))


def f32(ptr, count):
    a = _np(ptr, count, C.c_float)
    return None if a is None else torch.from_numpy(a)


def bf16(ptr, count):
    a = _np(ptr, count, C.c_uint16)
    return None if a is None else torch.from_numpy(a.view(np.int16)).view(ops.H16)


def rows16(ptr, n_rows, pitch, cols):
    """[n_rows, cols] view of 16-bit rows `pitch` elements apart that may be a column slice of a wider buffer: only
    (n_rows - 1) * pitch + cols elements are touched."""
    flat = bf16(ptr, (n_rows - 1) * pitch + cols)
    return torch.as_strided(flat, (n_rows, cols), (pitch, 1))


def dense16(ptr, n_rows, pitch, cols):
    """rows16 copied to a flat buffer of `cols`-element rows (pass `cols` as the pitch)."""
    return rows16(ptr, n_rows, pitch, cols).reshape(-1)


def i64(ptr, count):
    a = _np(ptr, count, C.c_int64)
    return None if a is None else torch.from_numpy(a)


# Optional observer of every store of an emulator result: RECORDER(view, result) with the host view the result was
# stored into (shaped like result.out) and the emulator's Result / Affine, which carries the bound.  tests/abi_shadow.py
# installs one to compare the stand-in's stores with a real library's; None (the default) costs nothing.
RECORDER = None


def put(view, r):
    """Store the emulator result r (a Result, or a tensor of exact values) into the host view; report it."""
    view.copy_((r.out if hasattr(r, "out") else r).reshape(view.shape).to(view.dtype))
    if RECORDER is not None:
        RECORDER(view, r if hasattr(r, "out") else W.copy(r.to(F64)))


def report(view, r):
    """Report a store the caller made itself, of a result that is not compared element by element (the partial slots
    of b200_ssim); see tests/abi_shadow.py."""
    if RECORDER is not None:
        RECORDER(view, r)


def store16(ptr, r):
    out = r.out if hasattr(r, "out") else r
    put(bf16(ptr, out.numel()).view(out.shape), r)


def store32(ptr, r):
    out = r.out if hasattr(r, "out") else r
    put(f32(ptr, out.numel()).view(out.shape), r)


def _sources(p):
    """The two channels-last sources of a GroupNorm / SPADE parameter block as the norm reading takes them."""
    rows = p.N * p.spatial
    C1 = p.x_C[1] if p.x_ptr[1] else 0
    x1 = bf16(p.x_ptr[1], rows * p.x_pitch[1]) if C1 else None
    return bf16(p.x_ptr[0], rows * p.x_pitch[0]), x1, p.x_C[0], C1, p.x_pitch[0], p.x_pitch[1]


def _store_table(ptr, t):
    view = f32(ptr, t.a.numel() * 2).view(*t.a.shape, 2)
    view.copy_(torch.stack([t.a, t.b], -1))
    if RECORDER is not None:
        RECORDER(view, t)


def _table_affine(tab):
    """A [N, C, 2] affine table read from memory as the norm reading's Affine (one group per channel, no error)."""
    a, b = tab[..., 0].to(F64), tab[..., 1].to(F64)
    z = torch.zeros_like(a)
    return N.Affine(a, b, z, z, z, z, z, z, z[:1])


_CTYPES = {_lib.DT_F32: (C.c_float, np.float32, None), _lib.DT_F64: (C.c_double, np.float64, None),
           _lib.DT_FP16: (C.c_uint16, np.int16, torch.float16), _lib.DT_BF16: (C.c_uint16, np.int16, torch.bfloat16)}


def _strided(ptr, dt, strides, shape):
    """A strided host view of a B200_DT_* buffer: h16 (the flavour's 16-bit type), fp32, fp64, fp16 or bf16."""
    count = 1 + sum((s - 1) * st for s, st in zip(shape, strides))
    if dt == _lib.DT_H16:
        return torch.as_strided(bf16(ptr, count), tuple(shape), tuple(strides))
    ctype, npt, as_dtype = _CTYPES[dt]
    flat = torch.from_numpy(_np(ptr, count, ctype).view(npt))
    return torch.as_strided(flat.view(as_dtype) if as_dtype else flat, tuple(shape), tuple(strides))


def _pos(pos_dev):
    return int(_np(pos_dev, 1, C.c_int32)[0]) if pos_dev else None


class FakeLib:
    def b200_igemm(self, p, stream):
        E.emulate(_obj(p))
        return 0

    def b200_groupnorm_workspace_bytes(self, N_, spatial, C_):
        return 16

    def b200_nchw_to_nhwc(self, x, N_, C_, sp, y, pitch, stream):
        store16(y, W.nchw_to_nhwc(f32(x, N_ * C_ * sp), N_, C_, sp, pitch))
        return 0

    def b200_nhwc_to_nchw(self, x, dt, N_, C_, sp, pitch, y, stream):
        src = (bf16 if dt == _lib.DT_H16 else f32)(x, N_ * sp * pitch)
        store32(y, W.nhwc_to_nchw(src, N_, C_, sp, pitch))
        return 0

    def b200_groupnorm_stats(self, p, stream):
        p = _obj(p)
        Cc = p.x_C[0] + (p.x_C[1] if p.x_ptr[1] else 0)
        t = N.gn_stats(*_sources(p), p.N, p.spatial, p.groups, p.eps, f32(p.gamma, Cc), f32(p.beta, Cc))
        _store_table(p.affine, t)
        return 0

    def b200_groupnorm_fused(self, sp, ap, stream):
        sp, ap = _obj(sp), _obj(ap)
        Cc = sp.x_C[0] + (sp.x_C[1] if sp.x_ptr[1] else 0)
        assert Cc % sp.groups == 0 and (not sp.x_ptr[1] or sp.x_C[0] % (Cc // sp.groups) == 0)
        r, _ = N.groupnorm(*_sources(sp), sp.N, sp.spatial, sp.groups, sp.eps, f32(sp.gamma, Cc), f32(sp.beta, Cc),
                           ap.act, ap.y_pitch)
        store16(ap.y_ptr, r)
        return 0

    def b200_groupnorm_from_partials_ex(self, p, partial, slots, group, stream):
        p = _obj(p)
        Cs = [p.x_C[0], p.x_C[1] if partial[1] else 0]
        sl = [int(v) for v in slots]
        gws = [(int(v) or 8) for v in group] if group is not None else [8, 8]
        cpg = sum(Cs) // p.groups
        assert all(cpg % gw == 0 and gw in (8, 4) for gw, Ci in zip(gws, Cs) if Ci) and Cs[0] % cpg == 0
        parts = [f32(partial[i], p.N * sl[i] * (Cs[i] // gws[i]) * 2) if Cs[i] else None for i in range(2)]
        t = N.gn_from_partials(parts, sl, gws, *Cs, p.N, p.spatial, p.groups, p.eps, f32(p.gamma, sum(Cs)),
                               f32(p.beta, sum(Cs)))
        _store_table(p.affine, t)
        return 0

    def b200_spade_apply(self, p, gb, gb_pitch, gb_affine, stream):
        p = _obj(p)
        src = _sources(p)
        Cc, S = src[2] + src[3], p.N * p.spatial
        ax = f32(p.affine, p.N * Cc * 2).view(p.N, Cc, 2)
        gba = f32(gb_affine, p.N * 2 * Cc * 2).view(p.N, 2 * Cc, 2)
        r = N.spade(*src, p.N, p.spatial, ax, bf16(gb, S * gb_pitch), gb_pitch, gba, p.act, p.y_pitch)
        store16(p.y_ptr, r)
        return 0

    def b200_groupnorm_apply(self, p, stream):
        p = _obj(p)
        src = _sources(p)
        Cc = src[2] + src[3]
        X = N.concat(*src, p.N, p.spatial)
        tab = f32(p.affine, p.N * Cc * 2).view(p.N, Cc, 2)
        store16(p.y_ptr, N.gn_output(X, _table_affine(tab), p.act, p.y_pitch))
        return 0

    def b200_layernorm(self, x, M, C_, xp, g, b, eps, y, yp, stream):
        store16(y, N.layernorm(bf16(x, M * xp), M, C_, xp, f32(g, C_), f32(b, C_), eps, yp))
        return 0

    def b200_upsample2x_interp(self, x, N_, H, W_, pitch, mode, y, stream):
        store16(y, R.upsample2x_interp(bf16(x, N_ * H * W_ * pitch), N_, H, W_, pitch, mode))
        return 0

    def b200_pool_s2(self, x, N_, D, H, W_, pitch, dims, k, pad, mode, y, stream):
        store16(y, R.pool_s2(bf16(x, N_ * D * H * W_ * pitch), N_, D, H, W_, pitch, dims, k, pad, mode))
        return 0

    def b200_interpolate(self, x, xdt, xs, y, ydt, ys, N_, C_, D, H, W_, OD, OH, OW, dims, mode, rd, rh, rw, stream):
        xs, ys = [int(v) for v in xs[:5]], [int(v) for v in ys[:5]]
        if R.vector_path(C_, xdt, xs, ys, int(x), int(y)):
            C_ = (C_ + 7) // 8 * 8
        src = _strided(x, xdt, xs, (N_, C_, D, H, W_))
        r = R.interpolate(src, (OD, OH, OW)[3 - dims:], (rd, rh, rw)[3 - dims:], mode, ydt == _lib.DT_H16)
        dst = _strided(y, ydt, ys, (N_, C_, OD, OH, OW))
        put(dst, r)
        return 0

    def b200_axpy_h16(self, a, b, alpha, y, n, stream):
        store16(y, W.axpy_h16(bf16(a, n), bf16(b, n), alpha, n))
        return 0

    @staticmethod
    def _geom(g):
        return [int(v) for v in (g if not hasattr(g, "_obj") else g._obj)][:16]

    def b200_tap_gather(self, x, C_, xp, geom, out, op, stream):
        g = self._geom(geom)
        store16(out, W.tap_gather(bf16(x, g[0] * g[1] * g[2] * g[3] * xp), C_, xp, g, op))
        return 0

    def b200_tap_sum(self, y, yp, geom, cout, bias, out, op, odt, stream):
        g = self._geom(geom)
        r = W.tap_sum(f32(y, g[0] * g[1] * g[2] * g[3] * yp), yp, g, cout, f32(bias, cout), op, odt == _lib.DT_H16)
        (store16 if odt == _lib.DT_H16 else store32)(out, r)
        return 0

    def b200_copy_channels(self, src, C_, sp, dst, dp, off, rows, stream):
        r = W.copy_channels(bf16(src, rows * sp), C_, sp, rows)
        put(bf16(dst, rows * dp).view(rows, dp)[:, off:off + C_], r)
        return 0

    def b200_geglu(self, x, M, H, xp, y, yp, stream):
        put(rows16(y, M, yp, H), W.geglu(bf16(x, M * xp), M, H, xp))
        return 0

    def b200_softmax_rows_partials(self, s, M, S, sp, part, n_tiles, p, pp, stream):
        r = A.softmax_rows_partials(f32(s, M * sp), M, S, sp, f32(part, M * n_tiles * 2), n_tiles, pp)
        store16(p, r)
        return 0

    def b200_sm_count(self):
        return 2

    def b200_attention_flash_workspace_bytes(self, a):
        return 0

    def b200_igemm_split_workspace_bytes(self, a):
        return 0            # splitting the reduction is a scheduling decision of the CUDA library; results are the same

    def b200_attention_flash(self, a, stream):
        a = _obj(a)
        B, T, S, Cc = a.B, a.T, a.S, a.heads * a.dh
        res = dense16(a.res, B * T, a.res_pitch, Cc) if a.res else None
        r = A.flash(dense16(a.q, B * T, a.q_pitch, Cc), dense16(a.k, B * S, a.k_pitch, Cc),
                    dense16(a.vt, B * Cc, a.vt_pitch, S), res, B, T, S, a.heads, a.dh, Cc, Cc, S, Cc, a.scale)
        put(rows16(a.out, B * T, a.out_pitch, Cc), r)
        return 0

    def b200_attention_small_ex(self, q, k, v, o, B, T, S, heads, dh, qp, kp, vp, op, scale, kv_rows, causal, q_pos0,
                                pos_dev, stream):
        Cc = heads * dh
        r = A.small(dense16(q, B * T, qp, Cc), dense16(k, B * kv_rows, kp, Cc), dense16(v, B * kv_rows, vp, Cc), B, T,
                    S, heads, dh, Cc, Cc, Cc, scale, kv_rows, causal, q_pos0, _pos(pos_dev))
        put(rows16(o, B * T, op, Cc), r)
        return 0

    def b200_attention_small(self, q, k, v, o, B, T, S, heads, dh, qp, kp, vp, op, scale, stream):
        return self.b200_attention_small_ex(q, k, v, o, B, T, S, heads, dh, qp, kp, vp, op, scale, S, 0, 0, None,
                                            stream)

    def b200_attention_decode(self, q, k, v, o, B, S, heads, dh, qp, kp, vp, op, scale, kv_rows, pos_dev, stream):
        Cc = heads * dh
        r = A.decode(dense16(q, B, qp, Cc), dense16(k, B * kv_rows, kp, Cc), dense16(v, B * kv_rows, vp, Cc), B, S,
                     heads, dh, Cc, Cc, Cc, scale, kv_rows, _pos(pos_dev))
        put(rows16(o, B, op, Cc), r)
        return 0

    def b200_rows_linear(self, x, xp, M, K, g, b, eps, w, wp, O, bias, act, res, rp, out, op, odt, stream):
        r = W.rows_linear(dense16(x, M, xp, K), K, M, K, f32(g, K), f32(b, K), eps, dense16(w, O, wp, K), K, O,
                          f32(bias, O), act, dense16(res, M, rp, O) if res else None, O, odt == _lib.DT_H16)
        if odt == _lib.DT_F32:
            put(f32(out, M * op).view(M, op)[:, :O], r)
        else:
            put(rows16(out, M, op, O), r)
        return 0

    def b200_cache_append(self, src, cache, B, T, L, pitch, pos_dev, stream):
        r = W.cache_append(bf16(src, B * T * pitch), bf16(cache, B * L * pitch), B, T, L, pitch, _pos(pos_dev))
        store16(cache, r)
        return 0

    def b200_advance_i32(self, p, delta, stream):
        pos = torch.from_numpy(_np(p, 1, C.c_int32))
        put(pos, (pos + delta).to(F64))
        return 0

    def b200_embed_tokens(self, tokens, M, seq_len, pos0, tok_emb, pos_emb, C_, out, pitch, pos_dev, stream):
        if pos_dev:
            pos0 = _pos(pos_dev)
        tk = i64(tokens, M)
        V, Lmax = int(tk.max()) + 1, pos0 + seq_len
        r = W.embed_tokens(tk, M, seq_len, pos0, f32(tok_emb, V * C_), f32(pos_emb, Lmax * C_), C_, pitch)
        store16(out, r)
        return 0

    def b200_timestep_embedding(self, t, N_, dim, max_period, emb, stream):
        store32(emb, W.timestep_embedding(f32(t, N_), N_, dim, max_period))
        return 0

    def b200_small_linear(self, x, M, K, W_, b, O_, act_in, act_out, y, stream):
        r = W.small_linear(f32(x, M * K), M, K, f32(W_, O_ * K), f32(b, O_), O_, act_in, act_out)
        store32(y, r)
        return 0

    def b200_ddim_step(self, m, s, nz, c, prev, x0o, n, stream):
        rp, rx = W.ddim_step(f32(m, n), f32(s, n), f32(nz, n), _obj(c), n)
        store32(prev, rp)
        if x0o:
            store32(x0o, rx)
        return 0

    def b200_ddpm_step(self, m, s, nz, pv, c, prev, x0o, n, stream):
        rp, rx = W.ddpm_step(f32(m, n), f32(s, n), f32(nz, n), f32(pv, n), _obj(c), n)
        store32(prev, rp)
        if x0o:
            store32(x0o, rx)
        return 0

    def b200_ddpm_kl(self, x0, xt, mo, c, kl_out, ssum, N_, per, stream):
        r, sums, err = W.ddpm_kl(*(f32(p, N_ * per) for p in (x0, xt, mo)), _obj(c), N_, per)
        if kl_out:
            store32(kl_out, r)
        acc = torch.from_numpy(_np(ssum, N_, C.c_double))
        put(acc, W.Result(acc + sums, acc + sums, err + W.U52 * (acc + sums).abs(), "copy"))
        return 0

    def b200_pndm_step(self, hist, s, c, prev, eps_out, n, stream):
        c = _obj(c)
        rp, re = W.pndm_step([f32(hist[k], n) for k in range(c.n_hist)], f32(s, n) if prev else None, c, n)
        if eps_out:
            store32(eps_out, re)
        if prev:
            store32(prev, rp)
        return 0

    def b200_add_noise(self, x0, nz, ca, cb, sign_b, N_, per, out, stream):
        r = W.add_noise(f32(x0, N_ * per), f32(nz, N_ * per), f32(ca, N_), f32(cb, N_), sign_b, N_, per)
        store32(out, r)
        return 0

    def b200_exp_half_clamped(self, x, lo, hi, y, n, stream):
        store32(y, W.exp_half_clamped(f32(x, n), lo, hi, n))
        return 0

    def b200_fma_f32(self, a, b, c, y, n, stream):
        store32(y, W.fma_f32(f32(a, n), f32(b, n), f32(c, n), n))
        return 0

    def b200_scale_f32(self, x, mul, div, y, n, stream):
        store32(y, W.scale_f32(f32(x, n), mul, div, n))
        return 0

    def b200_vae_reparam_kld(self, mu, lv, eps, z, kld, n, stream):
        rz, rk = W.vae_reparam_kld(f32(mu, n), f32(lv, n), f32(eps, n), n)
        store32(z, rz)
        store32(kld, rk)
        return 0

    def b200_vq_argmin_gather(self, x, M, D, xp, cb, K, idx, q16, qp, q32, ste, sq, hist, stream):
        v = W.vq_argmin_gather(f32(x, M * xp), M, D, xp, f32(cb, K * D), K, qp, ste)
        put(i64(idx, M), v.idx.to(F64))
        if q16:
            store16(q16, v.q16)
        if q32:
            store32(q32, v.q32)
        if sq:
            s = torch.from_numpy(_np(sq, 1, C.c_double))
            put(s, W.Result(s + v.sqerr, s + v.sqerr, torch.tensor([v.sqerr_err + W.U52 * float(s.abs())]), "copy"))
        if hist:
            h = torch.from_numpy(_np(hist, K, C.c_int32))
            put(h, (h + v.hist).to(F64))
        return 0

    def b200_vq_gather(self, idx, M, cb, K, D, q16, qp, stream):
        store16(q16, W.vq_gather(i64(idx, M), M, f32(cb, K * D), K, D, qp))
        return 0

    def b200_repack_weight(self, src, cout, cin, taps, transposed, mode, blocks, n_blocks, dst, rows_pad, pitch, stream):
        """include/b200gen.h, b200_repack_weight — literal restatement (fp32 sums in tap order, then one rounding)."""
        w = f32(src, cout * cin * taps)
        w = w.view(cin, cout, taps).transpose(0, 1) if transposed else w.view(cout, cin, taps)      # [co][c][tap]
        out = torch.zeros(rows_pad, pitch, dtype=torch.float32)
        if mode == _lib.REPACK_TAP_IN:
            out[:cout, :taps * cin] = w.permute(0, 2, 1).reshape(cout, taps * cin)
        elif mode == _lib.REPACK_TAP_OUT:
            out[:taps * cout, :cin] = w.permute(2, 0, 1).reshape(taps * cout, cin)
        else:
            for i in range(n_blocks):
                b = blocks[i]
                acc = torch.zeros(cout, b.cs)
                for t in range(b.ntaps):
                    acc = acc + w[:, b.cin0:b.cin0 + b.cs, b.tap[t]]
                out[:cout, b.col0:b.col0 + b.cs] = acc
        if ops.H16 == torch.float16:
            out = out.clamp(-65504.0, 65504.0)
        put(bf16(dst, rows_pad * pitch).view(rows_pad, pitch), out.to(ops.H16).to(F64))
        return 0

    def b200_batchnorm_fold(self, w, b, gamma, beta, mean, var, eps, cout, per, w_out, b_out, stream):
        rw, rb = W.batchnorm_fold(f32(w, cout * per), f32(b, cout), *(f32(p, cout) for p in (gamma, beta, mean, var)),
                                  eps, cout, per)
        store32(w_out, rw)
        store32(b_out, rb)
        return 0


def install(monkeypatch):
    """Route the product's C-ABI calls to the CPU stand-in and lift its CUDA-only guards (tests only)."""
    fake = FakeLib()
    monkeypatch.setattr(_lib, "require_device", lambda: fake)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "igemm_raw", E.emulate)
    import generativemodels_b200.networks._holders as H
    import generativemodels_b200.networks.blocks.encoder_modules as EM
    import generativemodels_b200.networks.nets.autoencoderkl as AK
    import generativemodels_b200.networks.nets.controlnet as CN
    import generativemodels_b200.networks.nets.diffusion_model_unet as U
    import generativemodels_b200.networks.nets.patchgan_discriminator as PG
    import generativemodels_b200.networks.nets.spade_network as SN
    import generativemodels_b200.networks.nets.vqvae as V
    import generativemodels_b200.networks.schedulers.scheduler as S
    import generativemodels_b200.networks.schedulers.ddim as S1
    import generativemodels_b200.networks.schedulers.ddpm as S2
    import generativemodels_b200.networks.schedulers.pndm as S3
    for mod in (H, AK, CN, U, V, PG, SN, EM):
        monkeypatch.setattr(mod, "require_cuda", lambda x, m: None, raising=False)

    def prep(*tensors):
        return [None if t is None else (t if (t.dtype == torch.float32 and t.is_contiguous()) else t.float().contiguous())
                for t in tensors]
    for mod in (S, S1, S2, S3):
        monkeypatch.setattr(mod, "_prep", prep, raising=False)
    return fake

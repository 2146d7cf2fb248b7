"""CPU emulator of b200_igemm's documented semantics (include/b200gen.h), reading the very ctypes struct the
host code hands to the library.  Test infrastructure only: lets the `-m "not gpu"` suite verify tap tables, weight
packing, strides, phases and epilogue plumbing of generativemodels_b200.ops without a GPU.
"""
import ctypes as C

import numpy as np

from generativemodels_b200._lib import (ACT_DTYPE, ACT_GEGLU, ACT_GELU, ACT_LEAKYRELU, ACT_RELU, ACT_SIGMOID, ACT_SILU, ACT_TANH,
                                         DT_H16, IgemmParams)


def _bf16_view(ptr, count):
    raw = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint16)), shape=(count,))
    return raw


# the library's 16-bit storage type ("h16"): IEEE fp16 (saturating stores) unless B200_ACT_DTYPE=bf16
if ACT_DTYPE == "fp16":
    def _bf16_to_f32(u16):
        return np.ascontiguousarray(u16).view(np.float16).astype(np.float32)

    def _f32_to_bf16(x):
        x = np.clip(np.ascontiguousarray(x, dtype=np.float32), -65504.0, 65504.0)
        return x.astype(np.float16).view(np.uint16)
else:
    def _bf16_to_f32(u16):
        return (u16.astype(np.uint32) << 16).view(np.float32)

    def _f32_to_bf16(x):
        u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
        rounded = (u + 0x7FFF + ((u >> 16) & 1)) >> 16          # round to nearest even
        return rounded.astype(np.uint16)


def _f32_view(ptr, count):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(count,))


def _act(x, a):
    if a == ACT_RELU:
        return np.maximum(x, 0)
    if a == ACT_SILU:
        return x / (1 + np.exp(-x))
    if a == ACT_LEAKYRELU:
        return np.where(x > 0, x, np.float32(0.01) * x)
    if a == ACT_TANH:
        return np.tanh(x)
    if a == ACT_SIGMOID:
        return (1 / (1 + np.exp(-x))).astype(np.float32)
    if a == ACT_GELU:
        from scipy.special import erf      # float64 erf of the float32 argument, as math.erf would give
        return (0.5 * x * (1.0 + erf(np.asarray(x * 0.7071067811865476).astype(np.float64)))).astype(np.float32)
    return x


def emulate(p: IgemmParams) -> None:
    N, ID, IH, IW = p.in_N, p.in_D, p.in_H, p.in_W
    srcs = []
    for s in range(2):
        if not p.a_ptr[s]:
            srcs.append(None)
            continue
        NA = 1 if p.a_broadcast else N          # a_broadcast: one A sample shared by all N
        cnt = NA * ID * IH * IW * p.a_pitch[s]
        a = _bf16_to_f32(_bf16_view(p.a_ptr[s], cnt).copy()).reshape(NA, ID, IH, IW, p.a_pitch[s])
        srcs.append(a)
    wK = p.w_K if p.w_K > 0 else p.w_pitch
    nwb = N if p.w_batched else 1
    bstride = p.w_bstride if p.w_bstride else p.w_rows * p.w_pitch
    span = (nwb - 1) * bstride + p.w_rows * p.w_pitch
    wraw = _bf16_to_f32(_bf16_view(p.w_ptr, span).copy())
    OD, OH, OW = p.out_D, p.out_H, p.out_W
    geglu = p.act1 == ACT_GEGLU          # [32 a | 32 gate] column groups of the GEMM -> a * gelu(gate), cout / 2 channels
    if geglu:
        assert p.cout % 64 == 0 and p.out_cols == p.cout // 2 and not p.res_ptr and p.scale == 1.0 and not p.row_bias
    cols = p.cout if geglu else p.out_cols
    acc = np.zeros((N, OD, OH, OW, cols), dtype=np.float64)
    od = np.arange(OD)[:, None, None]
    oh = np.arange(OH)[None, :, None]
    ow = np.arange(OW)[None, None, :]
    for n in range(N):
        wb = n if p.w_batched else 0
        W = wraw[wb * bstride: wb * bstride + p.w_rows * p.w_pitch].reshape(p.w_rows, p.w_pitch)
        kglob = 0
        for si in range(p.n_seg):
            sg = p.seg[si]
            a = srcs[sg.src]
            idd = od * p.stride_d + sg.dd
            ihh = oh * p.stride_h + sg.dh
            iww = ow * p.stride_w + sg.dw
            ok = (idd >= 0) & (idd < ID) & (ihh >= 0) & (ihh < IH) & (iww >= 0) & (iww < IW)
            g = a[0 if p.a_broadcast else n][np.clip(idd, 0, ID - 1), np.clip(ihh, 0, IH - 1), np.clip(iww, 0, IW - 1)]   # [OD,OH,OW,pitch]
            g = g * ok[..., None]
            for c in range(sg.nchunks):
                ch0 = (sg.c0 + c) * 64
                k0 = kglob * 64
                kglob += 1
                nch = max(0, min(64, p.a_C[sg.src] - ch0))
                nk = max(0, min(64, wK - k0))
                m = min(nch, nk)
                if m <= 0:
                    continue
                rows = min(p.w_rows, cols)
                acc[n, ..., :rows] += g[..., ch0:ch0 + m].astype(np.float64) @ W[:rows, k0:k0 + m].T.astype(np.float64)
    v = acc.astype(np.float32)
    col = np.arange(cols)
    valid = col < p.cout
    if p.bias:
        b = _f32_view(p.bias, p.cout).copy()
        v[..., :p.cout] += b
    if p.rowvec:
        for n in range(N):
            rv = _f32_view(p.rowvec, n * p.rowvec_bstride + p.cout)[n * p.rowvec_bstride:].copy()
            v[n, ..., :p.cout] += rv[:p.cout]
    if p.row_bias:
        rb = _f32_view(p.row_bias, OW).copy()
        v += rb[None, None, None, :, None]
    if geglu:
        H = p.cout // 2
        vv = v.reshape(*v.shape[:-1], p.cout // 64, 2, 32)
        gated = (vv[..., 0, :] * _act(vv[..., 1, :], ACT_GELU)).astype(np.float32).reshape(*v.shape[:-1], H)
        cols = p.out_cols
        v = np.zeros((*gated.shape[:-1], cols), dtype=np.float32)
        v[..., :H] = gated
        col = np.arange(cols)
        valid = col < H
    else:
        v = _act(v, p.act1) * np.float32(p.scale)

    def strided_index(sN, sD, sH, sW):
        n = np.arange(N)[:, None, None, None, None]
        return (n * sN + od[None, ..., None] * sD + oh[None, ..., None] * sH + ow[None, ..., None] * sW
                + col[None, None, None, None, :])

    if p.res_ptr:
        idx = strided_index(p.res_sN, p.res_sD, p.res_sH, p.res_sW)
        if p.res_dtype == DT_H16:
            r = _bf16_to_f32(_bf16_view(p.res_ptr, int(idx.max()) + 1)[idx])
        else:
            r = _f32_view(p.res_ptr, int(idx.max()) + 1)[idx]
        v = v + r
    v = _act(v, p.act2)
    if p.stat_ptr:       # softmax partials per 128-column tile (GEMM-shaped calls) of the fp32 output: (max, sum exp(v - max))
        assert N == OD == OH == 1
        nt = (cols + 127) // 128
        st = _f32_view(p.stat_ptr, OW * nt * 2).reshape(OW, nt, 2)
        rows2d = v.reshape(OW, cols)
        for t in range(nt):
            seg = rows2d[:, t * 128:min((t + 1) * 128, p.cout)]
            if seg.shape[1] == 0:
                st[:, t, 0], st[:, t, 1] = -np.inf, 0.0
                continue
            mx = seg.max(1)
            st[:, t, 0] = mx
            st[:, t, 1] = np.exp(seg - mx[:, None]).sum(1)
    v[..., ~valid] = 0
    idx = strided_index(p.out_sN, p.out_sD, p.out_sH, p.out_sW)
    if p.out_dtype == DT_H16:
        dst = _bf16_view(p.out_ptr, int(idx.max()) + 1)
        dst[idx] = _f32_to_bf16(v)
        if p.gn_partial:
            # (sum, sum of squares) of the stored 16-bit values per gn_group-channel group (8 or 4), all in slot gn_slot0
            assert p.cout % 32 == 0 and 0 <= p.gn_slot0 < p.gn_slots and p.gn_group in (0, 4, 8)
            gw = p.gn_group or 8
            stored = _bf16_to_f32(_f32_to_bf16(v))[..., :p.cout].reshape(N, -1, p.cout // gw, gw).astype(np.float64)
            part = _f32_view(p.gn_partial, N * p.gn_slots * (p.cout // gw) * 2).reshape(N, p.gn_slots, p.cout // gw, 2)
            part[:, p.gn_slot0, :, 0] += stored.sum((1, 3)).astype(np.float32)
            part[:, p.gn_slot0, :, 1] += (stored * stored).sum((1, 3)).astype(np.float32)
    else:
        dst = _f32_view(p.out_ptr, int(idx.max()) + 1)
        dst[idx] = v

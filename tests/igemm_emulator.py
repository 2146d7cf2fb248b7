"""CPU emulator of b200_igemm's documented semantics (include/b200gen.h), reading the very ctypes struct the
host code hands to the library.  Test infrastructure only: lets the `-m "not gpu"` suite verify tap tables, weight
packing, strides, phases and epilogue plumbing of generativemodels_b200.ops without a GPU.
"""
import ctypes as C

import numpy as np

from generativemodels_b200._lib import (ACT_DTYPE, ACT_GEGLU, ACT_GELU, ACT_LEAKYRELU, ACT_LEAKYRELU02, ACT_RELU, ACT_SIGMOID,
                                         ACT_SILU, ACT_TANH, DT_H16, IgemmParams)


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
    if a == ACT_LEAKYRELU02:
        return np.where(x > 0, x, np.float32(0.2) * x)
    if a == ACT_TANH:
        return np.tanh(x)
    if a == ACT_SIGMOID:
        return (1 / (1 + np.exp(-x))).astype(np.float32)
    if a == ACT_GELU:
        from scipy.special import erf      # float64 erf of the float32 argument, as math.erf would give
        return (0.5 * x * (1.0 + erf(np.asarray(x * 0.7071067811865476).astype(np.float64)))).astype(np.float32)
    return x


def sample_voxels(p: IgemmParams, limit: int = 8192):
    """None (every output voxel) for calls of at most `limit` voxels per sample; else a deterministic subset of the
    flat [OD, OH, OW] voxel indices: the first and last 128 and every 37th (37 is prime to the extents, so the subset
    walks every row and column offset, the volume's borders included)."""
    V = p.out_D * p.out_H * p.out_W
    if V <= limit:
        return None
    return np.array(sorted(set(range(128)) | set(range(V - 128, V)) | set(range(128, V, 37))))


def _a_count(p: IgemmParams, s: int) -> int:
    """16-bit elements the call reads from a_ptr[s]: up to channel a_C of the last row.  a_ptr may be a channel
    offset into a wider tensor (a concatenated skip connection), whose last row ends before a full pitch does."""
    NA = 1 if p.a_broadcast else p.in_N
    return (NA * p.in_D * p.in_H * p.in_W - 1) * p.a_pitch[s] + p.a_C[s]


def emulate(p: IgemmParams, voxels=None) -> None:
    """The call p on host pointers: every output voxel, or only the flat [OD, OH, OW] indices `voxels` (the same for
    every sample; the GroupNorm partials then cover those voxels only and softmax partials are not written)."""
    N, ID, IH, IW = p.in_N, p.in_D, p.in_H, p.in_W
    srcs = []
    for s in range(2):
        if not p.a_ptr[s]:
            srcs.append(None)
            continue
        NA = 1 if p.a_broadcast else N          # a_broadcast: one A sample shared by all N
        a = np.zeros(NA * ID * IH * IW * p.a_pitch[s], dtype=np.float32)
        cnt = _a_count(p, s)
        a[:cnt] = _bf16_to_f32(_bf16_view(p.a_ptr[s], cnt).copy())
        srcs.append(a.reshape(NA, ID, IH, IW, p.a_pitch[s]))
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
    if voxels is None:
        od = np.arange(OD)[:, None, None]
        oh = np.arange(OH)[None, :, None]
        ow = np.arange(OW)[None, None, :]
        grid = (OD, OH, OW)
    else:
        vx = np.asarray(voxels)
        od, oh, ow = vx // (OH * OW), (vx // OW) % OH, vx % OW
        grid = (len(vx),)
    acc = np.zeros((N, *grid, cols), dtype=np.float64)
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
            g = a[0 if p.a_broadcast else n][np.clip(idd, 0, ID - 1), np.clip(ihh, 0, IH - 1), np.clip(iww, 0, IW - 1)]   # [*grid, pitch]
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
        v += rb[ow][None, ..., None]
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
        n = np.arange(N).reshape(N, *([1] * len(grid)), 1)
        return n * sN + od[None, ..., None] * sD + oh[None, ..., None] * sH + ow[None, ..., None] * sW + col

    if p.res_ptr:
        idx = strided_index(p.res_sN, p.res_sD, p.res_sH, p.res_sW)
        if p.res_dtype == DT_H16:
            r = _bf16_to_f32(_bf16_view(p.res_ptr, int(idx.max()) + 1)[idx])
        else:
            r = _f32_view(p.res_ptr, int(idx.max()) + 1)[idx]
        v = v + r
    v = _act(v, p.act2)
    if p.stat_ptr and voxels is None:       # softmax partials per 128-column tile (GEMM-shaped calls) of the fp32 output: (max, sum exp(v - max))
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


# ------------------------------------------------------------------------------------------------------------------
# the value bound of the GPU tests (tests/test_igemm_contract_gpu.py's docstring derives it)
#     |got - want| <= ulp16(max(|got|, |want|)) + C_LIP |scale| 2^-16 mag + REL (|want| + 1)
# with mag the emulator on |A| and |W| without epilogue, on the parameter struct of the call over host pointers
# ------------------------------------------------------------------------------------------------------------------
C_LIP = 1.5
ACC = 2.0 ** -16
REL = 2.0 ** -17


def footprint(p: IgemmParams) -> np.ndarray:
    """Element offsets from out_ptr of the output footprint, [N, OD, OH, OW, out_cols]."""
    n, d, h, w, k = np.ix_(np.arange(p.out_N), np.arange(p.out_D), np.arange(p.out_H), np.arange(p.out_W),
                           np.arange(p.out_cols))
    return n * p.out_sN + d * p.out_sD + h * p.out_sH + w * p.out_sW + k


def _abs16(ptr, count):
    """A copy of `count` 16-bit values at ptr with the sign bit cleared (|x|, NaN stays NaN)."""
    return (_bf16_view(ptr, count).copy() & np.uint16(0x7FFF))


def gemm_only(p: IgemmParams, with_bias: bool = False, voxels=None) -> np.ndarray:
    """The emulator's fp32 [N, OD, OH, OW, GEMM columns] (or [N, len(voxels), GEMM columns]) of the call with no
    epilogue, as float64: on |A| and |W| (mag), or on the operands themselves plus the bias (the GEGLU inputs a and
    gate).  p is left untouched."""
    m = IgemmParams.from_buffer_copy(p)
    keep = []
    if not with_bias:
        NA = 1 if p.a_broadcast else p.in_N
        for s in range(2):
            if p.a_ptr[s]:
                a = np.zeros(NA * p.in_D * p.in_H * p.in_W * p.a_pitch[s], dtype=np.uint16)
                a[:_a_count(p, s)] = _abs16(p.a_ptr[s], _a_count(p, s))
                keep.append(a)
                m.a_ptr[s] = keep[-1].ctypes.data
        nwb = p.in_N if p.w_batched else 1
        bstride = p.w_bstride if p.w_bstride else p.w_rows * p.w_pitch
        keep.append(_abs16(p.w_ptr, (nwb - 1) * bstride + p.w_rows * p.w_pitch))
        m.w_ptr = keep[-1].ctypes.data
        m.bias = None
    ncols = p.cout if p.act1 == ACT_GEGLU else p.out_cols
    N, OD, OH, OW = p.out_N, p.out_D, p.out_H, p.out_W
    out = np.full(N * OD * OH * OW * ncols, np.nan, dtype=np.float32)
    m.out_ptr, m.out_dtype, m.out_cols = out.ctypes.data, 1, ncols
    m.out_sW, m.out_sH, m.out_sD, m.out_sN = ncols, OW * ncols, OH * OW * ncols, OD * OH * OW * ncols
    m.res_ptr = m.stat_ptr = m.gn_partial = m.rowvec = m.row_bias = m.split_ws = None
    m.act1 = m.act2 = 0
    m.scale = 1.0
    emulate(m, voxels)
    if voxels is not None:
        return out.reshape(N, OD * OH * OW, ncols)[:, voxels].astype(np.float64)
    return out.reshape(N, OD, OH, OW, ncols).astype(np.float64)


def ulp16(x):
    mant, emin = (10, -14) if ACT_DTYPE == "fp16" else (7, -126)
    m = np.maximum(np.abs(x), 2.0 ** emin)
    return np.exp2(np.floor(np.log2(m)) - mant)


def bound(p: IgemmParams, got, want, scale=None, voxels=None):
    """The per-element tolerance of got against want ([N, OD, OH, OW, out_cols], or [N, len(voxels), out_cols],
    float64) for the call p (host pointers to the call's inputs).  `scale`: the epilogue scale as the caller chose it
    (default: p.scale, fp32)."""
    mag = gemm_only(p, voxels=voxels)
    if p.act1 == ACT_GEGLU:
        # out[j] = a * gelu(gate) with a, gate the [32 a | 32 gate] column groups of the GEMM (+ bias)
        pre = gemm_only(p, with_bias=True, voxels=voxels)
        sel = lambda x, off: x.reshape(*x.shape[:-1], -1, 2, 32)[..., off, :].reshape(*x.shape[:-1], -1)
        a, gate, ea, eg = sel(pre, 0), sel(pre, 1), ACC * sel(mag, 0), ACC * sel(mag, 1)
        from scipy.special import erf
        gelu = 0.5 * gate * (1 + erf(gate / 2 ** 0.5))
        acc_err = np.abs(gelu) * ea + (np.abs(a) + ea) * 1.2 * eg
    else:
        acc_err = abs(p.scale if scale is None else scale) * ACC * mag
    tol = C_LIP * acc_err + REL * (np.abs(want) + 1)
    if p.out_dtype == DT_H16:
        tol = tol + ulp16(np.maximum(np.abs(got), np.abs(want)))
    return tol
